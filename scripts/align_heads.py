"""Rank the codec LM's attention heads as aligners against a known word alignment (for a maintainer with a checkpoint).

For each (layer, head), the prompt (--wav) is prefilled with alignment={layer: [head]}; the prompt frames' rows go through
the device monotonic alignment search and are grouped into words at the phonemizer's word separator `_`
(Alignment.words).  The score is the mean absolute difference, in seconds, between those word boundaries and the
`words` rows of --mfa-csv (the reference's Begin,End,Label,Type,Speaker layout), lower is better.  Prints one JSON line
per head, best first.  Reads only the paths it is given.

--ckpt: a reference VoiceCraft checkpoint (torch.save of {"config", "model", "phn2num"}); --encodec: the audiocraft
EnCodec checkpoint it was trained with (its "best_state"); --text: the phonemized transcript of the wav as the reference's
tokenize_text yields it, phonemes separated by spaces with `_` between words (no phonemizer runs here).

usage: align_heads.py --ckpt CKPT --encodec ENCODEC --wav WAV --mfa-csv CSV --text "h @ l oU _ w 3 l d" [--device cuda:0]"""
import argparse
import json
import os
import sys
from argparse import Namespace


def mfa_words(path):
    """(begin, end) of the `words` rows of an MFA CSV, as inference_speech_editing_scale.py:get_mask_interval reads it"""
    with open(path) as f:
        rows = [line.strip().split(",") for line in f.readlines()][1:]
    return [(float(r[0]), float(r[1])) for r in rows if len(r) >= 4 and r[3] == "words"]


def main():
    ap = argparse.ArgumentParser()
    for a in ("--ckpt", "--encodec", "--wav", "--mfa-csv", "--text"):
        ap.add_argument(a, required=True)
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args()
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import torch
    from voicecraft_b200.tokenizer import AudioTokenizer, default_codec_config, state_dict_from_audiocraft, tokenize_audio
    from voicecraft_b200.voicecraft import VoiceCraft, _read_alignment

    ck = torch.load(args.ckpt, map_location="cpu")
    cfg = ck["config"] if isinstance(ck["config"], Namespace) else Namespace(**ck["config"])
    phn2num = ck["phn2num"]
    model = VoiceCraft(cfg)
    model.load_state_dict(ck["model"])
    model = model.to(args.device).eval()
    ccfg = default_codec_config()
    enc = torch.load(args.encodec, map_location="cpu")
    tok = AudioTokenizer(device=args.device, config=ccfg, state_dict=state_dict_from_audiocraft(enc["best_state"], ccfg))
    codes = tokenize_audio(tok, args.wav)                                   # [1, K, T]
    phones = [p for p in args.text.split() if p in phn2num]
    x = torch.tensor([[phn2num[p] for p in phones]], dtype=torch.long)
    y = codes.transpose(1, 2).contiguous()
    sep = phn2num["_"]
    want = mfa_words(args.mfa_csv)
    T, x_len = int(y.shape[1]), int(x.shape[1])
    model.configure_engine(max_slots=1, align_text_cap=x_len, max_seq_len=(x_len + 2 * T + 64 + 255) // 256 * 256)
    scores = []
    for layer in range(cfg.num_decoder_layers):
        for head in range(cfg.nhead):
            sess = model.open_tts_session([x], [y], seeds=[0], alignment={layer: [head]})
            try:
                al = _read_alignment(model, sess.eng, sess.slots[0], sess.prompts[0], T, sess.stream)
            finally:
                sess.close()
            got = [(s, e) for _, _, s, e in al.words(sep)]
            n = min(len(got), len(want))
            err = sum(abs(a[0] - b[0]) + abs(a[1] - b[1]) for a, b in zip(got[:n], want[:n])) / max(1, 2 * n)
            scores.append(dict(layer=layer, head=head, mean_boundary_err_s=err, words=len(got), mfa_words=len(want)))
    for s in sorted(scores, key=lambda s: s["mean_boundary_err_s"]):
        print(json.dumps(s))


if __name__ == "__main__":
    main()
