"""Prompt audio -> codes: the CUDA-core encoder (encode_codes, enc_encode) against the tensor-core encoder
(encode_many, enc_encode_ragged), and audio tickets in the ContinuousBatcher.  JSON lines.

- `encode`: 32 x 10 s, 32 ragged prompts of 3..10 s, 1 x 3 s and 1 x 10 s at 16 kHz.  CUDA-core: encode_codes over the
  batch (the ragged batch one prompt per call, as a server has to); tensor-core: one encode_many.  CUDA events around
  `--iters` calls after a warm-up.  GFLOP from the encoder plan (oracle encoder_plan: every conv, the LSTM's W_ih and
  W_hh products, the RVQ scores) and the achieved TFLOP/s; for the tensor-core path also the FLOP its padded chunk runs.
- `--queue N`: a ContinuousBatcher.stream() queue of N bench.py-shaped tickets (830M, text 80, prompt 3 s) whose prompts
  arrive as 44.1 kHz audio, against the same tickets given the codes (encoded before the clock starts): first-audio
  p50 / p90 and time to all audio, rounds alternating; the tokens are checked equal.
The card's name and power limit are read in the same run.
usage: bench_encode.py [--iters 10] [--queue 64 --rounds 2]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402


def card():
    from bench_resample import gpu_identity
    return gpu_identity(0)


def timed_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def plan_flops(cfg, n):
    """FLOP of encoding one prompt of n samples, from oracle encoder_plan (multiply-add = 2)"""
    from oracle import encodec_oracle as eo
    T, f = n, 0.0
    for L in eo.encoder_plan(cfg):
        if L["kind"] == "conv":
            T = -(-T // L["stride"])
            f += 2.0 * L["cin"] * L["cout"] * L["k"] * T
        elif L["kind"] == "res":
            f += 2.0 * T * (L["dim"] * L["hidden"] * L["k"] + L["hidden"] * L["dim"] + L["dim"] * L["dim"])
        else:
            f += 2.0 * T * L["layers"] * 2 * 4 * L["dim"] * L["dim"]
    return f + 2.0 * T * cfg.dimension * cfg.bins * cfg.n_q


def encode(args):
    from oracle import encodec_oracle as eo
    from voicecraft_b200.tokenizer import AudioTokenizer
    cfg = eo.default_config()
    tok = AudioTokenizer(device="cuda:0", config=cfg, state_dict=eo.make_state_dict(cfg, seed=0, encoder=True))
    g = torch.Generator().manual_seed(0)
    lens3_10 = [int(16000 * (3 + 7 * i / 31)) for i in range(32)]
    cases = {"32x10s": [160000] * 32, "32x3-10s": lens3_10, "1x3s": [48000], "1x10s": [160000]}
    for name, lens in cases.items():
        wavs = [(torch.rand(1, n, generator=g) * 2 - 1).cuda() for n in lens]
        flops = sum(plan_flops(cfg, n) for n in lens)
        same_len = len(set(lens)) == 1
        batch = torch.stack(wavs) if same_len else None
        cc = timed_ms((lambda: tok.encode_codes(batch)) if same_len else (lambda: [tok.encode_codes(w[None]) for w in wavs]),
                      max(1, args.iters // 4))
        tc = timed_ms(lambda: tok.encode_many(wavs), args.iters)
        padded = len(lens) * plan_flops(cfg, max(lens))
        got = tok.encode_many(wavs)
        agree = sum(int((a == tok.encode_codes(w[None])).all(dim=1).sum()) for a, w in zip(got[:4], wavs[:4]))
        print(json.dumps({"measure": "encode", "case": name, "prompts": len(lens), "audio_s": round(sum(lens) / 16000, 2),
                          "cuda_core_ms": round(cc, 3), "tensor_core_ms": round(tc, 3), "speedup": round(cc / tc, 2),
                          "gflop": round(flops / 1e9, 1), "cuda_core_tflops": round(flops / cc / 1e9, 2),
                          "tensor_core_tflops": round(flops / tc / 1e9, 2),
                          "tensor_core_tflops_padded": round(padded / tc / 1e9, 2),
                          "frames_equal_first4": f"{agree}/{sum(x.shape[-1] for x in got[:4])}",
                          "iters": args.iters, "gpu": card()}), flush=True)


def queue(args):
    from oracle import encodec_oracle as eo
    from voicecraft_b200 import synthetic
    from voicecraft_b200.tokenizer import AudioTokenizer
    from voicecraft_b200.voicecraft import ContinuousBatcher
    from bench_kv_pool import model_830m
    B, N, text, seconds, rate = 32, args.queue, 80, 3.0, 44100
    cap = text * 10
    seq = (text + cap + 64 + 255) // 256 * 256
    cfg, m = model_830m("bf16", B, seq, cap + 64, codec_safe=True)
    ccfg = eo.default_config()
    tok = AudioTokenizer(device="cuda:0", config=ccfg, state_dict=eo.make_state_dict(ccfg, seed=0, encoder=True))
    g = torch.Generator().manual_seed(1)
    xs = [synthetic.synthetic_utterance(cfg, 100 + i, text, 8)[0].cuda() for i in range(N)]
    audio = [torch.rand(1, int(seconds * rate) - 37 * i, generator=g) * 2 - 1 for i in range(N)]
    ys = [c.transpose(1, 2) for c in tok.encode_many(audio, rate)]
    kw = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)

    def run(with_audio):
        cb = ContinuousBatcher(m, max_concurrency=B, poll_every=8, tokenizer=tok, **kw)
        for i in range(N):
            if with_audio:
                cb.submit(xs[i], audio=audio[i], sample_rate=rate, seed=1 + i)
            else:
                cb.submit(xs[i], ys[i], seed=1 + i)
        first = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for t, _, _ in cb.stream(tok, chunk_frames=25):
            first.setdefault(t, time.perf_counter() - t0)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        fa = sorted(first.values())
        return dict(seconds_to_all_audio=round(total, 3), first_audio_ms_p50=round(statistics.median(fa) * 1e3, 1),
                    first_audio_ms_p90=round(fa[int(0.9 * (len(fa) - 1))] * 1e3, 1), steps=cb.stats["steps"]), \
            [r[1] for r in cb.results]
    for arm in (True, False):                                  # warm-up of each arm
        run(arm)
    gens = {}
    for r in range(args.rounds):
        for arm in (True, False):
            rec, gen = run(arm)
            gens.setdefault(arm, gen)
            print(json.dumps({"measure": "queue", "round": r, "prompts": "audio 44.1 kHz" if arm else "codes", "tickets": N,
                              "max_concurrency": B, "prompt_s": seconds, **rec, "gpu": card()}), flush=True)
    print(json.dumps({"measure": "queue", "equal_tokens": all(torch.equal(a, b) for a, b in zip(gens[True], gens[False]))}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--queue", type=int, default=0)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_encode.py needs a CUDA device")
    encode(args)
    if args.queue:
        queue(args)


if __name__ == "__main__":
    main()
