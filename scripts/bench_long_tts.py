#!/usr/bin/env python
"""Long TTS benchmark: long texts as ContinuousBatcher long tickets, streamed, against sequential loops of single calls.

The workload: --texts long texts of --sentences sentences each (text lengths drawn by a fixed seed from
[--text-len-min, --text-len]), one 150-frame prompt per text, at bench.py's giga830M shape with random weights, into the
real-shape 16 kHz EnCodec decoder (seeded random weights).  As in bench.py only the length cap ends a sentence, and every
other non-audio token is suppressed too, so every generated frame has a waveform.  Two arms:
  batcher     every text submitted as one long ticket to ContinuousBatcher(max_concurrency=--slots).stream();
  sequential  the reference's Long TTS loop: per text, torch.manual_seed(seed) and one inference_tts per sentence, each
              sentence then decoded (tokenizer.decode), texts one after another.  It takes about --texts times as long
              as one text, so only the first --seq-texts texts run, and their time is reported with its per-text mean.

Reported (wall clock from the arm's start): time to first audio (median / max over the texts), the largest gap between two
consecutive chunks of one ticket across a sentence boundary and inside a sentence, total seconds and codec tokens/s;
card name, power limit and SM clock read in the same call.

    python scripts/bench_long_tts.py [--texts 32] [--sentences 5] [--slots 32] [--seq-texts 2]   -> one JSON line
"""
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

import bench  # noqa: E402  (model / NVML clock sampler of the headline benchmark)
from bench_stream import gpu_identity  # noqa: E402


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--texts", type=int, default=32)
    ap.add_argument("--sentences", type=int, default=5)
    ap.add_argument("--slots", type=int, default=32)
    ap.add_argument("--text-len-min", type=int, default=30)
    ap.add_argument("--text-len", type=int, default=60)
    ap.add_argument("--prompt", type=int, default=150)
    ap.add_argument("--model", default="830M")
    ap.add_argument("--codebooks", type=int, default=4)
    ap.add_argument("--kv", default="bf16", choices=["bf16", "fp32"])
    ap.add_argument("--chunk-frames", type=int, default=25)
    ap.add_argument("--poll-every", type=int, default=8)
    ap.add_argument("--seq-texts", type=int, default=2, help="texts the sequential arm runs (0: skip it)")
    a = ap.parse_args()
    a.workload, a.batch = "tts", a.slots
    return a


def main():
    args = parse()
    if not torch.cuda.is_available():
        raise SystemExit("bench_long_tts.py needs a CUDA device")
    from oracle import encodec_oracle as eo
    from voicecraft_b200 import synthetic
    from voicecraft_b200.tokenizer import AudioTokenizer
    from voicecraft_b200.voicecraft import ContinuousBatcher, VoiceCraft
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg, sd = bench.make_model(args)
    for k in range(cfg.n_codebooks):            # no frame may hold a token without a waveform
        for t in (cfg.empty_token, cfg.audio_pad_token):
            sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    K, N, S = cfg.n_codebooks, args.texts, args.sentences
    g = torch.Generator().manual_seed(0)
    lens = torch.randint(args.text_len_min, args.text_len + 1, (N, S), generator=g)
    texts = [[synthetic.synthetic_utterance(cfg, 1000 * i + j, int(lens[i, j]), 1)[0].to(dev) for j in range(S)]
             for i in range(N)]
    prompts = [synthetic.synthetic_utterance(cfg, 100 + i, 1, args.prompt)[2].to(dev) for i in range(N)]
    seeds = [1 + i for i in range(N)]
    model = VoiceCraft(cfg)
    model.load_state_dict(sd)
    model = model.to(dev).eval()
    cap = args.text_len * (cfg.encodec_sr // 5)
    model.configure_engine(max_slots=args.slots, max_seq_len=(args.text_len + cap + 64 + 255) // 256 * 256,
                           kv_dtype=args.kv, max_new_tokens=cap + 64)
    ccfg = eo.default_config()
    tok = AudioTokenizer(device=dev, config=ccfg, state_dict=eo.make_state_dict(ccfg, seed=0))
    kw = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)

    def batcher(n):
        first, last_at, gaps = {}, {}, {"boundary": [], "inside": []}
        t0 = time.perf_counter()
        cb = ContinuousBatcher(model, max_concurrency=args.slots, poll_every=args.poll_every, **kw)
        for i in range(n):
            cb.submit(texts[i], prompts[i], seed=seeds[i])
        it = cb.stream(tok, chunk_frames=args.chunk_frames)
        for t, _, _ in it:
            now = time.perf_counter() - t0
            # sentences finished when the chunk came: a chain appends a sentence's result after its last chunk
            sent = len(cb._live.jobs[t].chain.results)
            first.setdefault(t, now)
            if t in last_at:
                gaps["boundary" if sent != last_at[t][1] else "inside"].append(now - last_at[t][0])
            last_at[t] = (now, sent)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        frames = sum(int(gen.shape[-1]) for r in cb.results[:n] for _, gen in r)
        return [first[t] for t in range(n)], dt, frames, gaps, dict(cb.stats)

    def sequential(n):
        first, frames = {}, 0
        t0 = time.perf_counter()
        for i in range(n):
            torch.manual_seed(seeds[i])
            for x in texts[i]:
                _, gen = model.inference_tts(x, torch.tensor([x.shape[1]], device=dev), prompts[i], **kw)
                tok.decode([(gen, None)])
                torch.cuda.synchronize()
                first.setdefault(i, time.perf_counter() - t0)
                frames += int(gen.shape[-1])
        dt = time.perf_counter() - t0
        return [first[i] for i in range(n)], dt, frames

    batcher(2)                                   # untimed warm-up (allocations, codec workspace, both arms' shapes)
    if args.seq_texts:
        sequential(1)
    clocks = bench.ClockSampler(0)
    clocks.start()
    fa, dt, frames, gaps, stats = batcher(N)
    seq = sequential(min(args.seq_texts, N)) if args.seq_texts else None
    clk = clocks.stop()
    out = {
        "metric": f"codec tokens/s (giga{args.model} Long TTS, {N} texts x {S} sentences, {args.slots} slots, streamed)",
        "value": frames * K / dt, "unit": "codec tokens/s", "n_gpus": 1, "higher_is_better": True, "dtype": "bf16",
        "data": "synthetic",
        "config": dict(texts=N, sentences=S, slots=args.slots, text_len=[args.text_len_min, args.text_len],
                       prompt_frames=args.prompt, model=args.model, kv=args.kv, chunk_frames=args.chunk_frames,
                       poll_every=args.poll_every,
                       codec="16 kHz EnCodec decoder (4 x 2048, n_filters 64, LSTM 2), seeded random weights"),
        "batcher": {"first_audio_ms": {"median": statistics.median(fa) * 1e3, "max": max(fa) * 1e3},
                    "chunk_gap_ms": {k: {"max": max(v) * 1e3 if v else None,
                                         "median": statistics.median(v) * 1e3 if v else None, "n": len(v)}
                                     for k, v in gaps.items()},
                    "seconds": dt, "generated_frames": frames, "codec_tokens_per_s": frames * K / dt, "stats": stats},
        "gpu": gpu_identity(0), "clocks": clk,
        "note": "one timed call per arm after an untimed warm-up; wall clock from the arm's start"}
    if seq is not None:
        n = len(seq[0])
        out["sequential"] = {"texts_run": n, "seconds": seq[1], "seconds_per_text": seq[1] / n,
                             "first_audio_ms": {"median": statistics.median(seq[0]) * 1e3},
                             "generated_frames": seq[2], "codec_tokens_per_s": seq[2] * K / seq[1]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
