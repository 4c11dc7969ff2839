#!/usr/bin/env python
"""Streaming TTS benchmark: time to first audio, streaming vs batch, on one GPU.

The tts utterances of bench.py (B per GPU, 80 phoneme ids, 150-frame / 3 s prompt -> 800 frames / 16 s, the giga830M
shape with random weights) decoded two ways, the arms alternating in one call:
  streaming  VoiceCraft.inference_tts_many_stream into the real-shape 16 kHz EnCodec decoder (seeded random weights of
             oracle.encodec_oracle.make_state_dict: there is no codec checkpoint offline);
  batch      inference_tts_many, then one decode_codes of every utterance.
Every non-audio token except the length cap's end token is suppressed, so every generated frame has a waveform.

    python scripts/bench_stream.py [--batch 32] [--chunk-frames 25] [--poll-every 8] [--repeats 2]   -> one JSON line

--queue N instead serves N utterances with B slots, their text lengths spread by a fixed seed over
[--text-len-min, --text-len] (with equal lengths every utterance ends at the same step and continuous batching has nothing
to gain), two arms alternating in one call:
  batcher  all N submitted to ContinuousBatcher(max_concurrency=B).stream(), its cb.stats reported;
  static   ceil(N/B) consecutive inference_tts_many_stream calls of B utterances.

value = codec tokens/s of the streaming arm, tokens to waveform end to end; first_audio_ms (median / max over the
utterances) and seconds_to_all_audio for both arms, wall clock from the call's start; card name, power limit and SM clock
read in the same call.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402  (model / utterances / NVML clock sampler of the headline benchmark)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--text-len", type=int, default=80)
    ap.add_argument("--prompt", type=int, default=150)
    ap.add_argument("--model", default="830M")
    ap.add_argument("--codebooks", type=int, default=4)
    ap.add_argument("--kv", default="bf16", choices=["bf16", "fp32"])
    ap.add_argument("--chunk-frames", type=int, default=25)
    ap.add_argument("--poll-every", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=2, help="timed calls per arm after one untimed warm-up of each")
    ap.add_argument("--queue", type=int, default=0, help="serve this many utterances: batcher stream vs static batches")
    ap.add_argument("--text-len-min", type=int, default=40, help="--queue: shortest text (the longest is --text-len)")
    a = ap.parse_args()
    a.workload = "tts"
    return a


def gpu_identity(index):
    """card name, enforced power limit (W) and current SM clock (MHz), read through NVML"""
    out = {"name": torch.cuda.get_device_name(index), "power_limit_w": None, "sm_mhz": None}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        out["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
        out["sm_mhz"] = pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception as e:  # pragma: no cover
        out["error"] = repr(e)
    return out


def main():
    args = parse()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream.py needs a CUDA device")
    from oracle import encodec_oracle as eo
    from voicecraft_b200.tokenizer import AudioTokenizer
    from voicecraft_b200.voicecraft import VoiceCraft
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg, sd = bench.make_model(args)
    for k in range(cfg.n_codebooks):            # no frame may hold a token without a waveform
        for t in (cfg.empty_token, cfg.audio_pad_token):
            sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    K, B = cfg.n_codebooks, args.batch
    if args.queue:
        from voicecraft_b200 import synthetic
        lens = torch.randint(args.text_len_min, args.text_len + 1, (args.queue,), generator=torch.Generator().manual_seed(0))
        utts = [synthetic.synthetic_utterance(cfg, 100 + i, int(n), args.prompt) for i, n in enumerate(lens)]
    else:
        utts = bench.make_utterances(args, cfg, range(B))
    seeds = [1 + i for i in range(len(utts))]
    model = VoiceCraft(cfg)
    model.load_state_dict(sd)
    model = model.to(dev).eval()
    cap = args.text_len * (cfg.encodec_sr // 5)
    model.configure_engine(max_slots=B, max_seq_len=(args.text_len + cap + 64 + 255) // 256 * 256, kv_dtype=args.kv,
                           max_new_tokens=cap + 64)
    ccfg = eo.default_config()
    tok = AudioTokenizer(device=dev, config=ccfg, state_dict=eo.make_state_dict(ccfg, seed=0))
    xs = [u[0].to(dev) for u in utts]
    ys = [u[2].to(dev) for u in utts]
    kw = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
    if args.queue:
        return queue(args, cfg, model, tok, xs, ys, seeds, kw)

    def streaming():
        first = {}
        t0 = time.perf_counter()
        ts = model.inference_tts_many_stream(xs, ys, tok, chunk_frames=args.chunk_frames, poll_every=args.poll_every,
                                             seeds=seeds, **kw)
        for i, _ in ts:                          # a chunk is handed out once its waveform is complete on the device
            first.setdefault(i, time.perf_counter() - t0)
        torch.cuda.synchronize()
        return [first[i] for i in range(B)], time.perf_counter() - t0, sum(int(r[1].shape[-1]) for r in ts.results)

    def batch():
        t0 = time.perf_counter()
        out = model.inference_tts_many(xs, ys, poll_every=args.poll_every, seeds=seeds, **kw)
        gens = [r[1] for r in out]
        if len({g.shape[-1] for g in gens}) == 1:
            tok.decode_codes(torch.cat(gens, 0))
        else:
            for g in gens:
                tok.decode_codes(g)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        return [dt] * B, dt, sum(int(g.shape[-1]) for g in gens)

    streaming(), batch()                         # untimed warm-up (allocations, codec workspace)
    clocks = bench.ClockSampler(0)
    clocks.start()
    runs = {"streaming": [], "batch": []}
    for _ in range(max(1, args.repeats)):
        runs["streaming"].append(streaming())
        runs["batch"].append(batch())
    clk = clocks.stop()
    arms = {}
    for name, rs in runs.items():
        r = sorted(rs, key=lambda v: v[1])[len(rs) // 2]          # the median call by total time
        arms[name] = {"first_audio_ms": {"median": statistics.median(r[0]) * 1e3, "max": max(r[0]) * 1e3},
                      "seconds_to_all_audio": r[1], "generated_frames": r[2], "seconds_all": [v[1] for v in rs]}
    s = arms["streaming"]
    print(json.dumps({
        "metric": f"codec tokens/s (giga{args.model} streaming TTS, tokens to waveform)",
        "value": s["generated_frames"] * K / s["seconds_to_all_audio"], "unit": "codec tokens/s", "n_gpus": 1,
        "higher_is_better": True, "dtype": "bf16", "data": "synthetic",
        "config": dict(bench.workload_config(args, cfg, 1),
                       codec="16 kHz EnCodec decoder (4 x 2048, n_filters 64, LSTM 2), seeded random weights",
                       chunk_frames=args.chunk_frames, poll_every=args.poll_every),
        "streaming": s, "batch": arms["batch"], "gpu": gpu_identity(0), "clocks": clk,
        "note": "wall clock from the call's start, median of %d alternating calls per arm after one untimed warm-up of each; "
                "batch arm: first audio = all audio" % max(1, args.repeats)}))


def queue(args, cfg, model, tok, xs, ys, seeds, kw):
    from voicecraft_b200.voicecraft import ContinuousBatcher
    K, B, N = cfg.n_codebooks, args.batch, len(xs)

    def batcher():
        first = {}
        t0 = time.perf_counter()
        cb = ContinuousBatcher(model, max_concurrency=B, poll_every=args.poll_every, **kw)
        for x, y, s in zip(xs, ys, seeds):
            cb.submit(x, y, seed=s)
        it = cb.stream(tok, chunk_frames=args.chunk_frames)
        for t, _, _ in it:
            first.setdefault(t, time.perf_counter() - t0)
        torch.cuda.synchronize()
        return [first[t] for t in range(N)], time.perf_counter() - t0, sum(int(r[1].shape[-1]) for r in cb.results), \
            it.push_host_seconds, dict(cb.stats)

    def static():
        first, frames, push_s = {}, 0, 0.0
        t0 = time.perf_counter()
        for b in range(0, N, B):
            ts = model.inference_tts_many_stream(xs[b:b + B], ys[b:b + B], tok, chunk_frames=args.chunk_frames,
                                                 poll_every=args.poll_every, seeds=seeds[b:b + B], **kw)
            for i, _ in ts:
                first.setdefault(b + i, time.perf_counter() - t0)
            frames += sum(int(r[1].shape[-1]) for r in ts.results)
            push_s += ts.push_host_seconds
        torch.cuda.synchronize()
        return [first[t] for t in range(N)], time.perf_counter() - t0, frames, push_s, None

    batcher(), static()                          # untimed warm-up
    clocks = bench.ClockSampler(0)
    clocks.start()
    runs = {"batcher": [], "static": []}
    for _ in range(max(1, args.repeats)):
        runs["batcher"].append(batcher())
        runs["static"].append(static())
    clk = clocks.stop()
    arms = {}
    for name, rs in runs.items():
        r = sorted(rs, key=lambda v: v[1])[len(rs) // 2]          # the median call by total time
        fa = sorted(r[0])
        arms[name] = {"first_audio_ms": {"median": statistics.median(fa) * 1e3, "p90": fa[int(0.9 * (len(fa) - 1))] * 1e3,
                                         "max": fa[-1] * 1e3},
                      "seconds_to_all_audio": r[1], "generated_frames": r[2],
                      "codec_tokens_per_s": r[2] * K / r[1], "push_host_ms": r[3] * 1e3, "seconds_all": [v[1] for v in rs]}
        if r[4] is not None:
            arms[name]["stats"] = r[4]
    print(json.dumps({
        "metric": f"seconds to all audio (giga{args.model} streaming TTS, {N} queued utterances, {B} slots)",
        "value": arms["batcher"]["seconds_to_all_audio"], "unit": "s", "n_gpus": 1, "higher_is_better": False,
        "dtype": "bf16", "data": "synthetic",
        "config": dict(bench.workload_config(args, cfg, 1), queue=N, text_len_min=args.text_len_min,
                       codec="16 kHz EnCodec decoder (4 x 2048, n_filters 64, LSTM 2), seeded random weights",
                       chunk_frames=args.chunk_frames, poll_every=args.poll_every),
        "batcher": arms["batcher"], "static": arms["static"], "gpu": gpu_identity(0), "clocks": clk,
        "note": "wall clock from the call's start, median of %d alternating calls per arm after one untimed warm-up of each; "
                "push_host_ms: host time in the push step outside the device waits" % max(1, args.repeats)}))


if __name__ == "__main__":
    main()
