#!/usr/bin/env python
"""Streaming speech editing and the mixed batcher queue, on one GPU.  One JSON line.

edit arm (scripts/bench_edit.py's shape): 830M, B = 16 independent utterances, T = 800 frames each, 160 phoneme ids, one
masked span [300, 400); every non-audio token is suppressed, so every span runs to the reference's length cap
(y_len > 10 * x_len) and every frame has a waveform.  Two arms alternating in one call:
  streaming  VoiceCraft.inference_many_stream into the real-shape 16 kHz EnCodec decoder (seeded random weights);
  batch      inference_many, then one decode_codes of every edited utterance.
  Time to first audio (the leading original piece: 300 frames final before the first step) and to all audio.

queue arm: --queue N tickets, half TTS and half edit (40 phoneme ids, 150-frame prompts, edits mask [60, 100)), served by
ContinuousBatcher(max_concurrency=--slots).run(), two arms alternating in one call:
  per_ticket  each ticket with its own top_k / top_p / temperature / stop_repetition (the group table of the sampler);
  shared      the same tickets, every one with the batcher's parameters.
  ms per decode step (wall clock over the call / steps) and, in a separate profiled call of each arm, the sampler's
  device ms per step (vcb_profile_read class 4).

The card name, power limit and SM clock are read in the same call.

    python scripts/bench_edit_stream.py [--batch 16] [--queue 16] [--slots 8] [--repeats 2]
"""
import argparse
import ctypes as C
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

QUEUE_PARAMS = [dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3),
                dict(top_k=-100, top_p=0.9, temperature=0.8, stop_repetition=-1),
                dict(top_k=20, top_p=0.95, temperature=1.1, stop_repetition=2),
                dict(top_k=1, top_p=1.0, temperature=1.0, stop_repetition=3)]


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--chunk-frames", type=int, default=25)
    ap.add_argument("--poll-every", type=int, default=8)
    ap.add_argument("--queue", type=int, default=16, help="tickets of the mixed batcher queue (0: skip it)")
    ap.add_argument("--slots", type=int, default=8, help="max_concurrency of the mixed batcher queue")
    ap.add_argument("--repeats", type=int, default=2, help="timed calls per arm after one untimed warm-up of each")
    a = ap.parse_args()
    a.model, a.codebooks, a.text_len, a.prompt, a.kv, a.workload = "830M", 4, 160, 800, "bf16", "edit"
    return a


def median_call(rs, key):
    return sorted(rs, key=key)[len(rs) // 2]


def main():
    args = parse()
    if not torch.cuda.is_available():
        raise SystemExit("bench_edit_stream.py needs a CUDA device")
    from oracle import encodec_oracle as eo
    from voicecraft_b200 import _lib, synthetic
    from voicecraft_b200.tokenizer import AudioTokenizer
    from voicecraft_b200.voicecraft import ContinuousBatcher, VoiceCraft
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg, sd = bench.make_model(args)
    for k in range(cfg.n_codebooks):            # no frame may hold a token without a waveform; spans end at the cap
        for t in (cfg.empty_token, cfg.eog, cfg.audio_pad_token, cfg.eos):
            sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    K, B = cfg.n_codebooks, args.batch
    model = VoiceCraft(cfg)
    model.load_state_dict(sd)
    model = model.to(dev).eval()
    model.configure_engine(max_slots=max(B, args.slots), max_seq_len=2048, max_new_tokens=1200)
    ccfg = eo.default_config()
    tok = AudioTokenizer(device=dev, config=ccfg, state_dict=eo.make_state_dict(ccfg, seed=0))
    utts = [synthetic.synthetic_utterance(cfg, 100 + i, args.text_len, args.prompt) for i in range(B)]
    xs, ys = [u[0].to(dev) for u in utts], [u[2].to(dev) for u in utts]
    spans = [torch.tensor([[[300, 400]]]) for _ in range(B)]
    seeds = [1 + i for i in range(B)]
    kw = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=-1)

    def streaming():
        first = {}
        t0 = time.perf_counter()
        ts = model.inference_many_stream(xs, ys, spans, tok, chunk_frames=args.chunk_frames, poll_every=args.poll_every,
                                         seeds=seeds, **kw)
        for i, _ in ts:
            first.setdefault(i, time.perf_counter() - t0)
        torch.cuda.synchronize()
        return [first[i] for i in range(B)], time.perf_counter() - t0, sum(int(r.shape[-1]) for r in ts.results)

    def batch():
        t0 = time.perf_counter()
        res = model.inference_many(xs, ys, spans, poll_every=args.poll_every, seeds=seeds, **kw)
        if len({r.shape[-1] for r in res}) == 1:
            tok.decode_codes(torch.cat(res, 0))
        else:
            for r in res:
                tok.decode_codes(r)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        return [dt] * B, dt, sum(int(r.shape[-1]) for r in res)

    streaming(), batch()                         # untimed warm-up (allocations, codec workspace)
    clocks = bench.ClockSampler(0)
    clocks.start()
    runs = {"streaming": [], "batch": []}
    for _ in range(max(1, args.repeats)):
        runs["streaming"].append(streaming())
        runs["batch"].append(batch())
    edit = {}
    for name, rs in runs.items():
        r = median_call(rs, lambda v: v[1])
        edit[name] = {"first_audio_ms": {"median": statistics.median(r[0]) * 1e3, "max": max(r[0]) * 1e3},
                      "seconds_to_all_audio": r[1], "output_frames": r[2], "seconds_all": [v[1] for v in rs]}
    out = {"metric": "seconds to first audio (giga830M streaming speech editing, B=%d, T=800, span [300,400))" % B,
           "value": edit["streaming"]["first_audio_ms"]["median"] / 1e3, "unit": "s", "n_gpus": 1,
           "higher_is_better": False, "dtype": "bf16", "data": "synthetic",
           "config": dict(bench.workload_config(args, cfg, 1), span=[300, 400], chunk_frames=args.chunk_frames,
                          poll_every=args.poll_every,
                          codec="16 kHz EnCodec decoder (4 x 2048, n_filters 64, LSTM 2), seeded random weights"),
           "edit": edit}
    if args.queue:
        out["queue"] = queue(args, cfg, model, _lib, ContinuousBatcher, synthetic, dev)
    out["clocks"] = clocks.stop()
    out["gpu"] = gpu_identity(0)
    out["note"] = ("wall clock from the call's start, median of %d alternating calls per arm after one untimed warm-up of "
                   "each; batch arm: first audio = all audio; queue sampler_ms_per_step from one profiled call per arm"
                   % max(1, args.repeats))
    print(json.dumps(out))


def queue(args, cfg, model, _lib, ContinuousBatcher, synthetic, dev):
    N, lib = args.queue, _lib.load()
    tickets = []
    for i in range(N):
        x, _, y = synthetic.synthetic_utterance(cfg, 300 + i, 40, 150)
        tickets.append((x.to(dev), y.to(dev), torch.tensor([[[60, 100]]]) if i % 2 else None, 7 + i,
                        QUEUE_PARAMS[i % len(QUEUE_PARAMS)]))

    def serve(per_ticket, profile=False):
        cb = ContinuousBatcher(model, max_concurrency=args.slots, poll_every=args.poll_every, **QUEUE_PARAMS[0])
        for x, y, mi, seed, params in tickets:
            cb.submit(x, y, seed=seed, mask_interval=mi, **(params if per_ticket else {}))
        eng = model._engine()
        ms, cnt = (C.c_double * 7)(), (C.c_int64 * 7)()
        if profile:
            _lib.check(lib.vcb_set_option(eng, b"profile", 1))
            lib.vcb_profile_read(eng, ms, cnt, 7)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        cb.run()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        steps = cb.stats["steps"]
        if profile:
            _lib.check(lib.vcb_profile_read(eng, ms, cnt, 7))
            _lib.check(lib.vcb_set_option(eng, b"profile", 0))
            return ms[4] / steps
        return dt * 1e3 / steps, steps

    serve(True), serve(False)
    runs = {"per_ticket": [], "shared": []}
    for _ in range(max(1, args.repeats)):
        runs["per_ticket"].append(serve(True))
        runs["shared"].append(serve(False))
    arms = {}
    for name, rs in runs.items():
        r = median_call(rs, lambda v: v[0])
        arms[name] = {"ms_per_step": r[0], "steps": r[1], "ms_per_step_all": [v[0] for v in rs],
                      "sampler_ms_per_step": serve(name == "per_ticket", profile=True)}
    return dict(arms, tickets=N, slots=args.slots, tts_tickets=(N + 1) // 2, edit_span=[60, 100], text_len=40,
                prompt_frames=150)


if __name__ == "__main__":
    main()
