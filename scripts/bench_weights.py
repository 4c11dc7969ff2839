"""bf16 against int8 GEMM weights at bench.py's 830M TTS workload (text 80, 150-frame prompts), the timed window centred on
the mean context as bench.py (and scripts/bench_kv.py) centre it, under both KV policies.  For each batch size, KV policy
and weight policy, alternating the weight policies in every round, one JSON line with
  step_ms, tokens_per_s      device time of --steps decode steps (events), codec tokens / s
  gemm_ms_per_step           decode GEMMs (profile class 0) per step, from a separate profile-mode pass after the window
  weight_gbs                 weight bytes the decode GEMMs stream per step (weight_bytes without the prefill scratch and the
                             scales) / gemm_ms_per_step
  prefill_ms                 host time of the session's prefill of the B prompts, ending in a device synchronise
  weight_bytes               vcb_counter after the prefill (int8: the prefill scratch included)
Then the split sweep (--sweep): the int8 engine with every decode GEMM of the layers at one split count (VCB_SPLITS),
beside the bf16 rule's pick per shape (vcb_gemm_launch_shape).  First and last a line with the card name, power limit and
SM clocks.

  python scripts/bench_weights.py --batches 32 64 --rounds 2 --sweep
Needs a GPU; no fall-back."""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_kv import card  # noqa: E402


def run(model, cfg, B, kv, wd, args):
    import torch
    import bench
    from voicecraft_b200 import _lib
    lib = _lib.load()
    text_len, prompt = 80, 150
    cap = text_len * (cfg.encodec_sr // 5)
    S_total = cap - (prompt + 1) - 2
    start = max(args.warmup, (S_total - args.steps) // 2)
    max_seq_len = (text_len + cap + 64 + 255) // 256 * 256
    model.configure_engine(max_slots=B, max_seq_len=max_seq_len, kv_dtype=kv, weight_dtype=wd, max_new_tokens=cap + 64)
    model._engine()
    a = argparse.Namespace(text_len=text_len, prompt=prompt)
    utts = bench.make_utterances(a, cfg, range(B))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sess = model.open_tts_session([u[0].cuda() for u in utts], [u[2].cuda() for u in utts], seeds=[1 + i for i in range(B)],
                                  top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
    torch.cuda.synchronize()
    prefill_ms = (time.perf_counter() - t0) * 1e3
    try:
        eng = sess.eng
        sess.sample()
        for _ in range(start):
            sess.step()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(args.steps):
            sess.step()
        ev1.record()
        torch.cuda.synchronize()
        ms = ev0.elapsed_time(ev1) / args.steps
        nprof = 8
        msb, cnt = bench.profile_pass(lib, eng, sess, nprof)
        wb = lib.vcb_counter(eng, b"weight_bytes")
        d, F, Hh = cfg.d_model, 4 * cfg.d_model, int(cfg.audio_vocab_size) // 2
        V = int(cfg.audio_vocab_size) + cfg.n_special
        K = cfg.n_codebooks
        elems = cfg.num_decoder_layers * (3 * d * d + d * d + 2 * F * d) + K * Hh * d + K * ((V + 127) // 128 * 128) * Hh
        streamed = elems * (1 if wd == "int8" else 2)
        gemm_ms = msb[0] / nprof
        return dict(weights=wd, kv=kv, B=B, steps=args.steps, step_ms=ms, tokens_per_s=B * cfg.n_codebooks / (ms * 1e-3),
                    gemm_ms_per_step=gemm_ms, gemm_launches_per_step=cnt[0] / nprof, weight_bytes_streamed=streamed,
                    weight_gbs=streamed / (gemm_ms * 1e-3) / 1e9, prefill_ms=prefill_ms, weight_bytes=wb)
    finally:
        sess.close()


def decode_shapes(cfg):
    d = cfg.d_model
    return [(3 * d, d), (d, d), (4 * d, d), (d, 4 * d)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--kv", nargs="+", default=["bf16", "fp8"])
    ap.add_argument("--sweep", action="store_true", help="int8 split sweep of the layer GEMMs (VCB_SPLITS), KV bf16")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_weights needs a GPU")
    import bench
    from voicecraft_b200 import _lib
    from voicecraft_b200.voicecraft import VoiceCraft
    lib = _lib.load()
    print(json.dumps({"card": card()}), flush=True)
    cfg, sd = bench.make_model(argparse.Namespace(model="830M", codebooks=4))
    model = VoiceCraft(cfg)
    model.load_state_dict(sd)
    model = model.cuda().eval()
    for r in range(args.rounds):
        for B in args.batches:
            for kv in args.kv:
                for wd in (("bf16", "int8") if r % 2 == 0 else ("int8", "bf16")):
                    print(json.dumps(dict(run(model, cfg, B, kv, wd, args), round=r)), flush=True)
    if args.sweep:
        for B in args.batches:
            pick = {}
            for N, K in decode_shapes(cfg):
                out = (C.c_int32 * 2)()
                _lib.check(lib.vcb_gemm_launch_shape(N, K, B, 0, 0, 0, out))
                pick[f"{N}x{K}"] = out[0]
            for s in (1, 2, 4, 8, 16):
                os.environ["VCB_SPLITS"] = ",".join(f"{N}x{K}:{s}" for N, K in decode_shapes(cfg))
                model._drop_engine()
                try:
                    res = run(model, cfg, B, "bf16", "int8", args)
                except _lib.VcbError as exc:
                    res = dict(B=B, error=str(exc))
                print(json.dumps(dict(res, sweep_splits=s, bf16_rule=pick)), flush=True)
            os.environ.pop("VCB_SPLITS", None)
            model._drop_engine()
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
