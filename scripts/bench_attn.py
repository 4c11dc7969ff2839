"""Decode attention with and without its early start (VCB_ATT_EARLY, DESIGN.md section 7) at bench.py's 830M TTS workload
(text 80, 150-frame prompts, bf16 KV).  For each batch size, one generation per knob setting, the settings alternating in
every round; in each generation three windows (early, middle and late contexts), each with
  step_ms              device time of --steps decode steps (events; the launches overlap under PDL as in bench.py)
  attn_ms_per_step     attention (profile class 1) per step from a profile-mode pass of 8 steps after the window; that pass
                       serialises launches, so it holds the copy and compute time, not the overlap with the QKV GEMM
  attn_bytes_per_step  K / V bytes the TMA copies per step at the profiled contexts, computed from shapes: whole 64-token
                       slabs with the knob at 0, the live tokens of the last page with it at 1
Then per knob a least-squares line attn_ms = fixed + bytes / rate over all its windows (the fixed cost per step and per
launch, the marginal rate), and finally --bench-runs runs of bench.py with the knob at 0 and at 1, alternating.
The first line and the last line give the card name, power limit and SM clocks.

  python scripts/bench_attn.py --batches 16 32 64 --rounds 1 --bench-runs 3
Needs a GPU; no fall-back."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TEXT_LEN, PROMPT = 80, 150


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [s.strip() for s in out.stdout.splitlines()[0].split(",")])) if out.returncode == 0 else {}


def copied_bytes(per_tok, positions, early):
    """K / V bytes the attention copies for rows at these positions (one layer's share times the layers is in per_tok)"""
    if early:
        return sum(per_tok * (p + 1) for p in positions)
    return sum(per_tok * 64 * (p // 64 + 1) for p in positions)


def run(model, cfg, B, early, args):
    import torch
    import bench
    from voicecraft_b200 import _lib
    lib = _lib.load()
    cap = TEXT_LEN * (cfg.encodec_sr // 5)
    S_total = cap - (PROMPT + 1) - 2
    nprof = 8
    starts = [args.warmup, (S_total - args.steps) // 2, S_total - args.steps - nprof - 12]
    os.environ["VCB_ATT_EARLY"] = str(int(early))
    model.configure_engine(max_slots=B, max_seq_len=(TEXT_LEN + cap + 64 + 255) // 256 * 256, kv_dtype="bf16",
                           max_new_tokens=cap + 64)
    a = argparse.Namespace(text_len=TEXT_LEN, prompt=PROMPT)
    utts = bench.make_utterances(a, cfg, range(B))
    sess = model.open_tts_session([u[0].cuda() for u in utts], [u[2].cuda() for u in utts], seeds=[1 + i for i in range(B)],
                                  top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
    out = []
    try:
        eng = sess.eng
        got = lib.vcb_counter(eng, b"att_early")
        if got != int(early):
            raise SystemExit(f"VCB_ATT_EARLY={int(early)}: the engine runs {got}")
        per_tok = lib.vcb_counter(eng, b"kv_bytes_per_token")
        sess.sample()
        done = 0                                                       # decode steps so far
        for start in starts:
            for _ in range(start - done):
                sess.step()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for _ in range(args.steps):
                sess.step()
            ev1.record()
            torch.cuda.synchronize()
            ms = ev0.elapsed_time(ev1) / args.steps
            ctx = TEXT_LEN + PROMPT + 1 + start + args.steps          # context of the first profiled step
            msb, cnt = bench.profile_pass(lib, eng, sess, nprof)
            done = start + args.steps + nprof
            attn_bytes = B * copied_bytes(per_tok, [ctx + s for s in range(nprof)], early) / nprof
            out.append(dict(early=int(early), B=B, ctx_window=[TEXT_LEN + PROMPT + 1 + start, ctx], step_ms=ms,
                            attn_ms_per_step=msb[1] / nprof, attn_launches_per_step=cnt[1] / nprof,
                            attn_bytes_per_step=attn_bytes))
    finally:
        sess.close()
    return out


def fit(points):
    """least squares attn_ms = fixed + bytes * slope: fixed ms per step, marginal TB/s"""
    import numpy as np
    x = np.array([p["attn_bytes_per_step"] for p in points])
    y = np.array([p["attn_ms_per_step"] for p in points])
    slope, fixed = np.polyfit(x, y, 1)
    launches = points[0]["attn_launches_per_step"]
    return dict(fixed_ms_per_step=float(fixed), fixed_us_per_launch=float(fixed) * 1e3 / launches,
                marginal_tbs=float(1.0 / slope / 1e9) if slope > 0 else None, points=len(points))


def bench_runs(args):
    res = {0: [], 1: []}
    for r in range(args.bench_runs):
        for early in ((0, 1) if r % 2 == 0 else (1, 0)):
            env = dict(os.environ, VCB_ATT_EARLY=str(early))
            cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "100", "--warmup", "10",
                   "--no-cpu", "--no-e2e"] + (["--batch", str(args.bench_batch)] if args.bench_batch else [])
            p = subprocess.run(cmd, env=env, capture_output=True, text=True)
            lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
            if p.returncode != 0 or not lines:
                raise SystemExit(f"bench.py failed ({p.returncode}): {p.stderr[-2000:]}")
            d = json.loads(lines[-1])
            res[early].append(d["ms_per_step"])
            print(json.dumps(dict(bench_py=True, early=early, run=r, ms_per_step=d["ms_per_step"], clocks=d.get("clocks"))),
                  flush=True)
    print(json.dumps(dict(bench_py_summary={k: dict(min=min(v), max=max(v), all=v) for k, v in res.items()})), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[16, 32, 64])
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--bench-runs", type=int, default=3, help="bench.py runs per knob setting (0: none)")
    ap.add_argument("--bench-batch", type=int, default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_attn needs a GPU")
    import bench
    from voicecraft_b200.voicecraft import VoiceCraft
    print(json.dumps({"card": card()}), flush=True)
    cfg, sd = bench.make_model(argparse.Namespace(model="830M", codebooks=4))
    model = VoiceCraft(cfg)
    model.load_state_dict(sd)
    model = model.cuda().eval()
    pts = {0: [], 1: []}
    for r in range(args.rounds):
        for B in args.batches:
            for early in ((1, 0) if r % 2 == 0 else (0, 1)):
                for p in run(model, cfg, B, early, args):
                    pts[early].append(p)
                    print(json.dumps(dict(p, round=r)), flush=True)
    print(json.dumps({"fit": {f"early={k}": fit(v) for k, v in pts.items()}}), flush=True)
    del model
    torch.cuda.empty_cache()
    if args.bench_runs > 0:
        bench_runs(args)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
