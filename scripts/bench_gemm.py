"""Sweep of the decode GEMM (gemm_w_xT_cluster) over the split count at the 830M decode shapes.

Each point is vcb_bench_gemm: `iters` launches of one shape back to back on one stream, PDL on, so every launch has the
previous launch of the same chain as its predecessor, as in a decode step; the weights rotate over enough copies that
they stream from HBM.  The median of --repeats such runs is reported, with the weight bytes over that time.
The shape that was launched is read back through vcb_gemm_launch_shape (a cluster the device cannot place falls back
to a smaller one); points the launcher rejects are left out.  The card, its power limit and its SM clock are recorded
beside the numbers.  The pipeline depth is the one the kernel for the batch's row padding is built with (gemm_stages);
the table in DESIGN.md section 4.1 also covers depths 2 / 3 / 6 / 8, timed the same way on a build that instantiated them.

    python scripts/bench_gemm.py [--batch 32 64 128] [--out sweep.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = [("qkv", 6144, 2048), ("out", 2048, 2048), ("ff1", 8192, 2048), ("ff2", 2048, 8192), ("h1", 4096, 2048),
          ("h2", 2052, 1024)]       # h2: one codebook's second head (the step launches the four as one grouped launch)
SPLITS = (1, 2, 4, 8, 16)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[32, 64, 128])
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from voicecraft_b200 import _lib
    lib = _lib.load()
    torch.zeros(1, device="cuda")
    info = gpu_info()
    print("# " + info, flush=True)
    rows = []
    for B in args.batch:
        for name, N, K in SHAPES:
            mb = N * K * 2 / 1e6
            ncop = max(2, int(400 / mb) + 1)
            rule = (C.c_int32 * 2)()
            _lib.check(lib.vcb_gemm_launch_shape(N, K, B, 0, 0, 0, rule))
            line = []
            for s in SPLITS:
                shape = (C.c_int32 * 2)()
                if lib.vcb_gemm_launch_shape(N, K, B, s, 0, 0, shape) != 0:
                    continue
                ts = []
                for _ in range(args.repeats):
                    us = C.c_float()
                    _lib.check(lib.vcb_bench_gemm(N, K, B, s, 0, 1, args.iters, ncop, C.byref(us)))
                    ts.append(us.value)
                us = sorted(ts)[len(ts) // 2]
                rows.append(dict(B=B, gemm=name, N=N, K=K, splits=shape[0], stages=shape[1], asked_splits=s,
                                 us=us, us_all=ts, gbs=mb / us * 1e3, rule=shape[0] == rule[0]))
                line.append(f"S={shape[0]:2d}:{us:6.2f}us{'*' if rows[-1]['rule'] else ' '}")
            print(f"B={B:3d} {name:4s} {N}x{K} stages={rule[1]}  " + "  ".join(line), flush=True)
    print("# * = the split count the engine picks (gemm_pick_splits)")
    print("# " + gpu_info(), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"gpu_before": info, "gpu_after": gpu_info(), "points": rows}, f, indent=1)


if __name__ == "__main__":
    main()
