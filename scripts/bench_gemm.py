"""Micro-benchmark of the wgmma GEMM kernel over the 830M decode shapes (run on the GPU box)."""
import ctypes as C
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from voicecraft_b200 import _lib
lib = _lib.load()
torch.zeros(1, device="cuda")
shapes = [("qkv", 6144, 2048), ("out", 2048, 2048), ("ff1", 8192, 2048), ("ff2", 2048, 8192), ("h1", 4096, 2048), ("h2", 2052, 1024)]
B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
for name, N, K in shapes:
    mb = N * K * 2 / 1e6
    ncop = max(2, int(400 / mb) + 1)
    for stages in (3, 4, 6, 8):
        for pdl in (0, 1):
            row = []
            for s in (1, 2, 4, 8):
                us = C.c_float()
                rc = lib.vcb_bench_gemm(N, K, B, s, stages, pdl, 200, ncop, C.byref(us))
                row.append(f"S={s}:{us.value:6.1f}us({mb / us.value * 1e3:5.0f}GB/s)" if rc == 0 else f"S={s}: err")
            print(f"{name:4s} N={N} K={K} B={B} stages={stages} pdl={pdl} " + "  ".join(row), flush=True)
