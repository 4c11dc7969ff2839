"""The decode GEMM at 16 K splits (a non-portable cluster of 16 CTAs), and the launcher's split validation and fallback.

  * -m gpu: vcb_debug_gemm and vcb_debug_fold_chain at split 16 against the same fp64 references and bounds as
    test_gpu_parity / test_kernel_numerics, for every row padding and K where 16 splits are legal.
  * -m gpu: where the device cannot place a cluster of 16, the launch falls back to the largest cluster it can
    (vcb_gemm_launch_shape with a cap stands in for the occupancy API's answer: the launcher takes the same path).
  * no GPU: split counts the reduce-scatter cannot run are rejected before anything is launched.
"""
import ctypes as C

import pytest
import torch

from test_kernel_numerics import CLASSES, PREFILL_BOUND, _bpad, _fold_bound, _fold_ref, _fold_rows, _fold_run, _fold_weights


def _lib():
    from voicecraft_b200 import _lib
    return _lib, _lib.load()


def _shape(N, K, B, splits, stages=0, cap=0):
    """(splits, stages) the launcher would use, or None where it rejects the call"""
    _, lib = _lib()
    out = (C.c_int32 * 2)()
    if lib.vcb_gemm_launch_shape(N, K, B, splits, stages, cap, out) != 0:
        return None
    return out[0], out[1]


def _split16_legal(B, K):
    bpad, kb = _bpad(B), K // 64
    return bpad // 16 >= 2 and 15 * ((kb + 15) // 16) < kb


@pytest.mark.parametrize("N,K,B,splits", [
    (2048, 2048, 32, 32),      # more than 16
    (2048, 2048, 32, 12),      # not a power of two
    (2048, 2048, 32, 3),
    (2048, 2048, 16, 16),      # one token row per CTA (the reduce-scatter sends pairs of rows)
    (2048, 2048, 5, 16),
    (2048, 512, 32, 16),       # 8 k-blocks: splits past the last k-block
    (2048, 1088, 32, 16),      # 17 k-blocks: 2 per split leaves the 16th without one
    (2048, 100, 32, 1),        # K not a multiple of 64
])
def test_launcher_rejects_illegal_splits(N, K, B, splits):
    _, lib = _lib()
    assert _shape(N, K, B, splits) is None
    assert b"gemm:" in lib.vcb_last_error()


@pytest.mark.gpu
def test_one_pipeline_depth_per_row_padding():
    """gemm_stages: 4 stages, 3 where 4 do not fit into shared memory (bpad 128); no other depth is built"""
    _, lib = _lib()
    for B, stages in ((16, 4), (32, 4), (64, 4), (128, 3)):
        assert _shape(2048, 2048, B, 4) == (4, stages)
        assert _shape(2048, 2048, B, 4, stages=stages) == (4, stages)
        assert _shape(2048, 2048, B, 4, stages=stages - 1) is None
        assert b"no kernel" in lib.vcb_last_error()


@pytest.mark.gpu
@pytest.mark.parametrize("B", [20, 32, 64, 128])
def test_split16_falls_back_to_the_largest_placeable_cluster(B):
    assert _shape(2048, 2048, B, 16) is not None and _shape(2048, 2048, B, 16)[0] == 16, "H100: 16 must be placeable"
    for cap, want in ((8, 8), (4, 4), (2, 2), (1, 1), (16, 16), (32, 16)):
        s = _shape(2048, 2048, B, 16, cap=cap)
        assert s is not None and s[0] == want, (cap, s)
    assert _shape(2048, 2048, B, 4, cap=8)[0] == 4          # a cap above the split count changes nothing


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(2048, 2048, 32), (2048, 8192, 32), (6144, 2048, 20), (2052, 1024, 32), (768, 1024, 64),
                                   (256, 4096, 128), (1000, 3072, 48)])
def test_gemm_split16_vs_fp64(shape):
    """vcb_debug_gemm at 16 splits against fp64 W x^T, with test_gpu_parity's bound"""
    _l, lib = _lib()
    N, K, B = shape
    assert _split16_legal(B, K)
    assert _shape(N, K, B, 16) == (16, _shape(N, K, B, 4)[1]), "the launch must run 16 CTAs per cluster"
    g = torch.Generator(device="cpu").manual_seed(N + K + B + 16)
    W = torch.randn(N, K, generator=g).to(torch.bfloat16).float().cuda()
    X = torch.randn(B, K, generator=g).cuda()
    ref = X.double() @ W.double().t()
    out = torch.zeros(B, N, device="cuda")
    _l.check(lib.vcb_debug_gemm(W.data_ptr(), X.data_ptr(), out.data_ptr(), N, K, B, 16, 0))
    torch.cuda.synchronize()
    scale = ref.abs().max().item()
    err = (out.double() - ref).abs().max().item()
    assert err <= 2e-4 * max(scale, 1.0), f"shape={shape} err={err} scale={scale}"


@pytest.mark.gpu
@pytest.mark.parametrize("d", [1024, 2048, 4096])
@pytest.mark.parametrize("B", [20, 32, 48, 64, 128])
def test_folded_layernorm_split16_vs_fp64(B, d):
    """vcb_debug_fold_chain with both GEMMs at 16 splits, rows of every mean / std class, fold = 1 and 0: the bounds of
    test_kernel_numerics.test_folded_layernorm_vs_fp64"""
    assert _split16_legal(B, d) and _shape(d, d, B, 16)[0] == 16
    w = _fold_weights(d)
    bad = []
    x, a, cls = _fold_rows(B, d, 0, seed=B * 7919 + d + 16)
    for relu in (0, 1):
        xr, yr = _fold_ref(w, x, a, relu)
        for fold in (1, 0):
            xn, y = _fold_run(w, x, a, B, d, relu, fold, 16, 16)
            xerr = float((xn.double() - xr).abs().max() / xr.abs().max())
            if xerr > 2e-5:
                bad.append(f"x_new fold={fold}: {xerr:.3g}")
            for c in set(cls):
                rows = [i for i, ci in enumerate(cls) if ci == c]
                err = float((y[rows].double() - yr[rows]).abs().max() / yr[rows].abs().max())
                if err > (_fold_bound(c, d) if fold else PREFILL_BOUND):
                    bad.append(f"y fold={fold} mean/std={c} relu={relu}: {err:.3g}")
    assert not bad, bad
