"""The fp8 KV policy (kv_dtype="fp8", DESIGN.md sections 2.2 and 3): e4m3 K / V with a power-of-two fp32 scale per token and
head, written by both QKV epilogues and read by the paged attention.

CPU: the torch restatement of the quantizer against bytes written out by hand, and the rejection of unknown policies.
GPU (-m gpu): the device quantizer and both epilogues bit-exact against it, the attention against fp64 over the dequantized
pools and bit-reproducible, best-of-N forks, batch independence, token parity with the CPU oracle under the same policy,
the pool bytes, and the paths fp8 does not take (persistent step kernel, CUDA-core GEMM)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import golden_util as gu
from kv_fp8_ref import OracleLMFp8, dequantize_kv_fp8, quantize_kv_fp8, split_slabs, to_slabs

ULP_ABOVE_448 = float(np.nextafter(np.float32(448.0), np.float32(np.inf)))
TINY = 2.0 ** -126                                   # smallest normal fp32

# (row, e4m3 bytes, scale) written out by hand.  e4m3fn: sign, 4 exponent bits (bias 7), 3 mantissa bits; 448 = 0x7e,
# 1.0 = 0x38, 2.0 = 0x40, 0.5 = 0x30, 224 = 0x76; subnormals k * 2^-9 = k for k < 8.
HAND = [
    ([448.0, 1.0, -2.0, 0.0], [0x7E, 0x38, 0xC0, 0x00], 1.0),                       # amax exactly 448 * 2^0
    ([ULP_ABOVE_448, 1.0, -0.0, 0.0], [0x76, 0x30, 0x80, 0x00], 2.0),               # one ulp above: e = 1, 224 and 0.5
    ([896.0, -3.0, 0.0, 0.0], [0x7E, 0xBC, 0x00, 0x00], 2.0),                       # 896 = 448 * 2; -1.5 = 0xbc
    ([0.0, 0.0, 0.0, 0.0], [0x00] * 4, TINY),                                       # all zero: e = -126
    ([-0.0, -1e-10, 448.0, -0.0], [0x80, 0x80, 0x7E, 0x80], 1.0),                    # -0 and a negative underflow keep the sign
    ([448.0, 2.0 ** -9, 3 * 2.0 ** -9, 2.0 ** -10], [0x7E, 0x01, 0x03, 0x00], 1.0),  # subnormals; half the smallest -> 0 (even)
    ([448.0, 1.5 * 2.0 ** -9, 2.5 * 2.0 ** -9, -7 * 2.0 ** -9], [0x7E, 0x02, 0x02, 0x87], 1.0),   # ties to even
    ([TINY, 0.0, -TINY, 0.5 * TINY], [0x38, 0x00, 0xB8, 0x30], TINY),               # amax 2^-126: e clamped to -126
    ([448 * TINY, 0.0, 0.0, 0.0], [0x7E, 0x00, 0x00, 0x00], TINY),                  # exactly 448 * 2^-126
    ([449 * TINY, 0.0, 0.0, 0.0], [0x76, 0x00, 0x00, 0x00], 2 * TINY),              # 224.5 -> 224 at e = -125
    ([1e-45, 0.0, 0.0, 0.0], [0x00, 0x00, 0x00, 0x00], TINY),                       # fp32 subnormal amax
]


def _hand_rows(hd):
    """the hand rows padded with zeros to hd values (padding does not change amax)"""
    x = torch.zeros(len(HAND), hd)
    for i, (row, _, _) in enumerate(HAND):
        x[i, :4] = torch.tensor(row, dtype=torch.float32)
    return x


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_quantizer_matches_hand_written_bytes():
    x = _hand_rows(8)
    q, s = quantize_kv_fp8(x)
    for i, (row, want, scale) in enumerate(HAND):
        got = q[i, :4].view(torch.uint8).tolist()
        assert got == want, f"row {row}: bytes {[hex(b) for b in got]} != {[hex(b) for b in want]}"
        assert float(s[i]) == scale, f"row {row}: scale {float(s[i])!r} != {scale!r}"
        assert q[i, 4:].view(torch.uint8).tolist() == [0] * 4
    # dequantization is exact: q * 2^e reproduces every value e4m3 can hold at that scale
    assert torch.equal(dequantize_kv_fp8(q, s)[0, :4], torch.tensor([448.0, 1.0, -2.0, 0.0]))


def test_quantizer_relative_error_and_scale_rule():
    g = torch.Generator().manual_seed(5)
    x = torch.randn(512, 128, generator=g) * torch.logspace(-30, 30, 512).unsqueeze(1)
    q, s = quantize_kv_fp8(x)
    amax = x.abs().amax(-1)
    assert torch.all(amax <= 448 * s) and torch.all(amax > 224 * s)          # e is the smallest that fits
    err = (dequantize_kv_fp8(q, s) - x).abs()
    assert torch.all(err <= 2.0 ** -4 * x.abs() + 2.0 ** -10 * s[:, None])    # half an ulp of 3 mantissa bits, or subnormal


def test_fp8_oracle_restates_oracle_attention():
    """OracleLMFp8 restates OracleLM._mha with a storage step; with that step the identity it must compute exactly what
    the oracle computes (a change to the oracle's attention that the restatement misses fails here)"""
    from oracle import lm_oracle
    from voicecraft_b200 import synthetic
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=12)
    x, xl, y = synthetic.synthetic_utterance(cfg, 5, text_len=5, prompt_frames=9)
    kw = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3, silence_tokens=gu.SILENCE, max_steps=6,
              trace_logits=True)
    a = lm_oracle.OracleLM(cfg, sd)
    b = OracleLMFp8(cfg, sd)
    b.store_kv = lambda t: t
    ra = a.inference_tts(x, xl, y, noise_fn=gu.cpu_noise_fn(3), **kw)
    rb = b.inference_tts(x, xl, y, noise_fn=gu.cpu_noise_fn(3), **kw)
    assert torch.equal(ra, rb)
    assert all(torch.equal(p, q) for p, q in zip(a.logit_trace, b.logit_trace)) and len(a.logit_trace) == 6


def test_configure_engine_rejects_unknown_kv_dtype():
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    m = VoiceCraft(synthetic.make_config("tiny"))
    with pytest.raises(ValueError):
        m.configure_engine(kv_dtype="fp16")
    m.configure_engine(kv_dtype="fp8")
    assert m._eng_opts["kv_dtype"] == "fp8"


def _config(kv_dtype):
    from voicecraft_b200 import _lib
    return _lib.vcb_config(d_model=256, nhead=2, num_layers=1, n_codebooks=4, audio_vocab_size=2048, n_special=4,
                           text_vocab_rows=101, empty_token=2048, eog=2049, audio_pad_token=2050, eos=2051, encodec_sr=50,
                           max_n_spans=3, max_slots=1, max_seq_len=256, max_new_tokens=64, kv_dtype=kv_dtype)


def test_create_rejects_unknown_kv_dtype():
    """checked before the device is touched, so this holds on any machine"""
    from voicecraft_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    for bad in (3, -1):
        assert lib.vcb_create(C.byref(_config(bad)), C.byref(h)) != 0
        assert b"kv_dtype" in lib.vcb_last_error()


def test_create_rejects_simt_gemm_with_fp8(monkeypatch):
    from voicecraft_b200 import _lib
    lib = _lib.load()
    monkeypatch.setenv("VCB_GEMM_IMPL", "simt")
    h = C.c_void_p()
    assert lib.vcb_create(C.byref(_config(2)), C.byref(h)) != 0
    assert b"simt" in lib.vcb_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _lib():
    from voicecraft_b200 import _lib
    return _lib, _lib.load()


def _device_quantize(x):
    _l, lib = _lib()
    rows, hd = x.shape
    xd = x.contiguous().cuda()
    out = torch.zeros(rows * hd + 4 * rows, dtype=torch.uint8, device="cuda")
    _l.check(lib.vcb_debug_kv_quantize(xd.data_ptr(), rows, hd, out.data_ptr()))
    out = out.cpu()
    return out[:rows * hd].reshape(rows, hd), out[rows * hd:].view(torch.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("hd", [64, 128])
def test_device_quantizer_is_bit_exact(hd):
    g = torch.Generator().manual_seed(hd)
    rand = torch.randn(300, hd, generator=g) * torch.logspace(-40, 35, 300).unsqueeze(1)
    spiky = torch.randn(64, hd, generator=g) * 1e-3
    spiky[torch.arange(64), torch.randint(0, hd, (64,), generator=g)] = 1e3      # one large value per row
    for x in (_hand_rows(hd), rand, spiky):
        q, s = quantize_kv_fp8(x)
        bq, bs = _device_quantize(x)
        assert torch.equal(bq, q.view(torch.uint8)), f"{int((bq != q.view(torch.uint8)).sum())} bytes differ"
        assert torch.equal(bs.view(torch.int32), s.view(torch.int32)), "scales differ"


def _model(kv, nhead=2, max_slots=8, seed=3, **over):
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny", nhead=nhead, **over)
    sd = synthetic.make_state_dict(cfg, seed=seed)
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    m = m.to("cuda").eval()
    m.configure_engine(kv_dtype=kv, max_slots=max_slots, max_seq_len=512)
    return cfg, sd, m


def _layer0_pages(m, cfg, prompts):
    """prefill the prompts (one slot each) and read every slot's layer-0 slabs"""
    from voicecraft_b200.voicecraft import DecodeSession
    _l, lib = _lib()
    sp = m._sampling(silence_tokens=(1388, 1898, 131), top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
    sess = DecodeSession(m, [p[0] for p in prompts], [p[1] for p in prompts], sp)
    H, hd = cfg.nhead, cfg.d_model // cfg.nhead
    slab = 64 * hd * 4 if m._eng_opts["kv_dtype"] == "fp32" else 64 * (hd + 4)
    out = []
    try:
        for slot, (_, _, total) in zip(sess.slots, prompts):
            n = (total + 63) // 64
            k = np.zeros(n * H * slab, np.uint8)
            v = np.zeros_like(k)
            _l.check(lib.vcb_debug_kv_pages(sess.eng, 0, slot, 0, n, k.ctypes.data, v.ctypes.data))
            out.append((torch.from_numpy(k), torch.from_numpy(v), total))
    finally:
        sess.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("wide", ["1", "0"])
@pytest.mark.parametrize("nhead", [2, 4])
def test_epilogues_write_quantized_layer0_kv(nhead, wide, monkeypatch):
    """Layer 0's K / V do not depend on the cache: an fp8 engine's layer-0 slabs are quantize_kv_fp8 of an fp32 engine's
    layer-0 values, byte for byte, scales included.  Wide prefill (rows-as-M GEMM) and the decode GEMM's epilogue
    (VCB_PREFILL_WIDE=0); head dims 128 and 64; prompts ending mid-page and on a page boundary."""
    from test_best_of import _utt
    monkeypatch.setenv("VCB_PREFILL_WIDE", wide)
    cfg, sd, m32 = _model("fp32", nhead=nhead)
    H, hd = cfg.nhead, cfg.d_model // cfg.nhead
    prompts = [(*_utt(cfg, 70 + i, total)[::2], total) for i, total in enumerate((100, 128, 77, 191))]
    ref = _layer0_pages(m32, cfg, prompts)
    del m32
    m8 = _model("fp8", nhead=nhead)[2]
    _assert_quantized(ref, _layer0_pages(m8, cfg, prompts), H, hd)


SHAPES = {"hd128": dict(nhead=2), "hd64": dict(nhead=4), "hd64_straddle": dict(nhead=3, d_model=192, audio_embedding_dim=192)}


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
def test_decode_gemm_epilogue_at_every_row_padding(shape, monkeypatch):
    """The decode GEMM's fp8 QKV epilogue at every row padding it is built for: prompts of 12, 30, 60 and 200 positions
    through the decode GEMM (VCB_PREFILL_WIDE=0), one prompt per prefill, run in passes of 12, 30, 60, 128 + 72 rows, i.e.
    bpad 16, 32, 64 and 128 (the four KV8 instantiations; decode steps at B = 32 and 64 take the bpad 32 and 64 ones).
    Layer-0 slabs byte-identical to quantize_kv_fp8 of an fp32 engine's.  "hd64_straddle" (d = 192, three heads of 64):
    a 128-feature tile spans the Q | K boundary, and the last tile has 64 valid features (the rows-as-M prefill does not
    take this width, so every prompt goes through the decode GEMM)."""
    from voicecraft_b200 import synthetic
    monkeypatch.setenv("VCB_PREFILL_WIDE", "0")
    over = SHAPES[shape]
    cfg, _, m32 = _model("fp32", **over)
    H, hd = cfg.nhead, cfg.d_model // cfg.nhead
    prompts = []
    for i, total in enumerate((12, 30, 60, 200)):
        x, _, y = synthetic.synthetic_utterance(cfg, 90 + i, text_len=6, prompt_frames=total - 7)
        prompts.append((x.cuda(), y.cuda(), total))
    ref = [_layer0_pages(m32, cfg, [p])[0] for p in prompts]
    del m32
    m8 = _model("fp8", **over)[2]
    _assert_quantized(ref, [_layer0_pages(m8, cfg, [p])[0] for p in prompts], H, hd)


def _assert_quantized(ref, got, H, hd):
    """fp8 slabs `got` are quantize_kv_fp8 of the fp32 slabs `ref`, over each prompt's positions"""
    for (k32, v32, total), (k8, v8, _) in zip(ref, got):
        for a32, a8, what in ((k32, k8, "K"), (v32, v8, "V")):
            x = a32.view(torch.float32).reshape(-1, H, 64, hd).transpose(1, 2).reshape(-1, H, hd)[:total]
            q, s = quantize_kv_fp8(x)
            gq, gs = split_slabs(a8, H, hd)
            gq = gq.transpose(1, 2).reshape(-1, H, hd)[:total]
            gs = gs.transpose(1, 2).reshape(-1, H)[:total]
            assert torch.equal(gq, q.view(torch.uint8)), f"{what}, {total} positions: {int((gq != q.view(torch.uint8)).sum())} bytes differ"
            assert torch.equal(gs, s), f"{what}, {total} positions: scales differ"


def _fp8_case(c):
    """an attention case of test_kernel_numerics with its pools as fp8 slabs; Kp / Vp become the dequantized pools"""
    ks, kd = to_slabs(c["Kp"].float())
    vs, vd = to_slabs(c["Vp"].float())
    return dict(c, Kp=kd, Vp=vd, Ks=ks, Vs=vs)


def _attn_fp8(c, chunk_pages, via="row_pages", balance=1, repeats=1, rows=None):
    _l, lib = _lib()
    sel = torch.arange(len(c["pos"])) if rows is None else torch.as_tensor(rows)
    q = c["q"][sel].contiguous().cuda()
    pos = c["pos"][sel].contiguous().cuda()
    slot = c["row_slot"][sel].contiguous().cuda()
    pt = c["page_table"].contiguous().cuda()
    rp = pt[slot.long()].contiguous()
    Ks, Vs = c["Ks"].cuda(), c["Vs"].cuda()
    n, H, hd = len(sel), c["H"], c["hd"]
    out = torch.full((n, H * hd), 12345.0, device="cuda")
    args = (rp.data_ptr(), None, None) if via == "row_pages" else (None, pt.data_ptr(), slot.data_ptr())
    _l.check(lib.vcb_debug_attention(q.data_ptr(), Ks.data_ptr(), Vs.data_ptr(), 2, *args, pos.data_ptr(), n, H, hd,
                                     c["max_pages"], chunk_pages, balance, repeats, out.data_ptr()))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("chunk_pages", [1, 3, 16])
@pytest.mark.parametrize("hd", [64, 128])
def test_paged_attention_fp8_vs_fp64(hd, chunk_pages):
    """test_paged_attention_vs_fp64's positions (to 4100 tokens), score distributions and chunk sizes, on fp8 slabs:
    within 1e-5 * max|V| of fp64 attention over the dequantized pools (the conversion e4m3 -> f16 -> f32 is exact)."""
    from test_kernel_numerics import _attn_case, _attn_ref
    c = _fp8_case(_attn_case(hd, "fp32", chunk_pages))
    got = _attn_fp8(c, chunk_pages)
    ref = _attn_ref(c)
    vmax = float(c["Vp"].abs().max())
    active = c["pos"] >= 0
    assert torch.all(got[~active] == 12345.0), "an inactive row's output was written"
    for r in torch.nonzero(active).flatten().tolist():
        err = float((got[r].double() - ref[r]).abs().max())
        assert err <= 1e-5 * vmax, (f"row {r} pos {int(c['pos'][r])} ({c['kinds'][r]}): max err {err:.3g} "
                                    f"> 1e-5 * max|V| = {1e-5 * vmax:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("chunk_pages", [1, 3, 16])
@pytest.mark.parametrize("hd", [64, 128])
def test_paged_attention_fp8_is_bit_reproducible(hd, chunk_pages):
    """repeated launches, balance off, page_table + row_slot, row subsets and single rows: the same bits; and the grouped
    kernel (best-of-N decode) equals the per-row kernel bit for bit"""
    from test_kernel_numerics import _attn_case
    c = _fp8_case(_attn_case(hd, "fp32", chunk_pages, seed=1))
    base = _attn_fp8(c, chunk_pages)
    assert torch.equal(_attn_fp8(c, chunk_pages, repeats=3), base), "repeated launches differ"
    assert torch.equal(_attn_fp8(c, chunk_pages, balance=0), base), "result depends on the work balance"
    assert torch.equal(_attn_fp8(c, chunk_pages, via="page_table"), base), "row_pages and page_table + row_slot differ"
    subset = list(range(len(c["pos"]) - 1, -1, -3))
    assert torch.equal(_attn_fp8(c, chunk_pages, rows=subset), base[subset]), "a row depends on the other rows"
    for r in (int(np.argmax(c["pos"].numpy())), 7):
        assert torch.equal(_attn_fp8(c, chunk_pages, rows=[r]), base[[r]]), f"row {r} alone differs"

    from test_best_of import _group_case
    gc = _group_case(hd, "fp32", chunk_pages)
    Ks, _ = to_slabs(gc["Kp"].float().cpu())
    Vs, _ = to_slabs(gc["Vp"].float().cpu())
    Ks, Vs = Ks.cuda(), Vs.cuda()
    _l, lib = _lib()
    rows, H = gc["pos"].shape[0], gc["H"]
    outs = []
    for grouped in (False, True):
        out = torch.full((rows, H * hd), 12345.0, device="cuda")
        common = (gc["q"].data_ptr(), Ks.data_ptr(), Vs.data_ptr(), 2)
        tail = (rows, H, hd, gc["max_pages"], chunk_pages, 1, 1, out.data_ptr())
        if grouped:
            ng = len(gc["shared"])
            rc = lib.vcb_debug_attention_groups(*common, gc["pages"].data_ptr(), gc["pos"].data_ptr(), *tail,
                                                (C.c_int32 * (ng + 1))(*gc["first"]), (C.c_int32 * ng)(*gc["shared"]), ng)
        else:
            rc = lib.vcb_debug_attention(*common, gc["pages"].data_ptr(), None, None, gc["pos"].data_ptr(), *tail)
        torch.cuda.synchronize()
        assert rc == 0
        outs.append(out)
    assert torch.equal(outs[0], outs[1]), f"{int((outs[0] != outs[1]).any(dim=1).sum())} rows differ (grouped)"


@pytest.mark.gpu
@pytest.mark.parametrize("total", [128, 100])
def test_fp8_group_equals_independent_rows(total):
    """A best-of-3 group on an fp8 engine (forked tail page: bytes and scales) against 3 independent utterances of the same
    prompt fed the same noise: the same logits and tokens, bit for bit, up to the first end token."""
    from test_best_of import _model as bo_model, _trace, _utt
    cfg, m = bo_model("fp8", nhead=2, eos_bias=0.0)
    x, _, y = _utt(cfg, 43, total)
    lg, rg = _trace(m, cfg, x, y, 3, True)
    li, ri = _trace(m, cfg, x, y, 3, False)
    end = cfg.eos if cfg.eos > 0 else cfg.eog
    hit = [s for s in range(min(len(lg), len(li))) if any(int(r[s, 0]) == end for r in rg + ri if s < r.shape[0])]
    upto = hit[0] + 1 if hit else min(len(lg), len(li))
    assert upto >= 8
    for s in range(upto):
        assert torch.equal(lg[s], li[s]), f"step {s}: logits differ"
    for a, b in zip(rg, ri):
        assert torch.equal(torch.as_tensor(a[:upto]), torch.as_tensor(b[:upto])), "tokens differ"


@pytest.mark.gpu
def test_fp8_batch_rows_equal_single_calls():
    from voicecraft_b200 import synthetic
    cfg, sd, m = _model("fp8", seed=44)
    sd["predict_layer.0.2.bias"][cfg.eos] += 4.0
    m.load_state_dict(sd)
    m.configure_engine(max_slots=8, max_seq_len=512, kv_dtype="fp8")
    utts = [synthetic.synthetic_utterance(cfg, 600 + i, text_len=4 + i % 3, prompt_frames=12 + 5 * i) for i in range(8)]
    seeds = [900 + 17 * i for i in range(8)]
    kw = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
    singles = []
    for (x, xl, y), s in zip(utts, seeds):
        torch.manual_seed(s)
        singles.append(m.inference_tts(x.cuda(), xl.cuda(), y.cuda(), **kw)[0])
    many = m.inference_tts_many([u[0] for u in utts], [u[2] for u in utts], seeds=seeds, poll_every=3, **kw)
    for i, (a, (b, _)) in enumerate(zip(singles, many)):
        assert torch.equal(a, b), f"utterance {i}: batched row differs from its single call"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tts_topk40", "tts_topp", "edit2", "batch3"])
def test_tokens_match_oracle_kv_fp8(name):
    """The fp8 engine against the CPU oracle under the same policy (OracleLMFp8): identical token ids."""
    from test_gpu_parity import CASES, _run_case
    case = CASES[name]
    cfg, sd, x, x_lens, y, g = gu.build_case(name, case)
    oracle = OracleLMFp8(cfg, sd)
    kw = dict(case["kw"], silence_tokens=gu.SILENCE, kvcache=1, noise_fn=gu.cpu_noise_fn(case["seed"]))
    if case["kind"] == "tts":
        ores = oracle.inference_tts(x, x_lens, y, **kw)[0]
    elif case["kind"] == "batch":
        ores = oracle.inference_tts_batch(x, x_lens, y, batch_size=case["batch_size"], **kw)[0]
    else:
        ores = oracle.inference(x, x_lens, y, torch.from_numpy(g["mask_interval"]), **kw)
    res, _, _ = _run_case(name, case, "fp8")
    assert np.array_equal(res.cpu().numpy(), ores.numpy())


@pytest.mark.gpu
def test_fp8_pool_bytes():
    """kv_bytes_per_token = L * 2 * H * (64 * hd + 256) / 64 = L * 2 * (d + 4H) (67 584 B at 830M: d 2048, 16 heads, 16
    layers), and a bf16 engine holds exactly the pool bytes it differs by more than an fp8 engine of the same config"""
    from voicecraft_b200 import synthetic
    _l, lib = _lib()
    c830 = synthetic.make_config("830M")
    assert c830.num_decoder_layers * 2 * (c830.d_model + 4 * c830.nhead) == 67584
    cfg, sd, m = _model("bf16", max_slots=5)
    live = {}
    for kv in ("bf16", "fp8"):
        m.configure_engine(kv_dtype=kv)
        base = lib.vcb_counter(None, b"live_bytes")
        eng = m._engine()
        live[kv] = lib.vcb_counter(None, b"live_bytes") - base
        per_tok = lib.vcb_counter(eng, b"kv_bytes_per_token")
        L, d, H = cfg.num_decoder_layers, cfg.d_model, cfg.nhead
        assert per_tok == L * 2 * (d * 2 if kv == "bf16" else d + 4 * H)
        m._drop_engine()
    pages = 5 * (512 // 64)
    H, hd, L = cfg.nhead, cfg.d_model // cfg.nhead, cfg.num_decoder_layers
    assert live["bf16"] - live["fp8"] == 2 * L * pages * H * (64 * hd * 2 - 64 * (hd + 4))


@pytest.mark.gpu
def test_fp8_paths_it_does_not_take(monkeypatch):
    """VCB_MEGA=1 falls back to the per-kernel step for fp8 (mega_grid 0, the same tokens), and the CUDA-core GEMM is
    refused on an fp8 engine"""
    from voicecraft_b200 import synthetic
    _l, lib = _lib()
    toks = {}
    for mega in ("0", "1"):
        monkeypatch.setenv("VCB_MEGA", mega)
        cfg, sd, m = _model("fp8", seed=9)
        x, xl, y = synthetic.synthetic_utterance(cfg, 77, text_len=6, prompt_frames=20)
        m.noise_fn = gu.cpu_noise_fn(5)
        toks[mega] = m.inference_tts(x.cuda(), xl.cuda(), y.cuda(), top_k=40, stop_repetition=3)[0]
        assert lib.vcb_counter(m._eng, b"mega_grid") == 0
        if mega == "1":
            assert lib.vcb_set_option(m._eng, b"gemm_simt", 1) != 0
            assert b"fp8" in lib.vcb_last_error()
            assert lib.vcb_set_option(m._eng, b"gemm_simt", 0) == 0
    assert torch.equal(toks["0"], toks["1"])
    # control: a bf16 engine of the same config does take the persistent kernel under VCB_MEGA=1
    cfg, sd, m = _model("bf16", seed=9)
    m.noise_fn = gu.cpu_noise_fn(5)
    m.inference_tts(x.cuda(), xl.cuda(), y.cuda(), top_k=40, stop_repetition=3)
    assert lib.vcb_counter(m._eng, b"mega_grid") > 0


# ---------------------------------------------------------------------------------------------------------------------
# Headline shape under the fp8 policy: 830M, B = 32, 64 sampled steps, against tests/golden/lm_830m_b32_fp8.npz
# (make_golden_830m_fp8.py: OracleLMFp8 on make_golden_830m.py Part B's checkpoint, utterances and noise)
# ---------------------------------------------------------------------------------------------------------------------
# DESIGN.md section 2.2, from the first H100 run: max |logit - oracle| 6.6e-3 on the traced steps of still-identical
# utterances, 17 of 32 utterances identical throughout, every first divergence at a sensitivity <= 1.4e-3; 475 of the 8192
# fixture samples have a sensitivity below 1e-2
LOGIT_TOL_FP8 = 1e-2
M_IDENTICAL_FP8 = 12


@pytest.mark.gpu
def test_headline_830M_b32_fp8_matches_oracle():
    """The bf16 policy's rule (test_gpu_parity.test_headline_830M_b32_matches_oracle) under fp8: (a) raw logits within
    LOGIT_TOL_FP8 of the oracle on the traced steps of still-identical utterances, (b) every utterance identical up to its
    first differing sample, whose sensitivity is below LOGIT_TOL_FP8, (c) at least M_IDENTICAL_FP8 of 32 utterances
    identical throughout.  Also printed, not asserted: the fp8 and bf16 policies' distance from the fp32 policy in the
    oracle fixtures (max |logit difference| on the traced points, first divergent step per utterance)."""
    import os
    from test_gpu_parity import _headline_run
    meta, g, rows, logits = _headline_run("fp8")
    g.update(np.load(os.path.join(gu.GOLDEN, "lm_830m_b32_fp8.npz")))
    ref, margin = g["rows_fp8"].astype(np.int64), g["sens_fp8"]
    identical, first_div = 0, {}
    for i in range(32):
        neq = np.argwhere(rows[i] != ref[i])
        if len(neq) == 0:
            identical += 1
            continue
        s, k = (int(v) for v in neq[0])
        first_div[i] = (s, k, float(margin[i, s, k]))
    worst = 0.0
    for ui, u in enumerate(meta["trace_utts"]):
        for si, s in enumerate(meta["trace_steps"]):
            if u in first_div and first_div[u][0] < s:
                continue
            refl = g["logits_fp8"][ui, si]
            live = refl > -9999
            worst = max(worst, float(np.abs(logits[s][u] - refl)[live].max()))
    for pol in ("bf16", "fp8"):                     # the policies' cost against fp32, from the oracle fixtures
        d = np.abs(g[f"logits_{pol}"] - g["logits_fp32"])[g["logits_fp32"] > -9999]
        div = [int(np.argwhere(g[f"rows_{pol}"][i] != g["rows_fp32"][i])[0][0]) if (g[f"rows_{pol}"][i] != g["rows_fp32"][i]).any()
               else None for i in range(32)]
        print(f"oracle {pol} vs fp32: max |logit diff| {d.max():.3g} on the traced points (incl. after divergence); "
              f"{div.count(None)}/32 identical; first divergent step {div}")
    print(f"kv=fp8: {identical}/32 identical, divergences {first_div}, max |logit - oracle| {worst:.3g}")
    assert worst <= LOGIT_TOL_FP8, f"max |logit - oracle| = {worst}"
    for i, (s, k, mg) in first_div.items():
        assert mg < LOGIT_TOL_FP8, f"utterance {i} differs at step {s} codebook {k} where the oracle's decision is robust to {mg:.3g}"
    assert identical >= M_IDENTICAL_FP8, f"{identical}/32 utterances token-identical ({first_div})"
