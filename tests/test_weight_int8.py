"""Int8 GEMM weights (weight_dtype="int8", DESIGN.md section 2.2): every matrix the decode GEMM streams as int8 with a
power-of-two scale per output feature, multiplied as exact bf16 values by the same wgmmas as the bf16 engine.

CPU: the torch restatement of the rule against rows written out by hand and its bounds on random rows; the rejection of
unknown policies.  GPU (-m gpu): the device quantizer bit-exact against it; the int8 decode GEMM bit-identical to the bf16
GEMM on W_deq; an int8 engine bit-identical to a bf16 engine loaded with the dequantized state dict (logits and tokens);
split counts, weight bytes and the paths int8 does not take."""
import ctypes as C

import numpy as np
import pytest
import torch

import golden_util as gu
from weight_int8_ref import dequantize_rows, dequantize_state_dict, quantize_rows, quantized_keys

ULP_ABOVE_127 = float(np.nextafter(np.float32(127.0), np.float32(np.inf)))
TINY = 2.0 ** -126

# (row, q, e) written out by hand
HAND = [
    ([127.0, 1.0, -2.0, 0.0], [127, 1, -2, 0], 0),                      # amax exactly 127 * 2^0
    ([ULP_ABOVE_127, 1.0, -3.0, 0.0], [64, 0, -2, 0], 1),               # one ulp above: e = 1; 0.5 -> 0, -1.5 -> -2 (even)
    ([0.0, 0.0, 0.0, 0.0], [0, 0, 0, 0], -126),                         # all zero: e = -126
    ([127.0, 2.5, -2.5, 3.5], [127, 2, -2, 4], 0),                      # ties to even, both signs
    ([127.0, -0.5, 0.5, -1.5], [127, 0, 0, -2], 0),
    ([254.0, 3.0, -5.0, 1.0], [127, 2, -2, 0], 1),                      # 1.5 -> 2, -2.5 -> -2, 0.5 -> 0
    ([TINY, -TINY, 0.5 * TINY, 0.0], [1, -1, 0, 0], -126),              # amax 2^-126: e clamped; 0.5 -> 0 (even)
    ([127 * TINY, 1.5 * TINY, 0.0, 0.0], [127, 2, 0, 0], -126),         # exactly 127 * 2^-126
    ([128 * TINY, 0.0, 0.0, 0.0], [64, 0, 0, 0], -125),                 # just above: e = -125
    ([1e-45, 0.0, 0.0, 0.0], [0, 0, 0, 0], -126),                       # fp32 subnormal amax
]


def _hand_rows(k):
    x = torch.zeros(len(HAND), k)
    for i, (row, _, _) in enumerate(HAND):
        x[i, :4] = torch.tensor(row, dtype=torch.float32)
    return x


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_quantizer_matches_hand_written_rows():
    q, e = quantize_rows(_hand_rows(8))
    for i, (row, want, ew) in enumerate(HAND):
        assert q[i, :4].tolist() == want, f"row {row}: q {q[i, :4].tolist()} != {want}"
        assert int(e[i]) == ew, f"row {row}: e {int(e[i])} != {ew}"
        assert q[i, 4:].tolist() == [0] * 4


def test_quantizer_bounds_on_random_rows():
    g = torch.Generator().manual_seed(7)
    W = torch.randn(512, 256, generator=g) * torch.logspace(-30, 30, 512).unsqueeze(1)
    q, e = quantize_rows(W)
    s = torch.pow(2.0, e.double())
    amax = W.abs().amax(1).double()
    assert torch.all(amax <= 127 * s) and torch.all(amax > 63.5 * s)       # e is the smallest that fits
    assert int(q.abs().max()) <= 127
    deq = dequantize_rows(q, e)
    assert torch.all((W.double() - deq.double()).abs() <= 0.5 * s.unsqueeze(1))
    assert torch.equal(deq.bfloat16().float(), deq), "W_deq is not bf16-exact"


def test_dequantize_state_dict_covers_the_streamed_matrices():
    from voicecraft_b200 import synthetic
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=1)
    keys = quantized_keys(sd)
    assert len(keys) == 4 * cfg.num_decoder_layers + 2 * cfg.n_codebooks
    dq = dequantize_state_dict(sd)
    for k in sd:
        if k in keys:
            assert not torch.equal(dq[k], sd[k])
        else:
            assert dq[k] is sd[k]


def test_configure_engine_rejects_unknown_weight_dtype():
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    m = VoiceCraft(synthetic.make_config("tiny"))
    for bad in ("fp8", "int4", None):
        with pytest.raises(ValueError):
            m.configure_engine(weight_dtype=bad)
    m.configure_engine(weight_dtype="int8")
    assert m._eng_opts["weight_dtype"] == "int8"


def _config(weight_dtype, kv_dtype=0, d_model=256):
    from voicecraft_b200 import _lib
    return _lib.vcb_config(d_model=d_model, nhead=2, num_layers=1, n_codebooks=4, audio_vocab_size=2048, n_special=4,
                           text_vocab_rows=101, empty_token=2048, eog=2049, audio_pad_token=2050, eos=2051, encodec_sr=50,
                           max_n_spans=3, max_slots=1, max_seq_len=256, max_new_tokens=64, kv_dtype=kv_dtype,
                           weight_dtype=weight_dtype)


def test_create_rejects_unknown_weight_dtype():
    """checked before the device is touched, so this holds on any machine"""
    from voicecraft_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    for bad in (2, -1):
        assert lib.vcb_create(C.byref(_config(bad)), C.byref(h)) != 0
        assert b"weight_dtype" in lib.vcb_last_error()


def test_create_rejects_simt_gemm_and_narrow_shapes_with_int8(monkeypatch):
    from voicecraft_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.vcb_create(C.byref(_config(1, d_model=192)), C.byref(h)) != 0
    assert b"int8" in lib.vcb_last_error()
    monkeypatch.setenv("VCB_GEMM_IMPL", "simt")
    assert lib.vcb_create(C.byref(_config(1)), C.byref(h)) != 0
    assert b"simt" in lib.vcb_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _lib():
    from voicecraft_b200 import _lib
    return _lib, _lib.load()


def _device_quantize(W):
    _l, lib = _lib()
    N, K = W.shape
    Wd = W.contiguous().cuda()
    q = torch.zeros(N, K, dtype=torch.int8, device="cuda")
    e = torch.zeros(N, dtype=torch.int32, device="cuda")
    _l.check(lib.vcb_debug_weight_quantize(Wd.data_ptr(), N, K, q.data_ptr(), e.data_ptr()))
    return q.cpu(), e.cpu()


@pytest.mark.gpu
def test_device_quantizer_is_bit_exact():
    from voicecraft_b200 import synthetic
    g = torch.Generator().manual_seed(3)
    mats = [_hand_rows(64), torch.randn(600, 384, generator=g) * torch.logspace(-30, 30, 600).unsqueeze(1)]
    sd = synthetic.make_state_dict(synthetic.make_config("tiny"), seed=5)
    mats += [sd[k] for k in quantized_keys(sd)]
    for W in mats:
        q, e = quantize_rows(W)
        dq, de = _device_quantize(W)
        assert torch.equal(dq, q), f"{int((dq != q).sum())} bytes differ"
        assert torch.equal(de, e), "exponents differ"


def _legal_splits(bpad, K):
    kb = K // 64
    return [s for s in (1, 2, 4, 8, 16) if bpad // s >= 2 and (s - 1) * ((kb + s - 1) // s) < kb]


def _gemm(fn, W, X, N, K, B, splits, *extra):
    _l, lib = _lib()
    out = torch.full((B, N), 7.0, device="cuda")
    _l.check(fn(W.data_ptr(), X.data_ptr(), out.data_ptr(), N, K, B, splits, *extra))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1024, 2048, 8192])
@pytest.mark.parametrize("B", [16, 32, 64, 128])
def test_gemm_w8_equals_bf16_gemm_on_w_deq(B, K):
    """vcb_debug_gemm_w8(W) == vcb_debug_gemm(W_deq) bit for bit, at every split count the kernel for B rows can run;
    N = 2052 ends in a partial tile.  Rows span many magnitudes, so the scales differ from feature to feature."""
    _l, lib = _lib()
    g = torch.Generator().manual_seed(B * 7 + K)
    N = 2052
    W = torch.randn(N, K, generator=g) * torch.logspace(-3, 2, N).unsqueeze(1)
    X = torch.randn(B, K, generator=g)
    W_deq = dequantize_rows(*quantize_rows(W))
    Wd, Wq, Xd = W.cuda(), W_deq.cuda(), X.cuda()
    for s in _legal_splits(B, K) + [0]:
        ref = _gemm(lib.vcb_debug_gemm, Wq, Xd, N, K, B, s, 0)
        got = _gemm(lib.vcb_debug_gemm_w8, Wd, Xd, N, K, B, s)
        assert torch.equal(got, ref), f"splits {s}: {int((got != ref).sum())} outputs differ, max {float((got - ref).abs().max()):.3g}"


def _model(sd, cfg, wd, kv, **opts):
    from voicecraft_b200.voicecraft import VoiceCraft
    m = VoiceCraft(cfg)
    m.load_state_dict(sd if wd == "int8" else dequantize_state_dict(sd))
    m = m.to("cuda").eval()
    m.configure_engine(**dict(dict(kv_dtype=kv, weight_dtype=wd, max_slots=8, max_seq_len=512), **opts))
    return m


def _run_case(name, wd, kv):
    from test_gpu_parity import CASES
    case = CASES[name]
    cfg, sd, x, x_lens, y, g = gu.build_case(name, case)
    m = _model(sd, cfg, wd, kv)
    m.noise_fn = gu.cpu_noise_fn(case["seed"])
    m.trace_logits = []
    kw = dict(case["kw"], silence_tokens=gu.SILENCE, kvcache=1)
    if case["kind"] == "tts":
        res = m.inference_tts(x.cuda(), x_lens.cuda(), y.cuda(), **kw)[0]
    elif case["kind"] == "batch":
        res = m.inference_tts_batch(x.cuda(), x_lens.cuda(), y.cuda(), batch_size=case["batch_size"], **kw)[0]
    else:
        res = m.inference(x.cuda(), x_lens.cuda(), y.cuda(), torch.from_numpy(g["mask_interval"]).cuda(), **kw)
    return res.cpu(), [t.cpu() for t in m.trace_logits]


def _assert_same(a, b):
    (ra, la), (rb, lb) = a, b
    assert len(la) == len(lb) and len(la) > 0
    for s, (p, q) in enumerate(zip(la, lb)):
        assert torch.equal(p, q), f"step {s}: logits differ (max {float((p - q).abs().max()):.3g})"
    assert torch.equal(ra, rb), "tokens differ"


@pytest.mark.gpu
@pytest.mark.parametrize("kv", ["bf16", "fp8"])
@pytest.mark.parametrize("name", ["tts_topk40", "tts_topp", "edit2", "batch3"])
def test_engine_equals_bf16_engine_on_w_deq(name, kv):
    """an int8 engine loaded with sd against a bf16 engine loaded with dequantize_state_dict(sd): the same logits at every
    sampling step and the same tokens, bit for bit (prefill through the rows-as-M GEMM on the expanded W_deq, decode through
    the int8 kernel)"""
    _assert_same(_run_case(name, "int8", kv), _run_case(name, "bf16", kv))


@pytest.mark.gpu
@pytest.mark.parametrize("kv", ["bf16", "fp8"])
def test_best_of_group_equals_bf16_engine(kv):
    from test_best_of import _trace, _utt
    from voicecraft_b200 import synthetic
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=3)
    sd["predict_layer.0.2.bias"][cfg.eos] += 3.0
    x, _, y = _utt(cfg, 43, 100)
    out = {}
    for wd in ("int8", "bf16"):
        m = _model(sd, cfg, wd, kv, max_slots=24)
        out[wd] = _trace(m, cfg, x, y, 3, True)
        del m
    (li, ri), (lb, rb) = out["int8"], out["bf16"]
    assert len(li) == len(lb) > 0
    for s, (p, q) in enumerate(zip(li, lb)):
        assert torch.equal(p, q), f"step {s}: logits differ"
    for a, b in zip(ri, rb):
        assert np.array_equal(np.asarray(a), np.asarray(b)), "tokens differ"


@pytest.mark.gpu
def test_mega_falls_back_for_int8(monkeypatch):
    """VCB_MEGA=1: an int8 engine takes the per-kernel step (mega_grid 0) and stays bit-identical to the bf16 engine on W_deq
    without it; the CUDA-core GEMM is refused on an int8 engine"""
    from voicecraft_b200 import synthetic
    _l, lib = _lib()
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=9)
    x, xl, y = synthetic.synthetic_utterance(cfg, 77, text_len=6, prompt_frames=20)
    res = {}
    for wd, mega in (("int8", "1"), ("bf16", "0")):
        monkeypatch.setenv("VCB_MEGA", mega)
        m = _model(sd, cfg, wd, "bf16")
        m.noise_fn = gu.cpu_noise_fn(5)
        m.trace_logits = []
        toks = m.inference_tts(x.cuda(), xl.cuda(), y.cuda(), top_k=40, stop_repetition=3)[0]
        res[wd] = (toks.cpu(), [t.cpu() for t in m.trace_logits])
        if wd == "int8":
            assert lib.vcb_counter(m._eng, b"mega_grid") == 0
            assert lib.vcb_set_option(m._eng, b"gemm_simt", 1) != 0
            assert b"int8" in lib.vcb_last_error()
            assert lib.vcb_set_option(m._eng, b"gemm_simt", 0) == 0
        del m
    _assert_same(res["int8"], res["bf16"])


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["330M", "830M"])
def test_decode_shapes_take_the_bf16_split_count(size):
    """every decode GEMM of the 330M / 830M shapes at bpad 16..128: the int8 kernel runs the split count the bf16 rule
    picks (vcb_gemm_launch_shape), and with that count its output equals the bf16 GEMM's on W_deq -- a different K
    slicing would sum in a different order"""
    from voicecraft_b200 import synthetic
    _l, lib = _lib()
    cfg = synthetic.make_config(size)
    d, Hh, K = cfg.d_model, int(cfg.audio_vocab_size) // 2, cfg.n_codebooks
    shapes = [(3 * d, d), (d, d), (4 * d, d), (d, 4 * d), (K * Hh, d), (int(cfg.audio_vocab_size) + cfg.n_special, Hh)]
    g = torch.Generator().manual_seed(11)
    for N, Kd in shapes:
        assert Kd % 128 == 0
        W = torch.randn(N, Kd, generator=g).cuda()
        W_deq = dequantize_rows(*quantize_rows(W.cpu())).cuda()
        for B in (16, 32, 64, 128):
            shape = (C.c_int32 * 2)()
            _l.check(lib.vcb_gemm_launch_shape(N, Kd, B, 0, 0, 0, shape))
            X = torch.randn(B, Kd, generator=g).cuda()
            got = _gemm(lib.vcb_debug_gemm_w8, W, X, N, Kd, B, 0)
            ref = _gemm(lib.vcb_debug_gemm, W_deq, X, N, Kd, B, shape[0], 0)
            print(f"{size} N={N} K={Kd} B={B}: splits {shape[0]}")
            assert torch.equal(got, ref), f"N={N} K={Kd} B={B} splits {shape[0]}: outputs differ"


@pytest.mark.gpu
def test_weight_bytes_and_release():
    """int8 weight_bytes (before any prefill, so without the scratch) <= 0.51 of bf16's; the scratch is the largest layer
    matrix in bf16; after destroy, live bytes and handles return to their values before the engine"""
    from voicecraft_b200 import synthetic
    _l, lib = _lib()
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=2)
    x, xl, y = synthetic.synthetic_utterance(cfg, 5, text_len=6, prompt_frames=20)
    wb = {}
    for wd in ("bf16", "int8"):
        base = (lib.vcb_counter(None, b"live_bytes"), lib.vcb_counter(None, b"live_handles"))
        m = _model(sd, cfg, wd, "bf16")
        wb[wd] = lib.vcb_counter(m._engine(), b"weight_bytes")
        if wd == "int8":
            m.noise_fn = gu.cpu_noise_fn(1)
            m.inference_tts(x.cuda(), xl.cuda(), y.cuda(), top_k=40, stop_repetition=3)
            d = cfg.d_model
            assert lib.vcb_counter(m._eng, b"weight_bytes") - wb[wd] == 2 * max(3 * d * d, 4 * d * d)
        m._drop_engine()
        del m
        assert (lib.vcb_counter(None, b"live_bytes"), lib.vcb_counter(None, b"live_handles")) == base
    print(f"weight_bytes: bf16 {wb['bf16']}, int8 {wb['int8']} ({wb['int8'] / wb['bf16']:.4f})")
    assert wb["int8"] <= 0.51 * wb["bf16"]


@pytest.mark.gpu
def test_headline_830M_b32_int8_equals_bf16_engine():
    """the 830M B = 32 headline shape over 64 steps: an int8 engine and a bf16 engine on W_deq give the same logits on the
    traced steps and the same tokens"""
    import test_gpu_parity as tp
    meta, _ = gu.headline_fixture()
    cfg, sd = gu.headline_checkpoint(meta["ckpt_seed"])
    runs = {}
    orig = tp._model
    try:
        for wd in ("int8", "bf16"):
            tp._model = lambda cfg_, sd_, kv, wd=wd: _model(sd_, cfg_, wd, kv)
            _, _, rows, logits = tp._headline_run("bf16")
            runs[wd] = (rows, logits)
    finally:
        tp._model = orig
    (ri, li), (rb, lb) = runs["int8"], runs["bf16"]
    for s in li:
        assert np.array_equal(li[s], lb[s]), f"step {s}: logits differ"
    assert np.array_equal(ri, rb), "tokens differ"


def _batcher_sd():
    """test_batcher_edit._lm's checkpoint: heads that put no mass on non-audio tokens except codebook 0's end tokens"""
    from voicecraft_b200 import synthetic
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=3)
    for k in range(cfg.n_codebooks):
        for t in (cfg.empty_token, cfg.eog, cfg.audio_pad_token, cfg.eos):
            if not (k == 0 and t == cfg.eos):
                sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    sd["predict_layer.0.2.bias"][cfg.eog] = 2.5
    return cfg, sd


@pytest.mark.gpu
@pytest.mark.parametrize("kv", ["bf16", "fp8"])
def test_batcher_stream_mixed_queue_equals_bf16_engine(kv):
    """ContinuousBatcher.stream over a queue of TTS and edit tickets with their own sampling parameters, two of them
    submitted from inside the loop (so wide prefills of the int8 engine interleave with its decode steps): the int8 engine
    on sd and the bf16 engine on dequantize_state_dict(sd) yield the same chunks (ticket, audio, last) in the same order,
    the same last-step logits at every chunk, and the same results, bit for bit"""
    from test_batcher_edit import DEFAULTS, _codec, _queue, _submit
    from voicecraft_b200.voicecraft import ContinuousBatcher
    _l, lib = _lib()
    cfg, sd = _batcher_sd()
    tok = _codec()
    queue = _queue(cfg, 10, 1300)
    conc, K = 4, cfg.n_codebooks
    runs = {}
    for wd in ("int8", "bf16"):
        m = _model(sd, cfg, wd, kv)
        V = m.n_audio_tokens[0]
        cb = ContinuousBatcher(m, max_concurrency=conc, poll_every=4, **DEFAULTS)
        for q in queue[:8]:
            _submit(cb, q)
        chunks, logits = [], []
        t = torch.empty(conc * K, V, device="cuda")
        for i, (tk, w, last) in enumerate(cb.stream(tok, chunk_frames=6)):
            chunks.append((tk, None if w is None else w.cpu(), last))
            _l.check(lib.vcb_debug_logits(m._eng, t.data_ptr(), conc * K))
            logits.append(t.cpu())
            if i == 3:
                for q in queue[8:]:
                    _submit(cb, q)
        assert cb.errors == {} and len(cb.results) == len(queue)
        runs[wd] = (chunks, logits, [cb.results[i] for i in range(len(queue))])
        del cb, m
    (ci, li, ri), (cb_, lb, rb) = runs["int8"], runs["bf16"]
    assert len(ci) == len(cb_) > len(queue)
    for n, ((ta, wa, la), (tb, wb, lb_)) in enumerate(zip(ci, cb_)):
        assert ta == tb and la == lb_, f"chunk {n}: ticket / last differ"
        assert (wa is None and wb is None) or torch.equal(wa, wb), f"chunk {n} (ticket {ta}): audio differs"
    for n, (p, q) in enumerate(zip(li, lb)):
        assert torch.equal(p, q), f"chunk {n}: logits differ"
    for i, (a, b) in enumerate(zip(ri, rb)):
        for x, y in zip(a, b):
            assert (x is None and y is None) or torch.equal(x, y), f"ticket {i}: result differs"


def test_oracle_drift_of_int8_weights_830M():
    """Printed, not asserted (the weights are random: this bounds arithmetic drift, not speech quality): at the 830M
    B = 32 headline shape, the oracle under the bf16 KV policy on the checkpoint (lm_830m_b32*.npz) against the oracle on its
    dequantized int8 weights (lm_830m_b32_int8.npz, make_golden_830m_int8.py): max |logit difference| on the traced points
    of still-identical utterances, and the utterances whose 64 sampled steps stay identical."""
    import os
    meta, g = gu.headline_fixture()
    g.update(np.load(os.path.join(gu.GOLDEN, "lm_830m_b32_int8.npz")))
    ref, got = g["rows_bf16"].astype(np.int64), g["rows_int8"].astype(np.int64)
    assert ref.shape == got.shape == (32, meta["n_steps"], 4)
    first = {}
    for i in range(32):
        neq = np.argwhere(got[i] != ref[i])
        if len(neq):
            first[i] = int(neq[0][0])
    worst, worst_all = 0.0, 0.0
    for ui, u in enumerate(meta["trace_utts"]):
        for si, s in enumerate(meta["trace_steps"]):
            a, b = g["logits_int8"][ui, si], g["logits_bf16"][ui, si]
            live = (a > -9999) & (b > -9999)
            d = float(np.abs(a - b)[live].max())
            worst_all = max(worst_all, d)
            if u not in first or first[u] >= s:
                worst = max(worst, d)
    print(f"oracle, int8 weights vs bf16: max |logit diff| {worst:.3g} on the traced points of still-identical utterances "
          f"({worst_all:.3g} incl. after divergence); {32 - len(first)}/32 utterances identical over {meta['n_steps']} "
          f"steps; first divergent step {sorted(first.values())}")
