"""Text-speech alignment: the attention probe, the monotonic alignment search and the Alignment object.

Probe bound.  For a row with context keys j <= pos, the probe computes s_j = fl(fl(sum_i q_i k_ij) * c_j * scale) in fp32
(k_ij the stored bf16 / fp32 / e4m3 value, exact in fp32; c_j the fp8 scale or 1), then p_j = exp(s_j - M) / S with M the
max and S the fp32 sum of exp(s_i - M).  The fp64 reference takes the same stored K.  With hd terms, the dot product's
relative error is at most hd * u * sum |q_i k_ij| (u = 2^-24), so |ds_j| <= (hd + 2) u |scale| sum_i |q_i k_ij| =: e_j.
exp and the division add a few ulps, and the sum S of n terms adds n u relatively; so
    |p_j - p_j*| <= p_j* (2 max_i e_i + n u + 8 u) + 1e-30,
which the tests use with a factor 2 of headroom (p* from fp64).  The mean over heads adds u relatively per head.

Monotonic alignment search.  The device sums fp32 values frame by frame and compares them exactly; the fp32 restatement
below performs the same additions in the same order, so its path (and durations) equal the device's bit for bit.  The
fp64 restatement agrees with both wherever the best path beats every other by more than the fp32 rounding of the sums
(checked on planted matrices whose path wins by a wide margin).
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

# ---- CPU restatements ----------------------------------------------------------------------------------------------


def mas_durations(logp, dtype=np.float64):
    """Monotonic alignment search over logp [T, X] as vcb_align_monotonic states it: durations [X]."""
    lp = np.asarray(logp, dtype=dtype)
    T, X = lp.shape
    if T < X:
        raise ValueError("T < X")
    ninf = dtype(-np.inf)
    q = np.full(X, ninf, dtype=dtype)
    q[0] = lp[0, 0]
    down = np.zeros((T, X), dtype=bool)
    for t in range(1, T):
        cur = np.full(X, ninf, dtype=dtype)
        for x in range(min(X, t + 1)):
            stay = q[x] if x < t else ninf
            dn = q[x - 1] if x > 0 else ninf
            d = x == t or (x > 0 and dn > stay)
            down[t, x] = d
            cur[x] = dtype((dn if d else stay) + lp[t, x])
        q = cur
    dur = np.zeros(X, dtype=np.int32)
    x = X - 1
    for t in range(T - 1, -1, -1):
        dur[x] += 1
        if t > 0 and down[t, x]:
            x -= 1
    return dur


def read_mfa_csv(path):
    """the reader of inference_speech_editing_scale.py:get_mask_interval: header dropped, comma-split rows"""
    with open(path) as f:
        rows = [line.strip().split(",") for line in f.readlines()]
    assert rows[0] == ["Begin", "End", "Label", "Type", "Speaker"]
    return rows[1:]


# ---- CPU tests ------------------------------------------------------------------------------------------------------


def test_mas_hand_worked():
    # 3 frames, 2 tokens: the second frame prefers token 1
    lp = np.log(np.array([[0.9, 0.1], [0.2, 0.8], [0.3, 0.7]]))
    assert mas_durations(lp).tolist() == [1, 2]
    # prefers token 0 for two frames
    lp = np.log(np.array([[0.9, 0.1], [0.8, 0.2], [0.3, 0.7]]))
    assert mas_durations(lp).tolist() == [2, 1]
    # T == X: one frame each whatever the values
    assert mas_durations(np.zeros((4, 4))).tolist() == [1, 1, 1, 1]
    # X == 1: every frame on the one token
    assert mas_durations(np.zeros((5, 1))).tolist() == [5]


def test_mas_ties_stay():
    # all equal: at each backtracking step both predecessors tie, so the path stays on the later token as long as it can
    assert mas_durations(np.zeros((6, 3))).tolist() == [1, 1, 4]
    # -inf everywhere off the planted path is no obstacle: ties of -inf stay too
    lp = np.full((5, 2), -np.inf)
    lp[:3, 0] = 0
    lp[3:, 1] = 0
    assert mas_durations(lp).tolist() == [3, 2]


def test_mas_refuses_short():
    with pytest.raises(ValueError):
        mas_durations(np.zeros((2, 3)))


def test_words_and_mfa_csv(tmp_path):
    from voicecraft_b200.alignment import Alignment
    SEP = 7
    ids = np.array([1, 2, SEP, 3, SEP, 4, 5, 6])
    dur = torch.tensor([2, 3, 1, 5, 2, 4, 1, 7], dtype=torch.int32)
    al = Alignment(torch.zeros(25, 8), dur, 50, ids)
    assert al.token_frames()[:3] == [(0, 2), (2, 5), (5, 6)]
    words = al.words(SEP)
    assert words == [(0, 1, 0.0, 0.1), (3, 3, 0.12, 0.22), (5, 7, 0.26, 0.5)]
    p = os.path.join(tmp_path, "a.csv")
    al.to_mfa_csv(p, ["one", "two", "three"], SEP)
    rows = read_mfa_csv(p)
    assert [r[2] for r in rows] == ["one", "two", "three"] and all(r[3] == "words" for r in rows)
    for (_, _, s, e), r in zip(words, rows):
        assert abs(float(r[0]) - s) < 1e-9 and abs(float(r[1]) - e) < 1e-9
    with pytest.raises(ValueError):
        al.to_mfa_csv(p, ["one"], SEP)


def test_abi_offsets():
    from voicecraft_b200 import _lib
    cfg = _lib.vcb_config
    # align_text_cap takes the 4 bytes of padding after the 19 older int32: kv_pool_bytes and the size stay where they were
    assert cfg.align_text_cap.offset == 76 and cfg.kv_pool_bytes.offset == 80 and C.sizeof(cfg) == 88
    pr = _lib.vcb_prompt
    assert pr.align_heads.offset == pr.sampling.offset + 8 and C.sizeof(pr) == pr.align_heads.offset + 8


def test_head_masks():
    from voicecraft_b200.alignment import head_masks
    assert head_masks(None, 4, 16) is None
    assert head_masks(True, 2, 16).tolist() == [0xFFFF, 0xFFFF]
    assert head_masks({1: [0, 3]}, 2, 16).tolist() == [0, 9]
    for bad in ({2: [0]}, {0: [16]}, {0: []}, {}, "all", {-1: [0]}):
        with pytest.raises(ValueError):
            head_masks(bad, 2, 16)


def test_configure_engine_cap():
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    m = VoiceCraft(synthetic.make_config("tiny"))
    for bad in (-1, 4097, 1.5):
        with pytest.raises(ValueError, match="align_text_cap"):
            m.configure_engine(align_text_cap=bad)
    m.configure_engine(align_text_cap=64)


# ---- GPU: the probe against fp64 --------------------------------------------------------------------------------------

def _lib():
    from voicecraft_b200 import _lib as l
    return l, l.load()


def _pool(K, kv, hd):
    """K [pages, H, 64, hd] fp32 -> (pool bytes on the device, the stored values as fp64 [pages, H, 64, hd], scales)"""
    if kv == "fp32":
        return K.float().contiguous().cuda(), K.double(), None
    if kv == "bf16":
        b = K.to(torch.bfloat16).contiguous()
        return b.cuda(), b.double(), None
    amax = K.abs().amax(-1).clamp_min(1e-30)
    e = torch.ceil(torch.log2(amax / 448.0)).clamp_min(-126)
    sc = torch.pow(2.0, e)
    qb = (K / sc.unsqueeze(-1)).to(torch.float8_e4m3fn)
    P, H = K.shape[:2]
    raw = torch.cat([qb.view(torch.uint8).reshape(P, H, -1), sc.float().contiguous().view(torch.uint8).reshape(P, H, -1)], -1)
    return raw.contiguous().cuda(), qb.double() * sc.double().unsqueeze(-1), sc


def _probe_ref(q, Kd, pages, pos, heads, x_len, hd):
    """fp64 mean softmax weights on the text keys and the bound of the module docstring"""
    u = 2.0 ** -24
    ref, bound = [], []
    for r in range(q.shape[0]):
        j = torch.arange(pos[r] + 1)
        keys = Kd[pages[r][j // 64].long(), :, j % 64]
        acc, b = 0, 0
        for h in heads:
            qh = q[r, h].double()
            s = (keys[:, h] @ qh) / hd ** 0.5
            e = (hd + 2) * u * (keys[:, h].abs() @ qh.abs()) / hd ** 0.5
            p = torch.softmax(s, 0)
            acc = acc + p[:x_len]
            b = b + p[:x_len] * (2 * e.max() + (pos[r] + 1) * u + 8 * u)
        ref.append(acc / len(heads))
        bound.append(b / len(heads) + 1e-30 + 4 * u * acc / len(heads))
    return torch.stack(ref), torch.stack(bound)


@pytest.mark.gpu
@pytest.mark.parametrize("kv", ["bf16", "fp32", "fp8"])
@pytest.mark.parametrize("hd", [64, 128])
def test_probe_fp64(kv, hd):
    l, lib = _lib()
    g = torch.Generator().manual_seed(hd + len(kv))
    H, rows, max_pages, x_len = 4, 6, 72, 40
    pos = [40, 63, 64, 200, 4100, 4607]           # page boundaries, past 4096 keys
    n_pages = rows * max_pages
    K = torch.randn(n_pages, H, 64, hd, generator=g)
    q = torch.randn(rows, H, hd, generator=g)
    # planted scores: row 1 head 0 has +80 on key 5 (a text key), row 3 head 2 a maximum outside the text (key 150)
    perm = torch.randperm(n_pages, generator=g)[: rows * max_pages].reshape(rows, max_pages)
    pages = perm.int()
    for r, h, j, v in ((1, 0, 5, 80.0), (3, 2, 150, 80.0), (4, 1, 7, -80.0)):
        k = K[pages[r, j // 64], h, j % 64]
        q[r, h] = k * (v * hd ** 0.5 / float(k @ k))
    pool, Kd, _ = _pool(K, kv, hd)
    heads = [0, 1, 2]
    mask = sum(1 << h for h in heads)
    out = torch.full((rows, x_len), float("nan"), device="cuda")
    qd = q.float().contiguous().cuda()
    pages_d, pos_d = pages.cuda(), torch.tensor(pos, dtype=torch.int32).cuda()     # held: the call reads them
    l.check(lib.vcb_debug_align_probe(qd.data_ptr(), pool.data_ptr(), {"bf16": 0, "fp32": 1, "fp8": 2}[kv],
                                      pages_d.data_ptr(), pos_d.data_ptr(), rows, H, hd, max_pages, mask, x_len,
                                      out.data_ptr()))
    ref, bound = _probe_ref(q.float(), Kd, pages, pos, heads, x_len, hd)
    err = (out.cpu().double() - ref).abs()
    assert torch.isfinite(out).all()
    assert (err <= 2 * bound).all(), f"worst {float((err / bound).max()):.3g} x bound"


@pytest.mark.gpu
def test_probe_refusals():
    l, lib = _lib()
    x = torch.zeros(64, device="cuda")
    p = torch.zeros(4, dtype=torch.int32, device="cuda")
    for mask, H, hd, x_len in ((0, 2, 128, 4), (4, 2, 128, 4), (1, 2, 96, 4), (1, 2, 128, 0), (1, 33, 128, 4)):
        assert lib.vcb_debug_align_probe(x.data_ptr(), x.data_ptr(), 0, p.data_ptr(), p.data_ptr(), 1, H, hd, 1, mask,
                                         x_len, x.data_ptr()) != 0


# ---- GPU: the monotonic alignment search ------------------------------------------------------------------------------

def _device_mas(lp):
    from voicecraft_b200.alignment import monotonic_durations
    return monotonic_durations(torch.as_tensor(lp, dtype=torch.float32).cuda()).cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("T,X", [(5, 2), (37, 11), (800, 120), (4096, 300), (1100, 1100), (2000, 1500)])
def test_mas_device_equals_cpu(T, X):
    rng = np.random.default_rng(T * 7 + X)
    lp = np.log(rng.dirichlet(np.ones(X), size=T)).astype(np.float32)
    dev = _device_mas(lp)
    assert dev.sum() == T and (dev >= 1).all()
    assert dev.tolist() == mas_durations(lp, np.float32).tolist()
    # planted: a path with a wide margin, which the fp64 restatement finds too
    dur = rng.multinomial(T - X, np.ones(X) / X) + 1
    planted = np.full((T, X), -30.0, np.float32)
    t = 0
    for x, d in enumerate(dur):
        planted[t:t + d, x] = 0.0
        t += d
    assert _device_mas(planted).tolist() == dur.tolist() == mas_durations(planted).tolist()


@pytest.mark.gpu
def test_mas_refusals():
    l, lib = _lib()
    x = torch.zeros(16, device="cuda")
    d = torch.zeros(8, dtype=torch.int32, device="cuda")
    for T, X in ((2, 3), (4, 0), (5000, 4097)):
        assert lib.vcb_align_monotonic(x.data_ptr(), T, X, d.data_ptr(), None) != 0


# ---- GPU: the engine -------------------------------------------------------------------------------------------------

def _model(kv="bf16", weights="bf16", cap=48, seed=3, no_end=False, audio_only=False, **opts):
    """tiny LM; no_end: no special token is ever drawn, so every utterance runs to its length cap; audio_only: none but
    codebook 0's end token (every frame decodes to audio)"""
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=seed)
    sd["predict_layer.0.2.bias"][cfg.eos] += 3.0
    for k in range(cfg.n_codebooks if no_end or audio_only else 0):
        for t in (cfg.empty_token, cfg.eog, cfg.audio_pad_token, cfg.eos):
            if no_end or not (k == 0 and t == cfg.eos):
                sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    m = m.to("cuda").eval()
    m.configure_engine(**{**dict(kv_dtype=kv, weight_dtype=weights, max_slots=8, max_seq_len=512, align_text_cap=cap),
                          **opts})
    return cfg, m


def _utt(cfg, seed, text_len=12, frames=30):
    from voicecraft_b200 import synthetic
    x, xl, y = synthetic.synthetic_utterance(cfg, seed, text_len=text_len, prompt_frames=frames)
    return x.cuda(), xl.cuda(), y.cuda()


def _run(m, x, xl, y, seed, **kw):
    torch.manual_seed(seed)
    return m.inference_tts(x, xl, y, top_k=40, logprobs=True, **kw)


KV_W = [("bf16", "bf16"), ("fp32", "bf16"), ("fp8", "bf16"), ("bf16", "int8")]


@pytest.mark.gpu
@pytest.mark.parametrize("kv,w", KV_W)
def test_inert_and_recorded(kv, w):
    """alignment on: tokens and log-probabilities are those of a run without it; soft rows are distributions over the
    text restricted to it (sum <= 1), the durations tile the frames, and the result is reproducible bit for bit"""
    cfg, m = _model(kv, w)
    x, xl, y = _utt(cfg, 5)
    res0, gen0, lp0 = _run(m, x, xl, y, 11)
    res1, gen1, lp1, al = _run(m, x, xl, y, 11, alignment=True)
    assert torch.equal(res0, res1) and torch.equal(gen0, gen1) and torch.equal(lp0, lp1)
    T = res1.shape[-1]
    assert al.soft.shape == (T, x.shape[1])
    s = al.soft.sum(1)
    assert torch.isfinite(al.soft).all() and (al.soft >= 0).all() and (s <= 1 + 1e-5).all() and (s > 0).all()
    assert int(al.durations.sum()) == T and int(al.durations.min()) >= 1
    *_, al2 = _run(m, x, xl, y, 11, alignment=True)
    assert torch.equal(al.soft, al2.soft) and torch.equal(al.durations, al2.durations)
    # one layer's heads: a different average, same tokens
    *_, al3 = _run(m, x, xl, y, 11, alignment={1: [0]})
    assert not torch.equal(al.soft, al3.soft)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["wide", "narrow"])
def test_probe_in_engine_fp64(route, monkeypatch):
    """the last layer's probe in a decode step and in the prompt's prefill (rows-as-M wide route, or the narrow
    128-row route) against fp64 from the pass's own q and K"""
    l, lib = _lib()
    if route == "narrow":
        monkeypatch.setenv("VCB_PREFILL_WIDE", "0")
    cfg, m = _model("bf16")
    x, xl, y = _utt(cfg, 9, text_len=10, frames=20)
    L, H, hd = cfg.num_decoder_layers, cfg.nhead, cfg.d_model // cfg.nhead
    sess = m.open_tts_session([x], [y], seeds=[1], alignment={L - 1: [0, 1]})
    try:
        x_len, total, slot = x.shape[1], sess.prompts[0].total, sess.slots[0]

        def check(first, n, q_rows):
            npg = (first + n + 63) // 64
            kb = np.zeros(npg * H * 64 * hd * 2, np.uint8)
            vb = np.zeros_like(kb)
            l.check(lib.vcb_debug_kv_pages(sess.eng, L - 1, slot, 0, npg, kb.ctypes.data, vb.ctypes.data))
            Kd = torch.from_numpy(kb).view(torch.bfloat16).reshape(npg, H, 64, hd).double()
            q = torch.empty(q_rows, cfg.d_model, device="cuda")
            l.check(lib.vcb_debug_stage_read(sess.eng, b"q", q.data_ptr(), q_rows))
            got = np.empty((n, x_len), np.float32)
            l.check(lib.vcb_read_alignment(sess.eng, slot, got.ctypes.data_as(C.POINTER(C.c_float)), first, n,
                                           sess.stream))
            return Kd, q.cpu().reshape(q_rows, H, hd), torch.from_numpy(got).double()

        # prefill: rows are positions 0 .. total-1; the audio rows x_len .. total-1 were probed
        Kd, q, got = check(x_len, total - x_len, total)
        pages = torch.arange((total + 63) // 64).repeat(total - x_len, 1)
        ref, bound = _probe_ref(q[x_len:], Kd, pages, list(range(x_len, total)), [0, 1], x_len, hd)
        assert ((got - ref).abs() <= 2 * bound).all()
        sess.sample()
        sess.step()
        Kd, q, got = check(total, 1, 1)
        ref, bound = _probe_ref(q, Kd, torch.arange((total + 64) // 64)[None], [total], [0, 1], x_len, hd)
        assert ((got - ref).abs() <= 2 * bound).all()
    finally:
        sess.close()


@pytest.mark.gpu
def test_prefill_straddling_row_4096():
    """a prompt of more than 4096 rows runs two wide passes: the second pass's rows (positions 4096 ..) read keys the
    first pass wrote; their probe against fp64 from the pass's q and the slot's K"""
    l, lib = _lib()
    cfg, m = _model("bf16", max_seq_len=4608)
    L, H, hd = cfg.num_decoder_layers, cfg.nhead, cfg.d_model // cfg.nhead
    x, xl, y = _utt(cfg, 12, text_len=20, frames=4150)
    sess = m.open_tts_session([x], [y], seeds=[1], alignment={L - 1: [1]})
    try:
        x_len, total, slot = x.shape[1], sess.prompts[0].total, sess.slots[0]
        assert total > 4096 and l.load().vcb_counter(sess.eng, b"wide_rows") == 4096
        rows = total - 4096
        npg = (total + 63) // 64
        kb = np.zeros(npg * H * 64 * hd * 2, np.uint8)
        vb = np.zeros_like(kb)
        l.check(lib.vcb_debug_kv_pages(sess.eng, L - 1, slot, 0, npg, kb.ctypes.data, vb.ctypes.data))
        Kd = torch.from_numpy(kb).view(torch.bfloat16).reshape(npg, H, 64, hd).double()
        q = torch.empty(rows, cfg.d_model, device="cuda")
        l.check(lib.vcb_debug_stage_read(sess.eng, b"q", q.data_ptr(), rows))
        got = np.empty((rows, x_len), np.float32)
        l.check(lib.vcb_read_alignment(sess.eng, slot, got.ctypes.data_as(C.POINTER(C.c_float)), 4096, rows, sess.stream))
        ref, bound = _probe_ref(q.cpu().reshape(rows, H, hd), Kd, torch.arange(npg).repeat(rows, 1),
                                list(range(4096, total)), [1], x_len, hd)
        assert ((torch.from_numpy(got).double() - ref).abs() <= 2 * bound).all()
    finally:
        sess.close()


@pytest.mark.gpu
def test_prefill_decode_agreement():
    """The rows recorded for generated frames agree with the rows a prefill records when its prompt is extended by the
    very columns the decode steps fed (the original prompt's columns, then the sampled delayed rows): Alignment.soft row
    t (frame t) equals the prefill's row at position x_len + t.  The two paths compute q and K through different kernels
    (rounding-level differences, fp32 KV here), so they agree within a tolerance; the comparison shifted by one frame
    must be far off, which pins the mapping."""
    from voicecraft_b200 import voicecraft as vc
    l, lib = _lib()
    cfg, m = _model("fp32", audio_only=True)
    x, xl, y = _utt(cfg, 21, text_len=10, frames=25)
    sess = m.open_tts_session([x], [y], seeds=[4], alignment=True)
    try:
        sess.sample()
        while not (sess.steps % 4 == 0 and sess.all_done()):
            sess.step()
        rows = sess.raw_tokens(0)
        res, gen, al = sess.results()[0]
    finally:
        sess.close()
    T, g = y.shape[1], min(rows.shape[0] - 1, 20)
    assert g > 8
    p = vc._Prompt(m, x, y)
    p.y_tok = torch.cat([p.y_tok, torch.from_numpy(rows[:g]).to(p.y_tok)]).contiguous()
    p.total = int(x.shape[1]) + int(p.y_tok.shape[0])
    p.align = vc._align_heads(m, True, [x])
    eng, held = m._take_slots(1, p.total + 8)
    try:
        vc._prefill(eng, [(p, held[0], 1, 0, 0)], torch.cuda.current_stream().cuda_stream)
        b = vc._read_alignment(m, eng, held[0], p, T + g, torch.cuda.current_stream().cuda_stream).soft.double()
    finally:
        m._release_slots(held)
    a = al.soft.double()
    lo, hi = T + 1, T + g                       # decode-step rows (row x_len + T is the prompt's last, on both paths)
    diff = (a[lo:hi] - b[lo:hi]).abs().max().item()
    shifted = (a[lo + 1:hi] - b[lo:hi - 1]).abs().max().item()
    assert diff < 1e-4 and shifted > 10 * diff, (diff, shifted)
    assert (a[:lo] - b[:lo]).abs().max().item() < 1e-4          # prompt rows: prefills of the same columns


@pytest.mark.gpu
@pytest.mark.parametrize("kv", ["bf16", "fp8"])
def test_inert_logits_and_kv(kv):
    """alignment on: every step's raw logits (vcb_debug_logits) and every layer's KV bytes equal a run without it"""
    l, lib = _lib()
    cfg, m = _model(kv)
    x, xl, y = _utt(cfg, 5)
    K, V, L, H, hd = cfg.n_codebooks, m.n_audio_tokens[0], cfg.num_decoder_layers, cfg.nhead, cfg.d_model // cfg.nhead
    slab = 64 * (hd + 4) if kv == "fp8" else 64 * hd * 2
    runs = []
    for align in (None, True):
        sess = m.open_tts_session([x], [y], seeds=[3], alignment=align)
        try:
            logits = []
            t = torch.empty(K, V, device="cuda")
            sess.sample()
            for _ in range(12):
                l.check(lib.vcb_debug_logits(sess.eng, t.data_ptr(), K))
                logits.append(t.clone())
                sess.step()
            sess.poll()
            npg = (sess.prompts[0].total + 12 + 63) // 64
            kv_bytes = []
            for layer in range(L):
                kb = np.zeros(npg * H * slab, np.uint8)
                vb = np.zeros_like(kb)
                l.check(lib.vcb_debug_kv_pages(sess.eng, layer, sess.slots[0], 0, npg, kb.ctypes.data, vb.ctypes.data))
                kv_bytes += [kb, vb]
            runs.append((torch.stack(logits), kv_bytes))
        finally:
            sess.close()
    assert torch.equal(runs[0][0].view(torch.int32), runs[1][0].view(torch.int32))
    assert all(np.array_equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))


@pytest.mark.gpu
def test_batcher_run_stream_long():
    """ContinuousBatcher: with alignment (the constructor's, one ticket opting out), run() and stream() return the tokens
    and log-probabilities of a batcher without it; each ticket's Alignment equals its seeded single call's bit for bit;
    a long ticket's alignments equal inference_long_tts's per sentence; the streams' .alignments likewise"""
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, m = _model("bf16", audio_only=True)
    utts = [_utt(cfg, 30 + i, text_len=8 + 2 * i, frames=20 + 5 * i) for i in range(3)]
    kw = dict(top_k=40)

    def batch(align, stream=False):
        cb = ContinuousBatcher(m, max_concurrency=2, poll_every=4, alignment=align, **kw)
        for i, (x, _, y) in enumerate(utts):
            cb.submit(x, y, seed=50 + i, alignment=False if i == 2 else None)
        if stream:
            for _ in cb.stream(_codec()):
                pass
            return cb, cb.results
        return cb, cb.run()
    plain, r0 = batch(None)
    on, r1 = batch(True)
    son, r2 = batch(True, stream=True)
    for i in range(3):
        assert torch.equal(r0[i][0], r1[i][0]) and torch.equal(r0[i][0], r2[i][0])
        assert torch.equal(plain.logprobs[i], on.logprobs[i]) and torch.equal(plain.logprobs[i], son.logprobs[i])
    assert on.alignments[2] is None and son.alignments[2] is None
    for i in range(2):
        x, xl, y = utts[i]
        torch.manual_seed(50 + i)
        res, gen, al = m.inference_tts(x, xl, y, alignment=True, **kw)
        assert torch.equal(res, r1[i][0])
        for got in (on.alignments[i], son.alignments[i]):
            assert torch.equal(got.soft, al.soft) and torch.equal(got.durations, al.durations)
    # long TTS: per sentence, as the loop of seeded inference_tts calls returns it
    xs = [u[0] for u in utts[:2]]
    y = utts[0][2]
    torch.manual_seed(9)
    out = m.inference_long_tts(xs, y, alignment=True, **kw)
    torch.manual_seed(9)
    loop = [m.inference_tts(xi, torch.tensor([xi.shape[1]]), y, alignment=True, **kw) for xi in xs]
    for (res, gen, al), (res2, gen2, al2) in zip(out, loop):
        assert torch.equal(res, res2) and torch.equal(al.soft, al2.soft)
    torch.manual_seed(9)
    st = m.inference_long_tts_stream(xs, y, _codec(), alignment=True, **kw)
    for _ in st:
        pass
    assert all(torch.equal(a.soft, b[2].soft) for a, b in zip(st.alignments, out))
    # the single-utterance stream
    torch.manual_seed(50)
    s1 = m.inference_tts_stream(utts[0][0], utts[0][1], utts[0][2], _codec(), alignment=True, **kw)
    for _ in s1:
        pass
    assert torch.equal(s1.alignment.soft, on.alignments[0].soft)


def _codec():
    from oracle import encodec_oracle as eo
    from voicecraft_b200.tokenizer import AudioTokenizer
    cfg = eo.default_config()
    return AudioTokenizer(device="cuda:0", config=cfg, state_dict=eo.make_state_dict(cfg, seed=5))


@pytest.mark.gpu
def test_batch_and_best_of_independence():
    """an utterance's alignment is the same bits alone and in a session with others; best-of-N keeps the tokens of a run
    without alignment, and its kept copy's prompt rows are the one-copy prefill's"""
    cfg, m = _model("bf16")
    utts = [_utt(cfg, s, text_len=8 + s, frames=20 + 3 * s) for s in range(3)]
    alone = []
    for i, (x, xl, y) in enumerate(utts):
        (r, g, al), = m.inference_tts_many([x], [y], seeds=[100 + i], alignment=True)
        alone.append((r, al))
    many = m.inference_tts_many([u[0] for u in utts], [u[2] for u in utts], seeds=[100, 101, 102], alignment=True)
    for (r0, a0), (r1, g1, a1) in zip(alone, many):
        assert torch.equal(r0, r1) and torch.equal(a0.soft, a1.soft) and torch.equal(a0.durations, a1.durations)
    # best-of-N: tokens as without alignment, the kept copy's alignment covers its result
    x, xl, y = utts[0]
    torch.manual_seed(5)
    r0, g0 = m.inference_tts_batch(x, xl, y, top_k=40, batch_size=3)
    torch.manual_seed(5)
    r1, g1, al = m.inference_tts_batch(x, xl, y, top_k=40, batch_size=3, alignment=True)
    assert torch.equal(r0, r1) and al.soft.shape[0] == r1.shape[-1]
    # prompt rows of the kept copy equal the one-copy prefill's (copied with the fork)
    T0 = y.shape[1]
    assert torch.equal(al.soft[:T0], alone[0][1].soft[:T0])


@pytest.mark.gpu
def test_swap_carries_alignment():
    """a session under a KV budget swaps an utterance out and back: alignments equal a run without the budget.  Two
    utterances of ~440 positions (8 pages each) on a 9-page pool: the prefill takes 4 + 4 pages, growth forces a swap"""
    cfg, m = _model("bf16", no_end=True)
    utts = [_utt(cfg, s, text_len=40, frames=10) for s in range(2)]
    xs, ys = [u[0] for u in utts], [u[2] for u in utts]
    ref = m.inference_tts_many(xs, ys, seeds=[1, 2], alignment={0: [1], 1: [0]})
    from voicecraft_b200 import _lib as l
    pb = l.load().vcb_counter(m._engine(), b"kv_page_bytes")
    m.configure_engine(kv_pool_gb=9.5 * pb / 1e9)
    from voicecraft_b200 import voicecraft as vc
    swaps, orig = [], vc.KvPoolPolicy.close

    def close(pool):                               # count the session's swaps as its pool closes
        swaps.append((pool.swap_outs, pool.swap_ins))
        return orig(pool)
    vc.KvPoolPolicy.close = close
    try:
        out = m.inference_tts_many(xs, ys, seeds=[1, 2], alignment={0: [1], 1: [0]})
    finally:
        vc.KvPoolPolicy.close = orig
    assert swaps and swaps[0][0] >= 1 and swaps[0][1] >= 1, swaps
    for (r0, _, a0), (r1, _, a1) in zip(ref, out):
        assert torch.equal(r0, r1) and torch.equal(a0.soft, a1.soft)


@pytest.mark.gpu
def test_refusals_hold_nothing():
    l, lib = _lib()
    cfg, m = _model("bf16", cap=8)
    x, xl, y = _utt(cfg, 5, text_len=12)
    with pytest.raises(ValueError, match="align_text_cap"):
        m.inference_tts(x, xl, y, alignment=True)
    with pytest.raises(ValueError):
        m.inference_tts(x, xl, y, alignment={0: [2]})
    eng = m._engine()
    free = lib.vcb_counter(eng, b"kv_pages_free")
    # the engine refuses what the Python layer lets through: a mask bit >= nhead, x_len over the cap, an edit, no bit
    from voicecraft_b200.voicecraft import _Prompt
    x6 = x[:, :6]
    for mask, xx, mode in (([4, 0], x6, 0), ([1, 0], x, 0), ([1, 0], x6, 1), ([0, 0], x6, 0)):
        p = _Prompt(m, xx, y)
        P = p.fill(0, 1)
        P.mode = mode
        P.align_heads = (C.c_uint32 * 2)(*mask)
        assert lib.vcb_prefill(eng, C.byref(P), 1, None) != 0
    assert lib.vcb_counter(eng, b"kv_pages_free") == free
    assert all(lib.vcb_release(eng, s, 1) == 0 for s in range(8))
    # a zero cap refuses every alignment
    cfg, m0 = _model("bf16", cap=0)
    with pytest.raises(ValueError, match="align_text_cap"):
        m0.inference_tts(x, xl, y, alignment=True)


@pytest.mark.gpu
def test_mega_same_alignment(monkeypatch):
    """VCB_MEGA=1: steps with alignment rows run the per-kernel chain, so the alignment and the tokens are the default's"""
    cfg, m = _model("bf16")
    x, xl, y = _utt(cfg, 4)
    a = _run(m, x, xl, y, 3, alignment=True)
    monkeypatch.setenv("VCB_MEGA", "1")
    cfg, m1 = _model("bf16")
    b = _run(m1, x, xl, y, 3, alignment=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[3].soft, b[3].soft)


@pytest.mark.gpu
def test_no_launch_without_alignment():
    """an engine with a cap but no aligning prompt launches the kernels of one without a cap, and allocates no log"""
    l, lib = _lib()
    counts = []
    for cap in (0, 32):
        cfg, m = _model("bf16", cap=cap)
        x, xl, y = _utt(cfg, 4)
        eng = m._engine()
        lib.vcb_set_option(eng, b"profile", 1)
        torch.manual_seed(1)
        m.inference_tts(x, xl, y, top_k=40)
        ms = (C.c_double * 7)()
        n = (C.c_int64 * 7)()
        l.check(lib.vcb_profile_read(eng, ms, n, 7))
        counts.append(list(n))
        assert lib.vcb_counter(eng, b"align_bytes") == 0
    assert counts[0] == counts[1]
