"""Repetition-aware sampling (RAS) and per-request length bounds in the fused sampler (include/vcb200.h vcb_sampling,
DESIGN.md section 2.2).

RAS is not in the reference, so the oracle here is a restatement of the rule on top of the pinned sampling step
(lm_oracle.sample_rows and the state machine of OracleLM._span_step): draw t with the reference's masks, temperature,
top-k, top-p and argmax(p / q1); count t in the last min(W, cur) tokens of its codebook in the current generation (the
tokens written, forced ones included); at >= c redraw t = argmax(p_full / q2), p_full the softmax of the row after the
masks and temperature only.  Forced tokens and the end-token triggers follow on the final t.  min_frames masks the end
token on codebook 0 while cur < min_frames; max_frames forces it at cur == max_frames like the length cap.

CPU: argument checks of every entry point and of the hook, c = ceil(tau * W), the restatement's window edges, need_seq,
the ABI.  GPU (-m gpu): the kernel through vcb_debug_sampler_ras against the restatement (probe noise for exact
thresholds, random rows outside the fp64 margin, the state machine with bounds); the device generator's two draws; the
engine against the oracle LM; every entry point with the controls on against its seeded single call; off bit for bit
equal to omitting the keywords; the bounds on frame counts and on admission.
"""
import ctypes as C
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import lm_oracle
from oracle.lm_oracle import OracleLM

MARGIN = 1e-5


def _lib():
    from voicecraft_b200 import _lib
    return _lib, _lib.load()


def _sp(top_k=-100, top_p=1.0, temperature=1.0, stop_repetition=0, silence=(), W=0, c=0, lo=0, hi=0):
    _l, _ = _lib()
    return _l.vcb_sampling(top_k=top_k, top_p=top_p, temperature=temperature, stop_repetition=stop_repetition,
                           n_silence=len(silence), silence_tokens=(C.c_int32 * 8)(*silence), ras_window=W,
                           ras_threshold=c, min_frames=lo, max_frames=hi)


# ==========================================================================================================================
# the restatement
# ==========================================================================================================================
def window_count(hist, k, tok, W, cur):
    """occurrences of tok among the last min(W, cur) entries of codebook k of hist (rows [K], oldest first)"""
    h = min(W, cur)
    return sum(int(r[k]) == int(tok) for r in hist[len(hist) - h:]) if h > 0 else 0


def redraw(row, temperature, q2):
    """argmax(p_full / q2), p_full = softmax(row / temperature) of the edited row, no top-k / top-p"""
    x = row / temperature if temperature != 1.0 else row.clone()
    return int(torch.argmax(F.softmax(x, dim=-1) / q2))


def span_step(c, st, logits, samp, ctl, y_cur_len, x_len, q1, q2, hist):
    """One step of OracleLM._span_step with RAS and the length bounds.  c: (n_codebooks, empty_token, eog, eos,
    encodec_sr); st as _span_step's (updated); logits [K, V] (edited in place); ctl = (W, thr, min_frames, max_frames);
    hist: the rows [K] this generation wrote so far.  Returns (tokens [K] int64, redrew [K] bool)."""
    K = c.n_codebooks
    W, thr, lo, hi = ctl
    tts = st["mode"] == "tts"
    E = (c.eos if c.eos > 0 else c.eog) if tts else c.eog
    n_eog, cur = sum(st["eog"]), st["cur"]
    if n_eog == 0:
        for k in range(1, K):
            logits[k][E] = -10000
            logits[k][c.empty_token] = -10000
        if tts and cur <= c.encodec_sr // 5:
            logits[0][E] = -10000
        if cur < lo:
            logits[0][E] = -10000
        OracleLM._silence_penalty(logits[0], st["prev"], st["consec"], samp)
    else:
        for k in range(n_eog + 1, K):
            logits[k][E] = -10000
            logits[k][c.empty_token] = -10000
    # a copy: sample_rows filters its argument in place at temperature 1, and the redraw needs the unfiltered row
    s = lm_oracle.sample_rows(logits.clone(), samp["top_k"], samp["top_p"], samp["temperature"], lambda shape: q1).view(-1)
    redrew = [False] * K
    if W > 0:
        for k in range(K):
            if window_count(hist, k, int(s[k]), W, cur) >= thr:
                s[k] = redraw(logits[k], samp["temperature"], q2[k])
                redrew[k] = True
    if n_eog == 0:
        if cur < K - 1:
            for jj in range(1, K - cur):
                s[-jj] = c.empty_token
        cap = x_len * (c.encodec_sr // 5) if tts else x_len * 10
        if (int(s[0]) == E or int(torch.argmax(logits[0], dim=-1)) == E or y_cur_len > cap
                or (hi > 0 and cur >= hi)):
            s[0] = E
            st["eog"][0] = True
        tok0 = int(s[0])
        st["consec"] = st["consec"] + 1 if (tok0 in samp["silence_tokens"] and tok0 == st["prev"]) else 0
        st["prev"] = tok0
    else:
        for k in range(n_eog):
            s[k] = c.empty_token
        s[n_eog] = E
        st["eog"][n_eog] = True
    return s, redrew


# ==========================================================================================================================
# CPU
# ==========================================================================================================================
def test_threshold_is_the_ceiling_of_tau_times_w_in_float64():
    from voicecraft_b200.voicecraft import sampling_controls
    assert sampling_controls(10, 0.1) == (10, 1, 0, 0)
    assert sampling_controls(10, 0.3) == (10, 3, 0, 0)
    assert sampling_controls(10, 0.31) == (10, 4, 0, 0)
    assert sampling_controls(32, 1.0) == (32, 32, 0, 0)
    assert sampling_controls(256, 1e-9) == (256, 1, 0, 0)
    assert sampling_controls() == (0, 0, 0, 0)
    assert sampling_controls(0, 0.5, 3, 7) == (0, 0, 3, 7)
    assert sampling_controls(min_frames=5, max_frames=5) == (0, 0, 5, 5)


BAD = [dict(ras_window=-1), dict(ras_window=257), dict(ras_window=2.0), dict(ras_window=True), dict(ras_tau=0.0),
       dict(ras_tau=1.5), dict(ras_tau=float("nan")), dict(min_frames=-1), dict(max_frames=0), dict(max_frames=-3),
       dict(min_frames=8, max_frames=7)]


def _cpu_model():
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny")
    m = VoiceCraft(cfg)
    m.load_state_dict(synthetic.make_state_dict(cfg, seed=0))
    x, xl, y = synthetic.synthetic_utterance(cfg, 0, text_len=6, prompt_frames=10)
    return cfg, m, x, xl, y


def _entry_points(m, x, xl, y):
    """every public entry point that takes sampling parameters, as callables of the control keywords"""
    from voicecraft_b200.voicecraft import ContinuousBatcher
    mi = torch.tensor([[[2, 5]]])
    return {
        "inference_tts": lambda **kw: m.inference_tts(x, xl, y, **kw),
        "inference_tts_batch": lambda **kw: m.inference_tts_batch(x, xl, y, batch_size=2, **kw),
        "inference": lambda **kw: m.inference(x, xl, y, mi, **kw),
        "inference_tts_many": lambda **kw: m.inference_tts_many([x], [y], **kw),
        "inference_many": lambda **kw: m.inference_many([x], [y], [mi], **kw),
        "open_tts_session": lambda **kw: m.open_tts_session([x], [y], **kw),
        "open_edit_session": lambda **kw: m.open_edit_session([x], [y], [mi], **kw),
        "inference_tts_stream": lambda **kw: m.inference_tts_stream(x, xl, y, None, **kw),
        "inference_stream": lambda **kw: m.inference_stream(x, xl, y, mi, None, **kw),
        "inference_tts_many_stream": lambda **kw: m.inference_tts_many_stream([x], [y], None, **kw),
        "inference_many_stream": lambda **kw: m.inference_many_stream([x], [y], [mi], None, **kw),
        "inference_long_tts": lambda **kw: m.inference_long_tts([x, x], y, **kw),
        "inference_long_tts_stream": lambda **kw: m.inference_long_tts_stream([x, x], y, None, **kw),
        "ContinuousBatcher": lambda **kw: ContinuousBatcher(m, **kw),
        "submit": lambda **kw: ContinuousBatcher(m).submit(x, y, seed=1, **kw),
        "submit long": lambda **kw: ContinuousBatcher(m).submit([x, x], y, seed=1, **kw),
        "submit edit": lambda **kw: ContinuousBatcher(m).submit(x, y, seed=1, mask_interval=mi, **kw),
    }


def test_every_entry_point_rejects_bad_controls_before_the_engine():
    """the checks run on the host before any slot is taken, so they need no GPU"""
    _, m, x, xl, y = _cpu_model()
    for name, call in _entry_points(m, x, xl, y).items():
        for kw in BAD:
            with pytest.raises(ValueError):
                call(**kw)
            assert m._eng is None, f"{name} {kw}: an engine was created"


def test_ras_with_host_noise_is_rejected():
    _, m, x, xl, y = _cpu_model()
    m.noise_fn = lambda shape, device=None: torch.ones(shape)
    calls = _entry_points(m, x, xl, y)
    for name, call in calls.items():
        if name == "ContinuousBatcher":
            continue                           # the batcher refuses host noise when it runs (existing behaviour)
        with pytest.raises(ValueError, match="device generator"):
            call(ras_window=8, ras_tau=0.5)
        assert m._eng is None, name
    m.noise_fn = None
    fns = [lambda shape, device=None: torch.ones(shape)]
    with pytest.raises(ValueError, match="device generator"):
        m.open_tts_session([x], [y], noise_fns=fns, ras_window=4)
    with pytest.raises(ValueError, match="device generator"):
        m.open_edit_session([x], [y], [torch.tensor([[[2, 5]]])], noise_fns=fns, ras_window=4)
    assert m._eng is None


def test_need_seq_with_and_without_max_frames():
    from voicecraft_b200.voicecraft import _Prompt
    cfg, m, x, xl, y = _cpu_model()
    K, x_len, rows = cfg.n_codebooks, x.shape[1], y.shape[1] + 1
    cap = x_len * (cfg.encodec_sr // 5)
    assert _Prompt(m, x, y).need_seq == x_len + max(rows, cap + 1) + K + 8
    assert _Prompt(m, x, y, max_frames=0).need_seq == _Prompt(m, x, y).need_seq
    for mf in (1, 5, cap - rows, cap, 10 * cap):
        assert _Prompt(m, x, y, max_frames=mf).need_seq == x_len + max(rows, min(cap, rows + mf) + 1) + K + 8, mf
    spans = [(1, 3), (5, 8)]
    full = _Prompt(m, x, y, spans)
    extra = (K + 3) * 3
    assert full.need_seq == x_len + max(int(full.y_tok.shape[0]), 10 * x_len + 1) + extra + 8
    for mf in (1, 4, 100):
        p = _Prompt(m, x, y, spans, max_frames=mf)
        r = int(p.y_tok.shape[0])
        assert p.need_seq == x_len + max(r, min(10 * x_len, r + 2 * mf) + 1) + extra + 8
        # conservative: each span writes at most mf + K sampled columns and 2 hand-over columns, up to the cap
        assert p.need_seq >= x_len + min(r + 2 * (mf + K + 2), 10 * x_len + K + 2) + 1


def _cfg(K=4, eos=0):
    return SimpleNamespace(n_codebooks=K, empty_token=252, eog=253, eos=eos, encodec_sr=75)


def test_restatement_window_edges():
    """fewer than W steps so far, count c - 1 against c, forced tokens inside the window"""
    c, K, V = _cfg(), 4, 256
    samp = dict(top_k=1, top_p=1.0, temperature=1.0, stop_repetition=0, silence_tokens=[])
    g = torch.Generator().manual_seed(0)
    lg = torch.randn(K, V, generator=g)
    a = [int(i) for i in lg.argmax(-1)]                     # top_k = 1: the first draw is the argmax
    q1 = torch.ones(K, V)
    q2 = torch.ones(K, V)
    probe = [(t + 1) % V for t in a]
    for k in range(K):
        q2[k, probe[k]] = 1e-30

    def step(hist, cur, W=6, thr=3, lo=0, hi=0):
        st = dict(eog=[False] * K, cur=cur, prev=None, consec=0, mode="tts")
        return span_step(c, st, lg.clone(), samp, (W, thr, lo, hi), 0, 100, q1, q2, hist)

    row = lambda t: torch.tensor(t)
    other = [(t + 7) % V for t in a]
    # count c - 1 = 2 inside the window: no redraw; c = 3: redraw picks the probe
    hist = [row(other)] * 4 + [row(a)] * 2
    s, red = step(hist, cur=40)
    assert not any(red) and s.tolist() == a
    s, red = step(hist + [row(a)], cur=40)
    assert all(red) and s.tolist() == probe
    # fewer than W steps so far: only the last cur rows count; older copies of the token are outside the window
    hist = [row(a)] * 3 + [row(other)] * 2
    s, red = step(hist, cur=2)
    assert not any(red)
    s, red = step(hist, cur=5)
    assert all(red)
    # the window ends W rows back
    hist = [row(a)] * 3 + [row(other)] * 6
    assert not any(step(hist, cur=40)[1])
    # forced tokens count: the empty token the first steps wrote for k > cur
    lg2 = torch.full((K, V), -5.0)
    lg2[:, c.empty_token] = 5.0                             # codebooks >= 1 mask it; codebook 0 draws it
    st = dict(eog=[False] * K, cur=3, prev=None, consec=0, mode="edit")
    hist = [row([c.empty_token] * K)] * 3
    s, red = span_step(c, st, lg2, samp, (4, 3, 0, 0), 0, 100, q1, q2, hist)
    assert red == [True, False, False, False] and int(s[0]) == probe[0]
    # the bounds: E masked below min_frames, forced at max_frames
    lgE = lg.clone()
    lgE[0, c.eog] = 50.0
    for cur, want in ((19, False), (20, True)):
        st = dict(eog=[False] * K, cur=cur, prev=None, consec=0, mode="tts")
        span_step(c, st, lgE.clone(), samp, (0, 0, 20, 0), 0, 100, q1, q2, [])
        assert st["eog"][0] == want, cur
    for cur, want in ((29, False), (30, True)):
        st = dict(eog=[False] * K, cur=cur, prev=None, consec=0, mode="edit")
        span_step(c, st, lg.clone(), samp, (0, 0, 0, 30), 0, 100, q1, q2, [])
        assert st["eog"][0] == want, cur


def _ras_call(lib, logits_ptr, sp, n=1, K=4, V=16, state=(0, 0, 3, -1, 0, 1, 0), hist=True, redrew=True, noise=(None, None),
              threads=1):
    P = C.POINTER(C.c_int32)
    W = max(sp.ras_window, 1)
    st = np.array(state * n, np.int32)
    h = np.zeros(n * K * W, np.int32)
    tok, out, red = np.zeros(64, np.int32), np.zeros(64, np.int32), np.zeros(64, np.int32)
    return lib.vcb_debug_sampler_ras(logits_ptr, noise[0], noise[1], 1, 0, threads, C.byref(sp), n, K, V, 16, 17, 0, 50,
                                     st.ctypes.data_as(P), h.ctypes.data_as(P) if hist else None, tok.ctypes.data_as(P),
                                     out.ctypes.data_as(P), None, red.ctypes.data_as(P) if redrew else None)


def test_debug_sampler_ras_rejects_bad_arguments():
    """decided on the host before any allocation or launch"""
    _l, lib = _lib()
    logits = np.zeros(64, np.float32)
    ptr = logits.ctypes.data
    cases = {
        "W=0": (_sp(W=0), {}), "W=257": (_sp(W=257, c=1), {}), "c=0": (_sp(W=4, c=0), {}), "c>W": (_sp(W=4, c=5), {}),
        "min<0": (_sp(W=4, c=1, lo=-1), {}), "max<0": (_sp(W=4, c=1, hi=-1), {}), "min>max": (_sp(W=4, c=1, lo=5, hi=4), {}),
        "hist": (_sp(W=4, c=1), dict(hist=False)), "redrew": (_sp(W=4, c=1), dict(redrew=False)),
        "one noise plane": (_sp(W=4, c=1), dict(noise=(ptr, None))), "cur<0": (_sp(W=4, c=1), dict(state=(0, 0, -1, -1, 0, 1, 0))),
        "K=9": (_sp(W=4, c=1), dict(K=9)), "V=3073": (_sp(W=4, c=1), dict(V=3073)), "no noise": (_sp(W=4, c=1), dict(threads=0)),
    }
    for name, (sp, kw) in cases.items():
        rc = _ras_call(lib, ptr, sp, **kw)
        msg = (lib.vcb_last_error() or b"").decode()
        assert rc != 0 and msg.startswith("vcb_debug_sampler_ras"), f"{name}: rc {rc}, {msg!r}"
    # the other hooks reject controls the engine rejects too
    P = C.POINTER(C.c_int32)
    st, tok, out = np.array([0, 0, 3, -1, 0, 1, 0], np.int32), np.zeros(8, np.int32), np.zeros(8, np.int32)
    rc = lib.vcb_debug_sampler(ptr, None, 1, 0, 1, C.byref(_sp(lo=3, hi=2)), 1, 4, 16, 16, 17, 0, 50, st.ctypes.data_as(P),
                               tok.ctypes.data_as(P), out.ctypes.data_as(P))
    assert rc != 0 and b"sampling controls" in lib.vcb_last_error()


def test_abi_new_fields_and_symbol():
    """vcb_sampling ends with the four controls (17 32-bit fields) and vcb_debug_sampler_ras is declared and exported"""
    import os
    import re
    _l, lib = _lib()
    assert C.sizeof(_l.vcb_sampling) == 17 * 4
    names = [f[0] for f in _l.vcb_sampling._fields_]
    assert names[-4:] == ["ras_window", "ras_threshold", "min_frames", "max_frames"]
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vcb200.h")).read()
    struct = re.search(r"typedef struct \{([^}]*)\} vcb_sampling;", hdr).group(1)
    assert re.findall(r"int32_t (\w+);", struct)[-4:] == names[-4:]
    assert "vcb_debug_sampler_ras" in _l.PROTOTYPES and hasattr(lib, "vcb_debug_sampler_ras")
    assert re.search(r"\bvcb_debug_sampler_ras\s*\(", hdr)


# ==========================================================================================================================
# GPU: the kernel through the hook
# ==========================================================================================================================
def _hook(logits, q1, q2, sp, specials, state, hist, seed=0, offset=0, threads=0, lp=False):
    """logits [n][K][V] (device), q1 / q2 [n*K][V] or None, hist [n][K][W] -> (tokens [n][K], state [n][4], redrew [n][K])"""
    _l, lib = _lib()
    n, K, V = logits.shape
    P = C.POINTER(C.c_int32)
    st = np.ascontiguousarray(state, dtype=np.int32)
    h = np.ascontiguousarray(hist, dtype=np.int32)
    assert h.shape == (n, K, sp.ras_window)
    tok, out, red = np.zeros((n, K), np.int32), np.zeros((n, 4), np.int32), np.zeros((n, K), np.int32)
    lpa = np.zeros((n, K), np.float32)
    _l.check(lib.vcb_debug_sampler_ras(logits.data_ptr(), None if q1 is None else q1.data_ptr(),
                                       None if q2 is None else q2.data_ptr(), seed, offset, threads, C.byref(sp), n, K, V,
                                       *specials, st.ctypes.data_as(P), h.ctypes.data_as(P), tok.ctypes.data_as(P),
                                       out.ctypes.data_as(P), lpa.ctypes.data_as(C.POINTER(C.c_float)) if lp else None,
                                       red.ctypes.data_as(P)))
    return (tok, out, red.astype(bool)) + ((lpa,) if lp else ())


@pytest.mark.gpu
@pytest.mark.parametrize("V", [4, 257, 1023, 2053, 3072])
@pytest.mark.parametrize("K", [4, 8])
def test_redraw_fires_at_exactly_the_threshold(V, K):
    """top_k = 1 makes the first draw the argmax; the second plane probes one index (1e-30 there, 1 elsewhere), so a
    redraw returns that index (chosen outside the top-k, as unlikely as the row allows).  Per row the argmax occurs
    0, c-1, c or W times among the visible window, with copies outside it (cur < W) that must not count."""
    W, thr = 8, 3
    g = torch.Generator().manual_seed(V * 10 + K)
    cases = [(cnt, cur) for cnt in (0, thr - 1, thr, W) for cur in (40, W)] + [(thr - 1, 5), (thr, 5), (1, 2)]
    n = len(cases)
    logits = torch.randn(n, K, V, generator=g) * 2.0
    a = logits.argmax(-1)
    probe = logits.argmin(-1) if V > 4 else (a + 1) % V
    q2 = torch.ones(n * K, V)
    q2[torch.arange(n * K), probe.view(-1)] = 1e-30
    hist = np.zeros((n, K, W), np.int32)
    state, want_red = [], np.zeros((n, K), bool)
    for i, (cnt, cur) in enumerate(cases):
        h = min(W, cur)
        for k in range(K):
            t = int(a[i, k])
            col = [(t + 1 + j % (V - 1)) % V for j in range(W)]     # never t
            for j in range(min(cnt, h)):                # copies inside the visible window (the last h entries)
                col[W - 1 - j] = t
            for j in range(W - h):                      # and copies in the part the window does not reach
                col[j] = t
            hist[i, k] = col
            want_red[i, k] = min(cnt, h) >= thr
        state.append([0, 0, cur, -1, 0, 1, 0])
    sp = _sp(top_k=1, W=W, c=thr)
    tok, _, red = _hook(logits.cuda(), torch.ones(n * K, V).cuda(), q2.cuda(), sp, (V, V + 1, 0, 50), state, hist)
    assert np.array_equal(red, want_red), f"redraw flags\n{red.astype(int)}\nwant\n{want_red.astype(int)}"
    want = np.where(want_red, probe.numpy(), a.numpy())
    for i, (cnt, cur) in enumerate(cases):
        if cur < K - 1:
            want[i, cur + 1:] = V                       # forced empty tokens overwrite the draw
    assert np.array_equal(tok, want), f"tokens\n{tok}\nwant\n{want}"
    assert want_red.any() and not want_red.all()


@pytest.mark.gpu
@pytest.mark.parametrize("V", [4, 257, 1023, 3072])
@pytest.mark.parametrize("K", [4, 8])
def test_random_rows_match_the_restatement(V, K):
    """random rows, random q1 / q2 and histories seeded with the restatement's first draw so that about half the rows
    redraw; tokens equal wherever every fp64 p/q decision involved clears the runner-up by more than 1 + 1e-5"""
    W, thr, n = 6, 2, 24
    g = torch.Generator().manual_seed(V + 100 * K)
    failures, checked, fired = [], 0, 0
    for top_k, temp in ((-100, 1.0), (40, 0.7), (3, 1.3)):
        logits = torch.randn(n, K, V, generator=g) * 3.0
        q1 = torch.empty(n * K, V).exponential_(1, generator=g)
        q2 = torch.empty(n * K, V).exponential_(1, generator=g)
        first = lm_oracle.sample_rows(logits.view(n * K, V).clone(), top_k, 1.0, temp, lambda s: q1).view(n, K)
        hist = torch.randint(0, V, (n, K, W), generator=g)
        for i in range(0, n, 2):
            hist[i, :, :thr] = first[i][:, None]
        tok, _, red = _hook(logits.cuda(), q1.cuda(), q2.cuda(), _sp(top_k=top_k, temperature=temp, W=W, c=thr),
                            (V, V + 1, 0, 50), [[0, 0, 40, -1, 0, 1, 0]] * n, hist.numpy())
        x = logits.view(n * K, V) / temp if temp != 1.0 else logits.view(n * K, V)
        kept = torch.isfinite(lm_oracle.filter_top_k_top_p(x.clone(), top_k=top_k))

        def gap(keep, q):
            s = torch.where(keep, torch.softmax(torch.where(keep, x.double(), torch.tensor(-np.inf, dtype=torch.float64)), -1)
                            / q.double(), torch.tensor(-1.0, dtype=torch.float64))
            t2 = s.topk(min(2, V), -1).values
            return torch.where(t2[:, -1] > 0, t2[:, 0] / t2[:, -1] - 1, torch.tensor(np.inf, dtype=torch.float64))
        g1, g2 = gap(kept, q1), gap(torch.ones_like(kept), q2)
        for r in range(n * K):
            i, k = divmod(r, K)
            cnt = int((hist[i, k] == first[i, k]).sum())
            want_red = cnt >= thr
            if g1[r] <= MARGIN or (want_red and g2[r] <= MARGIN):
                continue
            checked += 1
            fired += want_red
            want = redraw(logits.view(n * K, V)[r], temp, q2[r]) if want_red else int(first[i, k])
            if bool(red[i, k]) != want_red or int(tok[i, k]) != want:
                failures.append(f"top_k={top_k} T={temp} row {i} k {k}: kernel {int(tok[i, k])} redrew {bool(red[i, k])}, "
                                f"restatement {want} redrew {want_red}")
    assert not failures, "\n".join(failures[:20])
    assert checked > 0.9 * 3 * n * K and fired > 0.2 * checked, (checked, fired)


SM_V, SM_EMPTY, SM_EOG, SM_SR, SM_XLEN = 256, 252, 253, 75, 3        # encodec_sr // 5 = 15; caps: tts 45, edit 30


@pytest.mark.gpu
@pytest.mark.parametrize("K", [4, 8])
@pytest.mark.parametrize("eos", [254, 0])
def test_state_machine_with_bounds_and_ras_matches_the_restatement(K, eos):
    """the end token masked on codebook 0 below min_frames and forced at max_frames, exactly there, in TTS and in an edit
    span; RAS on the same rows with forced tokens in the histories"""
    g = torch.Generator().manual_seed(K * 31 + eos)
    V, lo, hi, W, thr = SM_V, 20, 30, 4, 1
    c = _cfg(K, eos)
    c.empty_token, c.eog, c.encodec_sr = SM_EMPTY, SM_EOG, SM_SR
    rows = []
    for mode in (0, 1):
        E = (eos if eos > 0 else SM_EOG) if mode == 0 else SM_EOG
        for cur in (lo - 1, lo, hi - 1, hi, hi + 1, 1, K):
            for boost in (True, False):
                lg = torch.randn(K, V, generator=g) * 2.0
                q1 = torch.empty(K, V).exponential_(1, generator=g)
                q2 = torch.empty(K, V).exponential_(1, generator=g)
                if boost:                       # the end token would win codebook 0 unless masked
                    lg[0, E] = 12.0
                    q1[0, E] = 1e-3
                else:                           # ... or is never drawn unless forced
                    lg[0, E] = -5.0
                    q1[0, E] = 1e3
                if eos > 0:
                    lg[:, SM_EOG if mode == 0 else eos] = -10000.0       # the callers' edit (lm_oracle.py:321, :508)
                hist = lg.topk(W, -1).indices.T.contiguous()              # each row's W favourites: most draws repeat
                if cur < K:
                    hist[-2, 1:] = SM_EMPTY                                # forced empties in the window
                rows.append((mode, cur, lg, q1, q2, hist))
    n = len(rows)
    state = [[m_, 0, cur, -1, 0, SM_XLEN, 5] for (m_, cur, *_r) in rows]
    tok, out, red = _hook(torch.stack([r[2] for r in rows]).cuda(), torch.cat([r[3] for r in rows]).cuda(),
                          torch.cat([r[4] for r in rows]).cuda(), _sp(40, 0.9, 0.8, W=W, c=thr, lo=lo, hi=hi),
                          (SM_EMPTY, SM_EOG, eos, SM_SR), state, np.stack([r[5].T.numpy() for r in rows]))
    samp = dict(top_k=40, top_p=0.9, temperature=0.8, stop_repetition=0, silence_tokens=[])
    failures, ended = [], {}
    for i, (mode, cur, lg, q1, q2, hist) in enumerate(rows):
        st = dict(eog=[False] * K, cur=cur, prev=None, consec=0, mode="tts" if mode == 0 else "edit")
        s, rr = span_step(c, st, lg.clone(), samp, (W, thr, lo, hi), 5, SM_XLEN, q1, q2, [h for h in hist])
        n_after = sum(st["eog"])
        ended[(mode, cur, i % 2 == 0)] = n_after == 1
        if tok[i].tolist() != s.tolist() or red[i].tolist() != rr or int(out[i, 2]) != n_after:
            failures.append(f"mode={mode} cur={cur} row {i}: tokens {tok[i].tolist()} / {s.tolist()}, redrew "
                            f"{red[i].astype(int).tolist()} / {[int(v) for v in rr]}, n_eog {out[i, 2]} / {n_after}")
    assert not failures, "\n".join(failures)
    for mode in (0, 1):
        assert not ended[(mode, lo - 1, True)] and ended[(mode, lo, True)]        # min_frames: masked until cur == lo
        assert not ended[(mode, hi - 1, False)] and ended[(mode, hi, False)]      # max_frames: forced at cur == hi
    assert red.any()


@pytest.mark.gpu
def test_device_noise_is_two_consecutive_torch_draws():
    """noise pointers null: q1 at (seed, offset) and q2 at the next offset of the stream equal two consecutive
    torch.empty(K*V, device="cuda").exponential_(1) under that generator state"""
    from voicecraft_b200.voicecraft import VoiceCraft
    V, K, n, W = 2053, 4, 12, 64
    seed, offset = 0x5EED1234ABC, 8
    logits = (torch.randn(n, K, V, generator=torch.Generator().manual_seed(3)) * 0.5).cuda()
    gen = torch.cuda.default_generators[0]
    saved = gen.get_state()
    try:
        gen.manual_seed(seed)
        gen.set_offset(offset)
        d1 = torch.empty(K * V, device="cuda").exponential_(1)
        d2 = torch.empty(K * V, device="cuda").exponential_(1)
        after = gen.get_offset()
    finally:
        gen.set_state(saved)
    threads = VoiceCraft._rng_threads(torch.device("cuda", 0), K * V)
    step = ((K * V - 1) // (4 * threads) + 1) * 4
    assert after == offset + 2 * step
    # the top 64 tokens of each row in the history of even rows (the first draw, in the top 40, always repeats), tokens
    # far below them in odd rows (never)
    order = logits.argsort(-1, descending=True).cpu()
    hist = np.where((np.arange(n) % 2 == 0)[:, None, None], order[:, :, :W].numpy(), order[:, :, -W:].numpy())
    sp = _sp(40, 0.9, 0.8, W=W, c=1)
    specials = (V, V + 1, 0, 50)
    state = [[0, 0, 70, -1, 0, 1, 0]] * n
    dev, _, rd = _hook(logits, None, None, sp, specials, state, hist, seed=seed, offset=offset, threads=threads)
    fed, _, rf = _hook(logits, d1.view(K, V).repeat(n, 1).contiguous(), d2.view(K, V).repeat(n, 1).contiguous(), sp,
                       specials, state, hist)
    assert np.array_equal(dev, fed) and np.array_equal(rd, rf), f"device\n{dev}\nfed\n{fed}"
    assert rd[0::2].all() and not rd[1::2].any()


# ==========================================================================================================================
# GPU: the engine
# ==========================================================================================================================
KW = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)


def _lm(kv="bf16", weights="bf16", eos_bias=3.0, eog_bias=None, max_slots=8, seed=3, no_end=False, repeat=None,
        max_seq_len=512, kv_pool_gb=None, audio_only=False):
    """tiny LM; codebook 0's end token gets eos_bias (TTS ends) and eog eog_bias (edit spans end); no_end: the heads put no
    mass on the non-audio tokens (only a forced end ends); audio_only: none on the non-audio tokens but the end tokens of
    codebook 0 (every generated frame decodes to audio); repeat: a logit bias on audio token 5 in every codebook, so
    that draws repeat"""
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=seed)
    if no_end:
        for k in range(cfg.n_codebooks):
            for t in (cfg.empty_token, cfg.eog, cfg.audio_pad_token, cfg.eos):
                sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    else:
        if audio_only:
            for k in range(cfg.n_codebooks):
                for t in (cfg.empty_token, cfg.eog, cfg.audio_pad_token, cfg.eos):
                    if not (k == 0 and t in (cfg.eos, cfg.eog)):
                        sd[f"predict_layer.{k}.2.bias"][t] = -1e4
        sd["predict_layer.0.2.bias"][cfg.eos] += eos_bias
        if eog_bias is not None:
            sd["predict_layer.0.2.bias"][cfg.eog] = eog_bias
    if repeat is not None:
        for k in range(cfg.n_codebooks):
            sd[f"predict_layer.{k}.2.bias"][5] += repeat
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    m = m.to("cuda").eval()
    m.configure_engine(kv_dtype=kv, weight_dtype=weights, max_slots=max_slots, max_seq_len=max_seq_len,
                       kv_pool_gb=kv_pool_gb)
    return cfg, sd, m


def _utt(cfg, seed, text_len=12, frames=30):
    from voicecraft_b200 import synthetic
    x, xl, y = synthetic.synthetic_utterance(cfg, seed, text_len=text_len, prompt_frames=frames)
    return x.cuda(), xl.cuda(), y.cuda()


def _bits(t):
    return t.cpu().contiguous().view(torch.int32)


def _flat(r):
    return [r] if torch.is_tensor(r) else [t for x in r for t in _flat(x)]


def _same(p, q):
    """bit for bit, NaN included"""
    return p.dtype == q.dtype and p.shape == q.shape and p.cpu().numpy().tobytes() == q.cpu().numpy().tobytes()


def _draw_step(m, n_copies=1):
    K, V = m.args.n_codebooks, m.n_audio_tokens[0]
    threads = m._rng_threads(torch.device("cuda", 0), n_copies * K * V)
    return ((n_copies * K * V - 1) // (4 * threads) + 1) * 4


@pytest.mark.gpu
def test_rng_offset_advances_two_draws_per_step_under_ras():
    cfg, _, m = _lm(no_end=True)
    x, _, y = _utt(cfg, 7, 10, 20)
    for W, per in ((0, 1), (8, 2)):
        sess = m.open_tts_session([x], [y], seeds=[11], ras_window=W, ras_tau=0.5, **KW)
        try:
            sess.sample()
            for _ in range(9):
                sess.step()
            st = sess.poll()
            assert st[0].n_steps == 10
            assert st[0].rng_offset == per * 10 * _draw_step(m), (W, st[0].rng_offset)
        finally:
            sess.close()


def _oracle_tts(o, x, y, samp, ctl, seed):
    """OracleLM.inference_tts with span_step, the noise two torch draws per step from a CUDA generator seeded `seed`.
    Returns (gen [1,K,G], redraws)."""
    c = o.c
    K, V = c.n_codebooks, o.sd["predict_layer.0.2.weight"].shape[0]
    g = torch.Generator(device="cuda").manual_seed(seed)
    draw = lambda: torch.empty(K, V, device="cuda").exponential_(1, generator=g).cpu()
    y = y.cpu().transpose(2, 1)
    x_in = o.embed_text(x.cpu())
    prompt = o._delay(y[0])[:, : -(K - 1)]
    emb = o.embed_codes(prompt.unsqueeze(-1)).transpose(1, 0)
    y_in = o.pos_audio(emb)
    st = dict(eog=[False] * K, cur=0, prev=None, consec=0, mode="tts")
    cache = dict(kv=None, on=True)
    rows, n_red = [], 0
    while True:
        out = o.dec_forward(x_in, y_in, cache)
        logits = o.heads(out[:, -1:]).squeeze(0)
        if c.eos > 0:
            logits[:, c.eog] = -10000.0
        q1, q2 = draw(), draw()
        s, red = span_step(c, st, logits, samp, ctl, y_in.shape[1], x.shape[1], q1, q2, rows)
        st["cur"] += 1
        rows.append(s.clone())
        n_red += sum(red)
        if sum(st["eog"]) == K:
            break
        emb = torch.cat([emb, o.embed_codes(s.view(K, 1)).sum(dim=0, keepdim=True).view(1, 1, -1)], dim=1)
        y_in = o.pos_audio(emb)
    return o._undelay(rows).unsqueeze(0), n_red


@pytest.mark.gpu
def test_engine_session_with_ras_equals_the_oracle_lm():
    cfg, sd, m = _lm(eos_bias=1.0, repeat=3.0)
    o = OracleLM(cfg, sd, kv_round_bf16=True)
    samp = dict(top_k=40, top_p=0.9, temperature=1.0, stop_repetition=3, silence_tokens=[1388, 1898, 131])
    total = 0
    for i, (W, tau, lo, hi) in enumerate(((10, 0.1, 0, 0), (4, 0.25, 12, 0), (10, 0.2, 0, 15))):
        x, _, y = _utt(cfg, 30 + i, 4, 12)
        want, n_red = _oracle_tts(o, x, y, samp, (W, math.ceil(tau * W), lo, hi), 70 + i)
        (res, gen), = m.inference_tts_many([x], [y], seeds=[70 + i], ras_window=W, ras_tau=tau, min_frames=lo,
                                           max_frames=hi or None, **{k: samp[k] for k in ("top_k", "top_p", "temperature",
                                                                                           "stop_repetition")})
        assert torch.equal(gen.cpu(), want), f"case {i}: engine {gen.shape} / oracle {want.shape}"
        total += n_red
    assert total > 5, f"the biased model should make RAS redraw ({total} redraws)"


RAS = dict(ras_window=8, ras_tau=0.25, min_frames=3, max_frames=24)


@pytest.mark.gpu
@pytest.mark.parametrize("kv,weights", [("bf16", "bf16"), ("fp8", "int8")])
def test_controls_off_are_bit_identical_to_omitting_them(kv, weights):
    from voicecraft_b200.voicecraft import ContinuousBatcher
    off = dict(ras_window=0, min_frames=0, max_frames=None)
    cfg, _, m = _lm(kv, weights, eog_bias=2.5)
    gen = torch.cuda.default_generators[0]
    x, xl, y = _utt(cfg, 95, 10, 30)
    mi = torch.tensor([[[5, 9], [14, 20]]])
    calls = [lambda **kw: m.inference_tts(x, xl, y, logprobs=True, **KW, **kw),
             lambda **kw: m.inference_tts_batch(x, xl, y, batch_size=3, logprobs=True, **KW, **kw),
             lambda **kw: m.inference(x, xl, y, mi, logprobs=True, **KW, **kw),
             lambda **kw: m.inference_long_tts([x, x[:, :6]], y, logprobs=True, **KW, **kw)]
    for j, call in enumerate(calls):
        got = []
        for kw in ({}, off):
            torch.manual_seed(21 + j)
            r = call(**kw)
            got.append((r, gen.get_offset()))
        (a, oa), (b, ob) = got
        assert oa == ob, j
        fa, fb = _flat(a), _flat(b)
        assert len(fa) == len(fb) and all(_same(p, q) for p, q in zip(fa, fb)), j
    # a session and a batcher under a KV budget that swaps
    _, _, m2 = _lm(kv, weights, no_end=True, max_slots=4)
    utts = [_utt(cfg, 70 + i, 40, 9 + 3 * i) for i in range(6)]
    pb = _lib()[1].vcb_counter(m2._engine(), b"kv_page_bytes")
    m2.configure_engine(kv_dtype=kv, weight_dtype=weights, kv_pool_gb=12.5 * pb / 1e9, max_slots=4, max_seq_len=512)
    outs = []
    for kw in ({}, off):
        cb = ContinuousBatcher(m2, max_concurrency=4, poll_every=5, **KW, **kw)
        for i, (x_, _, y_) in enumerate(utts):
            cb.submit(x_, y_, seed=500 + i)
        outs.append((cb.run(), cb.logprobs, cb.stats["swap_outs"]))
        sess = m2.open_tts_session([u[0] for u in utts[:2]], [u[2] for u in utts[:2]], seeds=[1, 2], **KW, **kw)
        sess.sample()
        for _ in range(12):
            sess.step()
        outs[-1] += ([m2._read_rows(sess.eng, s, sess.poll()[j].n_steps, sess.stream) for j, s in enumerate(sess.slots)],
                     [int(s.rng_offset) for s in sess.poll()])
        sess.close()
    (r0, l0, s0, t0, o0), (r1, l1, s1, t1, o1) = outs
    assert s0 > 0 and s0 == s1
    assert all(torch.equal(a[1], b[1]) and torch.equal(_bits(p), _bits(q)) for a, b, p, q in zip(r0, r1, l0, l1))
    assert all(np.array_equal(a, b) for a, b in zip(t0, t1)) and o0 == o1


@pytest.mark.gpu
def test_batcher_tickets_with_mixed_controls_equal_their_seeded_single_calls():
    """run(), stream() and a KV budget that swaps: every ticket equals its seeded single call, RAS, bounds or neither"""
    from voicecraft_b200.voicecraft import ContinuousBatcher
    from oracle import encodec_oracle as eo
    from voicecraft_b200.tokenizer import AudioTokenizer
    cfg, _, m = _lm(eos_bias=1.0, eog_bias=1.0, repeat=2.0, max_slots=4, audio_only=True)
    utts = [_utt(cfg, 100 + i, 6 + 2 * i, 14 + 5 * i) for i in range(5)]
    seeds = [40 + i for i in range(5)]
    per = [dict(RAS), {}, dict(ras_window=16, ras_tau=0.1), dict(min_frames=12), dict(max_frames=9)]
    singles = []
    for (x, xl, y), s, kw in zip(utts, seeds, per):
        torch.manual_seed(s)
        singles.append(m.inference_tts(x, xl, y, logprobs=True, **KW, **kw))
    assert singles[4][1].shape[-1] <= 9 and singles[3][1].shape[-1] >= 12

    def fill(cb):
        for (x, _, y), s, kw in zip(utts, seeds, per):
            cb.submit(x, y, seed=s, **kw)

    def check(results, lps):
        for i, (r, g, lp) in enumerate(singles):
            assert torch.equal(results[i][1], g) and torch.equal(_bits(lps[i]), _bits(lp)), i
    cb = ContinuousBatcher(m, max_concurrency=3, poll_every=3, **KW)
    fill(cb)
    check(cb.run(), cb.logprobs)
    ecfg = eo.default_config()
    tok = AudioTokenizer(device="cuda:0", config=ecfg, state_dict=eo.make_state_dict(ecfg, seed=5))
    cb = ContinuousBatcher(m, max_concurrency=3, poll_every=3, **KW)
    fill(cb)
    chunks = {}
    for i, wav, _ in cb.stream(tok, chunk_frames=8):
        chunks.setdefault(i, []).append(wav)
    check(cb.results, cb.logprobs)
    for i, (r, g, lp) in enumerate(singles):             # streams equal decoding the whole result
        if g.shape[-1]:
            want = tok.decode_codes(g)
            assert torch.equal(torch.cat(chunks[i], -1), want), i
    # through swaps under a KV budget: the tickets run to their bounds (no end token otherwise)
    _, _, m2 = _lm(no_end=True, max_slots=4)
    long_utts = [_utt(cfg, 70 + i, 40, 9 + 3 * i) for i in range(6)]
    kws = [dict(RAS), dict(ras_window=4, ras_tau=0.5), {}, dict(max_frames=150), dict(RAS), {}]

    def run():
        cb = ContinuousBatcher(m2, max_concurrency=4, poll_every=5, **KW)
        for i, ((x, _, y), kw) in enumerate(zip(long_utts, kws)):
            cb.submit(x, y, seed=500 + i, **kw)
        return cb, cb.run()
    free, plain = run()
    assert free.stats["swap_outs"] == 0
    pb = _lib()[1].vcb_counter(m2._engine(), b"kv_page_bytes")
    m2.configure_engine(kv_pool_gb=12.5 * pb / 1e9, max_slots=4, max_seq_len=512)
    cb, got = run()
    assert cb.stats["swap_outs"] > 0, cb.stats
    for i in range(6):
        assert torch.equal(got[i][1], plain[i][1]) and torch.equal(_bits(cb.logprobs[i]), _bits(free.logprobs[i])), i
    for i in range(6):
        x, xl, y = long_utts[i]
        torch.manual_seed(500 + i)
        assert torch.equal(m2.inference_tts(x, xl, y, **KW, **kws[i])[1], got[i][1]), i


@pytest.mark.gpu
def test_best_of_long_and_single_streams_with_controls():
    from voicecraft_b200.voicecraft import ContinuousBatcher
    from oracle import encodec_oracle as eo
    from voicecraft_b200.tokenizer import AudioTokenizer
    cfg, _, m = _lm(eos_bias=1.5, eog_bias=2.5, repeat=2.0, audio_only=True)
    gen = torch.cuda.default_generators[0]
    x, xl, y = _utt(cfg, 90, 10, 25)
    # a best-of group in the batcher equals inference_tts_batch
    torch.manual_seed(3)
    r1, g1, lp1 = m.inference_tts_batch(x, xl, y, batch_size=3, logprobs=True, **KW, **RAS)
    cb = ContinuousBatcher(m, max_concurrency=4, **KW)
    cb.submit(x, y, seed=3, best_of=3, **RAS)
    (r, g), = cb.run()
    assert torch.equal(g, g1) and torch.equal(_bits(cb.logprobs[0]), _bits(lp1))
    # a long ticket equals the loop of inference_tts calls, the offsets handed over
    xs = [x, x[:, :5], x[:, 3:9]]
    torch.manual_seed(8)
    loop = [m.inference_tts(xi, torch.tensor([xi.shape[1]]), y, **KW, **RAS) for xi in xs]
    off = gen.get_offset()
    torch.manual_seed(8)
    long = m.inference_long_tts(xs, y, **KW, **RAS)
    assert gen.get_offset() == off
    assert all(torch.equal(a[1], b[1]) for a, b in zip(loop, long))
    # streams equal decoding the whole result
    ecfg = eo.default_config()
    tok = AudioTokenizer(device="cuda:0", config=ecfg, state_dict=eo.make_state_dict(ecfg, seed=5))
    torch.manual_seed(8)
    s = m.inference_long_tts_stream(xs, y, tok, chunk_frames=6, **KW, **RAS)
    wav = torch.cat([c for c in s], -1)
    assert torch.equal(wav, torch.cat([tok.decode([(b[1], None)]) for b in long], -1))
    assert all(torch.equal(a[1], b[1]) for a, b in zip(s.results, long))
    torch.manual_seed(9)
    res, g9 = m.inference_tts(x, xl, y, **KW, **RAS)
    torch.manual_seed(9)
    s = m.inference_tts_stream(x, xl, y, tok, chunk_frames=5, **KW, **RAS)
    wav = torch.cat([c for c in s], -1)
    assert torch.equal(s.result[1], g9) and torch.equal(wav, tok.decode([(g9, None)]))
    mi = torch.tensor([[[4, 9], [15, 19]]])
    torch.manual_seed(10)
    e = m.inference(x, xl, y, mi, **KW, **RAS)
    torch.manual_seed(10)
    s = m.inference_stream(x, xl, y, mi, tok, chunk_frames=5, **KW, **RAS)
    wav = torch.cat([c for c in s], -1)
    assert torch.equal(s.result, e) and torch.equal(wav, tok.decode_codes(e))


@pytest.mark.gpu
def test_bounds_hold_exactly():
    cfg, _, m = _lm(no_end=True)
    x, xl, y = _utt(cfg, 5, 20, 12)
    for mf in (1, 7, 33):
        torch.manual_seed(mf)
        _, g = m.inference_tts(x, xl, y, max_frames=mf, **KW)
        assert g.shape[-1] == mf, (mf, g.shape)
        torch.manual_seed(mf)
        (_, gb), = m.inference_tts_many([x], [y], seeds=[mf], max_frames=mf, ras_window=8, ras_tau=0.3, **KW)
        assert gb.shape[-1] == mf
    T = y.shape[1]
    mi = torch.tensor([[[2, 5], [7, 11]]])
    for mf in (1, 6):
        res = m.inference(x, xl, y, mi, max_frames=mf, **KW)
        assert res.shape[-1] == T - 3 - 4 + 2 * mf, (mf, res.shape)    # each span generated mf frames
    # the end token favoured: min_frames holds it back
    cfg, _, m = _lm(eos_bias=12.0, eog_bias=12.0)
    x, xl, y = _utt(cfg, 6, 20, 12)
    torch.manual_seed(4)
    _, g = m.inference_tts(x, xl, y, **KW)
    assert g.shape[-1] < 40
    for lo in (g.shape[-1] + 5, 40):
        torch.manual_seed(4)
        _, g2 = m.inference_tts(x, xl, y, min_frames=lo, **KW)
        assert g2.shape[-1] >= lo, (lo, g2.shape)
    e = m.inference(x, xl, y, mi, **KW)
    e2 = m.inference(x, xl, y, mi, min_frames=9, **KW)
    assert e2.shape[-1] >= T - 7 + 2 * 9 > e.shape[-1]


@pytest.mark.gpu
def test_a_bounded_ticket_is_admitted_where_the_unbounded_one_does_not_fit():
    """a best-of-2 group holds its full reservation: ceil(max_seq_len / 64) pages per copy, the engine sized by the
    tickets' need_seq.  With 10 pages, the bounded ticket (need_seq <= 256: 4 + 4 pages) runs; the unbounded one (cap
    400 frames: 512 positions, 8 + 8 pages) cannot"""
    from voicecraft_b200 import _lib as L
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, _, m = _lm(no_end=True, max_slots=4, max_seq_len=256)
    pb = _lib()[1].vcb_counter(m._engine(), b"kv_page_bytes")
    m.configure_engine(kv_pool_gb=10.5 * pb / 1e9, max_slots=4, max_seq_len=256)
    x, _, y = _utt(cfg, 8, 40, 10)
    cb = ContinuousBatcher(m, max_concurrency=2, **KW)
    cb.submit(x, y, seed=1, best_of=2, max_frames=20)
    (_, g), = cb.run()
    assert g.shape[-1] == 20
    cb = ContinuousBatcher(m, max_concurrency=2, **KW)
    cb.submit(x, y, seed=1, best_of=2)
    with pytest.raises(L.VcbError, match="KV pool smaller"):
        cb.run()
