"""Token log-probabilities (DESIGN.md section 2.2): what the fused sampler stores next to every token it writes, and how
the results carry it.

The value.  For the token tok written for codebook k at a step, lp = (u_tok - M) - log sum_v exp(u_v - M) with u the raw
logit row of that step and codebook (bias included, before the reference's edits, temperature, top-k and top-p) and
M = max_v u_v.  The checks compare it to the fp64 log-softmax of the same fp32 row.

The bound.  With U = 2^-24 (half an fp32 ulp, relative), n_t = ceil(V / 256) entries per thread and L = 12 merges on any
path from a thread to the block (5 warp-shuffle levels, then thread 0 folds the 8 warp totals in order):
  * a thread sums exp(u - m_t) over its n_t entries in index order (m_t its own max, so its sum S_t >= 1): each expf is
    within 2 ulp (4U relative, the CUDA math library's bound), the rounded argument moves a term e^x by at most
    U |x| e^x <= U / e, and n_t - 1 additions add U each: relative error <= U (n_t - 1 + n_t (4 + 1/e));
  * a merge (m, s) + (m', s') -> (M, s + s' expf(m' - M)), m <= M = the part's max (exactly, fmaxf), costs expf 4U, the
    product U, the sum U, and the rounded argument U |x| of the scaled part, which is at most U ln V of the merged sum
    (the scaled part is at most n' e^x of it): <= U (6 + ln V) per merge;
  * so the sum S carries a relative error delta_S <= U (n_t - 1 + n_t (4 + 1/e) + L (6 + ln V)), which moves log S by
    at most delta_S; logf adds 1 ulp <= 2U log S <= 2U ln V; u_tok - M is rounded once (U |u_tok - M|) and the final
    difference once (U (|u_tok - M| + ln V)).
  B(gap, V) = 2U gap + delta_S + 3U ln V (times 1.01 for second-order terms), gap = |u_tok - M|.  At V = 3072 that is
  2.4e-7 gap + 1.6e-5; gap reaches 2e4 in the +-1e4 rows (B = 4.8e-3) and 1e4 for the forced tokens the engine writes
  against its -1e4 head biases.
Each check prints the worst fraction of B it reached.

CPU: the un-delay of the log-probability rows in _Prompt.result (TTS, edits of 1 to 3 spans, a truncated session), from
synthetic rows.  GPU (-m gpu): the kernel through vcb_debug_sampler_lp on planted rows; the engine at every step against
the step's vcb_debug_logits rows (KV bf16 / fp32 / fp8, int8 weights, the persistent step kernel, best-of-N, an edit of
two spans); the public calls, the batch and the batcher (run, stream, swaps) against seeded single calls, bit for bit; and
the 830M fixture's oracle logits.
"""
import ctypes as C
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

U = 2.0 ** -24
MERGES = 12
WORST = {}                      # check -> worst fraction of the bound reached (printed at the end of the module)


def lp_bound(gap, V):
    """the bound of the module docstring for |u_tok - M| = gap (array) and V entries"""
    n_t = -(-V // 256)
    d_s = U * (n_t - 1 + n_t * (4 + 1 / math.e) + MERGES * (6 + math.log(V)))
    return 1.01 * (2 * U * np.asarray(gap, np.float64) + d_s + 3 * U * math.log(V))


def lp_ref(L, tok):
    """fp64 log-softmax of fp32 rows L [..., V] at tok [...], and |u_tok - M|"""
    L = np.asarray(L, np.float64)
    M = L.max(-1)
    u = np.take_along_axis(L, np.asarray(tok, np.int64)[..., None], -1)[..., 0]
    lse = M + np.log(np.exp(L - M[..., None]).sum(-1))
    return u - lse, M - u


def check_lp(name, lp, L, tok):
    """lp [...] against lp_ref within lp_bound; records the worst fraction under `name`"""
    ref, gap = lp_ref(L, tok)
    err = np.abs(np.asarray(lp, np.float64) - ref)
    frac = err / lp_bound(gap, np.shape(L)[-1])
    worst = float(frac.max()) if frac.size else 0.0
    WORST[name] = max(WORST.get(name, 0.0), worst)
    assert np.isfinite(lp).all() and worst <= 1.0, f"{name}: worst {worst:.3g} of the bound, max err {err.max():.3g}"


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    for k, v in sorted(WORST.items()):
        print(f"[logprobs] {k}: worst |lp - fp64| = {v:.3g} of the bound")


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the un-delay in _Prompt.result
# ---------------------------------------------------------------------------------------------------------------------
def _cpu_model():
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny")
    return cfg, VoiceCraft(cfg)


def _tagged(rows):
    """log-probability rows that name their own (row, codebook): row r, codebook k -> -(r * 16 + k + 1)"""
    n, K = rows.shape
    return -(np.arange(n)[:, None] * 16 + np.arange(K)[None, :] + 1).astype(np.float32)


def _untag(lp):
    """(row, codebook) of every tagged entry of lp [K, n]"""
    v = (-lp - 1).astype(np.int64)
    return v // 16, v % 16


@pytest.mark.parametrize("done", [True, False])
def test_tts_logprobs_align_with_gen(done):
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import _Prompt
    cfg, m = _cpu_model()
    K = cfg.n_codebooks
    x, _, y = synthetic.synthetic_utterance(cfg, 5, 4, 9)
    p = _Prompt(m, x, y)
    rng = np.random.default_rng(3)
    G = 13
    rows = rng.integers(0, 2048, (G + K, K))
    if done:                                  # the end token in codebook 0, then the delayed ends
        for r in range(G, G + K):
            rows[r, : r - G] = cfg.empty_token
            rows[r, r - G] = cfg.eos
    else:                                     # a truncated session: no end yet, the still-delayed tail is dropped
        rows = rows[: G + K - 2]
    res, gen, lp = p.result(rows, SimpleNamespace(done=int(done)), _tagged(rows))
    n = G if done else G + K - 2 - K + 1
    assert gen.shape == lp.shape == (1, K, n) and lp.dtype == torch.float32
    r, k = _untag(lp[0].numpy())
    assert (k == np.arange(K)[:, None]).all()
    assert (r == np.arange(n)[None, :] + np.arange(K)[:, None]).all()       # frame t of codebook k: row t + k
    assert np.array_equal(gen[0].numpy(), rows[r, k])                       # element for element with gen
    assert torch.equal(p.result(rows, SimpleNamespace(done=int(done)))[1], gen)


@pytest.mark.parametrize("T,spans,gens", [
    (20, [(0, 5)], [7]),
    (24, [(3, 6), (6, 10)], [5, 0]),
    (30, [(0, 4), (9, 12), (25, 30)], [3, 6, 2]),
    (30, [(2, 4), (8, 12), (15, 21)], [0, 9, 1]),
])
def test_edit_logprobs_align_with_res(T, spans, gens):
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import _Prompt
    cfg, m = _cpu_model()
    K = cfg.n_codebooks
    x, _, y = synthetic.synthetic_utterance(cfg, 7, 4, T)
    p = _Prompt(m, x, y, spans)
    rng = np.random.default_rng(T)
    rows, ends = [], []
    for g in gens:
        for r in range(g + K):
            row = rng.integers(0, 2048, K)
            if r >= g:
                row[: r - g] = cfg.empty_token
                row[r - g] = cfg.eog
            rows.append(row)
        ends.append(len(rows))
    rows = np.array(rows, np.int64)
    st = SimpleNamespace(done=1, n_spans_done=len(spans), span_ends=ends + [0] * (8 - len(ends)))
    res, gen, lp = p.result(rows, st, _tagged(rows))
    assert gen is None and lp.shape == res.shape and lp.dtype == torch.float32
    lp, res = lp[0].numpy(), res[0].numpy()
    # NaN exactly on the frames copied from the original audio
    orig = np.zeros(res.shape[1], bool)
    f, c0 = 0, 0
    for (s0, s1), g in zip(spans + [(T, T)], gens + [0]):
        orig[f: f + s0 - c0] = True
        f, c0 = f + s0 - c0 + g, s1
    assert res.shape[1] == T - sum(e - s for s, e in spans) + sum(gens)
    assert (np.isnan(lp) == orig[None, :]).all()
    r, k = _untag(lp[:, ~orig])
    assert (k == np.arange(K)[:, None]).all()
    assert np.array_equal(res[:, ~orig], rows[r, k])                        # element for element with res


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the kernel through vcb_debug_sampler_lp
# ---------------------------------------------------------------------------------------------------------------------
def _lib():
    from voicecraft_b200 import _lib
    return _lib, _lib.load()


def _sp(top_k=-100, top_p=1.0, temperature=1.0, stop_repetition=0, silence=()):
    _l, _ = _lib()
    return _l.vcb_sampling(top_k=top_k, top_p=top_p, temperature=temperature, stop_repetition=stop_repetition,
                           n_silence=len(silence), silence_tokens=(C.c_int32 * 8)(*silence))


def _hook(logits, noise, sp, specials, state, lp=True, seed=0, threads=0):
    """logits [n][K][V] fp32 (device), noise [n*K][V] or None -> tokens [n][K], state [n][4], lp [n][K] (numpy)"""
    _l, lib = _lib()
    n, K, V = logits.shape
    st = np.ascontiguousarray(state, dtype=np.int32)
    tok, out, lps = np.zeros((n, K), np.int32), np.zeros((n, 4), np.int32), np.zeros((n, K), np.float32)
    P = C.POINTER(C.c_int32)
    args = (logits.data_ptr(), None if noise is None else noise.data_ptr(), seed, 0, threads, C.byref(sp), n, K, V,
            *specials, st.ctypes.data_as(P), tok.ctypes.data_as(P), out.ctypes.data_as(P))
    if lp:
        _l.check(lib.vcb_debug_sampler_lp(*args, lps.ctypes.data_as(C.POINTER(C.c_float))))
    else:
        _l.check(lib.vcb_debug_sampler(*args))
    return tok, out, lps


def _neutral(n, K, V):
    """state rows under which no edit or forced value touches [0, V): specials V (empty), V + 1 (eog), eos unused"""
    return np.tile(np.array([0, 0, K - 1, -1, 0, 1, 0], np.int32), (n, 1)), (V, V + 1, 0, 75)


def _planted(kind, n, K, V, g):
    L = torch.randn(n, K, V, generator=g)
    if kind == "scale30":
        L *= 30
    elif kind == "equal":
        L.fill_(0.7)
    elif kind == "ties":
        L = torch.randint(-3, 3, (n, K, V), generator=g).float()
        L[..., :: max(1, V // 5)] = 3.0                       # several entries tie at the maximum
    elif kind == "spread":
        L = (torch.rand(n, K, V, generator=g) * 2 - 1) * 1e4  # the losers' exp underflows to 0
    return L


@pytest.mark.gpu
@pytest.mark.parametrize("V", [4, 255, 257, 1023, 2052, 3072])
@pytest.mark.parametrize("K", [1, 4, 8])
@pytest.mark.parametrize("kind", ["normal", "scale30", "equal", "ties", "spread"])
def test_kernel_lp_matches_fp64(V, K, kind):
    """drawn tokens of planted rows; tokens and state equal vcb_debug_sampler's bit for bit"""
    g = torch.Generator().manual_seed(V * 10 + K + len(kind))
    n = 3
    L = _planted(kind, n, K, V, g)
    state, specials = _neutral(n, K, V)
    noise = torch.empty(n * K, V).exponential_(1, generator=g)
    sp = _sp(top_k=40 if kind == "normal" else -100, top_p=0.9 if kind == "scale30" else 1.0)
    tok, st, lp = _hook(L.cuda(), noise.cuda(), sp, specials, state)
    tok0, st0, _ = _hook(L.cuda(), noise.cuda(), sp, specials, state, lp=False)
    assert np.array_equal(tok, tok0) and np.array_equal(st, st0)
    check_lp(f"kernel {kind}", lp, L.numpy(), tok)
    if kind == "equal":
        assert np.abs(lp + math.log(V)).max() <= lp_bound(0.0, V)


@pytest.mark.gpu
@pytest.mark.parametrize("V", [257, 2052, 3072])
@pytest.mark.parametrize("gap", [20.0, 60.0])
def test_kernel_lp_of_a_token_far_below_the_max(V, gap):
    """the planted noise draws an index `gap` below the row's max (q = 1e-30 there, 1 elsewhere)"""
    K, n = 4, 2
    g = torch.Generator().manual_seed(V + int(gap))
    L = torch.randn(n, K, V, generator=g)
    L[..., 1] = 10.0
    target = V - 2
    L[..., target] = 10.0 - gap
    noise = torch.ones(n * K, V)
    noise[:, target] = 1e-30
    state, specials = _neutral(n, K, V)
    tok, _, lp = _hook(L.cuda(), noise.cuda(), _sp(), specials, state)
    assert (tok == target).all()
    check_lp("kernel far below the max", lp, L.numpy(), tok)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [4, 8])
def test_kernel_lp_ignores_the_edits_and_covers_forced_tokens(K):
    """the end / empty masks (-10000), the silence-repetition scaling and the forced empty / end tokens: lp is the raw
    row's log-softmax at the written token, whatever the edits made of the row"""
    V, SR = 256, 75
    EMPTY, EOG, EOS = 252, 253, 254
    g = torch.Generator().manual_seed(K)
    rows, states = [], []

    def add(state, boost=()):
        lg = torch.randn(K, V, generator=g)
        for idx, val in boost:
            lg[:, idx] = val
        rows.append(lg)
        states.append(state)
    # masked entries hold the raw maximum: the edited row's max is another entry
    add([0, 0, 20, -1, 0, 3, 5], [(EMPTY, 9.0), (EOS, 9.5), (EOG, 8.0)])    # k >= 1: end / empty masked; eog masked (eos)
    add([0, 0, 3, -1, 0, 3, 5], [(EOS, 9.0)])                               # codebook 0: end masked before sr / 5 steps
    add([1, 0, 20, -1, 0, 3, 5], [(EOG, 9.0), (EMPTY, 8.5)])                 # edit mode
    add([0, 0, 20, 10, 6, 3, 5], [(10, 7.0), (11, 5.0)])                     # silence token 10 repeated: 7 / 4 < 5
    add([0, 0, 0, -1, 0, 3, 5])                                              # cur 0: k >= 1 forced empty
    add([0, 0, 1, -1, 0, 3, 5])                                              # cur 1: k >= 2 forced empty
    add([0, 1, 20, -1, 0, 3, 5], [(EOS, 9.0)])                               # end cascade: empty, end, ...
    add([0, K - 1, 20, -1, 0, 3, 5])
    add([0, 0, 20, -1, 0, 3, 200])                                           # past the length cap: forced end
    L = torch.stack(rows)
    n = L.shape[0]
    noise = torch.empty(n * K, V).exponential_(1, generator=g)
    sp = _sp(stop_repetition=3, silence=(10, 20, 30))
    specials = (EMPTY, EOG, EOS, SR)
    tok, st, lp = _hook(L.cuda(), noise.cuda(), sp, specials, np.array(states, np.int32))
    tok0, st0, _ = _hook(L.cuda(), noise.cuda(), sp, specials, np.array(states, np.int32), lp=False)
    assert np.array_equal(tok, tok0) and np.array_equal(st, st0)
    check_lp("kernel edits and forced tokens", lp, L.numpy(), tok)
    # the forced values were written (so lp covers them)
    assert (tok[4, 1:] == EMPTY).all() and (tok[5, 2:] == EMPTY).all()
    assert tok[6, 0] == EMPTY and tok[6, 1] == EOS and tok[8, 0] == EOS
    assert tok[0, 1:].tolist() != [EMPTY] * (K - 1)                         # the masked maximum was not drawn


@pytest.mark.gpu
def test_kernel_lp_does_not_depend_on_sampling_parameters_or_noise():
    """the same index drawn under every temperature / top-k / top-p and three noises: the same lp bits"""
    K, V, n = 4, 2052, 2
    g = torch.Generator().manual_seed(11)
    L = torch.randn(n, K, V, generator=g)
    target = 1000
    L[..., 7], L[..., target] = 8.0, 7.0                  # the target ranks second in every row: kept by every filter below
    state, specials = _neutral(n, K, V)
    seen = []
    for temp in (0.3, 1.0, 1.7):
        for top_k, top_p in ((-100, 1.0), (5, 1.0), (40, 0.999), (-100, 0.999)):
            for s in range(3):
                noise = torch.empty(n * K, V).exponential_(1, generator=torch.Generator().manual_seed(s))
                noise[:, target] = 1e-30
                tok, _, lp = _hook(L.cuda(), noise.cuda(), _sp(top_k, top_p, temp), specials, state)
                assert (tok == target).all()
                seen.append(lp)
    assert all(np.array_equal(s.view(np.int32), seen[0].view(np.int32)) for s in seen)
    check_lp("kernel parameter independence", seen[0], L.numpy(), np.full((n, K), target))
    # the device generator's draw instead of the caller's noise: lp is that of whichever token it drew
    tok, _, lp = _hook(L.cuda(), None, _sp(), specials, state, threads=256 * 8)
    check_lp("kernel device noise", lp, L.numpy(), tok)


@pytest.mark.gpu
def test_debug_sampler_lp_rejects_bad_arguments():
    _l, lib = _lib()
    L = torch.zeros(1, 4, 16, device="cuda")
    st = np.array([0, 0, 3, -1, 0, 1, 0], np.int32)
    tok, out = np.zeros(4, np.int32), np.zeros(4, np.int32)
    P = C.POINTER(C.c_int32)
    sp = _sp()
    for V, lp in ((16, None), (4000, np.zeros(4, np.float32))):
        rc = lib.vcb_debug_sampler_lp(L.data_ptr(), None, 1, 0, 256, C.byref(sp), 1, 4, V, 16, 17, 0, 50,
                                      st.ctypes.data_as(P), tok.ctypes.data_as(P), out.ctypes.data_as(P),
                                      None if lp is None else lp.ctypes.data_as(C.POINTER(C.c_float)))
        assert rc != 0 and lib.vcb_last_error().decode().startswith("vcb_debug_sampler_lp:")


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the engine, every step
# ---------------------------------------------------------------------------------------------------------------------
KW = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)


def _lm(kv="bf16", weights="bf16", eos_bias=3.0, eog_bias=None, max_slots=8, seed=3, audio_only=False):
    """tiny LM; codebook 0's end token gets eos_bias (TTS ends) and eog eog_bias (edit spans end); audio_only: the heads
    put no mass on the other non-audio tokens (every generated frame decodes to audio)"""
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=seed)
    if audio_only:
        for k in range(cfg.n_codebooks):
            for t in (cfg.empty_token, cfg.eog, cfg.audio_pad_token, cfg.eos):
                if not (k == 0 and t == cfg.eos):
                    sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    sd["predict_layer.0.2.bias"][cfg.eos] += eos_bias
    if eog_bias is not None:
        sd["predict_layer.0.2.bias"][cfg.eog] = eog_bias
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    m = m.to("cuda").eval()
    m.configure_engine(kv_dtype=kv, weight_dtype=weights, max_slots=max_slots, max_seq_len=512)
    return cfg, m


def _utt(cfg, seed, text_len=12, frames=30):
    from voicecraft_b200 import synthetic
    x, xl, y = synthetic.synthetic_utterance(cfg, seed, text_len=text_len, prompt_frames=frames)
    return x.cuda(), xl.cuda(), y.cuda()


def _drive(sess, max_steps=160):
    """run a session step by step; returns per slot index {token-log row: that step's raw logits [K, V]}"""
    _l, lib = _lib()
    n, K, V = len(sess.slots), sess.K, sess.V
    t = torch.empty(n * K, V, device="cuda")
    seen, prev = [dict() for _ in range(n)], [0] * n
    sess.sample()
    for _ in range(max_steps):
        st = sess.poll()
        _l.check(lib.vcb_debug_logits(sess.eng, t.data_ptr(), n * K))
        rows = t.view(n, K, V).cpu().numpy()
        for j in range(n):
            if st[j].n_steps > prev[j]:            # this step sampled slot j (a forced hand-over step writes no row)
                assert st[j].n_steps == prev[j] + 1
                seen[j][prev[j]] = rows[j].copy()
                prev[j] = st[j].n_steps
        if all(s.done for s in st):
            break
        sess.step()
    return seen


def _check_session(name, sess, seen):
    m = sess.model
    st = sess.poll()
    for j, slot in enumerate(sess.slots):
        n = st[j].n_steps
        toks = m._read_rows(sess.eng, slot, n, sess.stream)
        lp = m._read_lp(sess.eng, slot, n, sess.stream)
        assert sorted(seen[j]) == list(range(n)), f"slot {slot}: rows {sorted(seen[j])[:5]}.. of {n}"
        L = np.stack([seen[j][r] for r in range(n)])
        check_lp(name, lp, L, toks)


@pytest.mark.gpu
@pytest.mark.parametrize("kv,weights,mega", [("bf16", "bf16", 0), ("fp32", "bf16", 0), ("fp8", "bf16", 0),
                                             ("bf16", "int8", 0), ("bf16", "bf16", 1)])
def test_engine_lp_every_step_matches_fp64(kv, weights, mega, monkeypatch):
    if mega:
        monkeypatch.setenv("VCB_MEGA", "1")
    cfg, m = _lm(kv, weights)
    utts = [_utt(cfg, 60 + i, 8 + 3 * i, 20 + 9 * i) for i in range(3)]
    sess = m.open_tts_session([u[0] for u in utts], [u[2] for u in utts], seeds=[5, 6, 7], **KW)
    try:
        if mega:
            assert _lib()[1].vcb_counter(sess.eng, b"mega_grid") > 0, "the persistent kernel did not run"
        seen = _drive(sess)
        _check_session(f"engine kv={kv} w={weights} mega={mega}", sess, seen)
        # the session's result carries the same rows, un-delayed
        out = sess.results(logprobs=True)
        for i, (res, gen, lp) in enumerate(out):
            rows = m._read_lp(sess.eng, sess.slots[i], sess.status[i].n_steps, sess.stream)
            K, G = gen.shape[1], gen.shape[2]
            want = np.stack([rows[k:k + G, k] for k in range(K)])
            assert lp.shape == gen.shape and np.array_equal(lp[0].cpu().numpy(), want)
    finally:
        sess.close()


@pytest.mark.gpu
def test_engine_lp_best_of_n_every_copy_and_the_kept_one():
    cfg, m = _lm(eos_bias=2.0, max_slots=8)
    x, _, y = _utt(cfg, 90, 10, 25)
    sess = m.open_tts_session([x], [y], seeds=[3], best_of=4, **KW)
    try:
        seen = _drive(sess)
        _check_session("engine best-of-4", sess, seen)
        (res, gen, lp), = sess.results(logprobs=True)
        j = sess._kept(0, sess.status)
        assert sess.status[0].keep >= 0
        rows = m._read_lp(sess.eng, sess.slots[j], sess.status[j].n_steps, sess.stream)
        K, G = gen.shape[1], gen.shape[2]
        assert np.array_equal(lp[0].cpu().numpy(), np.stack([rows[k:k + G, k] for k in range(K)]))
    finally:
        sess.close()
    torch.manual_seed(3)
    res1, gen1, lp1 = m.inference_tts_batch(x, torch.tensor([x.shape[1]]), y, batch_size=4, logprobs=True, **KW)
    assert torch.equal(gen1, gen) and np.array_equal(lp1.cpu().numpy().view(np.int32), lp.cpu().numpy().view(np.int32))


@pytest.mark.gpu
def test_engine_lp_edit_two_spans():
    cfg, m = _lm(eog_bias=2.5)
    x, _, y = _utt(cfg, 91, 10, 30)
    mi = torch.tensor([[[4, 9], [15, 19]]])
    sess = m.open_edit_session([x], [y], [mi], seeds=[4], **KW)
    try:
        seen = _drive(sess, max_steps=400)
        assert sess.status[0].done == 1 and sess.status[0].n_spans_done == 2
        _check_session("engine edit, 2 spans", sess, seen)
        (res, _, lp), = sess.results(logprobs=True)
    finally:
        sess.close()
    nan_cols = torch.isnan(lp[0]).all(0)
    assert lp.shape == res.shape and int(nan_cols.sum()) == y.shape[1] - 5 - 4       # the frames kept from y
    assert torch.isfinite(lp[0][:, ~nan_cols]).all()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the public calls
# ---------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.cpu().contiguous().view(torch.int32)


@pytest.mark.gpu
def test_logprobs_keyword_leaves_results_bit_identical():
    cfg, m = _lm(eog_bias=2.5)
    x, xl, y = _utt(cfg, 95, 10, 30)
    torch.manual_seed(21)
    res, gen = m.inference_tts(x, xl, y, **KW)
    off = torch.cuda.default_generators[0].get_offset()
    torch.manual_seed(21)
    res1, gen1, lp = m.inference_tts(x, xl, y, **KW, logprobs=True)
    assert torch.cuda.default_generators[0].get_offset() == off
    assert torch.equal(res, res1) and torch.equal(gen, gen1)
    assert lp.shape == gen.shape and lp.dtype == torch.float32 and bool((lp <= 0).all())
    torch.manual_seed(22)
    r2, g2 = m.inference_tts_batch(x, xl, y, batch_size=3, **KW)
    torch.manual_seed(22)
    r3, g3, lp3 = m.inference_tts_batch(x, xl, y, batch_size=3, **KW, logprobs=True)
    assert torch.equal(r2, r3) and torch.equal(g2, g3) and lp3.shape == g3.shape
    mi = torch.tensor([[[5, 9], [14, 20]]])
    torch.manual_seed(23)
    e = m.inference(x, xl, y, mi, **KW)
    torch.manual_seed(23)
    e1, elp = m.inference(x, xl, y, mi, **KW, logprobs=True)
    assert torch.equal(e, e1) and elp.shape == e1.shape


@pytest.mark.gpu
def test_batch_and_batcher_rows_equal_seeded_single_calls():
    """row i of inference_tts_many / inference_many / ContinuousBatcher.run / .stream: the seeded single call's lp bits"""
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, m = _lm(eog_bias=2.5, audio_only=True)
    utts = [_utt(cfg, 100 + i, 6 + 2 * i, 14 + 5 * i) for i in range(5)]
    seeds = [40 + i for i in range(5)]
    singles = []
    for (x, xl, y), s in zip(utts, seeds):
        torch.manual_seed(s)
        singles.append(m.inference_tts(x, xl, y, **KW, logprobs=True))
    many = m.inference_tts_many([u[0] for u in utts], [u[2] for u in utts], seeds=seeds, logprobs=True, **KW)
    for i, ((r, g, lp), (r1, g1, lp1)) in enumerate(zip(singles, many)):
        assert torch.equal(g, g1) and torch.equal(_bits(lp), _bits(lp1)), i
    mis = [torch.tensor([[[2, 6]]]), torch.tensor([[[3, 5], [8, 12]]])]
    eds = m.inference_many([u[0] for u in utts[3:]], [u[2] for u in utts[3:]], mis, seeds=[7, 8], logprobs=True, **KW)
    for j, (res, lp) in enumerate(eds):
        x, xl, y = utts[3 + j]
        torch.manual_seed(7 + j)
        res1, lp1 = m.inference(x, xl, y, mis[j], **KW, logprobs=True)
        assert torch.equal(res, res1) and torch.equal(_bits(lp), _bits(lp1)), j

    def fill(cb):
        for (x, _, y), s in zip(utts, seeds):
            cb.submit(x, y, seed=s)
    cb = ContinuousBatcher(m, max_concurrency=3, poll_every=3, **KW)
    fill(cb)
    out = cb.run()
    for i, (r, g, lp) in enumerate(singles):
        assert torch.equal(out[i][1], g) and torch.equal(_bits(cb.logprobs[i]), _bits(lp)), i
    from oracle import encodec_oracle as eo
    from voicecraft_b200.tokenizer import AudioTokenizer
    ecfg = eo.default_config()
    tok = AudioTokenizer(device="cuda:0", config=ecfg, state_dict=eo.make_state_dict(ecfg, seed=5))
    cb = ContinuousBatcher(m, max_concurrency=3, poll_every=3, **KW)
    fill(cb)
    for _ in cb.stream(tok, chunk_frames=8):
        pass
    for i, (r, g, lp) in enumerate(singles):
        assert torch.equal(cb.results[i][1], g) and torch.equal(_bits(cb.logprobs[i]), _bits(lp)), i


@pytest.mark.gpu
def test_batcher_logprobs_through_swaps_equal_an_unconstrained_run():
    from voicecraft_b200.voicecraft import ContinuousBatcher
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=3)
    for k in range(cfg.n_codebooks):                  # no early end: every utterance runs to its length cap
        for t in (cfg.empty_token, cfg.eog, cfg.audio_pad_token, cfg.eos):
            sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    m = m.to("cuda:0").eval()
    m.configure_engine(max_slots=4, max_seq_len=512)
    utts = [_utt(cfg, 70 + i, 40, 50 + 3 * i - 41) for i in range(6)]
    seeds = [500 + i for i in range(6)]

    def run():
        cb = ContinuousBatcher(m, max_concurrency=4, poll_every=5, **KW)
        for (x, _, y), s in zip(utts, seeds):
            cb.submit(x, y, seed=s)
        return cb, cb.run()
    free, plain = run()
    assert free.stats["swap_outs"] == 0
    pb = _lib()[1].vcb_counter(m._engine(), b"kv_page_bytes")
    m.configure_engine(kv_pool_gb=12.5 * pb / 1e9, max_slots=4, max_seq_len=512)
    cb, got = run()
    assert cb.stats["swap_outs"] > 0, cb.stats
    for i in range(6):
        assert torch.equal(got[i][1], plain[i][1]), i
        assert torch.equal(_bits(cb.logprobs[i]), _bits(free.logprobs[i])), i


# ---------------------------------------------------------------------------------------------------------------------
# GPU: against the oracle at 830M
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kv", ["fp32", "bf16"])
def test_830M_lp_against_the_oracle_logits(kv):
    """The 830M fixture (tests/golden/make_golden_830m.py): 32 utterances, 64 steps, the oracle's raw logits at 4 traced
    steps of 4 utterances.  On each traced row where the engine's tokens still equal the fixture's, the engine's lp must lie
    within 2 max|delta logit| + B of the oracle's log-softmax at the same token, delta measured on that row in this test
    (the log-sum-exp moves by at most max|delta|, the token's logit by at most that too).  The oracle stores its rows after
    its eog mask (-10000); that column takes the engine's raw value on both sides."""
    import golden_util as gu
    meta, g = gu.headline_fixture()
    cfg, sd = gu.headline_checkpoint(meta["ckpt_seed"])
    from voicecraft_b200.voicecraft import VoiceCraft
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    m = m.to("cuda").eval()
    m.configure_engine(kv_dtype=kv, max_slots=32, max_seq_len=1024, max_new_tokens=128)
    utts = [gu.headline_utterance(cfg, meta, i) for i in range(32)]
    sess = m.open_tts_session([u[0] for u in utts], [u[2] for u in utts], noise_fns=[gu.cpu_noise_fn(1 + i) for i in range(32)],
                              silence_tokens=gu.SILENCE, **meta["kw"])
    K, V, N = cfg.n_codebooks, m.n_audio_tokens[0], meta["n_steps"]
    _l, lib = _lib()
    t = torch.empty(32 * K, V, device="cuda")
    raw = {}
    try:
        for step in range(N):
            sess.sample() if step == 0 else sess.step()
            if step in meta["trace_steps"]:
                _l.check(lib.vcb_debug_logits(sess.eng, t.data_ptr(), 32 * K))
                raw[step] = t.view(32, K, V).cpu().numpy().copy()
        st = sess.poll()
        rows = [m._read_rows(sess.eng, s, st[i].n_steps, sess.stream)[:N] for i, s in enumerate(sess.slots)]
        lps = [m._read_lp(sess.eng, s, st[i].n_steps, sess.stream)[:N] for i, s in enumerate(sess.slots)]
    finally:
        sess.close()
    ref_rows = g[f"rows_{kv}"].astype(np.int64)
    checked, worst = 0, 0.0
    for ui, u in enumerate(meta["trace_utts"]):
        for si, s in enumerate(meta["trace_steps"]):
            if not np.array_equal(rows[u][: s + 1], ref_rows[u][: s + 1]):
                continue                              # inputs differ after a divergence
            o = g[f"logits_{kv}"][ui, si].astype(np.float32).copy()
            e = raw[s][u]
            o[:, cfg.eog] = e[:, cfg.eog]
            tok = rows[u][s]
            dlt = np.abs(o.astype(np.float64) - e).max(-1)
            ref, _ = lp_ref(o, tok)
            _, gap = lp_ref(e, tok)
            err = np.abs(lps[u][s] - ref)
            lim = 2 * dlt + lp_bound(gap, V)
            worst = max(worst, float((err / lim).max()))
            assert (err <= lim).all(), f"utt {u} step {s}: |lp - oracle| {err} > {lim}"
            check_lp(f"830M kv={kv} engine rows", lps[u][s], e, tok)
            checked += 1
    WORST[f"830M kv={kv} vs oracle (of 2 max|dlogit| + B)"] = worst
    assert checked >= 12, f"only {checked} traced rows comparable"
