"""The decode step across its tuning knobs (DESIGN.md section 7).

Two kinds of knob:
  * scheduling only: the persistent kernel's ring depths VCB_MEGA_NS / _NB, its loads in flight VCB_MEGA_FLIGHT and its L2
    prefetch distance VCB_MEGA_PF; on the per-kernel step VCB_PDL (and vcb_set_option("pdl")), VCB_PREFETCH and
    VCB_ATT_BALANCE; VCB_ATT_CHUNK_PAGES on the persistent kernel, which does not read it.  These change when bytes move,
    never the order of a sum (the persistent kernel's work split depends on the grid alone, partials are summed in
    contributor order), so every logit of every step, every K / V byte and every token must be bit-identical to the
    default engine's.
  * summation order: the persistent kernel's grid (VCB_MEGA_GRID), the decode GEMM's split count (VCB_SPLITS) and the
    per-kernel attention's chunk pages (VCB_ATT_CHUNK_PAGES).  These are held stage by stage to test_lm_numerics's fp64
    bounds, unchanged.

The ring rule itself (which (ns, nb) fit the shared-memory pool, and the loads in flight clamped to [1, ns]) is checked
without a GPU through vcb_mega_ring_config; engines built with a refused configuration fail on the host before anything
of theirs is launched.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import golden_util as gu

_HAS_GPU = torch.cuda.is_available()


def gpu(f):
    return pytest.mark.gpu(pytest.mark.skipif(not _HAS_GPU, reason="needs an H100")(f))


def _lib():
    from voicecraft_b200 import _lib
    return _lib, _lib.load()


# ==========================================================================================================================
# the ring rule (no GPU)
# ==========================================================================================================================
def _ring_legal(ns, nb):
    """2 <= ns, 3 <= nb <= 8 and ns 16 KB + nb 8 KB within the 224 KB pool (so ns <= 12)"""
    return ns >= 2 and 3 <= nb <= 8 and ns * 16 + nb * 8 <= 224


RING_PAIRS = [(ns, nb) for ns in range(2, 13) for nb in range(3, 9) if _ring_legal(ns, nb)]
RING_DEFAULT = (11, 6, 5, 0)        # ns, nb, flight, pf


def _ring_config(ns, nb, flight):
    _, lib = _lib()
    out = (C.c_int32 * 3)()
    if lib.vcb_mega_ring_config(ns, nb, flight, out) != 0:
        return None
    return tuple(out)


def test_ring_rule_has_sixty_pairs():
    assert len(RING_PAIRS) == 60
    assert max(ns for ns, _ in RING_PAIRS) == 12 and (11, 6) in RING_PAIRS


def test_ring_config_follows_the_rule():
    """every (ns, nb) in a box around the legal set: accepted exactly where the rule holds, with the loads in flight clamped
    to [1, ns] (more than ns in flight would wait on a slot's barrier with a parity that aliases a later phase)"""
    _, lib = _lib()
    for ns in range(-1, 16):
        for nb in range(-1, 11):
            for flight in (-3, 0, 1, 2, ns - 1, ns, ns + 1, 5, 40):
                got = _ring_config(ns, nb, flight)
                if not _ring_legal(ns, nb):
                    assert got is None, (ns, nb, flight)
                    err = lib.vcb_last_error()
                    assert f"= {ns} / {nb}:".encode() in err and b"ns <= 12" in err, err
                else:
                    assert got == (ns, nb, min(max(flight, 1), ns)), (ns, nb, flight, got)


# ==========================================================================================================================
# GPU: engines and what a few decode steps leave
# ==========================================================================================================================
SP = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3, silence_tokens=gu.SILENCE)
_MODELS = {}


def _model(name):
    """one VoiceCraft per config name on the GPU, kept for the module (each knob configuration builds its own engine)"""
    if name not in _MODELS:
        from voicecraft_b200 import synthetic
        from voicecraft_b200.voicecraft import VoiceCraft
        cfg = synthetic.make_config(name)
        sd = gu.suppress_end_tokens(cfg, synthetic.make_state_dict(cfg, seed=81))
        m = VoiceCraft(cfg)
        m.load_state_dict(sd)
        _MODELS[name] = m.to("cuda").eval()
    return _MODELS[name]


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    yield
    _MODELS.clear()


def _utts(cfg, totals, seed):
    from voicecraft_b200 import synthetic
    out = []
    for i, total in enumerate(totals):
        text = 6 + i % 5
        x, _, y = synthetic.synthetic_utterance(cfg, seed + 31 * i, text_len=text, prompt_frames=total - text - 1)
        out.append((x, y))
    return out


def _kv_positions(lib, m, eng, kv, slot, seq_len):
    """every layer's K and V bytes of a slot over positions 0 .. seq_len - 1, position-major"""
    _l = _lib()[0]
    a = m.args
    H, hd, L = a.nhead, a.d_model // a.nhead, a.num_decoder_layers
    npg = (seq_len + 63) // 64
    slab = {"fp32": 64 * hd * 4, "bf16": 64 * hd * 2, "fp8": 64 * (hd + 4)}[kv]
    out = []
    for l in range(L):
        kb = np.zeros(npg * H * slab, np.uint8)
        vb = np.zeros_like(kb)
        _l.check(lib.vcb_debug_kv_pages(eng, l, slot, 0, npg, kb.ctypes.data, vb.ctypes.data))
        for raw in (kb, vb):
            t = torch.from_numpy(raw)
            if kv == "fp8":
                from kv_fp8_ref import split_slabs
                q, s = split_slabs(t, H, hd)
                out.append(q.transpose(1, 2).reshape(-1, H, hd)[:seq_len].clone())
                out.append(s.view(torch.int32).transpose(1, 2).reshape(-1, H)[:seq_len].clone())
            else:
                out.append(t.reshape(npg, H, 64, -1).transpose(1, 2).reshape(npg * 64, H, -1)[:seq_len].clone())
    return out


def _build(m, env, kv="bf16", weight_dtype="bf16", max_slots=32, max_seq_len=4608, options=()):
    """a fresh engine of m built under env (the knobs are read when the engine is built), then vcb_set_option(options)"""
    _l, lib = _lib()
    with pytest.MonkeyPatch.context() as mp:
        for k, v in env.items():
            mp.setenv(k, str(v))
        m.configure_engine(kv_dtype=kv, weight_dtype=weight_dtype, max_slots=max_slots, max_seq_len=max_seq_len)
        eng = m._engine()
    for name, value in options:
        _l.check(lib.vcb_set_option(eng, name, value))
    return eng


def _counters(eng):
    _, lib = _lib()
    return {c: lib.vcb_counter(eng, c.encode()) for c in ("mega_grid", "mega_ns", "mega_nb", "mega_flight", "mega_pf")}


def _decode(m, eng, kv, row_sets, steps):
    """per row set (one session each, in order): the logits of the first sample and of every decode step, the tokens, and
    every layer's K / V of every slot over its written positions"""
    from voicecraft_b200.voicecraft import DecodeSession
    _l, lib = _lib()
    K, V = m.args.n_codebooks, m.n_audio_tokens[0]
    out = []
    for r, totals in enumerate(row_sets):
        utts = _utts(m.args, totals, 900 + 37 * r)
        sess = DecodeSession(m, [u[0] for u in utts], [u[1] for u in utts], m._sampling(**SP),
                             seeds=[2000 + 7 * r + i for i in range(len(totals))])
        try:
            assert sess.eng == eng, "the engine was rebuilt: its knobs are gone"
            n = len(totals)
            logits = []
            for s in range(steps + 1):
                sess.sample() if s == 0 else sess.step()
                t = torch.empty(n * K, V, device="cuda")
                _l.check(lib.vcb_debug_logits(eng, t.data_ptr(), n * K))
                logits.append(t)
            st = sess.poll()
            toks = [torch.from_numpy(np.asarray(sess.raw_tokens(i))) for i in range(n)]
            kvb = [_kv_positions(lib, m, eng, kv, sess.slots[i], sess.prompts[i].total + st[i].n_steps - 1)
                   for i in range(n)]
            out.append(dict(logits=logits, tokens=toks, kv=kvb))
        finally:
            sess.close()
    return out


def _differences(a, b):
    """what differs between two _decode results (empty: bit-identical)"""
    bad = []
    for r, (x, y) in enumerate(zip(a, b)):
        for s, (p, q) in enumerate(zip(x["logits"], y["logits"])):
            if not torch.equal(p, q):
                bad.append(f"rows {r} step {s}: {int((p != q).sum())} logits differ, max {float((p - q).abs().max()):.3g}")
        for i, (p, q) in enumerate(zip(x["tokens"], y["tokens"])):
            if not torch.equal(p, q):
                bad.append(f"rows {r} utterance {i}: tokens differ")
        for i, (p, q) in enumerate(zip(x["kv"], y["kv"])):
            for j, (u, v) in enumerate(zip(p, q)):
                if not torch.equal(u, v):
                    bad.append(f"rows {r} utterance {i}: layer {j // 2} {'KV'[j % 2]} bytes differ")
    return bad


def _compare_all(label, base, configs, run):
    """run(config) for every config, each against base; prints how many were compared"""
    bad = []
    for cfg in configs:
        diff = _differences(base, run(cfg))
        if diff:
            bad.append(f"{cfg}: {diff[:3]}")
    print(f"{label}: {len(configs)} configurations compared bit for bit with the default engine, {len(bad)} differ")
    assert not bad, f"{label}: {len(bad)} configurations differ (first: {bad[:4]})"


# ---- 1. the persistent kernel's ring configurations, bit for bit --------------------------------------------------------
# tiny: n = 1 (bpad 16; its context crosses the page boundary at 63 / 64 during the steps), n = 17 (bpad 32; rows at 63, 64
# and one past 4096 tokens: 17 attention chunks, the workspace fold), n = 32
MEGA_ROWS = [(61,), (61, 62, 4200) + tuple(30 + 5 * i for i in range(14)), tuple(40 + 3 * i for i in range(32))]
MEGA_GRID = 10          # the smallest grid tiny takes: every CTA's ring wraps many times per step
MEGA_STEPS = 8


def _ring_env(ns, nb, flight=None, pf=None):
    env = {"VCB_MEGA": 1, "VCB_MEGA_GRID": MEGA_GRID, "VCB_MEGA_NS": ns, "VCB_MEGA_NB": nb}
    if flight is not None:
        env["VCB_MEGA_FLIGHT"] = flight
    if pf is not None:
        env["VCB_MEGA_PF"] = pf
    return env


def _ring_run(m, kv, env, rows, grid=MEGA_GRID):
    eng = _build(m, env, kv=kv, max_slots=max(len(r) for r in rows))
    c = _counters(eng)
    ns, nb = int(env.get("VCB_MEGA_NS", RING_DEFAULT[0])), int(env.get("VCB_MEGA_NB", RING_DEFAULT[1]))
    flight, pf = int(env.get("VCB_MEGA_FLIGHT", RING_DEFAULT[2])), int(env.get("VCB_MEGA_PF", RING_DEFAULT[3]))
    want = dict(mega_grid=grid, mega_ns=ns, mega_nb=nb, mega_flight=min(max(flight, 1), ns), mega_pf=pf)
    assert c == want, f"{env}: the engine runs {c}, not {want} (a fallback to the per-kernel step cannot pass)"
    return _decode(m, eng, kv, rows, MEGA_STEPS)


RING_KNOB_PAIRS = [(2, 3), (3, 8), (11, 6), (12, 4)]


def _ring_knob_configs():
    out = [(ns, nb, None, None) for ns, nb in RING_PAIRS if (ns, nb) != (11, 6)]
    for ns, nb in RING_KNOB_PAIRS:
        out += [(ns, nb, f, None) for f in sorted({1, 2, ns - 1, ns})]
        out += [(ns, nb, None, pf) for pf in (1, 2, 4, 16)]
    return out


@gpu
@pytest.mark.parametrize("kv", ["bf16", "fp32"])
def test_ring_configurations_are_bit_identical(kv):
    """all 60 legal (ns, nb) at the default loads in flight and prefetch (flight 5 runs as ns for ns < 5), and at four
    pairs every flight in {1, 2, ns - 1, ns} and prefetch distance in {1, 2, 4, 16}: logits of every step, K / V bytes
    of every layer and tokens equal the default (11, 6, 5, 0) engine's at the same grid (a bf16 ring slot holds 64
    tokens of one head, an fp32 one 32)"""
    m = _model("tiny")
    base = _ring_run(m, kv, _ring_env(*RING_DEFAULT[:2]), MEGA_ROWS)
    _compare_all(f"ring kv={kv}", base, _ring_knob_configs(),
                 lambda c: _ring_run(m, kv, _ring_env(*c), MEGA_ROWS))


@gpu
def test_ring_configurations_830M():
    """a few pairs at d = 2048, 16 layers (82 phases), 32 rows, on a grid of 66"""
    m = _model("830M")
    rows = [tuple(60 + 7 * i for i in range(31)) + (1099,)]
    run = lambda c: _ring_run(m, "bf16", dict(_ring_env(*c), VCB_MEGA_GRID=66), rows, grid=66)
    base = run((11, 6, None, None))
    _compare_all("ring 830M", base, [(2, 3, None, None), (5, 8, 2, None), (12, 4, 12, 4), (8, 5, None, 16)], run)


@gpu
def test_att_chunk_pages_leave_the_persistent_kernel_unchanged():
    """the persistent kernel uses its own 4-page chunks and does not read VCB_ATT_CHUNK_PAGES.  The prefill's attention does
    read it, so the prompts here fit in one page: one chunk whatever the setting, and the same K / V for the decode steps"""
    m = _model("tiny")
    rows = [(61,), (61, 62) + tuple(30 + 2 * i for i in range(15)), tuple(20 + i for i in range(32))]
    env = _ring_env(*RING_DEFAULT[:2])
    base = _ring_run(m, "bf16", env, rows)
    _compare_all("persistent kernel VCB_ATT_CHUNK_PAGES", base, [1, 2, 5],
                 lambda cp: _ring_run(m, "bf16", dict(env, VCB_ATT_CHUNK_PAGES=cp), rows))


# ---- 2. ring knob validation ---------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("ns,nb", [(13, 3), (13, 2), (12, 5), (2, 2), (2, 9), (1, 3), (0, 6), (11, 7), (14, 0)])
def test_illegal_ring_is_refused_when_the_engine_is_built(ns, nb):
    """the engine build fails with the rule in its message; the check runs before the persistent kernel's buffers are
    allocated, so nothing of it is launched"""
    _l, _ = _lib()
    m = _model("tiny")
    with pytest.raises(_l.VcbError) as ei:
        _build(m, {"VCB_MEGA": 1, "VCB_MEGA_NS": ns, "VCB_MEGA_NB": nb}, max_slots=1, max_seq_len=256)
    assert f"VCB_MEGA_NS / VCB_MEGA_NB = {ns} / {nb}" in str(ei.value) and "ns <= 12" in str(ei.value)
    m.configure_engine(max_slots=1)             # leave a buildable configuration behind


@gpu
@pytest.mark.parametrize("ns,flight,want", [(4, 9, 4), (2, 5, 2), (12, 40, 12), (6, 0, 1), (6, -3, 1), (6, 6, 6)])
def test_flight_is_clamped_to_the_ring(ns, flight, want):
    eng = _build(_model("tiny"), {"VCB_MEGA": 1, "VCB_MEGA_NS": ns, "VCB_MEGA_NB": 3, "VCB_MEGA_FLIGHT": flight},
                 max_slots=1, max_seq_len=256)
    c = _counters(eng)
    assert c["mega_grid"] > 0 and c["mega_ns"] == ns and c["mega_flight"] == want, c


# ---- 3. per-kernel step knobs, bit for bit -------------------------------------------------------------------------------
STEP_ROWS = [(61,), (62, 63, 1099) + tuple(30 + 3 * i for i in range(14)), tuple(25 + 2 * i for i in range(32)) + (1099,),
             tuple(20 + i for i in range(127)) + (1099,)]
STEP_KNOBS = [("VCB_PDL=0", {"VCB_PDL": 0}, ()), ("pdl option 0", {}, ((b"pdl", 0),)), ("VCB_PREFETCH=1", {"VCB_PREFETCH": 1}, ()),
              ("VCB_PREFETCH=2", {"VCB_PREFETCH": 2}, ()), ("VCB_ATT_BALANCE=0", {"VCB_ATT_BALANCE": 0}, ())]
STEP_POLICIES = [("bf16", "bf16", "1"), ("bf16", "bf16", "0"), ("fp8", "bf16", "1"), ("fp8", "bf16", "0"),
                 ("fp32", "bf16", "1"), ("bf16", "int8", "1")]


@gpu
@pytest.mark.parametrize("kv,weights,wide", STEP_POLICIES, ids=[f"kv={k}-w={w}-wide={p}" for k, w, p in STEP_POLICIES])
def test_step_knobs_are_bit_identical(kv, weights, wide):
    """VCB_PDL=0, vcb_set_option("pdl", 0) on a live engine, VCB_PREFETCH=1 / 2 and VCB_ATT_BALANCE=0 on the per-kernel
    step at n = 1, 17, 33 and 128 (every bpad), after a wide or narrow prefill"""
    m = _model("tiny")

    def run(knob):
        _, env, opts = knob
        eng = _build(m, dict(env, VCB_PREFILL_WIDE=wide), kv=kv, weight_dtype=weights, max_slots=128, max_seq_len=1280,
                     options=opts)
        assert _counters(eng)["mega_grid"] == 0
        return _decode(m, eng, kv, STEP_ROWS, 3)

    base = run(("default", {}, ()))
    _compare_all(f"per-kernel step kv={kv} weights={weights} wide={wide}", base, STEP_KNOBS, run)


# ---- 4. the persistent kernel's grid against fp64, stage by stage ---------------------------------------------------------
GRIDS = [("tiny", (62,), g) for g in (10, 11, 33, 66, 131, None)] + \
        [("tiny", tuple(30 + i for i in range(31)) + (1099,), g) for g in (10, 11, 33, 66, 131, None)] + \
        [("830M", tuple(60 + 7 * i for i in range(31)) + (1099,), g) for g in (66, 131)]


@gpu
@pytest.mark.parametrize("cfg_name,totals,grid", GRIDS, ids=[f"{c}-n{len(t)}-grid{g}" for c, t, g in GRIDS])
def test_grid_against_fp64(cfg_name, totals, grid, monkeypatch):
    """grids where a CTA's block range splits output tiles unevenly (11, 33, 131 against the phases' tile counts) and where
    attention items span CTAs, with test_lm_numerics's bounds"""
    from test_lm_numerics import Case, _run_case
    _, lib = _lib()
    monkeypatch.setenv("VCB_MEGA", "1")
    if grid is not None:
        monkeypatch.setenv("VCB_MEGA_GRID", str(grid))
    case = Case(cfg_name, totals=totals, mode="decode", max_seq_len=2048)
    want = grid if grid is not None else lib.vcb_counter(case.eng, b"num_sms")
    assert lib.vcb_counter(case.eng, b"mega_grid") == want
    _run_case(case, f"persistent kernel {cfg_name} n={len(totals)} grid={want}", pre_steps=1, mega=True)


# ---- 5. split counts against fp64, stage by stage -----------------------------------------------------------------------
DIMS = {"tiny": 256, "330M": 1024, "830M": 2048}


def _split_shapes(cfg_name, n, s):
    """the decode GEMMs (N, K) -- QKV, out-projection, FFN1, FFN2, first head stage (4 codebooks x 1024) -- that can run
    s splits at n rows: a power of two <= 16 leaving each CTA two token rows and a k-block (test_gemm_split16)"""
    d = DIMS[cfg_name]
    bpad = 16 if n <= 16 else 32 if n <= 32 else 64 if n <= 64 else 128
    legal = lambda K: s <= 16 and bpad % s == 0 and bpad // s >= 2 and (s - 1) * ((K // 64 + s - 1) // s) < K // 64
    return [(N, K) for N, K in [(3 * d, d), (d, d), (4 * d, d), (d, 4 * d), (4 * 1024, d)] if legal(K)]


SPLITS = [("tiny", "bf16", "bf16", n, s) for n in (16, 32, 64, 128) for s in (1, 2, 4, 8, 16)] + \
         [("tiny", "fp8", "bf16", n, s) for n in (16, 128) for s in (2, 8, 16)] + \
         [("330M", "bf16", "bf16", 32, s) for s in (4, 16)] + \
         [("830M", "bf16", "bf16", 16, 8), ("830M", "bf16", "bf16", 128, 16), ("830M", "bf16", "int8", 32, 8)]
SPLITS = [c for c in SPLITS if _split_shapes(c[0], c[3], c[4])]


@gpu
@pytest.mark.parametrize("cfg_name,kv,weights,n,s", SPLITS, ids=[f"{c}-kv={k}-w={w}-n{n}-s{s}" for c, k, w, n, s in SPLITS])
def test_split_count_against_fp64(cfg_name, kv, weights, n, s, monkeypatch):
    """one split count on every decode GEMM that takes it, the decode step's stages with test_lm_numerics's bounds"""
    from test_lm_numerics import Case, _run_case
    _, lib = _lib()
    shapes = _split_shapes(cfg_name, n, s)
    out = (C.c_int32 * 2)()
    for N, K in shapes:
        assert lib.vcb_gemm_launch_shape(N, K, n, s, 0, 0, out) == 0 and out[0] == s, (N, K, n, s)
    env = ",".join(f"{N}x{K}:{s}" for N, K in shapes)
    monkeypatch.setenv("VCB_SPLITS", env)
    case = Case(cfg_name, kv=kv, totals=tuple(30 + 3 * (i % 23) for i in range(n)), mode="decode", weight_dtype=weights)
    print(f"VCB_SPLITS={env}")
    _run_case(case, f"decode {cfg_name} kv={kv} weights={weights} n={n} splits={s}", pre_steps=1)


@gpu
@pytest.mark.parametrize("splits", ["256x1024:16", "768x256:3"])
def test_rejected_split_leaves_the_step_undone(splits):
    """A VCB_SPLITS entry the launcher refuses for the step's bpad (16 splits at bpad 16, 3 anywhere) fails
    vcb_decode_step with a "gemm:" error before anything is enqueued: positions, step counts and K / V are as they were,
    and the same slots then step (at a bpad where the entry is legal) exactly as an engine that never saw the call."""
    from voicecraft_b200.voicecraft import DecodeSession
    _l, lib = _lib()
    m = _model("tiny")
    totals = (62, 63) + tuple(30 + 4 * i for i in range(15))
    env = {"VCB_SPLITS": splits}
    results = []
    for bad_call in (True, False):
        eng = _build(m, env, max_slots=17, max_seq_len=512)
        utts = _utts(m.args, totals, 4000)
        sess = DecodeSession(m, [u[0] for u in utts], [u[1] for u in utts], m._sampling(**SP),
                             seeds=[50 + i for i in range(17)])
        try:
            sess.sample()
            if not splits.endswith(":3"):       # (3 splits fail every step)
                sess.step()
            if bad_call:
                before = [(s.n_steps, s.done) for s in sess.poll()]
                written = [totals[i] + s.n_steps - 1 for i, s in enumerate(sess.poll())]
                kv0 = [_kv_positions(lib, m, eng, "bf16", sess.slots[i], written[i]) for i in range(16)]
                rc = lib.vcb_decode_step(eng, (C.c_int32 * 16)(*sess.slots[:16]), 16, None, C.byref(sess.sp), sess.stream)
                assert rc != 0 and b"gemm:" in lib.vcb_last_error(), lib.vcb_last_error()
                assert [(s.n_steps, s.done) for s in sess.poll()] == before
                kv1 = [_kv_positions(lib, m, eng, "bf16", sess.slots[i], written[i]) for i in range(16)]
                assert all(torch.equal(a, b) for p, q in zip(kv0, kv1) for a, b in zip(p, q)), "K / V changed"
            if splits.endswith(":3"):
                with pytest.raises(_l.VcbError, match="gemm:"):
                    sess.step()
                continue
            sess.step()                         # all 17 rows: bpad 32, where 16 splits are legal
            logits = torch.empty(17 * 4, m.n_audio_tokens[0], device="cuda")
            _l.check(lib.vcb_debug_logits(eng, logits.data_ptr(), 17 * 4))
            st = sess.poll()
            results.append((logits, [torch.from_numpy(np.asarray(sess.raw_tokens(i))) for i in range(17)],
                            [_kv_positions(lib, m, eng, "bf16", sess.slots[i], totals[i] + st[i].n_steps - 1)
                             for i in range(17)]))
        finally:
            sess.close()
    if results:
        (la, ta, ka), (lb, tb, kb) = results
        assert torch.equal(la, lb), "logits differ from an engine that never saw the refused step"
        assert all(torch.equal(a, b) for a, b in zip(ta, tb)), "tokens differ"
        assert all(torch.equal(a, b) for p, q in zip(ka, kb) for a, b in zip(p, q)), "K / V differ"


# ---- 6. the per-kernel attention's chunk pages against fp64 ---------------------------------------------------------------
@gpu
@pytest.mark.parametrize("chunk_pages", [1, 2, 5])
def test_att_chunk_pages_against_fp64(chunk_pages, monkeypatch):
    """VCB_ATT_CHUNK_PAGES through the folded decode chain at positions 63, 64 and 1099 (split-context merges of 1, 2 and
    5 pages per chunk)"""
    from test_lm_numerics import Case, _run_case
    monkeypatch.setenv("VCB_ATT_CHUNK_PAGES", str(chunk_pages))
    case = Case("tiny", totals=(61, 62, 1097), mode="decode", max_seq_len=2048)
    _run_case(case, f"decode VCB_ATT_CHUNK_PAGES={chunk_pages}", pre_steps=1)
