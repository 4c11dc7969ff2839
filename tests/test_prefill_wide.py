"""The wide prefill (the rows-as-M GEMM of csrc/gemm_rows.cu), which every prompt takes by default, against float64 and
against itself.

  * Stage by stage, with test_lm_numerics's stops, references and bounds as they are: several prompts packed into one
    pass with a ragged last row tile (703 rows: 703 % 128 = 63), an edit prompt packed with a TTS prompt (mask-embedding
    rows into gemm_rows), head dim 64, int8 weights (W_deq expanded before each GEMM), more rows than a pass holds (the
    last pass's rows attend to pages the first pass wrote; a prompt straddles row 4096), and d = 384, whose QKV (9 blocks
    of 128 features), out-projection and FFN2 (3 blocks) run 128-wide tiles: there a head of 128 features spans both
    epilogue halves, and the fp8 scale's amax must still be taken over the whole head.
  * The GEMM alone (vcb_debug_gemm_rows) per element against GEMM(K) |x| |W|^T: operands that hi + lo hold exactly, so
    the bound is the fp32 accumulation alone, and rows scaled by 2^-20 .. 2^20, so a lost lo plane or a mis-scaled row
    shows.  Both tile widths, K 64 .. 8192 (FFN2 at 830M), 1 .. 4096 rows.
  * Placement invariance, bit for bit: one probe prompt's K / V bytes (fp8 scales included) and first-sample logits are
    the same alone, packed first, in the middle and last, with the 4096-row pass boundary inside it at two rows, ending on
    a pass's last row, and as the leader of a best-of-N group (whose members' tail page must hold its own bytes).  Batcher
    results equal to seeded single calls, and best-of-N groups equal to independent utterances, rest on this.
"""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

from test_lm_numerics import Case, View, Worst, _checkpoint, _gemm_c, _lib, _run_case

PACKED = (63, 64, 65, 130, 381)           # ends at positions 62 .. 64, 703 rows: a last row tile of 63 rows
PASS = 4096                               # rows per pass once max_slots * max_seq_len reaches it


class Packed:
    """One vcb_prefill of several prompts, as a batcher admission round hands them to the engine: prompt i is TTS
    (spans[i] None) or an edit (its [1, M, 2] intervals), in a group of copies[i] slots.  slots[i]: its first slot."""

    def __init__(self, m, utts, spans=None, copies=None, seeds=None):
        from voicecraft_b200.voicecraft import _prefill, _Prompt
        n = len(utts)
        spans = spans or [None] * n
        self.m, self.copies = m, list(copies or [1] * n)
        self.prompts = [_Prompt(m, x, y, None if s is None else [(int(a), int(b)) for a, b in s[0].tolist()])
                        for (x, y), s in zip(utts, spans)]
        self.eng, self.held = m._take_slots(sum(self.copies), max(p.need_seq for p in self.prompts))
        self.slots = [self.held[int(s)] for s in np.cumsum([0] + self.copies[:-1])]
        self.stream = torch.cuda.current_stream().cuda_stream
        seeds = seeds or [1000 + i for i in range(n)]
        try:
            _prefill(self.eng, [(p, s, c, seed, 0) for p, s, c, seed in zip(self.prompts, self.slots, self.copies, seeds)],
                     self.stream)
        except BaseException:
            self.close()
            raise

    def close(self):
        _l, lib = _lib()
        for s, c in zip(self.slots, self.copies):
            lib.vcb_release(self.eng, s, c)
        self.m._release_slots(self.held, starts=[])


class WideCase(Case):
    """A prefill Case on the default (wide) path, its prompts in one packed call; `edit`: which prompts are edits.
    View checks the rows of the last pass, whose size is the engine's."""

    def __init__(self, cfg_name, edit=(), **kw):
        super().__init__(cfg_name, mode="prefill", edit=any(edit), **kw)
        if self.edit:
            self.spans = [s if e else None for s, e in zip(self.spans, edit)]
        self.rows_run = 0

    @property
    def chunk(self):
        _l, lib = _lib()
        n = lib.vcb_counter(self.eng, b"wide_rows")
        assert n > 0, "the prefill did not take the wide path"
        return n

    @contextlib.contextmanager
    def run(self, stop, pre_steps=0):
        _l, lib = _lib()
        _l.check(lib.vcb_set_option(self.eng, b"stop_stage", stop))
        sess = None
        try:
            before = lib.vcb_counter(self.eng, b"prefill_rows")
            sess = Packed(self.m, self.utts, self.spans if self.edit else None, seeds=self.seeds)
            assert sess.eng == self.eng, "the engine was rebuilt: its options are gone"
            self.rows_run = lib.vcb_counter(self.eng, b"prefill_rows") - before
            assert self.rows_run == sum(p.total for p in sess.prompts)
            torch.cuda.synchronize()
            yield View(self, sess)
        finally:
            _l.check(lib.vcb_set_option(self.eng, b"stop_stage", 0))
            if sess is not None:
                sess.close()


def _run_wide(case, label):
    _run_case(case, label, fold=False)
    return case.chunk


# ==========================================================================================================================
# 1. stage by stage against fp64
# ==========================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("kv", ["fp32", "bf16", "fp8"])
def test_packed_prompts(kv):
    """five prompts in one pass: ends at positions 62, 63, 64, text / audio boundaries, a ragged last row tile"""
    case = WideCase("tiny", kv=kv, totals=PACKED)
    assert _run_wide(case, f"wide packed {PACKED} kv={kv}") >= sum(PACKED)


@pytest.mark.gpu
def test_edit_prompt_packed_with_tts():
    """an edit prompt of two spans (embed_rows_kernel's mask-embedding rows) in the same pass as a TTS prompt"""
    case = WideCase("tiny", totals=(90, 130), edit=(True, False))
    _run_wide(case, "wide edit + TTS")


@pytest.mark.gpu
@pytest.mark.parametrize("kv", ["bf16", "fp8"])
def test_head_dim_64_packed(kv):
    case = WideCase("tiny", kv=kv, totals=PACKED, nhead=4)
    assert case.hd == 64
    _run_wide(case, f"wide packed hd 64 kv={kv}")


@pytest.mark.gpu
def test_int8_weights_packed():
    """int8 weights: every GEMM multiplies W_deq, expanded into the bf16 scratch just before it"""
    case = WideCase("tiny", kv="bf16", totals=PACKED, weight_dtype="int8")
    _run_wide(case, "wide packed int8 weights")


@pytest.mark.gpu
@pytest.mark.parametrize("kv,regime", [("bf16", "plain"), ("fp8", "plain"), ("bf16", "offset")])
def test_across_the_pass_boundary(kv, regime):
    """4400 rows in passes of 4096: the third prompt's rows 596 .. 899 run in the second pass and attend to its pages
    0 .. 595, which the first pass wrote"""
    totals = (2000, 1500, 900)
    case = WideCase("tiny", kv=kv, regime=regime, totals=totals, max_seq_len=2048)
    assert _run_wide(case, f"wide across the pass boundary kv={kv} {regime}") == PASS
    assert case.rows_run == sum(totals) > PASS
    start = totals[0] + totals[1]
    assert start < PASS < start + totals[2], "the third prompt does not straddle the boundary"


@pytest.mark.gpu
@pytest.mark.parametrize("nhead", [3, 6])
@pytest.mark.parametrize("kv", ["fp32", "bf16", "fp8"])
def test_128_wide_tiles(kv, nhead):
    """d = 384: QKV (N = 1152) and the out-projection and FFN2 (N = 384) have an odd number of 128-feature blocks, the
    shapes gemm_rows_launch runs as 128 x 128 tiles; at hd 128 each head is split over the two epilogue halves"""
    case = WideCase("tiny", kv=kv, totals=PACKED, d_model=384, audio_embedding_dim=384, nhead=nhead)
    d = case.d
    assert d == 384 and case.hd == 384 // nhead
    for N in (3 * d, d):                      # QKV, then out-projection and FFN2
        assert (N // 128) % 2 == 1, f"N = {N} runs 256-wide tiles"
    _run_wide(case, f"wide 128-wide tiles d=384 hd={case.hd} kv={kv}")


# ==========================================================================================================================
# 2. the rows-as-M GEMM per element
# ==========================================================================================================================
def _hilo_exact(x):
    """x with its 8 lowest mantissa bits cleared: 16 significant bits, which bf16 hi + lo (split_bf16) hold exactly"""
    return (x.view(torch.int32) & ~0xFF).view(torch.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [1, 127, 128, 129, 4096])
@pytest.mark.parametrize("K", [64, 1024, 8192])
@pytest.mark.parametrize("N", [256, 384, 1152, 1536])
def test_gemm_rows_elementwise(N, K, rows):
    """vcb_debug_gemm_rows against fp64 within GEMM(K) |x| |W|^T per element.  N / 128 even: 256-wide tiles, odd:
    128-wide.  Products of bf16 weights and hi / lo parts are exact in fp32, so all the error is the accumulation."""
    _l, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(N * 7 + K * 3 + rows)
    W = torch.randn(N, K, device="cuda", generator=g).to(torch.bfloat16).float()
    X = _hilo_exact(torch.randn(rows, K, device="cuda", generator=g))
    e = torch.randint(-20, 21, (rows, 1), device="cuda", generator=g)
    e[0] = 20
    e[-1] = -20
    X = torch.ldexp(X, e.float())
    out = torch.full((rows, N), float("nan"), device="cuda")
    _l.check(lib.vcb_debug_gemm_rows(W.data_ptr(), X.data_ptr(), out.data_ptr(), N, K, rows))
    Xd, Wd = X.double(), W.double()
    ref = Xd @ Wd.t()
    w = Worst(f"gemm_rows N={N} ({'256' if (N // 128) % 2 == 0 else '128'}-wide tiles) K={K} rows={rows}")
    w.check("out", out, ref, _gemm_c(K) * (Xd.abs() @ Wd.abs().t()))
    w.done()


# ==========================================================================================================================
# 3. placement invariance, bit for bit
# ==========================================================================================================================
def _kv_positions(eng, l, slot, T, kv, H, hd):
    """layer l's K and V bytes of a slot's positions 0 .. T-1, each [T, H, bytes] uint8 (fp8: the e4m3 bytes, then the
    position's scale)"""
    from kv_fp8_ref import split_slabs
    _l, lib = _lib()
    npg = (T + 63) // 64
    slab = {"fp32": 64 * hd * 4, "bf16": 64 * hd * 2, "fp8": 64 * (hd + 4)}[kv]
    kb = np.zeros(npg * H * slab, np.uint8)
    vb = np.zeros_like(kb)
    _l.check(lib.vcb_debug_kv_pages(eng, l, slot, 0, npg, kb.ctypes.data, vb.ctypes.data))
    out = []
    for raw in (kb, vb):
        t = torch.from_numpy(raw)
        if kv == "fp8":
            q, s = split_slabs(t, H, hd)
            t = torch.cat([q, s.unsqueeze(-1).contiguous().view(torch.uint8)], -1)
        else:
            t = t.reshape(npg, H, 64, -1)
        out.append(t.transpose(1, 2).reshape(npg * 64, H, -1)[:T].clone())
    return out


PROBE = 300                               # a partial tail page (300 % 64 = 44 positions)


def _placements():
    """name: ([(total, seed)] of the packed prompts with the probe as None, copies per prompt or None)"""
    P = PROBE
    a, b = (130, 21), (65, 22)
    big = (2000, 23)
    return {
        "alone": ([None], None),
        "first": ([None, a, b], None),
        "middle": ([a, None, b], None),
        "last": ([a, b, None], None),
        "pass boundary at its row 64": ([big, (PASS - 2000 - 64, 24), None, (200, 27)], None),
        "pass boundary at its row 171": ([big, (PASS - 2000 - 171, 25), None], None),
        "ending on a pass's last row": ([big, (PASS - 2000 - P, 26), None, (200, 27)], None),
        "best-of-3 leader": ([a, None, b], [1, 3, 1]),
    }


@pytest.mark.gpu
@pytest.mark.parametrize("kv,weights", [("fp32", "bf16"), ("bf16", "bf16"), ("fp8", "bf16"), ("bf16", "int8")])
def test_probe_prompt_bits_do_not_depend_on_its_placement(kv, weights):
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    import golden_util as gu
    _l, lib = _lib()
    cfg, sd = _checkpoint("tiny", 5)
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    m = m.to("cuda").eval()
    m.configure_engine(kv_dtype=kv, max_slots=8, max_seq_len=2048, weight_dtype=weights)
    eng = m._engine()
    L, H, K = cfg.num_decoder_layers, cfg.nhead, cfg.n_codebooks
    hd = cfg.d_model // H
    V = int(cfg.audio_vocab_size) + cfg.n_special
    sp = m._sampling(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3, silence_tokens=gu.SILENCE)

    def utt(total, seed, text=7):
        x, _, y = synthetic.synthetic_utterance(cfg, seed, text_len=text, prompt_frames=total - text - 1)
        return x, y

    probe = utt(PROBE, 11)
    scrub = [utt(1000, 90 + i) for i in range(8)]
    got = {}
    for name, (spec, copies) in _placements().items():
        # every slot's last hidden state and the pages released last overwritten first, so a placement cannot pass on
        # what an earlier one left behind
        Packed(m, scrub).close()
        utts = [probe if s is None else utt(*s) for s in spec]
        j = spec.index(None)
        first = sum(PROBE if s is None else s[0] for s in spec[:j])
        before = lib.vcb_counter(eng, b"prefill_rows")
        sess = Packed(m, utts, copies=copies)
        try:
            assert sess.eng == eng, "the engine was rebuilt"
            rows = lib.vcb_counter(eng, b"prefill_rows") - before
            assert rows == sum(p.total for p in sess.prompts) and sess.prompts[j].total == PROBE
            assert lib.vcb_counter(eng, b"wide_rows") == PASS, "not the wide path, or not passes of 4096 rows"
            if "boundary" in name:
                assert first < PASS < first + PROBE
            if "last row" in name:
                assert first + PROBE == PASS < rows
            lead, n = sess.slots[j], sess.copies[j]
            kvs = [_kv_positions(eng, l, lead, PROBE, kv, H, hd) for l in range(L)]
            for c in range(1, n):           # the forked members: shared full pages, their own copy of the tail page
                for l in range(L):
                    for part, t in enumerate(_kv_positions(eng, l, lead + c, PROBE, kv, H, hd)):
                        assert torch.equal(t, kvs[l][part]), f"{name}: member {c}'s layer {l} {'KV'[part]} differs"
            slots = (C.c_int32 * n)(*range(lead, lead + n))
            _l.check(lib.vcb_sample(eng, slots, n, None, C.byref(sp), sess.stream))
            logits = torch.empty(n * K, V, device="cuda")
            _l.check(lib.vcb_debug_logits(eng, logits.data_ptr(), n * K))
            logits = logits.cpu().reshape(n, K, V)
            for c in range(1, n):
                assert torch.equal(logits[c], logits[0]), f"{name}: member {c}'s first-sample logits differ"
            got[name] = (kvs, logits[0])
        finally:
            sess.close()
    kv0, lg0 = got.pop("alone")
    bad = []
    for name, (kvs, lg) in got.items():
        for l in range(L):
            for part in range(2):
                n_diff = int((kvs[l][part] != kv0[l][part]).any(-1).any(-1).sum())
                if n_diff:
                    bad.append(f"{name}: layer {l} {'KV'[part]} differs at {n_diff} positions")
        if not torch.equal(lg, lg0):
            bad.append(f"{name}: first-sample logits differ (max {float((lg - lg0).abs().max()):.3g})")
    print(f"placement invariance kv={kv} weights={weights}: {len(got)} placements against the probe alone, "
          f"{len(bad)} differ")
    assert not bad, "; ".join(bad)
