"""The fused sampler (sampler_kernel) on its own, through vcb_debug_sampler, against two restatements of the reference's
sampling step (voicecraft.py:26-86, 1018-1067, 718-787): the pinned fp32 oracle (lm_oracle.filter_top_k_top_p,
sample_rows, OracleLM._span_step) and an fp64 restatement of the same step, which measures how far each decision lies
from its boundary.  The GPU tests are marked `gpu`; the restatement itself and the hook's argument checks are pinned on
the CPU.

  * filter membership, every index of every case, by probe rows: probe row v carries the noise q_v = 1e-30 and q = 1
    elsewhere, so the kernel returns v if v survives temperature -> top-k -> top-p (and its probability is above 1e-20),
    else the most probable kept index (the lowest one at ties).  Vocabularies 4 .. 3072 (the kernel's ceiling, V % 4 != 0,
    V just above a multiple of 256), top_k from off to past V, top_p from 0 to 0.999, temperatures 0.3 / 1 / 1.7, on
    random rows of three scales, integer rows with heavy ties at the k-th value and across the nucleus cut, an all-equal
    row, rows holding -10000 entries and rows holding both +0.0 and -0.0.
      - top-k membership equals the oracle exactly: it involves no arithmetic beyond the IEEE temperature division.
      - top-p membership equals the oracle wherever the fp64 cumulative probability of every rank is more than 1e-5 from
        top_p.  The kernel's cumulative sums are fp32 scans of at most 3072 terms in a tree of depth <= 29 (16 sequential
        terms per thread, a 5-level warp scan, 8 warp totals), each term within 2 ulp, then one division by the fp32 total:
        under 29 * 2^-24 ~ 2e-6 off.  The oracle's fp32 cumsum is sequential; its rounding errors of random sign stay
        within a few 1e-6 over 3072 terms.  1e-5 covers both.
      - at ties straddling the cut the kept count equals the reference's, every value strictly above the tied one is
        kept, and the kept tied entries are the lowest indices (the kernel's rule).  The reference's own choice among tied
        entries is unspecified: torch's CPU sort(descending=True) is not stable.
  * exact nucleus boundaries: m equal logits among -10000 entries (each probability exactly 1/m, m a power of two), with
    top_p = j/m and one fp32 ulp below and above: the kept count follows the strict `cum > top_p` and the shift by one
    with no tolerance, and the kept entries are the lowest indices, for equal +-0.0 logits as well; with top_k = j too,
    whose k-th value all m entries tie.
  * the draw, argmax(p / q): random rows with random Exp(1) noise, 4 codebooks per row (column k*Vpad + v), over the same
    grid; the token equals the oracle's wherever the fp64 best p/q exceeds the runner-up by more than a factor 1 + 1e-5
    (and every kept count the top-p margin allows draws that same token).  And the device noise (noise pointer null)
    against the same rows fed torch's own draw under that generator state.
  * the state machine, one step, against OracleLM._span_step with the callers' eos edit: forced empties, the end token
    masked on codebook 0 until encodec_sr // 5 steps in TTS, the end-token trigger by sample / by argmax / by the length
    cap (first index wins a tie), the silence penalty and its bookkeeping, the end cascade for n_eog > 0, eos > 0 against
    eos <= 0.
"""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import lm_oracle
from oracle.lm_oracle import OracleLM

MARGIN = 1e-5
P_MIN = 1e-20                    # a kept index below this probability may lose its probe to the most probable one
VOCABS = [4, 255, 256, 257, 1023, 2052, 2053, 3071, 3072]
TOP_PS = [1.0, 0.0, 1e-6, 0.5, 0.8, 0.999]
TEMPS = [1.0, 0.3, 1.7]


def _top_ks(V):
    return [-100, 1, 2, 40, V - 1, V, V + 7]


def _grid(V):
    """every (top_k, top_p) pair, the temperature cycling through TEMPS"""
    pairs = [(k, p) for k in _top_ks(V) for p in TOP_PS]
    return [(k, p, TEMPS[i % len(TEMPS)]) for i, (k, p) in enumerate(pairs)]


def _lib():
    from voicecraft_b200 import _lib
    return _lib, _lib.load()


def _sp(top_k=-100, top_p=1.0, temperature=1.0, stop_repetition=0, silence=()):
    _l, _ = _lib()
    return _l.vcb_sampling(top_k=top_k, top_p=top_p, temperature=temperature, stop_repetition=stop_repetition,
                           n_silence=len(silence), silence_tokens=(C.c_int32 * 8)(*silence))


def _neutral(n, K):
    """state rows that let no edit, forced value or end trigger touch a sampled index: tts, n_eog 0, cur_num_gen K-1,
    no previous token, y_len 0 (under any length cap); used with empty_token = V, eog = V+1, eos = 0"""
    return np.tile(np.array([0, 0, K - 1, -1, 0, 1, 0], np.int32), (n, 1))


def _sample(logits, noise, sp, specials, state, seed=0, offset=0, threads=0):
    """logits [n][K][V] fp32 on the device, noise [n*K][V] or None -> tokens [n][K], state after [n][4] (numpy)"""
    _l, lib = _lib()
    n, K, V = logits.shape
    st = np.ascontiguousarray(state, dtype=np.int32)
    tok, out = np.zeros((n, K), np.int32), np.zeros((n, 4), np.int32)
    P = C.POINTER(C.c_int32)
    _l.check(lib.vcb_debug_sampler(logits.data_ptr(), None if noise is None else noise.data_ptr(), seed, offset, threads,
                                   C.byref(sp), n, K, V, *specials, st.ctypes.data_as(P), tok.ctypes.data_as(P),
                                   out.ctypes.data_as(P)))
    return tok, out


# ==========================================================================================================================
# the two restatements
# ==========================================================================================================================
def _temper(rows, temp):
    return rows / temp if temp != 1.0 else rows.clone()


def _oracle_kept(x, top_k, top_p):
    """the pinned fp32 oracle's filter on tempered rows [N][V]: the kept entries"""
    y = x.clone()
    lm_oracle.filter_top_k_top_p(y, top_k=top_k, top_p=top_p)
    return torch.isfinite(y)


def _ref64(x, top_k, top_p):
    """fp64 restatement of the filter on tempered fp32 rows [N][V] (the values the kernel sees), ties ranked lower index
    first.  Returns (order [N][V]: value descending, index ascending; n_topk [N]: entries the top-k keeps, a prefix of
    `order`; cum [N][V]: fp64 cumulative softmax over `order` after top-k; n_kept [N]; kept [N][V])."""
    N, V = x.shape
    srt, order = torch.sort(x, dim=1, descending=True, stable=True)
    srt = srt.double()
    keep = torch.ones(N, V, dtype=torch.bool)
    if top_k > 0:
        k = min(max(top_k, 1), V)
        keep &= srt >= srt[:, k - 1: k]                     # strict '<' removes: ties with the k-th value stay
    n_topk = keep.sum(1)
    cum = torch.softmax(torch.where(keep, srt, torch.tensor(-np.inf, dtype=torch.float64)), dim=1).cumsum(1)
    if top_p < 1.0:
        rm = cum > float(np.float32(top_p))                 # the oracle and the kernel both compare with fp32 top_p
        keep &= ~torch.cat([torch.zeros(N, 1, dtype=torch.bool), rm[:, :-1]], dim=1)
    kept = torch.zeros(N, V, dtype=torch.bool).scatter(1, order, keep)
    return order, n_topk, cum, keep.sum(1), kept


def _softmax_over(x, kept):
    return torch.softmax(torch.where(kept, x.double(), torch.tensor(-np.inf, dtype=torch.float64)), dim=-1)


def _prefix(order_row, L):
    m = torch.zeros(order_row.numel(), dtype=torch.bool)
    m[order_row[:L]] = True
    return m


# ==========================================================================================================================
# filter membership by probe rows
# ==========================================================================================================================
def _probe(rows, top_k, top_p, temp):
    """rows [m][V] fp32 -> t [m][V]: the token the kernel returns for probe row (r, v) (noise 1e-30 at v, 1 elsewhere)"""
    m, V = rows.shape
    logits = rows.cuda().repeat_interleave(V, dim=0).view(m * V, 1, V)
    noise = torch.ones(m * V, V, device="cuda")
    noise.view(m, V, V).diagonal(dim1=1, dim2=2).fill_(1e-30)
    tok, _ = _sample(logits, noise, _sp(top_k, top_p, temp), (V, V + 1, 0, 50), _neutral(m * V, 1))
    del logits, noise
    return torch.from_numpy(tok.reshape(m, V)).long()


def _probe_mismatch(t, x, kept, a_star):
    """probe results t [V] against the kept set `kept` [V]: kept with p > P_MIN -> v, removed -> a_star, kept below P_MIN
    -> either.  Returns the indices that break the rule."""
    V = t.numel()
    idx = torch.arange(V)
    p = _softmax_over(x, kept)
    want = torch.where(kept & (p > P_MIN), idx, torch.full_like(idx, a_star))
    either = kept & (p <= P_MIN) & ((t == idx) | (t == a_star))
    return idx[(t != want) & ~either]


def _rows(V, seed):
    """the logit rows every case is crossed with"""
    g = torch.Generator().manual_seed(seed)
    rows = [torch.randn(V, generator=g) * s for s in (0.5, 3.0, 30.0)]
    rows.append(torch.randint(-3, 4, (V,), generator=g).float())              # 7 tied classes: ties at most cuts
    rows.append(torch.randint(0, 3, (V,), generator=g).float() * 2.0)         # 3 classes of ~V/3 tied entries
    rows.append(torch.full((V,), 1.25))                                        # all equal
    r = torch.randn(V, generator=g) * 3.0
    r[torch.randperm(V, generator=g)[: max(2, V // 4)]] = -10000.0
    rows.append(r)
    z = torch.where(torch.rand(V, generator=g) < 0.5, torch.tensor(-0.0), torch.tensor(0.0))
    perm = torch.randperm(V, generator=g)
    z[perm[: max(1, V // 16)]] = 0.5
    z[perm[max(1, V // 16): max(1, V // 16) + V // 8]] = -1.0
    rows.append(z)                                                             # the cut falls among the +-0.0 entries
    return torch.stack(rows)


ROW_KINDS = ["randn*0.5", "randn*3", "randn*30", "int7", "int3", "equal", "-10000", "+-0"]

# what the GPU tests saw, printed at the end of the module: probed indices, decisions inside the margin (the nearest one's
# distance from its boundary, and the largest distance at which the kernel and the fp64 restatement decided differently)
_report = {"probed": 0, "topp_in_margin": 0, "topp_min_dist": float("inf"), "topp_max_disagree": 0.0, "draw_rows": 0,
           "draw_in_margin": 0, "draw_min_gap": float("inf"), "draw_max_disagree": 0.0}


@pytest.mark.gpu
@pytest.mark.parametrize("V", VOCABS)
def test_filter_membership_by_probe_rows(V):
    rows = _rows(V, 100 + V)
    idx = torch.arange(V)
    failures, in_margin = [], {}
    for ci, (top_k, top_p, temp) in enumerate(_grid(V)):
        x = _temper(rows, temp)
        t = _probe(rows, top_k, top_p, temp)
        ok32 = _oracle_kept(x, top_k, top_p)
        order, n_topk, cum, n_kept, kept64 = _ref64(x, top_k, top_p)
        for r in range(len(rows)):
            case = f"V={V} top_k={top_k} top_p={top_p} T={temp} row={ROW_KINDS[r]}"
            a_star = int((x[r] == x[r].max()).nonzero()[0])            # most probable, lowest index at ties
            stray = idx[(t[r] != idx) & (t[r] != a_star)]
            if len(stray):
                failures.append(f"{case}: probes {stray[:5].tolist()} returned neither themselves nor {a_star}")
                continue
            _report["probed"] += V
            if top_p >= 1.0:
                # top-k alone: exact, and the fp64 restatement agrees with the oracle
                assert torch.equal(ok32[r], kept64[r]), f"{case}: fp64 restatement differs from the oracle"
                bad = _probe_mismatch(t[r], x[r], ok32[r], a_star)
                if len(bad):
                    failures.append(f"{case}: top-k membership differs at {bad[:8].tolist()} ({len(bad)} indices)")
                continue
            dist = (cum[r] - float(np.float32(top_p))).abs()
            n_marg = int((dist <= MARGIN).sum())
            c64 = int(n_kept[r])
            if n_marg == 0:
                # outside the margin: the oracle's count, values above the tie all kept, the kept ties the lowest indices
                c32 = int(ok32[r].sum())
                vc = x[r][order[r, c64 - 1]]
                assert c32 == c64 and bool(ok32[r][x[r] > vc].all()) and bool((x[r][ok32[r]] >= vc).all()), \
                    f"{case}: the oracle keeps {c32}, the fp64 restatement {c64}"
                bad = _probe_mismatch(t[r], x[r], kept64[r], a_star)
                if len(bad):
                    failures.append(f"{case}: top-p membership differs at {bad[:8].tolist()} ({len(bad)} indices), "
                                    f"kept {c64}, nearest cum {float(dist.min()):.3g} from top_p")
                continue
            # inside the margin: the kernel keeps a prefix of the ranked order whose length is decided within the margin
            in_margin[case] = float(dist.min())
            _report["topp_in_margin"] += 1
            _report["topp_min_dist"] = min(_report["topp_min_dist"], float(dist.min()))
            lens = sorted(range(max(1, c64 - n_marg), min(int(n_topk[r]), c64 + n_marg) + 1), key=lambda L: abs(L - c64))
            L = next((L for L in lens if len(_probe_mismatch(t[r], x[r], _prefix(order[r], L), a_star)) == 0), None)
            if L is None:
                failures.append(f"{case}: within the margin, but the kept set is no prefix of {lens} ranks")
            elif L != c64:
                _report["topp_max_disagree"] = max(_report["topp_max_disagree"], float(dist.min()))
    print(f"\nV={V}: {len(_grid(V))} cases x {len(rows)} rows, {len(_grid(V)) * len(rows) * V} probed indices; "
          f"top-p boundaries inside the {MARGIN:g} margin: {len(in_margin)}")
    for case, d in in_margin.items():
        print(f"  in margin: {case}: nearest cumulative probability {d:.3g} from top_p")
    assert not failures, "\n".join(failures[:20])


# ==========================================================================================================================
# exact nucleus boundaries
# ==========================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("V", [257, 2053, 3072])
def test_exact_nucleus_boundaries(V):
    """m equal logits among -10000 entries: every kept probability is exactly 1/m and every cumulative sum j/m, in the
    kernel's scan as in the oracle's cumsum.  top_p = j/m keeps j + 1 (cum > top_p is strict, then the shift by one),
    one ulp below keeps j, one ulp above j + 1; the kept entries are the lowest indices of the m, for +-0.0 logits too.
    With top_k = j as well, the top-k keeps all m (they tie the k-th value) and the counts are the same."""
    g = torch.Generator().manual_seed(V)
    failures = []
    for m in (m for m in (2, 4, 8, 64, 256, 1024) if m <= V):
        pos = torch.sort(torch.randperm(V, generator=g)[:m]).values
        rows = torch.full((2, V), -10000.0)
        rows[0, pos] = 2.5
        rows[1, pos] = torch.where(torch.arange(m) % 2 == 0, torch.tensor(-0.0), torch.tensor(0.0))  # -0.0 at the lowest
        for j in sorted({1, m // 2, m - 1}):
            exact = np.float32(j / m)
            for top_p, want in ((exact, j + 1), (np.nextafter(exact, np.float32(0)), j),
                                (np.nextafter(exact, np.float32(1)), j + 1)):
                # top_k = j: the k-th value is tied by all m entries, and the strict '<' keeps every one of them
                for top_k in (-100, j):
                    top_p = float(top_p)
                    ok32 = _oracle_kept(rows, top_k, top_p)
                    assert ok32.sum(1).tolist() == [want, want] and bool(ok32[:, pos].sum(1).eq(want).all()), \
                        f"the oracle keeps {ok32.sum(1).tolist()} of m={m} at top_p={top_p!r}, not {want}"
                    t = _probe(rows, top_k, top_p, 1.0)
                    kept = torch.zeros(V, dtype=torch.bool)
                    kept[pos[:want]] = True
                    for r, kind in enumerate(("2.5", "+-0.0")):
                        bad = _probe_mismatch(t[r], rows[r], kept, int(pos[0]))
                        if len(bad):
                            failures.append(f"V={V} m={m} top_k={top_k} top_p={top_p!r} logits {kind}: keeps "
                                            f"{int((t[r][pos] == pos).sum())} (want the lowest {want}), wrong at "
                                            f"{bad[:6].tolist()}")
    assert not failures, "\n".join(failures[:20])


# ==========================================================================================================================
# the draw
# ==========================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("V", VOCABS)
def test_draw_matches_oracle(V):
    K, n = 4, 16
    g = torch.Generator().manual_seed(7 * V)
    failures, in_margin = [], []
    for ci, (top_k, top_p, temp) in enumerate(_grid(V)):
        scale = torch.tensor([0.5, 3.0, 30.0])[torch.randint(0, 3, (n, K, 1), generator=g)]
        logits = torch.randn(n, K, V, generator=g) * scale
        noise = torch.empty(n * K, V).exponential_(1, generator=g)
        tok, _ = _sample(logits.cuda(), noise.cuda(), _sp(top_k, top_p, temp), (V, V + 1, 0, 50), _neutral(n, K))
        tok = torch.from_numpy(tok).long().view(-1)
        rows = logits.view(n * K, V)
        ref = lm_oracle.sample_rows(rows.clone(), top_k, top_p, temp, lambda shape: noise).view(-1)
        x = _temper(rows, temp)
        order, n_topk, cum, n_kept, kept = _ref64(x, top_k, top_p)

        def scores(keep, xs=x, qs=noise):
            s = torch.where(keep, _softmax_over(xs, keep) / qs.double(), torch.tensor(-1.0, dtype=torch.float64))
            top2 = s.topk(min(2, V), dim=-1).values
            g = top2[..., 0] / top2[..., -1] - 1
            return s, torch.where(top2[..., -1] > 0, g, torch.tensor(np.inf, dtype=torch.float64))

        sc, gap = scores(kept)
        tp32 = float(np.float32(top_p))
        dist = (cum - tp32).abs().min(1).values if top_p < 1.0 else torch.full((n * K,), np.inf)
        _report["draw_rows"] += n * K
        for r in range(n * K):
            case = f"V={V} top_k={top_k} top_p={top_p} T={temp} row={r}"
            if dist[r] <= MARGIN and gap[r] > MARGIN:
                # the nucleus boundary is within the margin: decided all the same if every kept count the margin allows
                # draws the same token, each by more than the margin
                n_marg, c64 = int(((cum[r] - tp32).abs() <= MARGIN).sum()), int(n_kept[r])
                lens = range(max(1, c64 - n_marg), min(int(n_topk[r]), c64 + n_marg) + 1)
                alt = [scores(_prefix(order[r], L), x[r], noise[r]) for L in lens]
                if len({int(s.argmax()) for s, _ in alt}) == 1 and all(g > MARGIN for _, g in alt):
                    dist[r] = np.inf
            if gap[r] <= MARGIN or dist[r] <= MARGIN:
                same = int(tok[r]) == int(ref[r])
                in_margin.append(f"{case}: p/q gap {float(gap[r]):.3g}, nucleus {float(dist[r]):.3g}, "
                                 f"{'same token' if same else 'tokens differ'}")
                _report["draw_in_margin"] += 1
                if not same:
                    _report["draw_max_disagree"] = max(_report["draw_max_disagree"], float(min(gap[r], dist[r])))
                continue
            _report["draw_min_gap"] = min(_report["draw_min_gap"], float(gap[r]))
            assert int(ref[r]) == int(sc[r].argmax()), f"{case}: the oracle's token differs from the fp64 restatement"
            if int(tok[r]) != int(ref[r]):
                failures.append(f"{case}: kernel {int(tok[r])}, oracle {int(ref[r])} (p/q gap {float(gap[r]):.3g})")
    print(f"\nV={V}: {len(_grid(V)) * n * K} draws, {len(in_margin)} inside the {MARGIN:g} margin")
    for line in in_margin:
        print("  in margin:", line)
    assert not failures, "\n".join(failures[:20])


@pytest.mark.gpu
def test_device_noise_equals_torch_draw():
    """noise pointer null: row i, codebook k draws element k*V + v of the [K][V] draw of its one-member group's generator
    (the reference's multinomial over [size*K, V], member 0); every row's generator sits at the same (seed, offset), so the
    same tokens come from feeding every row torch.empty(K*V, device="cuda").exponential_(1) under that state"""
    from voicecraft_b200.voicecraft import VoiceCraft
    V, K, n = 2053, 4, 12
    seed, offset = 0x5EED1234ABC, 8
    logits = (torch.randn(n, K, V, generator=torch.Generator().manual_seed(3)) * 0.5).cuda()
    gen = torch.cuda.default_generators[0]
    saved = gen.get_state()
    try:
        gen.manual_seed(seed)
        gen.set_offset(offset)
        draw = torch.empty(K * V, device="cuda").exponential_(1)
    finally:
        gen.set_state(saved)
    threads = VoiceCraft._rng_threads(torch.device("cuda", 0), K * V)
    sp = _sp(40, 0.9, 0.8)
    dev, _ = _sample(logits, None, sp, (V, V + 1, 0, 50), _neutral(n, K), seed=seed, offset=offset, threads=threads)
    fed, _ = _sample(logits, draw.view(K, V).repeat(n, 1).contiguous(), sp, (V, V + 1, 0, 50), _neutral(n, K))
    assert np.array_equal(dev, fed), f"device noise tokens\n{dev}\nfed\n{fed}"
    assert len(np.unique(dev)) > n, "the rows should draw different tokens"


# ==========================================================================================================================
# the state machine, one step
# ==========================================================================================================================
SM_V, SM_EMPTY, SM_EOG, SM_SR, SM_XLEN = 256, 252, 253, 75, 3        # encodec_sr // 5 = 15; caps: tts 45, edit 30
SILENCE = [10, 20, 30]


def _sm_rows(K, eos, g):
    """(label, state, logits [K][V], noise [K][V]) rows for one (K, eos)"""
    V, E_tts = SM_V, (eos if eos > 0 else SM_EOG)
    rows = []

    def add(label, mode, n_eog=0, cur=20, prev=-1, consec=0, y_len=5, edit=None, ones=False):
        E = E_tts if mode == 0 else SM_EOG
        lg = torch.randn(K, V, generator=g) * 2.0
        q = torch.ones(K, V) if ones else torch.empty(K, V).exponential_(1, generator=g)
        if edit:
            edit(lg, q, E)
        rows.append((f"{label} mode={mode}", [mode, n_eog, cur, prev, consec, SM_XLEN, y_len], lg, q))

    def boost_end(lg, q, E):                      # end and empty token would win every codebook unless masked
        lg[:, E] = 9.0
        lg[:, SM_EMPTY] = 8.0
        lg[:, SM_EOG] = 8.5
        if eos > 0:
            lg[:, eos] = 8.7

    for mode in (0, 1):
        E = E_tts if mode == 0 else SM_EOG
        for cur in sorted({0, 1, K - 2, K - 1, K, 40}):                         # forced empties for k > cur
            add(f"cur={cur}", mode, cur=cur)
        for cur in (SM_SR // 5, SM_SR // 5 + 1):                                # end masked on codebook 0 (tts)
            add(f"end mask cur={cur}", mode, cur=cur, edit=boost_end)

        def by_sample(lg, q, E):
            lg[0, 5], lg[0, E] = 12.0, 11.5
            q[0, E] = 1e-3

        def by_argmax(lg, q, E):
            lg[0, E] = 12.0
            q[0, E] = 1e3

        def tie_lower(lg, q, E):                                                # index 7 < E ties the end token
            lg[0, 7] = lg[0, E] = 12.0
            q[0, E] = 1e3

        def tie_higher(lg, q, E):                                               # index 255 > E ties it
            lg[0, 255] = lg[0, E] = 12.0
            q[0, E] = q[0, 255] = 1e3

        for label, fn in (("trigger by sample", by_sample), ("trigger by argmax", by_argmax),
                          ("tie with a lower index", tie_lower), ("tie with a higher index", tie_higher)):
            add(label, mode, edit=fn)

        def quiet_end(lg, q, E):
            lg[0, E] = -5.0
            q[0, E] = 1e3

        cap = SM_XLEN * (SM_SR // 5) if mode == 0 else SM_XLEN * 10
        for y in (cap, cap + 1):                                                # the length cap
            add(f"y_len={y} cap={cap}", mode, y_len=y, edit=quiet_end)

        def sil_pos(lg, q, E):                                                  # 6 / 2 = 3 < 4: the penalty flips it
            lg[0] = torch.randn(V, generator=g) * 0.5 - 3.0
            lg[0, 10], lg[0, 11] = 6.0, 4.0

        def sil_neg(lg, q, E):                                                  # -1 * 2 = -2 < -1.5
            lg[0] = -3.0
            lg[0, 10], lg[0, 11] = -1.0, -1.5

        for label, fn in (("silence +", sil_pos), ("silence -", sil_neg)):
            for prev, consec in ((10, 3), (10, 4), (10, 6), (-1, 9), (11, 9)):
                add(f"{label} prev={prev} consec={consec}", mode, prev=prev, consec=consec, edit=fn, ones=True)
        for n_eog in sorted({1, K - 1}):                                        # the end cascade
            add(f"n_eog={n_eog}", mode, n_eog=n_eog, edit=boost_end)
            add(f"n_eog={n_eog} random", mode, n_eog=n_eog, prev=10, consec=5)
        add("eog boosted", mode, edit=lambda lg, q, E: lg[:, SM_EOG].fill_(9.0))   # eos > 0 moves the eog mask
        if eos > 0:
            add("eos boosted", mode, edit=lambda lg, q, E: lg[:, eos].fill_(9.0))
    return rows


def _span_step_ref(K, eos, samp, state, logits, noise):
    o = object.__new__(OracleLM)
    o.c = SimpleNamespace(n_codebooks=K, empty_token=SM_EMPTY, eog=SM_EOG, eos=eos, encodec_sr=SM_SR)
    mode, n_eog, cur, prev, consec, x_len, y_len = state
    lg = logits.clone()
    if eos > 0:                                                                 # the callers' edit (lm_oracle.py:321, :508)
        lg[:, SM_EOG if mode == 0 else eos] = -10000.0
    st = dict(eog=[True] * n_eog + [False] * (K - n_eog), cur=cur, prev=None if prev < 0 else prev, consec=consec,
              mode="tts" if mode == 0 else "edit")
    s = o._span_step(st, lg, samp, y_len, x_len, lambda shape: noise)
    n_after = sum(st["eog"])
    return s[:, 0].tolist(), [-1 if st["prev"] is None else st["prev"], st["consec"], n_after, int(n_after == K)]


@pytest.mark.gpu
@pytest.mark.parametrize("K", [4, 8])
@pytest.mark.parametrize("eos", [254, 0])
@pytest.mark.parametrize("filt", [(-100, 1.0, 1.0, 3), (40, 0.9, 0.8, 3), (-100, 1.0, 1.0, 0), (-100, 1.0, 1.0, -1)])
def test_state_machine_step_matches_span_step(K, eos, filt):
    top_k, top_p, temp, rep = filt
    rows = _sm_rows(K, eos, torch.Generator().manual_seed(K * 1000 + eos + 7 * rep + top_k))
    logits = torch.stack([r[2] for r in rows]).cuda()
    noise = torch.cat([r[3] for r in rows]).cuda()
    state = np.array([r[1] for r in rows], np.int32)
    tok, out = _sample(logits, noise, _sp(top_k, top_p, temp, rep, SILENCE), (SM_EMPTY, SM_EOG, eos, SM_SR), state)
    samp = dict(top_k=top_k, top_p=top_p, temperature=temp, stop_repetition=rep, silence_tokens=SILENCE)
    failures = []
    for i, (label, st, lg, q) in enumerate(rows):
        want_tok, want_st = _span_step_ref(K, eos, samp, st, lg, q)
        if tok[i].tolist() != want_tok or out[i].tolist() != want_st:
            failures.append(f"{label} state={st}: tokens {tok[i].tolist()} / {want_tok}, "
                            f"(prev, consec, n_eog, done) {out[i].tolist()} / {want_st}")
    assert not failures, "\n".join(failures)


# ==========================================================================================================================
# CPU: the fp64 restatement is pinned to the oracle, and the hook rejects bad arguments before any launch
# ==========================================================================================================================
@pytest.mark.parametrize("V", [257, 2053])
def test_fp64_restatement_matches_the_oracle(V):
    """on random rows (no ties), outside the margin: the kept set of the fp64 restatement equals lm_oracle's, and so does
    argmax(p64 / q) against sample_rows; plus the exact boundaries the GPU test relies on"""
    g = torch.Generator().manual_seed(V)
    checked = 0
    for top_k, top_p, temp in _grid(V):
        rows = torch.randn(24, V, generator=g) * torch.tensor([0.5, 3.0, 30.0]).repeat(8)[:, None]
        noise = torch.empty(24, V).exponential_(1, generator=g)
        x = _temper(rows, temp)
        _, _, cum, _, kept = _ref64(x, top_k, top_p)
        ok32 = _oracle_kept(x, top_k, top_p)
        ref = lm_oracle.sample_rows(rows.clone(), top_k, top_p, temp, lambda shape: noise).view(-1)
        sc = torch.where(kept, _softmax_over(x, kept) / noise.double(), torch.tensor(-1.0, dtype=torch.float64))
        top2 = sc.topk(2, dim=1).values
        for r in range(24):
            if top_p < 1.0 and float((cum[r] - float(np.float32(top_p))).abs().min()) <= MARGIN:
                continue
            assert torch.equal(kept[r], ok32[r]), (top_k, top_p, temp, r)
            if top2[r, 1] <= 0 or top2[r, 0] / top2[r, 1] > 1 + MARGIN:
                assert int(sc[r].argmax()) == int(ref[r]), (top_k, top_p, temp, r)
                checked += 1
    assert checked > 0.9 * 24 * len(_grid(V))
    # exact boundaries: 4 equal logits, top_p = 0.5 keeps 3 (the example of the docstring)
    row = torch.full((1, V), -10000.0)
    row[0, [3, 9, 100, 200]] = 1.0
    assert int(_oracle_kept(row, -100, 0.5).sum()) == 3
    assert int(_ref64(row, -100, 0.5)[3]) == 3
    assert int(_ref64(row, -100, float(np.nextafter(np.float32(0.5), np.float32(0))))[3]) == 2


def test_debug_sampler_rejects_bad_arguments():
    """every rejection is decided on the host, before any allocation, copy or launch (so this needs no GPU)"""
    _l, lib = _lib()
    logits = np.zeros(64, np.float32)            # never read: the call must return before touching it
    P = C.POINTER(C.c_int32)
    sp = _sp()

    def call(n=1, K=4, V=16, empty=16, eog=17, eos=0, state=(0, 0, 3, -1, 0, 1, 0), noise_threads=1):
        st = np.array(state * max(n, 1), np.int32)
        tok, out = np.zeros(64, np.int32), np.zeros(64, np.int32)
        rc = lib.vcb_debug_sampler(logits.ctypes.data, None, 1, 0, noise_threads, C.byref(sp), n, K, V, empty, eog, eos, 50,
                                   st.ctypes.data_as(P), tok.ctypes.data_as(P), out.ctypes.data_as(P))
        return rc, (lib.vcb_last_error() or b"").decode()

    cases = {
        "n": dict(n=0), "K=0": dict(K=0), "K=9": dict(K=9), "V=0": dict(V=0), "V=3073": dict(V=3073),
        "empty": dict(empty=18), "empty<0": dict(empty=-1), "eog": dict(eog=18), "eos": dict(eos=18),
        "mode": dict(state=(2, 0, 3, -1, 0, 1, 0)), "n_eog<0": dict(state=(0, -1, 3, -1, 0, 1, 0)),
        "n_eog=K": dict(state=(0, 4, 3, -1, 0, 1, 0)), "y_len<0": dict(state=(0, 0, 3, -1, 0, 1, -1)),
        "no noise": dict(noise_threads=0),
    }
    for name, kw in cases.items():
        rc, msg = call(**kw)
        assert rc != 0 and msg.startswith("vcb_debug_sampler:"), f"{name}: rc {rc}, {msg!r}"


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    r = _report
    if r["probed"] or r["draw_rows"]:
        print(f"\nsampler numerics: {r['probed']} probed indices, {r['topp_in_margin']} top-p boundaries inside the "
              f"margin (nearest {r['topp_min_dist']:.3g}, kernel and fp64 counts differing up to "
              f"{r['topp_max_disagree']:.3g}); {r['draw_rows']} draws, {r['draw_in_margin']} inside the margin (tokens "
              f"differing up to {r['draw_max_disagree']:.3g}), smallest p/q gap checked {r['draw_min_gap']:.3g}")
