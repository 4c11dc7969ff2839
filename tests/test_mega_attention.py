"""The persistent step kernel's attention phase (csrc/mega_step.cu, VCB_MEGA=1) on its own, through its cooperative launch
(vcb_debug_mega_attention), against fp64 and against itself.

The phase has its own attention implementation: work items of 4 pages of one (row, head) split between CTAs by a unit
range, scores in the log2 domain, 8 warp states folded per chunk and chunk states folded per item (on chip for up to 16
chunks of one CTA, else through a workspace by the last CTA to arrive), and the current position's key taken from the QKV
epilogue's knew / vnew buffers, not from the page.  The cases are test_kernel_numerics' planted ones cut into the
kernel's own chunks, at contexts up to 8201 keys, plus what only this kernel has:
  * underflow_cached: a cached key of a middle chunk dominates, so the key at pos (knew) underflows with every other chunk;
  * self_min: knew has logit -140;
  * max_other_cta: the maximum sits in a chunk whose CTA owns no other chunk of the item, so it reaches the result only
    through the workspace.  Ownership is the kernel's rule restated here, at grids where such chunks exist.
knew / vnew are the pool's slot at pos, so _attn_ref (softmax over keys 0..pos of the pages) is the reference unchanged.

CPU: the cases are as hostile as claimed (fp64).  GPU (-m gpu): every row against fp64 at every grid, KV policy and head
count; bit identity across grids 1 .. max, batch position, row padding, repeated and mixed-grid launches on one workspace;
only knew / vnew stand for position pos; inactive rows stay untouched; the hook's rejections.
"""
import math
from functools import lru_cache

import pytest
import torch

from test_kernel_numerics import KINDS, PAGE, _attn_case, _attn_ref

CHUNK = 4                                   # pages per work item (MG_CHUNK)
MAXCH = 16                                  # chunks an item may fold on chip (MG_MAXCH)
HD = 128
POSITIONS = [0, 1, 63, 64, 65, 255, 256, 257, 1023, 1024, 4095, 4096, 4100, 8200]
MEGA_KINDS = KINDS + ("underflow_cached", "self_min")
MOC_POSITIONS = [p for p in POSITIONS if p >= CHUNK * PAGE]        # items of at least 2 chunks
NOMINAL_MAX_GRID = 132                      # one CTA per SM of an H100 SXM; the GPU tests use the device's own count
GRIDS = [1, 2, 3, 7, 16, 33, 64, 131, "max"]
MOC_GRIDS = [7, 16, 33, 64, 131, "max"]     # grids at which the launches below have chunks owned alone (none at 2 and 3)
LOG2E = 1.4426950408889634
TINY = 2.0 ** -126                          # fp32's smallest normal


def _max_grid():
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(0).multi_processor_count
    return NOMINAL_MAX_GRID


def _grid(G):
    return _max_grid() if G == "max" else G


# --------------------------------------------------------------------------------------------------------------------------
# the kernel's work split, restated
# --------------------------------------------------------------------------------------------------------------------------
def _launches(pos, size=32):
    """the case's row indices in launches of at most `size` rows: its active rows in order, its two inactive rows at the
    front and in the middle of every launch"""
    act = [i for i, p in enumerate(pos) if p >= 0]
    ina = [i for i, p in enumerate(pos) if p < 0]
    per = size - len(ina)
    out = []
    for k in range(0, len(act), per):
        a = act[k:k + per]
        out.append([ina[0]] + a[:len(a) // 2] + ina[1:] + a[len(a) // 2:])
    return out


def _owner_rule(pos, H, G):
    """{(launch row, head): owner CTA of each chunk} by mg_owner: chunk start s belongs to ((s + 1) * Ge - 1) // U"""
    npg = [p // PAGE + 1 if p >= 0 else 0 for p in pos]
    U = H * sum(npg)
    Ge = min(U, G)
    out, u = {}, 0
    for r, n in enumerate(npg):
        for h in range(H):
            out[(r, h)] = [((s + 1) * Ge - 1) // U for s in range(u, u + n, CHUNK)]
            u += n
    return out


def _owner_ranges(pos, H, G):
    """the same from the ranges themselves (mg_range, mg_chunk_align): CTA c < Ge takes the chunks that start in
    [c * U / Ge, (c + 1) * U / Ge), in 32-bit unsigned arithmetic"""
    npg = [p // PAGE + 1 if p >= 0 else 0 for p in pos]
    U = H * sum(npg)
    Ge = min(U, G)
    bounds = [(U * c % 2 ** 32) // Ge for c in range(Ge + 1)]
    out, u = {}, 0
    for r, n in enumerate(npg):
        for h in range(H):
            out[(r, h)] = [next(c for c in range(Ge) if bounds[c] <= s < bounds[c + 1]) for s in range(u, u + n, CHUNK)]
            u += n
    return out


def _solo_chunks(owners):
    """chunks of an item shared between CTAs whose owner holds no other chunk of the item"""
    if len(set(owners)) < 2:
        return []
    return [j for j, o in enumerate(owners) if owners.count(o) == 1]


# --------------------------------------------------------------------------------------------------------------------------
# cases
# --------------------------------------------------------------------------------------------------------------------------
@lru_cache(maxsize=None)
def _case(kv, H):
    """every (position, kind) pair, chunks of the kernel's 4 pages"""
    return _attn_case(HD, kv, CHUNK, seed=7, positions=POSITIONS, kinds=MEGA_KINDS, H=H)


@lru_cache(maxsize=None)
def _moc_case(kv, H, G):
    """rows of MOC_POSITIONS launched together at grid G; the maximum of item (row, head) sits in a chunk its owner holds
    alone where the item has one (c["solo"]), else on the first key of a middle chunk"""
    solo = {}

    def plant(r, pos, kind):
        lrow = {i: k for k, i in enumerate(_launches(pos)[0])}
        owners = _owner_rule([pos[i] for i in _launches(pos)[0]], H, G)
        p, ts = pos[r], []
        for h in range(H):
            js = _solo_chunks(owners[(lrow[r], h)])
            if js:
                j = js[len(js) // 2]
                solo[(r, h)] = j
                ts.append(min(j * CHUNK * PAGE + 77, p))
            else:
                ts.append((p // (CHUNK * PAGE)) // 2 * CHUNK * PAGE)
        return ts, 40.0

    c = _attn_case(HD, kv, CHUNK, seed=100 + G, positions=MOC_POSITIONS, kinds=("max_other_cta",), H=H, plant=plant)
    c["solo"] = solo
    return c


def _scores(c, r, h):
    """fp64 logits of row r, head h over keys 0..pos (the key at pos last)"""
    p = int(c["pos"][r])
    pages = c["page_table"][int(c["row_slot"][r])][: p // PAGE + 1].long()
    K = c["Kp"][pages, h].double().reshape(-1, c["hd"])[: p + 1]
    q = c["q"][r, h].double()
    return (K @ q) / math.sqrt(c["hd"]), (K.abs() @ q.abs()) / math.sqrt(c["hd"])


def _chunk_weights(s):
    """softmax weight of each 4-page chunk relative to the largest weight"""
    w = torch.exp(s - s.max())
    n = (len(s) + CHUNK * PAGE - 1) // (CHUNK * PAGE)
    return torch.stack([w[j * CHUNK * PAGE:(j + 1) * CHUNK * PAGE].sum() for j in range(n)])


# --------------------------------------------------------------------------------------------------------------------------
# CPU: the cases are what their names say
# --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [2, 16])
@pytest.mark.parametrize("kv", ["fp32", "bf16"])
def test_hostile_cases_are_hostile(kv, H):
    """On fp64: in underflow / underflow_cached rows every chunk but the dominant one weighs less than fp32's smallest
    normal relative to the maximum (the dominant chunk being the self key's / a middle one); in self_min rows the key at
    pos does; and at every grid of MOC_GRIDS some max_other_cta items have their maximum in a chunk whose owner - by the
    kernel's range rule - holds no other chunk of the item, while mg_owner's closed form agrees with those ranges."""
    c = _case(kv, H)
    n_under = 0
    for r, (p, kind) in enumerate(zip(c["pos"].tolist(), c["kinds"])):
        if kind not in ("underflow", "underflow_cached", "self_min"):
            continue
        for h in range(H):
            s, _ = _scores(c, r, h)
            if kind == "self_min":
                if p > 0:
                    assert math.exp(float(s[-1] - s.max())) < TINY, (r, p, h)
                continue
            cw = _chunk_weights(s)
            top = int(torch.argmax(cw))
            span = CHUNK * PAGE
            want = p // span if kind == "underflow" or p == 0 else (p // span) // 2
            assert top == want, (kind, p, h, top, want)
            others = torch.cat([cw[:top], cw[top + 1:]])
            assert len(others) == 0 or float(others.max()) < TINY, (kind, p, h, float(others.max()))
            n_under += len(others) > 0
    assert n_under == 2 * len(MOC_POSITIONS) * H, n_under            # every row of 2 chunks or more
    for G in MOC_GRIDS:
        G = NOMINAL_MAX_GRID if G == "max" else G
        m = _moc_case(kv, H, G)
        launch = _launches(m["pos"].tolist())
        assert len(launch) == 1
        lpos = [int(m["pos"][i]) for i in launch[0]]
        by_rule, by_range = _owner_rule(lpos, H, G), _owner_ranges(lpos, H, G)
        assert by_rule == by_range, G
        lrow = {i: k for k, i in enumerate(launch[0])}
        assert m["solo"], f"grid {G}: no chunk owned alone"
        for (r, h), j in m["solo"].items():
            owners = by_range[(lrow[r], h)]
            s, _ = _scores(m, r, h)
            top = int(torch.argmax(s)) // (CHUNK * PAGE)
            assert top == j and owners.count(owners[j]) == 1 and len(set(owners)) >= 2, (G, r, h, j, top, owners)


def test_launch_layout():
    """every case row runs, launches hold at most 32 rows with inactive rows among them, and the position set reaches
    both chunk folds: 16 chunks (4095), 17 (4096, the last only the self key) and 33 (8200)"""
    c = _case("bf16", 2)
    pos = c["pos"].tolist()
    L = _launches(pos)
    assert sorted(i for l in L for i in l if pos[i] >= 0) == [i for i, p in enumerate(pos) if p >= 0]
    assert all(len(l) <= 32 and sum(pos[i] < 0 for i in l) == 2 and pos[l[0]] < 0 for l in L)
    nch = {p: (p // PAGE + CHUNK) // CHUNK for p in POSITIONS}
    assert nch[4095] == MAXCH and nch[4096] == MAXCH + 1 and nch[8200] == 33 and 4096 % (CHUNK * PAGE) == 0


# --------------------------------------------------------------------------------------------------------------------------
# GPU
# --------------------------------------------------------------------------------------------------------------------------
def _lib():
    from voicecraft_b200 import _lib
    return _lib, _lib.load()


def _dev(c):
    if "_dev" not in c:
        c["_dev"] = (c["Kp"].cuda(), c["Vp"].cuda())
    return c["_dev"]


def _call(c, sel, grids, Kp=None, Vp=None, page_table=None):
    """vcb_debug_mega_attention over case rows `sel` (in that order): fp32 [len(sel)][H*128] on the host, or the error"""
    _l, lib = _lib()
    Kd, Vd = _dev(c) if Kp is None else (Kp, Vp)
    pt = c["page_table"] if page_table is None else page_table
    sel = torch.as_tensor(sel, dtype=torch.long)
    H, n = c["H"], len(sel)
    pos = c["pos"][sel]
    rp = pt[c["row_slot"][sel].long()].contiguous()
    knew = torch.zeros(n, H, HD)
    vnew = torch.zeros(n, H, HD)
    Kh, Vh = c["Kp"], c["Vp"]
    for i, p in enumerate(pos.tolist()):
        if p >= 0:
            page = int(rp[i, p // PAGE])
            knew[i] = Kh[page, :, p % PAGE].float()
            vnew[i] = Vh[page, :, p % PAGE].float()
    q = c["q"][sel].float().contiguous().cuda()
    knew, vnew, rp, posd = knew.cuda(), vnew.cuda(), rp.cuda(), pos.contiguous().cuda()
    out = torch.full((n, H * HD), 12345.0, device="cuda")
    g = (_l.C.c_int32 * len(grids))(*[_grid(G) for G in grids])
    rc = lib.vcb_debug_mega_attention(q.data_ptr(), knew.data_ptr(), vnew.data_ptr(), Kd.data_ptr(), Vd.data_ptr(),
                                      int(Kd.dtype == torch.float32), rp.data_ptr(), posd.data_ptr(), n, H, c["max_pages"],
                                      g, len(grids), out.data_ptr())
    torch.cuda.synchronize()
    return rc, out.cpu()


def _run(c, sel, grids):
    rc, out = _call(c, sel, grids)
    if rc:
        _l, lib = _lib()
        raise AssertionError(lib.vcb_last_error().decode())
    return out


def _bits(x):
    return x.contiguous().view(torch.int32)


@lru_cache(maxsize=None)
def _reference(kv, H):
    """fp64 output and each (row, head)'s bound, see test_mega_attention_vs_fp64"""
    c = _case(kv, H)
    ref = _attn_ref(c)
    return ref, _bounds(c, ref)


def _bounds(c, ref):
    """[rows][H] bound of each head's 128 outputs"""
    vmax = float(c["Vp"].float().abs().max())
    u = 2.0 ** -24
    b = torch.full((len(c["pos"]), c["H"]), float("nan"), dtype=torch.float64)
    for r, p in enumerate(c["pos"].tolist()):
        if p < 0:
            continue
        for h in range(c["H"]):
            _, mass = _scores(c, r, h)
            S = float(mass.max()) * LOG2E
            o = float(ref[r, h * HD:(h + 1) * HD].abs().max())
            b[r, h] = vmax * (1e-5 + 2 * math.log(2) * 36 * u * S) + 2.0 ** -17 * o
    return b


def _check(c, got, ref, bound, rows, label, worst):
    """active rows within their bound, inactive rows still the image's fill (NaN)"""
    H = c["H"]
    for i, r in enumerate(rows):
        p = int(c["pos"][r])
        if p < 0:
            assert torch.isnan(got[i]).all(), f"{label}: inactive row {r} was written"
            continue
        for h in range(H):
            err = float((got[i, h * HD:(h + 1) * HD].double() - ref[r, h * HD:(h + 1) * HD]).abs().max())
            frac = err / float(bound[r, h])
            worst[0] = max(worst[0], frac)
            assert frac <= 1.0, (f"{label}: row {r} pos {p} ({c['kinds'][r]}) head {h}: err {err:.3g} = {frac:.3g} x bound "
                                 f"{float(bound[r, h]):.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("G", GRIDS)
@pytest.mark.parametrize("H", [2, 16])
@pytest.mark.parametrize("kv", ["fp32", "bf16"])
def test_mega_attention_vs_fp64(kv, H, G):
    """Every active row within its bound of the fp64 softmax, at every grid, and inactive rows untouched.

    Bound of head h of row r: max|V| * (1e-5 + 2 ln2 * 36 u S) + 2^-17 |o|.  1e-5 max|V| is the per-kernel attention's
    bound (test_kernel_numerics).  The kernel scores in the log2 domain: q' = fl(q * fl(scale * log2 e)), then a lane's
    32-term fma chain and 2 shuffle adds, so a score is off by at most 36 u S first order (u = 2^-24, S = max over keys of
    sum_d |q_d k_d| * scale * log2 e).  Scores off by at most e (log2 units) move every weight by a factor within
    2^(+-2e), so the output by at most 2 ln2 e max|V|.  The hi/lo split of the output adds 2^-17 |o|.  At the 140 plants
    the second term is ~3e-4 max|V|; in diffuse rows it is below 1e-5 max|V|, where one missing key of 8200 is 1e-4."""
    c = _case(kv, H)
    ref, bound = _reference(kv, H)
    worst = [0.0]
    for rows in _launches(c["pos"].tolist()):
        _check(c, _run(c, rows, [G]), ref, bound, rows, f"kv {kv} H {H} grid {G}", worst)
    if G in MOC_GRIDS:
        m = _moc_case(kv, H, _grid(G))
        assert m["solo"], f"grid {G}: no chunk owned alone"
        rows = _launches(m["pos"].tolist())[0]
        mref = _attn_ref(m)
        _check(m, _run(m, rows, [G]), mref, _bounds(m, mref), rows, f"max_other_cta kv {kv} H {H} grid {G}", worst)
    print(f"mega attention kv {kv} H {H} grid {G}: worst error / bound {worst[0]:.3g}")


@lru_cache(maxsize=None)
def _bit_case(kv, H):
    return _attn_case(HD, kv, CHUNK, seed=11, positions=[0, 64, 256, 1023, 4095, 4096, 4100, 8200],
                      kinds=("wide", "max_first_of_chunk", "underflow_cached"), H=H)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [2, 16])
@pytest.mark.parametrize("kv", ["fp32", "bf16"])
def test_mega_attention_is_bit_reproducible(kv, H):
    """A row's bits depend only on its own context (mega_step.cu): identical at every grid 1 .. max, alone or in a full
    batch at row 0 or 31, in a launch of 16 rows (BPAD 16) or 17 (BPAD 32), after 2 launches on one workspace and after
    launches at different grids in sequence on one workspace (the arrival counters reset themselves; the hook also
    checks each is back at 0 after every launch)."""
    c = _bit_case(kv, H)
    pos = c["pos"].tolist()
    act = [i for i, p in enumerate(pos) if p >= 0]
    ina = [i for i, p in enumerate(pos) if p < 0]
    rows = [ina[0]] + act[:10] + [ina[1]] + act[10:]                    # 26 rows: BPAD 32
    base = _run(c, rows, ["max"])
    ok = [i for i, r in enumerate(rows) if pos[r] >= 0]
    ref = _bits(base[ok])
    diff = [G for G in range(1, _max_grid() + 1) if not torch.equal(_bits(_run(c, rows, [G])[ok]), ref)]
    assert not diff, f"grids whose result differs from grid max: {diff}"
    assert torch.equal(_bits(_run(c, rows, ["max", "max"])[ok]), ref), "2 launches on one workspace differ"
    seq = [1, "max", 7, 131, 2, 64, 33, 3, 16]
    assert torch.equal(_bits(_run(c, rows, seq)[ok]), ref), "launches at different grids on one workspace differ"
    col = {r: base[rows.index(r)] for r in act}
    for r in [next(r for r in act if pos[r] == p) for p in (8200, 4096, 4095, 256)]:
        others = [o for o in act if o != r]
        for G in (1, 7, "max"):
            for sel, at, what in (([r], 0, "alone"), ([r] + (others * 2)[:31], 0, "row 0 of 32"),
                                  ((others * 2)[:31] + [r], 31, "row 31 of 32"), ((others * 2)[:15] + [r], 15, "row 15 of 16"),
                                  ((others * 2)[:16] + [r], 16, "row 16 of 17")):
                got = _run(c, sel, [G])[at]
                assert torch.equal(_bits(got), _bits(col[r])), f"row {r} (pos {pos[r]}) {what}, grid {G}: differs"


@pytest.mark.gpu
@pytest.mark.parametrize("kv", ["fp32", "bf16"])
def test_mega_attention_reads_knew_not_the_page(kv):
    """Only knew / vnew stand for position pos, and masked keys contribute exactly nothing: with every row's last page
    private, the page slots pos .. 63 of it zeroed, or filled with K entries of magnitude 1e30 and V entries of 1e4,
    give the same bits as the untouched pages."""
    c = _case(kv, 2)
    pos = c["pos"].tolist()
    Kp, Vp, pt = c["Kp"].clone(), c["Vp"].clone(), c["page_table"].clone()
    act = [r for r, p in enumerate(pos) if p >= 0]
    n0 = Kp.shape[0]
    Kp = torch.cat([Kp, torch.zeros((len(act),) + Kp.shape[1:], dtype=Kp.dtype)])
    Vp = torch.cat([Vp, torch.zeros((len(act),) + Vp.shape[1:], dtype=Vp.dtype)])
    for i, r in enumerate(act):                       # the last page of row r becomes a copy only row r reads
        slot, last = int(c["row_slot"][r]), pos[r] // PAGE
        Kp[n0 + i], Vp[n0 + i] = Kp[int(pt[slot, last])], Vp[int(pt[slot, last])]
        pt[slot, last] = n0 + i
    g = torch.Generator().manual_seed(5)
    variants = {}
    for name in ("untouched", "zero", "sentinel"):
        K, V = Kp.clone(), Vp.clone()
        for i, r in enumerate(act):
            t = pos[r] % PAGE
            if name == "zero":
                K[n0 + i, :, t:] = 0
                V[n0 + i, :, t:] = 0
            elif name == "sentinel":
                sk = torch.randint(0, 2, K[n0 + i, :, t:].shape, generator=g) * 2 - 1
                sv = torch.randint(0, 2, V[n0 + i, :, t:].shape, generator=g) * 2 - 1
                K[n0 + i, :, t:] = (sk * 1e30).to(K.dtype)
                V[n0 + i, :, t:] = (sv * 1e4).to(V.dtype)
        Kd, Vd = K.cuda(), V.cuda()
        for G in (1, 7, "max"):
            outs = []
            for rows in _launches(pos):
                rc, out = _call(dict(c, Kp=Kp, Vp=Vp), rows, [G], Kd, Vd, pt)
                assert rc == 0
                outs.append(out[[j for j, rr in enumerate(rows) if pos[rr] >= 0]])
            variants[(name, G)] = _bits(torch.cat(outs))
        del Kd, Vd
    for key, v in variants.items():
        assert torch.equal(v, variants[("untouched", key[1])]), f"{key} differs from the untouched pages"


@pytest.mark.gpu
def test_mega_attention_rejections():
    """Rejected on the host with a message, nothing launched (the output keeps its fill): rows outside [1, 32], fp8 KV,
    grids outside [1, max], H * rows * max_pages * (grid + 1) >= 2^31, a position beyond the pages."""
    _l, lib = _lib()
    C = _l.C
    gmax = _max_grid()
    H, max_pages = 2, 4
    Kp = torch.zeros(8, H, PAGE, HD, device="cuda")

    def call(rows=2, kv=1, grids=(1,), H=H, max_pages=max_pages, pos=0):
        q = torch.zeros(max(rows, 1), H, HD, device="cuda")
        rp = torch.zeros(max(rows, 1), min(max_pages, 64), dtype=torch.int32, device="cuda")
        p = torch.full((max(rows, 1),), pos, dtype=torch.int32, device="cuda")
        out = torch.full((max(rows, 1), H * HD), 7.0, device="cuda")
        g = (C.c_int32 * len(grids))(*grids)
        rc = lib.vcb_debug_mega_attention(q.data_ptr(), q.data_ptr(), q.data_ptr(), Kp.data_ptr(), Kp.data_ptr(), kv,
                                          rp.data_ptr(), p.data_ptr(), rows, H, max_pages, g, len(grids), out.data_ptr())
        torch.cuda.synchronize()
        return rc, (lib.vcb_last_error() or b"").decode(), bool((out == 7.0).all())

    assert call()[0] == 0 and call(grids=(gmax,))[0] == 0
    for kw, msg in ((dict(rows=0), "rows"), (dict(rows=33), "rows"), (dict(kv=2), "kv_dtype"), (dict(grids=(0,)), "grid"),
                    (dict(grids=(gmax + 1,)), "grid"), (dict(grids=(1, gmax + 1)), "grid"),
                    (dict(H=16, rows=32, max_pages=(2 ** 31) // (16 * 32 * (gmax + 1)) + 1, grids=(gmax,)), "2^31"),
                    (dict(pos=max_pages * PAGE), "beyond")):
        rc, err, untouched = call(**kw)
        assert rc != 0 and msg in err and untouched, (kw, rc, err)
