"""-m gpu: single kernels against plain fp64 references, at the shapes and edges where they go wrong, plus end-to-end runs
that reach the code paths only long contexts take.

  * paged attention (attn_rows_kernel) through vcb_debug_attention, with the engine's chunk / grid / balance decisions:
    contexts up to 4100 tokens, split-context merges with 1, 3 and 16 pages per chunk, shuffled and shared page tables,
    logits spanning +-80, chunks whose softmax weights all underflow, and diffuse rows where every key carries about
    1/context of the weight.  Bound 1e-5 * max|V|, far below one missing or duplicated key of a diffuse row.
  * the folded LayerNorm of the decode path (vcb_debug_fold_chain: residual GEMM emitting gamma * x and per-tile row
    statistics, then the consumer GEMM folding LN into its epilogue) against fp64 LN(x_new) W^T + b, at rows whose
    mean / std reaches 300 and rows with a few massive features; and the prefill arithmetic (two-pass LN) on the same data.
  * end to end against the CPU oracle past 1024 tokens (the split-context merge in decode and wide prefill) and past 4096
    tokens (the persistent kernel's chunk fold beyond its on-chip table), and on a checkpoint with a large residual offset.
"""
import math

import numpy as np
import pytest
import torch

import golden_util as gu

pytestmark = pytest.mark.gpu
LOGIT_TOL = 2e-3


def _lib():
    from voicecraft_b200 import _lib
    return _lib, _lib.load()


# ==========================================================================================================================
# paged attention
# ==========================================================================================================================
PAGE = 64
POSITIONS = [0, 1, 63, 64, 65, 1023, 1024, 1025, 2047, 2048, 4100]
KINDS = ("wide", "diffuse", "max_first_of_chunk", "max_last", "max_early_chunk", "underflow")
Q_SCALE = {"wide": 20.0, "diffuse": 0.3}         # logit std: "wide" spans +-80, "diffuse" spreads the weight over every key


def _attn_case(hd, kv, chunk_pages, seed=0, positions=POSITIONS, kinds=KINDS, H=2, plant=None):
    """rows of every (position, score distribution) pair plus two inactive rows; K / V pools [page][H][64][hd] shared by
    every row through shuffled page lists (one list per row, in a shuffled slot order).
    Kinds beyond KINDS: "underflow_cached" (logit 140 on a cached key of a middle chunk: every other chunk and the key at
    pos underflow against it) and "self_min" (logit -140 on the key at pos).  Any other kind is planted by
    plant(r, pos, kind) -> (key index, or one per head, logit) or None, with pos the case's positions (-1: inactive)."""
    g = torch.Generator(device="cpu").manual_seed(1000 * hd + 10 * chunk_pages + (kv == "bf16") + seed)
    max_pages = (max(positions) + PAGE) // PAGE + 1
    n_pool = max_pages + 14
    n_slots = len(positions) * len(kinds) + 2
    Kp = torch.randn(n_pool, H, PAGE, hd, generator=g)
    Vp = torch.randn(n_pool, H, PAGE, hd, generator=g)
    rows = [(p, k) for p in positions for k in kinds]
    pos = [p for p, _ in rows]
    q = torch.empty(len(rows), H, hd)
    for r, (p, kind) in enumerate(rows):
        q[r] = torch.randn(H, hd, generator=g) * Q_SCALE.get(kind, 5.0)
    # insert the two inactive rows in the middle and at the end
    pos = pos[:20] + [-1] + pos[20:] + [-1]
    q = torch.cat([q[:20], torch.randn(1, H, hd, generator=g), q[20:], torch.randn(1, H, hd, generator=g)])
    kinds = [k for _, k in rows]
    kinds = kinds[:20] + [None] + kinds[20:] + [None]
    row_slot = torch.randperm(n_slots, generator=g).int()
    # planted keys: key index t of row r gets k = c * q_hat with the logit it should produce; every planted (page, key) is
    # planted once (page lists are redrawn until no two plants land on the same key)
    span = chunk_pages * PAGE
    plants = {}
    for r, (p, kind) in enumerate(zip(pos, kinds)):
        if p < 0 or kind in Q_SCALE:
            continue
        if kind == "max_first_of_chunk":
            t, logit = (p // span) // 2 * span, 40.0          # first key of a middle chunk (chunk 0 when there is one)
        elif kind == "max_last":
            t, logit = p, 40.0
        elif kind == "max_early_chunk":
            t, logit = min(p, 5), 40.0                        # chunk 0, while the row has more chunks after it
        elif kind == "underflow":
            t, logit = p, 140.0                               # every other chunk's weights underflow in fp32
        elif kind == "underflow_cached":
            t, logit = min((p // span) // 2 * span + span // 2, max(p - 1, 0)), 140.0
        elif kind == "self_min":
            t, logit = p, -140.0
        else:
            planted = plant(r, pos, kind)
            if planted is None:
                continue
            t, logit = planted
        plants[r] = (t, logit)
    heads = {r: sorted(set(t)) if isinstance(t, list) else [t] for r, (t, _) in plants.items()}
    while True:
        page_table = torch.stack([torch.randperm(n_pool, generator=g)[:max_pages] for _ in range(n_slots)]).int()
        keys = [(int(page_table[row_slot[r], t // PAGE]), t % PAGE) for r in plants for t in heads[r]]
        if len(set(keys)) == len(keys):
            break
    for r, (t, logit) in plants.items():
        for h in range(H):
            th = t[h] if isinstance(t, list) else t
            page = int(page_table[row_slot[r], th // PAGE])
            qv = q[r, h]
            Kp[page, h, th % PAGE] = qv * (logit * math.sqrt(hd) / float(qv.dot(qv)))
    if kv == "bf16":
        Kp, Vp = Kp.to(torch.bfloat16), Vp.to(torch.bfloat16)
    return dict(H=H, hd=hd, q=q, Kp=Kp, Vp=Vp, page_table=page_table, row_slot=row_slot,
                pos=torch.tensor(pos, dtype=torch.int32), max_pages=max_pages, kinds=kinds)


def _attn_run(c, chunk_pages, via="row_pages", balance=1, repeats=1, rows=None):
    _l, lib = _lib()
    sel = torch.arange(len(c["pos"])) if rows is None else torch.as_tensor(rows)
    q = c["q"][sel].contiguous().cuda()
    pos = c["pos"][sel].contiguous().cuda()
    slot = c["row_slot"][sel].contiguous().cuda()
    pt = c["page_table"].contiguous().cuda()
    rp = pt[slot.long()].contiguous()
    Kp, Vp = c["Kp"].cuda(), c["Vp"].cuda()
    n, H, hd = len(sel), c["H"], c["hd"]
    out = torch.full((n, H * hd), 12345.0, device="cuda")
    args = (rp.data_ptr(), None, None) if via == "row_pages" else (None, pt.data_ptr(), slot.data_ptr())
    _l.check(lib.vcb_debug_attention(q.data_ptr(), Kp.data_ptr(), Vp.data_ptr(), int(Kp.dtype == torch.float32), *args,
                                     pos.data_ptr(), n, H, hd, c["max_pages"], chunk_pages, balance, repeats, out.data_ptr()))
    torch.cuda.synchronize()
    return out.cpu()


def _attn_ref(c):
    """fp64 softmax(q K^T / sqrt(hd)) V over keys 0..pos of each row, from the (bf16-rounded) pool values"""
    H, hd = c["H"], c["hd"]
    Kp, Vp = c["Kp"].double(), c["Vp"].double()
    out = torch.full((len(c["pos"]), H * hd), float("nan"), dtype=torch.float64)
    for r, p in enumerate(c["pos"].tolist()):
        if p < 0:
            continue
        pages = c["page_table"][int(c["row_slot"][r])][: p // PAGE + 1].long()
        for h in range(H):
            K = Kp[pages, h].reshape(-1, hd)[: p + 1]
            V = Vp[pages, h].reshape(-1, hd)[: p + 1]
            s = (K @ c["q"][r, h].double()) / math.sqrt(hd)
            out[r, h * hd:(h + 1) * hd] = torch.softmax(s, 0) @ V
    return out


@pytest.mark.parametrize("chunk_pages", [1, 3, 16])
@pytest.mark.parametrize("kv", ["fp32", "bf16"])
@pytest.mark.parametrize("hd", [64, 128])
def test_paged_attention_vs_fp64(hd, kv, chunk_pages):
    c = _attn_case(hd, kv, chunk_pages)
    got = _attn_run(c, chunk_pages)
    ref = _attn_ref(c)
    vmax = float(c["Vp"].float().abs().max())
    active = c["pos"] >= 0
    assert torch.all(got[~active] == 12345.0), "an inactive row's output was written"
    for r in torch.nonzero(active).flatten().tolist():
        err = float((got[r].double() - ref[r]).abs().max())
        assert err <= 1e-5 * vmax, (f"row {r} pos {int(c['pos'][r])} ({c['kinds'][r]}): max err {err:.3g} "
                                    f"> 1e-5 * max|V| = {1e-5 * vmax:.3g}")


@pytest.mark.parametrize("chunk_pages", [1, 3, 16])
@pytest.mark.parametrize("kv", ["fp32", "bf16"])
@pytest.mark.parametrize("hd", [64, 128])
def test_paged_attention_is_bit_reproducible(hd, kv, chunk_pages):
    """The same bits (1) after 3 launches on the same workspace and counters (the merging CTA resets its counter), (2) with
    the work balance off, (3) for a row whatever else is in the launch, and (4) whether its pages come as a per-row list
    (decode) or through page_table + row_slot (prefill)."""
    c = _attn_case(hd, kv, chunk_pages, seed=1)
    base = _attn_run(c, chunk_pages)
    assert torch.equal(_attn_run(c, chunk_pages, repeats=3), base), "repeated launches differ: arrival counters not reset"
    assert torch.equal(_attn_run(c, chunk_pages, balance=0), base), "result depends on the work balance"
    assert torch.equal(_attn_run(c, chunk_pages, via="page_table"), base), "row_pages and page_table + row_slot differ"
    n = len(c["pos"])
    subset = list(range(n - 1, -1, -3))                  # other rows, other order, another longest context
    assert torch.equal(_attn_run(c, chunk_pages, rows=subset), base[subset]), "a row depends on the other rows"
    for r in (int(np.argmax(c["pos"].numpy())), 7):
        assert torch.equal(_attn_run(c, chunk_pages, rows=[r]), base[[r]]), f"row {r} alone differs"


# ==========================================================================================================================
# folded LayerNorm (decode) and the two-pass LayerNorm (prefill) against fp64
# ==========================================================================================================================
RATIOS = [0.0, 4.0, 30.0, 100.0, 300.0]          # mean / std of a row of x_new
# max|err| / max|ref| of the decode path (fold = 1) per class of rows.  The fold merges per-tile centred statistics
# (tile sum, M2 about the tile mean) in tile order, so the variance keeps its precision at any mean; what remains grows
# with mean / std through the hi/lo split of gamma * x that the fold subtracts mean * cvec from (DESIGN.md section 4.1).
# That remainder is a sum over the d features of rounding errors of size 2^-17 * |gamma * x|, so it grows like sqrt(d): the
# bounds at mean / std 100 and 300 hold up to d = 2048 and scale with sqrt(d / 2048) beyond.  The prefill path (two-pass
# LayerNorm rows) is held to 2e-4 at every ratio.
FOLD_BOUND = {0.0: 2e-4, 4.0: 2e-4, 30.0: 5e-4, 100.0: 5e-4, 300.0: 2e-3, "massive": 2e-4}


def _fold_bound(c, d):
    return FOLD_BOUND[c] * (max(1.0, math.sqrt(d / 2048)) if c in (100.0, 300.0) else 1.0)
PREFILL_BOUND = 2e-4
CLASSES = RATIOS + ["massive"]


def _valid_splits(bpad, kdim):
    """split counts gemm_launch accepts for this bpad and K (what gemm_pick_splits may return, where it is legal)"""
    kb = kdim // 64
    return [s for s in (1, 2, 4, 8) if bpad % s == 0 and bpad // s >= 2 and (s - 1) * ((kb + s - 1) // s) < kb]


def _bpad(B):
    return 16 if B <= 16 else 32 if B <= 32 else 64 if B <= 64 else 128


_FOLD_W = {}


def _fold_weights(d):
    if d not in _FOLD_W:
        g = torch.Generator(device="cpu").manual_seed(d)
        bf = lambda t: t.to(torch.bfloat16).float()
        _FOLD_W.clear()
        _FOLD_W[d] = dict(W1=bf(torch.randn(d, d, generator=g) * (0.25 / math.sqrt(d))).cuda(),
                          b1=(0.05 * torch.randn(d, generator=g)).cuda(),
                          gamma=(1.0 + 0.1 * torch.randn(d, generator=g)).cuda(),
                          beta=(0.05 * torch.randn(d, generator=g)).cuda(),
                          W2=bf(torch.randn(d, d, generator=g) / math.sqrt(d)).cuda(),
                          b2=(0.05 * torch.randn(d, generator=g)).cuda())
    return _FOLD_W[d]


def _fold_rows(B, d, shift, seed, classes=CLASSES):
    """x rows of class classes[(i + shift) % n]: std 1 around mean / std = ratio, or std 1 with 4 features at 50..100"""
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(B, d, generator=g)
    cls = [classes[(i + shift) % len(classes)] for i in range(B)]
    for i, c in enumerate(cls):
        if c == "massive":
            idx = torch.randperm(d, generator=g)[:4]
            x[i, idx] = (50.0 + 50.0 * torch.rand(4, generator=g)) * torch.sign(torch.randn(4, generator=g))
        else:
            x[i] += c
    a = torch.randn(B, d, generator=g)
    return x.cuda(), a.cuda(), cls


def _fold_ref(w, x, a, relu):
    xn = x.double() + a.double() @ w["W1"].double().t() + w["b1"].double()
    ln = torch.nn.functional.layer_norm(xn, (xn.shape[1],), w["gamma"].double(), w["beta"].double(), eps=1e-5)
    y = ln @ w["W2"].double().t() + w["b2"].double()
    return xn, (torch.relu(y) if relu else y)


def _fold_run(w, x, a, B, d, relu, fold, s1, s2):
    _l, lib = _lib()
    xn = torch.empty(B, d, device="cuda")
    y = torch.empty(B, d, device="cuda")
    _l.check(lib.vcb_debug_fold_chain(x.data_ptr(), a.data_ptr(), w["W1"].data_ptr(), w["b1"].data_ptr(), w["gamma"].data_ptr(),
                                      w["beta"].data_ptr(), w["W2"].data_ptr(), w["b2"].data_ptr(), B, d, d, relu, fold, s1, s2,
                                      xn.data_ptr(), y.data_ptr()))
    torch.cuda.synchronize()
    return xn, y


def _fold_sweep(B, d, fold_bound, classes=CLASSES):
    """every legal split count (and the engine's choice) x rows of every class, fold = 1 and 0: the list of results over
    their bound, and the worst error per (fold, class)"""
    w = _fold_weights(d)
    splits = [(0, 0)] + [(s, s) for s in _valid_splits(_bpad(B), d)]
    shifts = range(len(classes)) if B < len(classes) else [0]
    worst, bad = {}, []
    for shift in shifts:
        x, a, cls = _fold_rows(B, d, shift, seed=B * 7919 + d + shift, classes=classes)
        for si, (s1, s2) in enumerate(splits):
            relu = (si + shift) % 2
            xr, yr = _fold_ref(w, x, a, relu)
            for fold in (1, 0):
                xn, y = _fold_run(w, x, a, B, d, relu, fold, s1, s2)
                xerr = float((xn.double() - xr).abs().max() / xr.abs().max())
                if xerr > 2e-5:
                    bad.append(f"x_new fold={fold} splits={s1}: {xerr:.3g}")
                for c in set(cls):
                    rows = [i for i, ci in enumerate(cls) if ci == c]
                    err = float((y[rows].double() - yr[rows]).abs().max() / yr[rows].abs().max())
                    key = (fold, c)
                    worst[key] = max(worst.get(key, 0.0), err)
                    if err > (fold_bound(c, d) if fold else PREFILL_BOUND):
                        bad.append(f"y fold={fold} mean/std={c} splits={s1} relu={relu}: {err:.3g}")
    summary = {f"fold={k[0]} {k[1]}": f"{v:.2g}" for k, v in sorted(worst.items(), key=str)}
    print("worst max|err|/max|ref|:", summary)
    return bad, summary


@pytest.mark.parametrize("d", [256, 1024, 2048, 4096])
@pytest.mark.parametrize("B", [1, 5, 16, 20, 32, 48, 64, 128])
def test_folded_layernorm_vs_fp64(B, d):
    """x_new = x + a W1^T + b1 and LN(x_new) W2^T + b2 (ReLU'd on alternate runs) through the decode path (fold = 1: both
    stats paths, bpad 16..128, every legal split count and the engine's own choice) and the prefill path (fold = 0)."""
    bad, summary = _fold_sweep(B, d, _fold_bound)
    assert not bad, f"{len(bad)} over the bound (first: {bad[:6]}); worst by class {summary}"


# ==========================================================================================================================
# end to end against the CPU oracle: contexts past 1024 and 4096 tokens, a residual stream with a large common offset
# ==========================================================================================================================
KW = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3, silence_tokens=gu.SILENCE)
N_STEPS = 16


def _oracle_traces(cfg, sd, utts, seed0):
    from oracle import lm_oracle
    torch.set_num_threads(max(1, min(16, torch.get_num_threads())))
    oracle = lm_oracle.OracleLM(cfg, sd)
    out = []
    for i, (x, xl, y) in enumerate(utts):
        rows = oracle.inference_tts(x, xl, y, noise_fn=gu.cpu_noise_fn(seed0 + i), max_steps=N_STEPS, trace_logits=True, **KW)
        assert rows.shape == (N_STEPS, cfg.n_codebooks), "the checkpoint must not end within the traced steps"
        out.append((rows.numpy(), [t.numpy() for t in oracle.logit_trace]))
    return out


def _gpu_traces(cfg, sd, utts, seed0, max_seq_len=None):
    """(rows, per-step logits) of every utterance through one DecodeSession, and the engine's persistent-kernel grid"""
    from voicecraft_b200.voicecraft import VoiceCraft
    _l, lib = _lib()
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    m = m.to("cuda").eval()
    m.configure_engine(kv_dtype="fp32", **({} if max_seq_len is None else dict(max_seq_len=max_seq_len)))
    B, K, V = len(utts), cfg.n_codebooks, m.n_audio_tokens[0]
    sess = m.open_tts_session([u[0].cuda() for u in utts], [u[2].cuda() for u in utts],
                              noise_fns=[gu.cpu_noise_fn(seed0 + i) for i in range(B)], **KW)
    t = torch.empty(B * K, V, device="cuda")
    traces = []
    try:
        for step in range(N_STEPS):
            sess.sample() if step == 0 else sess.step()
            _l.check(lib.vcb_debug_logits(sess.eng, t.data_ptr(), B * K))
            traces.append(t.cpu().numpy().reshape(B, K, V).copy())
        rows = [sess.raw_tokens(i)[:N_STEPS] for i in range(B)]
        mega_grid = lib.vcb_counter(sess.eng, b"mega_grid")
    finally:
        sess.close()
    return [(rows[i], [tr[i] for tr in traces]) for i in range(B)], mega_grid


def _assert_matches_oracle(got, ref, what):
    for i, ((grows, gtr), (rrows, rtr)) in enumerate(zip(got, ref)):
        worst = 0.0
        for s, (a, b) in enumerate(zip(gtr, rtr)):
            live = b > -9999
            worst = max(worst, float(np.abs(a - b)[live].max()))
        assert worst <= LOGIT_TOL, f"{what}: utterance {i}: max |logit - oracle| = {worst:.3g}"
        assert np.array_equal(np.asarray(grows), rrows), f"{what}: utterance {i}: token ids differ from the oracle"


def _long_checkpoint(cfg, seed):
    from voicecraft_b200 import synthetic
    return gu.suppress_end_tokens(cfg, synthetic.make_state_dict(cfg, seed=seed))


CFGS = {"hd128": ("tiny", {}), "hd64": ("tiny", {"nhead": 4})}


@pytest.mark.parametrize("wide,mega,cfg_name", [(w, g, c) for c in CFGS for w in ("0", "1") for g in ("0", "1")
                                                 if not (c == "hd64" and g == "1")])
def test_prompt_past_1024_tokens_matches_oracle(cfg_name, wide, mega, monkeypatch):
    """A 1110-token prompt (120 text tokens, 990 frames) on the default engine (max_seq_len 2048): prefill and decode
    attention merge two context chunks of 1024 tokens (the persistent kernel: 4-page chunks spread over CTAs)."""
    from voicecraft_b200 import synthetic
    monkeypatch.setenv("VCB_PREFILL_WIDE", wide)
    monkeypatch.setenv("VCB_MEGA", mega)
    name, over = CFGS[cfg_name]
    cfg = synthetic.make_config(name, **over)
    sd = _long_checkpoint(cfg, 71)
    utts = [synthetic.synthetic_utterance(cfg, 8100, text_len=120, prompt_frames=990)]
    got, grid = _gpu_traces(cfg, sd, utts, 5)
    if mega == "1":
        assert grid > 0, "the persistent decode kernel did not run"
    _assert_matches_oracle(got, _oracle_traces(cfg, sd, utts, 5), f"{cfg_name} wide={wide} mega={mega}")


@pytest.mark.parametrize("name", ["tts_topk40", "batch3", "edit2"])
def test_one_page_attention_chunks_match_reference_fixture(name, monkeypatch):
    """VCB_ATT_CHUNK_PAGES=1: every 64-token page is its own attention work item, so every prefill and decode row of the
    fixture cases goes through the split-context merge."""
    from test_gpu_parity import CASES, _run_case
    monkeypatch.setenv("VCB_ATT_CHUNK_PAGES", "1")
    res, trace, g = _run_case(name, CASES[name], "fp32")
    for step, ref in zip(g["trace_steps"], g["trace_logits"]):
        got = trace[int(step)].cpu().numpy()
        live = ref > -9999
        diff = np.abs(got - ref)[live]
        assert int((diff > LOGIT_TOL).sum()) <= 1, f"step {step}: max {diff.max()}"   # <=1: silence penalty slot
    assert np.array_equal(res.cpu().numpy(), g["res"]), "token ids differ from the reference fixture"


@pytest.mark.parametrize("n_utts,grid", [(1, None), (8, "10")])
def test_persistent_kernel_past_4096_tokens_matches_oracle(n_utts, grid, monkeypatch):
    """About 4200 tokens of context (66 pages = 17 chunks of 4 pages per (row, head), one more than the persistent kernel's
    on-chip chunk table holds).  One utterance: every item is shared between CTAs.  Eight utterances on 10 CTAs (the
    smallest grid mega_setup accepts for `tiny`): a CTA's share covers whole items, which then fold 17 chunks."""
    from voicecraft_b200 import synthetic
    monkeypatch.setenv("VCB_MEGA", "1")
    if grid:
        monkeypatch.setenv("VCB_MEGA_GRID", grid)
    cfg = synthetic.make_config("tiny")
    sd = _long_checkpoint(cfg, 72)
    utts = [synthetic.synthetic_utterance(cfg, 8200 + i, text_len=420, prompt_frames=3780 + 3 * i) for i in range(n_utts)]
    got, g = _gpu_traces(cfg, sd, utts, 9)
    assert g > 0, "the persistent decode kernel did not run"
    if grid:
        assert g == int(grid)
    _assert_matches_oracle(got, _oracle_traces(cfg, sd, utts, 9), f"{n_utts} utterances, grid {g}")


def test_persistent_kernel_grid_floor_for_tiny(monkeypatch):
    """mega_setup declines a grid whose per-CTA block range would touch more than MEGA_MAXSEG output tiles: for `tiny`
    (the 4 x 17-tile logit heads with 16 k-blocks each) 10 CTAs is the smallest grid it accepts."""
    from voicecraft_b200 import synthetic
    monkeypatch.setenv("VCB_MEGA", "1")
    cfg = synthetic.make_config("tiny")
    sd = _long_checkpoint(cfg, 73)
    utts = [synthetic.synthetic_utterance(cfg, 8300, text_len=4, prompt_frames=10)]
    for grid, accepted in (("9", False), ("10", True)):
        monkeypatch.setenv("VCB_MEGA_GRID", grid)
        _, g = _gpu_traces(cfg, sd, utts, 3)
        assert (g > 0) == accepted, f"VCB_MEGA_GRID={grid}: mega_grid = {g}"


@pytest.mark.parametrize("mega", ["0", "1"])
def test_residual_offset_checkpoint_matches_oracle(mega, monkeypatch):
    """+20 on out_proj.bias and linear2.bias of every layer: the residual stream carries a common offset of up to 80 over a
    spread of order one, where a one-pass variance E[x^2] - mean^2 would lose precision.  Decode logits against the oracle on the per-kernel path and on the persistent kernel."""
    from voicecraft_b200 import synthetic
    monkeypatch.setenv("VCB_MEGA", mega)
    cfg = synthetic.make_config("tiny")
    sd = _long_checkpoint(cfg, 74)
    for l in range(cfg.num_decoder_layers):
        sd[f"decoder.layers.{l}.self_attn.out_proj.bias"] += 20.0
        sd[f"decoder.layers.{l}.linear2.bias"] += 20.0
    utts = [synthetic.synthetic_utterance(cfg, 8400 + i, text_len=10, prompt_frames=40 + 7 * i) for i in range(3)]
    got, g = _gpu_traces(cfg, sd, utts, 13)
    if mega == "1":
        assert g > 0, "the persistent decode kernel did not run"
    _assert_matches_oracle(got, _oracle_traces(cfg, sd, utts, 13), f"offset checkpoint mega={mega}")
