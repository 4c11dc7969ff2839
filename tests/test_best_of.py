"""Best-of-N for sessions and the continuous batcher, with one prefill per group and the prompt's full KV pages shared
by the group's copies.  CPU: the batcher's slot-run admission.  GPU (-m gpu): a group against independent rows of the
same prompt fed the same noise (bit-identical logits and tokens), the page and prefill-row accounting, sessions against
seeded inference_tts_batch calls, and the batcher with mixed group sizes."""
import ctypes as C
import gc

import pytest
import torch

from voicecraft_b200.voicecraft import place_groups

KW = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: admission of ContinuousBatcher.run()
# ---------------------------------------------------------------------------------------------------------------------
def test_place_groups_fifo_lowest_run():
    free = set(range(8))
    new, nxt = place_groups(free, [1, 3, 2, 2], 0)
    assert new == [(0, 0), (1, 1), (4, 2), (6, 3)] and nxt == 4 and free == set()


def test_place_groups_head_waits_and_is_not_overtaken():
    free = {0, 2, 3, 5, 6}
    new, nxt = place_groups(free, [2, 3, 1], 0)
    assert new == [(2, 0)] and nxt == 1 and free == {0, 5, 6}      # ticket 1 needs 3 in a row: ticket 2 waits behind it
    new, nxt = place_groups(free, [2, 3, 1], nxt)
    assert new == [] and nxt == 1 and free == {0, 5, 6}
    free.update({3, 4})                                            # ticket 0's slots come back, with slot 4
    new, nxt = place_groups(free, [2, 3, 1], nxt)
    assert new == [(3, 1), (0, 2)] and nxt == 3 and free == {6}


def test_place_groups_reuses_released_runs():
    free = set(range(4))
    sizes = [4, 2, 2, 4]
    new, nxt = place_groups(free, sizes, 0)
    assert new == [(0, 0)] and not free
    free.update(range(4))
    new, nxt = place_groups(free, sizes, nxt)
    assert new == [(0, 1), (2, 2)] and nxt == 3
    free.update({2, 3})
    assert place_groups(free, sizes, nxt) == ([], 3)
    free.update({0, 1})
    assert place_groups(free, sizes, nxt) == ([(0, 3)], 4)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _model(kv="bf16", max_slots=24, nhead=2, seed=3, eos_bias=3.0):
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny", nhead=nhead)
    sd = synthetic.make_state_dict(cfg, seed=seed)
    sd["predict_layer.0.2.bias"][cfg.eos] += eos_bias
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    m = m.to("cuda").eval()
    m.configure_engine(kv_dtype=kv, max_slots=max_slots, max_seq_len=512)
    return cfg, m


def _utt(cfg, seed, total):
    """an utterance whose prompt fills `total` engine positions (text + the delayed prompt's T + 1 rows); 40 text ids let
    it generate up to 400 - T frames (the reference's length cap)"""
    from voicecraft_b200 import synthetic
    x, xl, y = synthetic.synthetic_utterance(cfg, seed, text_len=40, prompt_frames=total - 41)
    return x.cuda(), xl.cuda(), y.cuda()


def _cpu_noise(seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return lambda shape, device=None: torch.empty(shape).exponential_(1, generator=g).to(device or "cpu")


def _trace(m, cfg, x, y, n, grouped, max_steps=48):
    """pre-edit logits [n*K, V] of every sampling step and the token rows of each copy: one best-of-n group, or n
    independent utterances of the same prompt; both take the same [n*K, V] host draw per step (row c*K + k: copy c)"""
    from voicecraft_b200 import _lib
    from voicecraft_b200.voicecraft import DecodeSession
    m.noise_fn = _cpu_noise(11)
    sp = m._sampling(silence_tokens=(1388, 1898, 131), **KW)
    sess = DecodeSession(m, [x], [y], sp, best_of=n) if grouped else DecodeSession(m, [x] * n, [y] * n, sp)
    lib, rows_n = _lib.load(), n * cfg.n_codebooks
    logits = []
    try:
        with torch.cuda.device(sess.dev):
            sess.sample()
            while True:
                t = torch.empty(rows_n, sess.V, device="cuda")
                _lib.check(lib.vcb_debug_logits(sess.eng, t.data_ptr(), rows_n))
                logits.append(t)
                st = sess.poll()
                if len(logits) >= max_steps or any(s.done for s in st):
                    break
                sess.step()
            rows = [m._read_rows(sess.eng, s, st[i].n_steps, sess.stream) for i, s in enumerate(sess.slots)]
    finally:
        sess.close()
        m.noise_fn = None
    return logits, rows


def _group_case(hd, kv, seed):
    """row groups over one K / V pool: (size, position, shared pages) per group; members share their first S page ids and
    own the rest.  Groups of 1, 2, 3, 8, 9 and 20 rows (9 and 20 split into launch groups), contexts past 4096 tokens,
    S = 0 and S = all pages but the last, an inactive group, and independent rows between them."""
    g = torch.Generator(device="cpu").manual_seed(100 * hd + 7 * seed + (kv == "bf16"))
    H, n_pool = 2, 700
    groups = [(1, 900, 0), (2, 4500, 70), (1, 33, 0), (3, 200, 2), (8, 4200, 0), (1, -1, 0), (9, 5000, 40),
              (4, -1, 3), (20, 1300, 20), (3, 640, 10), (1, 4100, 0)]
    max_pages = max(p for _, p, _ in groups) // 64 + 2
    pages, pos, first, shared = [], [], [0], []
    for size, p, S in groups:
        prefix = torch.randperm(n_pool, generator=g)[:S]
        for _ in range(size):
            pages.append(torch.cat([prefix, torch.randperm(n_pool, generator=g)[:max_pages - S]]))
            pos.append(p)
        first.append(first[-1] + size)
        shared.append(S)
    rows = len(pos)
    Kp = torch.randn(n_pool, H, 64, hd, generator=g)
    Vp = torch.randn(n_pool, H, 64, hd, generator=g)
    if kv == "bf16":
        Kp, Vp = Kp.to(torch.bfloat16), Vp.to(torch.bfloat16)
    q = torch.randn(rows, H, hd, generator=g) * 3.0
    return dict(H=H, hd=hd, q=q.cuda(), Kp=Kp.cuda(), Vp=Vp.cuda(), pages=torch.stack(pages).int().cuda(),
                pos=torch.tensor(pos, dtype=torch.int32).cuda(), max_pages=max_pages, first=first, shared=shared)


def _attention(c, chunk_pages, grouped, repeats=1, pages=None, pos=None):
    from voicecraft_b200 import _lib
    lib = _lib.load()
    pages = c["pages"] if pages is None else pages
    pos = c["pos"] if pos is None else pos
    rows, H, hd = pos.shape[0], c["H"], c["hd"]
    out = torch.full((rows, H * hd), 12345.0, device="cuda")
    common = (c["q"].data_ptr(), c["Kp"].data_ptr(), c["Vp"].data_ptr(), int(c["Kp"].dtype == torch.float32))
    tail = (rows, H, hd, c["max_pages"], chunk_pages, 1, repeats, out.data_ptr())
    if grouped:
        ng = len(c["shared"])
        rc = lib.vcb_debug_attention_groups(*common, pages.data_ptr(), pos.data_ptr(), *tail,
                                            (C.c_int32 * (ng + 1))(*c["first"]), (C.c_int32 * ng)(*c["shared"]), ng)
    else:
        rc = lib.vcb_debug_attention(*common, pages.data_ptr(), None, None, pos.data_ptr(), *tail)
    torch.cuda.synchronize()
    return rc, out


@pytest.mark.gpu
@pytest.mark.parametrize("chunk_pages", [1, 3, 16])
@pytest.mark.parametrize("kv", ["fp32", "bf16"])
@pytest.mark.parametrize("hd", [64, 128])
def test_grouped_attention_equals_per_row(hd, kv, chunk_pages):
    """attn_rows_kernel over row groups (shared pages loaded once per group, head and chunk) against the per-row kernel on
    the same pools, queries, positions and page lists: every row's output is bit-identical, inactive rows stay untouched,
    and repeated launches on the same arrival counters give the same bits."""
    c = _group_case(hd, kv, chunk_pages)
    rc, ref = _attention(c, chunk_pages, grouped=False)
    assert rc == 0
    for repeats in (1, 3):
        rc, got = _attention(c, chunk_pages, grouped=True, repeats=repeats)
        assert rc == 0
        assert torch.equal(got, ref), f"{int((got != ref).any(dim=1).sum())} rows differ (repeats {repeats})"
    assert (ref[c["pos"] < 0] == 12345.0).all()


@pytest.mark.gpu
def test_grouped_attention_rejects_bad_groups():
    from voicecraft_b200 import _lib
    c = _group_case(128, "bf16", 0)
    pages = c["pages"].clone()
    pages[1, 5] = (pages[1, 5] + 1) % 700                  # row 1 is the second member of the group sharing 70 pages
    assert _attention(c, 16, True, pages=pages)[0] != 0
    assert b"pages differ" in _lib.load().vcb_last_error()
    pos = c["pos"].clone()
    pos[2] -= 1                                            # unequal positions inside that group
    assert _attention(c, 16, True, pos=pos)[0] != 0
    assert b"positions" in _lib.load().vcb_last_error()
    pos[2] = -1                                            # an inactive member is allowed
    assert _attention(c, 16, True, pos=pos)[0] == 0
    bad = dict(c, first=c["first"][:-1] + [c["first"][-1] - 1])
    assert _attention(bad, 16, True)[0] != 0               # groups that do not tile the rows


CASES = [(n, kv, total, {}, 2) for n in (2, 3, 8, 20) for kv in ("fp32", "bf16") for total in (128, 100)]
CASES += [(3, "bf16", 100, {}, 4), (8, "fp32", 128, {}, 4)]                               # head dim 64
CASES += [(n, "bf16", total, env, 2) for n in (3, 20) for total in (128, 100)
          for env in ({"VCB_ATT_CHUNK_PAGES": "1"}, {"VCB_MEGA": "1"})]


@pytest.mark.gpu
@pytest.mark.parametrize("n,kv,total,env,nhead", CASES)
def test_group_equals_independent_rows(n, kv, total, env, nhead, monkeypatch):
    """Until the first step at which any copy samples the end token, a best-of-n group (one prefill, shared full prompt
    pages, forked tail page and last hidden state) and n independent utterances of the same prompt produce the same
    pre-edit logits and tokens, bit for bit."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    cfg, m = _model(kv, nhead=nhead, eos_bias=0.0)
    x, _, y = _utt(cfg, 40 + n, total)
    lg, rg = _trace(m, cfg, x, y, n, True)
    li, ri = _trace(m, cfg, x, y, n, False)
    end = cfg.eos if cfg.eos > 0 else cfg.eog
    hit = [s for s in range(min(len(lg), len(li))) if any(int(r[s, 0]) == end for r in rg + ri if s < r.shape[0])]
    upto = hit[0] + 1 if hit else min(len(lg), len(li))
    assert upto >= 2
    for s in range(upto):
        assert torch.equal(lg[s], li[s]), f"step {s}: logits of the group differ from the independent rows"
    for c in range(n):
        assert (rg[c][:upto] == ri[c][:upto]).all(), f"copy {c}: tokens differ"
    if env.get("VCB_MEGA"):
        from voicecraft_b200 import _lib
        assert _lib.load().vcb_counter(m._engine(), b"mega_grid") > 0, "the persistent kernel did not run"


@pytest.mark.gpu
@pytest.mark.parametrize("total", [128, 100])
def test_group_prefill_and_page_accounting(total):
    from voicecraft_b200 import _lib
    from voicecraft_b200.voicecraft import _Prompt, _prefill
    lib = _lib.load()
    gc.collect()
    torch.cuda.synchronize()
    live0 = (lib.vcb_counter(None, b"live_bytes"), lib.vcb_counter(None, b"live_handles"))
    cfg, m = _model("bf16", max_slots=6)
    x, _, y = _utt(cfg, 5, total)
    eng = m._engine()
    stream = torch.cuda.current_stream().cuda_stream
    max_pages, shared, N = 512 // 64, total // 64, 4
    p = _Prompt(m, x, y)
    free0, rows0 = lib.vcb_counter(eng, b"kv_pages_free"), lib.vcb_counter(eng, b"prefill_rows")
    assert free0 == 6 * max_pages
    need = max_pages + (N - 1) * (max_pages - shared)
    for order in ([0, 1, 2, 3], [3, 1, 0, 2], [2, 0, 3, 1]):
        _prefill(eng, [(p, 1, N, 7, 0)], stream)
        assert lib.vcb_counter(eng, b"prefill_rows") - rows0 == total
        rows0 += total
        assert free0 - lib.vcb_counter(eng, b"kv_pages_free") == need
        for c in order:
            _lib.check(lib.vcb_release(eng, 1 + c, 1))
        assert lib.vcb_counter(eng, b"kv_pages_free") == free0
    # a failed prefill holds nothing.  The pool itself cannot run out: it has max_pages pages per slot and an open slot
    # holds at most max_pages of its own, so the KV-pool check in vcb_prefill is a safeguard no call reaches; the failure
    # here is a call that also names a slot that is open
    _prefill(eng, [(p, 0, 1, 7, 0)], stream)
    before = lib.vcb_counter(eng, b"kv_pages_free")
    with pytest.raises(_lib.VcbError, match="already open"):
        _prefill(eng, [(p, 1, 5, 7, 0), (p, 0, 1, 7, 0)], stream)
    assert lib.vcb_counter(eng, b"kv_pages_free") == before
    assert lib.vcb_counter(eng, b"prefill_rows") == rows0 + total
    _prefill(eng, [(p, 1, 5, 7, 0)], stream)                       # the group's slots were left closed
    assert before - lib.vcb_counter(eng, b"kv_pages_free") == max_pages + 4 * (max_pages - shared)
    for s in (4, 0, 1, 5, 2, 3):
        _lib.check(lib.vcb_release(eng, s, 1))
    assert lib.vcb_counter(eng, b"kv_pages_free") == free0
    m._drop_engine()
    del m
    torch.cuda.synchronize()
    assert (lib.vcb_counter(None, b"live_bytes"), lib.vcb_counter(None, b"live_handles")) == live0


@pytest.mark.gpu
def test_session_best_of_equals_inference_tts_batch():
    """Utterance i of inference_tts_many(best_of=3, seeds=s) equals torch.manual_seed(s_i); inference_tts_batch(x_i, ...,
    batch_size=3), with utterances of different lengths that end at different steps."""
    from voicecraft_b200 import synthetic
    cfg, m = _model("bf16")
    utts = [synthetic.synthetic_utterance(cfg, 300 + i, text_len=3 + i, prompt_frames=20 + 23 * i) for i in range(5)]
    utts = [(x.cuda(), xl.cuda(), y.cuda()) for x, xl, y in utts]
    seeds = [71 + 13 * i for i in range(5)]
    singles, steps = [], []
    for (x, xl, y), s in zip(utts, seeds):
        torch.manual_seed(s)
        singles.append(m.inference_tts_batch(x, xl, y, batch_size=3, **KW))
        steps.append(m.last_stats["steps"])
    assert len(set(steps)) > 1, "utterances should end at different steps"
    many = m.inference_tts_many([u[0] for u in utts], [u[2] for u in utts], seeds=seeds, best_of=3, poll_every=3, **KW)
    for i, ((a, ga), (b, gb)) in enumerate(zip(singles, many)):
        assert torch.equal(a, b) and torch.equal(ga, gb), f"utterance {i}"
    with pytest.raises(ValueError, match="best_of"):
        m.inference_tts_many_stream([utts[0][0]], [utts[0][2]], tokenizer=None, best_of=2)
    with pytest.raises(ValueError, match="best_of"):
        m.inference_tts_many([utts[0][0]], [utts[0][2]], best_of=0)
    assert not m._sessions


@pytest.mark.gpu
def test_batcher_mixed_best_of():
    """max_concurrency 8 with tickets of best_of 1, 2, 3 and 5: groups wait for consecutive free slots, and every ticket
    equals its single call under its seed."""
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, m = _model("bf16")
    sizes = [3, 1, 5, 2, 1, 5, 3, 2, 1, 1]
    utts = [synthetic.synthetic_utterance(cfg, 500 + i, text_len=3 + i % 4, prompt_frames=12 + 7 * (i % 5))
            for i in range(len(sizes))]
    seeds = [900 + i for i in range(len(sizes))]
    cb = ContinuousBatcher(m, max_concurrency=8, poll_every=4, **KW)
    with pytest.raises(ValueError, match="max_concurrency"):
        cb.submit(utts[0][0], utts[0][2], seed=1, best_of=9)
    for (x, _, y), s, n in zip(utts, seeds, sizes):
        cb.submit(x, y, seed=s, best_of=n)
    got = cb.run()
    assert cb.stats["max_active"] <= 8
    for i, ((x, xl, y), s, n) in enumerate(zip(utts, seeds, sizes)):
        torch.manual_seed(s)
        ref = m.inference_tts_batch(x.cuda(), xl.cuda(), y.cuda(), batch_size=n, **KW) if n > 1 else \
            m.inference_tts(x.cuda(), xl.cuda(), y.cuda(), **KW)
        assert torch.equal(got[i][0], ref[0]) and torch.equal(got[i][1], ref[1]), f"ticket {i} (best_of {n})"
    assert not m._sessions


@pytest.mark.gpu
def test_batcher_stream_refuses_best_of_and_serves_the_rest():
    from oracle import encodec_oracle as eo
    from voicecraft_b200 import synthetic
    from voicecraft_b200.tokenizer import AudioTokenizer
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, m = _model("bf16")
    ccfg = eo.default_config()
    tok = AudioTokenizer(device="cuda:0", config=ccfg, state_dict=eo.make_state_dict(ccfg, seed=5))
    utts = [synthetic.synthetic_utterance(cfg, 800 + i, text_len=3, prompt_frames=10 + 3 * i) for i in range(3)]
    cb = ContinuousBatcher(m, max_concurrency=4, poll_every=4, **KW)
    for i, ((x, _, y), n) in enumerate(zip(utts, [1, 2, 1])):
        cb.submit(x, y, seed=40 + i, best_of=n)
    lasts = {}
    for t, w, last in cb.stream(tok):
        if t == 0:
            with pytest.raises(ValueError, match="best_of"):
                cb.submit(utts[0][0], utts[0][2], seed=1, best_of=2)
        if last:
            lasts[t] = w
    assert set(lasts) == {0, 1, 2} and lasts[1] is None and "best_of" in cb.errors[1]
    assert cb.results[1] is None and cb.results[0] is not None and cb.results[2] is not None
    for i in (0, 2):
        x, xl, y = utts[i]
        torch.manual_seed(40 + i)
        ref = m.inference_tts(x.cuda(), xl.cuda(), y.cuda(), **KW)
        assert torch.equal(cb.results[i][1], ref[1])
    assert not m._sessions
