"""KV pool budget: pages taken as utterances grow, refusal of a step the pool cannot cover, and swapping an utterance to host
memory and back byte for byte.  CPU: the batcher's pool policy (KvPoolPolicy) and its admission round against a fake
engine, and the default vcb_config.  GPU (-m gpu): page accounting under a budget, a refused step against an engine that
was never refused, swaps against uninterrupted runs (logits, tokens, KV bytes) in every KV / weight policy, head dim and
step path, snapshot lifetimes, and ContinuousBatcher.run() under a budget that forces swaps."""
import ctypes as C
import gc
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from voicecraft_b200 import _lib
from voicecraft_b200.voicecraft import KvPoolPolicy

KW = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the pool policy against a fake engine
# ---------------------------------------------------------------------------------------------------------------------
class FakeEngine:
    """every listed slot takes one more page per step; a step the free pages cannot cover is refused and changes nothing"""
    stream = None                                      # the CUDA stream of _EngineOps, which the batcher's state takes

    def __init__(self, pool):
        self.pool, self.held, self.log = pool, {}, []

    def free_pages(self):
        return self.pool - sum(self.held.values())

    def step(self, slots):
        if len(slots) > self.free_pages():
            self.log.append(("refused", tuple(slots)))
            return _lib.VCB_ERR_KV_FULL
        for s in slots:
            self.held[s] += 1
        self.log.append(("step", tuple(slots)))
        return 0

    def swap_out(self, slot):
        self.log.append(("out", slot))
        return ["snap", self.held.pop(slot)]

    def swap_in(self, snap, slot):
        assert slot not in self.held and snap[0] == "snap"
        self.log.append(("in", slot))
        self.held[slot] = snap[1]

    def snapshot_pages(self, snap):
        return snap[1]

    def free(self, snap):
        snap[0] = "freed"


def test_policy_admission_is_fifo_with_a_chunk_per_active_slot():
    eng = FakeEngine(20)
    pol = KvPoolPolicy(eng, budget=True, max_swapped=4, chunk=4)
    # 4 <= 20; 4 + 4 <= 16; 4 + 8 <= 12; 4 + 12 > 8
    assert pol.admit_count([(4, 1)] * 4, 0) == 3
    # a large head ticket is not overtaken by the small one behind it
    assert pol.admit_count([(30, 1), (1, 1)], 1) == 0
    # a group counts its slots
    assert pol.admit_count([(4, 3), (8, 1)], 0) == 1
    # the default pool admits by slots alone
    assert KvPoolPolicy(eng, budget=False, max_swapped=4).admit_count([(99, 1)] * 3, 5) == 3


def test_policy_swaps_the_youngest_single_utterance():
    eng = FakeEngine(8)
    eng.held = {0: 2, 1: 2, 2: 2}                      # 2 free: a step of three is refused
    pol = KvPoolPolicy(eng, budget=True, max_swapped=4, chunk=1)
    live = [("a", 0, 0, True), ("b", 1, 1, True), ("c", 2, 2, True)]
    live, out = pol.step(live)
    assert out == [("c", 2)] and [u[0] for u in live] == ["a", "b"]
    assert eng.log == [("refused", (0, 1, 2)), ("out", 2), ("step", (0, 1))]
    assert pol.swap_outs == 1 and [t[1] for t in pol.swapped] == ["c"]
    # a best-of-N group is never the victim, however young
    eng = FakeEngine(7)
    eng.held = {0: 2, 1: 2, 2: 2}
    pol = KvPoolPolicy(eng, budget=True, max_swapped=4, chunk=1)
    live, out = pol.step([("g", 0, 9, False), ("g", 1, 9, False), ("b", 2, 1, True)])
    assert out == [("b", 2)] and [u[1] for u in live] == [0, 1]


def test_policy_resumes_oldest_first_before_admitting():
    eng = FakeEngine(10)
    eng.held = {0: 3, 1: 3, 2: 3}
    pol = KvPoolPolicy(eng, budget=True, max_swapped=4, chunk=1)
    pol.step([("a", 0, 0, True), ("b", 1, 1, True), ("c", 2, 2, True)])      # c out (1 free < 3), a and b step: 2 free
    eng.held[1] += 2                                                         # b grew: none free
    pol.step([("a", 0, 0, True), ("b", 1, 1, True)])                         # b out too (6 pages); a steps: 5 free
    assert [t[1] for t in pol.swapped] == ["b", "c"]
    assert pol.admit_count([(1, 1)], 1) == 0                                 # nothing new while anything is out
    free = {1, 2}
    assert pol.resume(free, 1) == []                                         # b: 6 pages + 2 chunks > 5 free
    del eng.held[0]                                                          # a finished: 10 free
    assert pol.resume(free, 0) == [("b", 1)] and eng.held[1] == 6            # c: 4 pages + 2 chunks > 4 free
    assert pol.swap_ins == 1 and free == {2}
    assert pol.admit_count([(1, 1)], 1) == 0                                 # c is still out
    pol.close()
    assert pol.swapped == []


def test_policy_pool_smaller_than_one_utterance():
    eng = FakeEngine(3)
    eng.held = {0: 3}
    pol = KvPoolPolicy(eng, budget=True, max_swapped=4, chunk=1)
    with pytest.raises(_lib.VcbError, match="smaller than one utterance"):
        pol.step([("a", 0, 0, True)])
    with pytest.raises(_lib.VcbError, match="smaller than one utterance"):
        KvPoolPolicy(FakeEngine(3), budget=True, max_swapped=4).admit_count([(4, 1)], 0)


def test_policy_waits_for_pages_of_finished_utterances():
    """a stream's finished ticket keeps its pages until the next round releases it: a refused step that no victim resolves
    (one ticket still running, or two whose survivor still lacks a page) then waits for those pages instead of failing"""
    eng = FakeEngine(6)
    eng.held = {0: 3, 1: 3}                            # slot 1 finished, not released yet; no page free
    pol = KvPoolPolicy(eng, budget=True, max_swapped=4, chunk=1)
    assert pol.step([("a", 0, 0, True)], leaving=True) == (None, [])
    assert pol.swapped == [] and eng.log == [("refused", (0,))]
    with pytest.raises(_lib.VcbError, match="smaller than one utterance"):
        pol.step([("a", 0, 0, True)])                  # nothing is leaving: the pool is too small
    eng = FakeEngine(5)
    eng.held = {0: 2, 1: 0, 2: 3}                      # slot 2 finished; swapping b out frees nothing
    pol = KvPoolPolicy(eng, budget=True, max_swapped=4, chunk=1)
    assert pol.step([("a", 0, 0, True), ("b", 1, 1, True)], leaving=True) == (None, [("b", 1)])
    assert [t[1] for t in pol.swapped] == ["b"]
    del eng.held[2]                                    # released: the next round steps a
    live, out = pol.step([("a", 0, 0, True)])
    assert [u[0] for u in live] == ["a"] and out == []
    # a refusal a victim resolves swaps as usual, finished tickets or not
    eng = FakeEngine(8)
    eng.held = {0: 2, 1: 2, 2: 2, 3: 1}                # slot 3 finished; 1 free
    pol = KvPoolPolicy(eng, budget=True, max_swapped=4, chunk=1)
    live, out = pol.step([("a", 0, 0, True), ("b", 1, 1, True), ("c", 2, 2, True)], leaving=True)
    assert out == [("c", 2)] and [u[0] for u in live] == ["a", "b"]


def test_policy_caps_the_swapped_out_utterances():
    eng = FakeEngine(7)
    eng.held = {0: 3, 1: 3, 2: 1}                      # no page free: two utterances have to leave
    pol = KvPoolPolicy(eng, budget=True, max_swapped=1, chunk=1)
    with pytest.raises(_lib.VcbError, match="swapped out already"):
        pol.step([("a", 0, 0, True), ("b", 1, 1, True), ("c", 2, 2, True)])
    assert [t[1] for t in pol.swapped] == ["c"]
    pol.close()


def _serving(eng, n_slots, tickets, cancelled=(), budget=True):
    """ContinuousBatcher's serving state over the fake engine, with no model: tickets lists (best_of, sentences), with
    sentences None for a plain ticket, whose prompt asks admission for a page per slot, and for a long ticket the pages
    each sentence's prompt asks per slot.  The prefill (_admit) takes one page per slot and logs ("admit", [(slot,
    ticket)]) next to the engine's steps and swaps; releasing a slot gives its pages back; every result is ("res", "gen")"""
    from voicecraft_b200.voicecraft import ContinuousBatcher, _Chain, _Ticket

    def prompt(pages):
        return SimpleNamespace(pages=lambda n, max_pages: n * pages, source=_lib.vcb_edit_source,
                               result=lambda *a: ("res", "gen", "lp"))

    def release(held, starts, n_copies=1, keep_held=False):
        for s in starts:
            for c in range(n_copies):
                eng.held.pop(s + c, None)

    def admit(s, new):
        eng.log.append(("admit", list(new)))
        eng.held.update({slot + c: 1 for slot, t in new for c in range(s.jobs[t].best_of)})
    model = SimpleNamespace(_eng_opts=dict(max_seq_len=64, kv_pool_gb=1.0 if budget else None), _release_slots=release,
                            _read_rows=lambda *a: None, _read_lp=lambda *a: None)
    cb = ContinuousBatcher(model, max_concurrency=n_slots, poll_every=1)
    cb._admit, cb.logprobs = admit, [None] * len(tickets)
    jobs = []
    for n, sentences in tickets:
        chain = None if sentences is None else _Chain(["x"] * len(sentences))
        if chain is not None:
            chain.start([prompt(pages) for pages in sentences])
        jobs.append(_Ticket(prompt(1) if chain is None else chain.prompt, None, n, None, chain=chain))
    s = SimpleNamespace(eng=None, slots=list(range(n_slots)), jobs=jobs, results=[None] * len(jobs),
                        cancelled=set(cancelled), cstream=None, pool=None)
    cb._open(s, eng)
    s.pool.chunk = 1                                   # the fake engine's slots grow a page per step
    return cb, s


def _ended(r, offset=0, keep=0):
    r.status = SimpleNamespace(n_steps=0, rng_offset=offset, keep=keep)
    return r.slot + keep, r.status


def test_batcher_round_order_under_a_budget():
    """One admission round, shared by run() and stream(): a held next sentence first, no swapped-out utterance back
    while it waits, then swapped-out utterances, then the queue in order, cancelled tickets skipped; freed slots are
    reused lowest first"""
    eng = FakeEngine(9)
    # ticket 0: a long ticket whose second sentence asks 6 pages; 3 is cancelled; 4 is a best-of-2 group
    cb, s = _serving(eng, 5, [(1, [1, 6]), (1, None), (1, None), (1, None), (2, None), (1, None)], cancelled={3})
    followed, new = cb._round(s)
    # 1 + 2 + 3 + (2 + 3) of 9 pages; ticket 5 would need 1 + 5 of the 4 left
    assert eng.log == [("admit", [(0, 0), (1, 1), (2, 2), (3, 4)])] and followed == []
    assert [(r.slot, r.ticket) for r in new] == [(0, 0), (1, 1), (2, 2), (3, 4)] and s.nxt == 5 and s.free == set()
    assert cb.stats["max_active"] == 5
    # five slots, four free pages: the step is refused and the youngest one-copy utterance (ticket 2) goes out
    r2 = s.active[2]
    assert cb._steps(s, [s.active[k] for k in sorted(s.active)]) == 1
    assert eng.log[1:] == [("refused", (0, 1, 2, 3, 4)), ("out", 2), ("step", (0, 1, 3, 4))]
    assert sorted(s.active) == [0, 1, 3] and s.free == {2} and [k for _, k, _ in s.pool.swapped] == [r2]
    assert cb._leave(s, s.active[1], _ended(s.active[1])) is True
    r0 = s.active[0]
    assert cb._leave(s, r0, _ended(r0, offset=480)) is False          # its next sentence keeps slot 0
    assert s.follow == [r0] and s.free == {1, 2} and s.results[:2] == [None, ("res", "gen")]
    assert s.jobs[0].chain.offset == 480
    # 5 pages free: the next sentence (6 + a chunk per active slot) waits, and ticket 2 (1 + 3), which the pool would take,
    # does not come back before it
    n_log = len(eng.log)
    assert cb._round(s) == ([], []) and len(eng.log) == n_log and s.follow == [r0] and s.nxt == 5
    r4 = s.active[3]
    assert cb._leave(s, r4, _ended(r4, keep=1)) is True and s.free == {1, 2, 3, 4} and eng.held == {}
    followed, new = cb._round(s)
    assert eng.log[n_log:] == [("admit", [(0, 0)]), ("in", 1), ("admit", [(2, 5)])]
    (r,) = followed
    assert (r.slot, r.cid, r.label, r.carry, r.more) == (0, r0.cid, "ticket 0 sentence 1", True, False)
    assert s.active[1] is r2 and r2.slot == 1                          # back into the lowest free slot, not its own
    assert [(r.slot, r.ticket) for r in new] == [(2, 5)] and s.nxt == 6 and s.free == {3, 4} and s.follow == []


def test_batcher_round_keeps_a_group_ahead_of_later_tickets():
    """a best-of-N group that finds no run of free slots stops the admission; a cancelled ticket is passed over"""
    eng = FakeEngine(0)
    cb, s = _serving(eng, 4, [(1, None), (1, None), (1, None), (2, None), (1, None), (1, None), (1, None)],
                     cancelled={5}, budget=False)
    cb._round(s)
    assert eng.log == [("admit", [(0, 0), (1, 1), (2, 2)])] and s.nxt == 3 and s.free == {3}
    cb._leave(s, s.active[1], _ended(s.active[1]))
    assert cb._round(s) == ([], []) and len(eng.log) == 1 and s.nxt == 3 and s.free == {1, 3}
    cb._leave(s, s.active[2], _ended(s.active[2]))
    _, new = cb._round(s)
    assert eng.log[1:] == [("admit", [(1, 3), (3, 4)])] and s.nxt == 6 and s.free == set()
    assert [r.label for r in new] == ["ticket 3", "ticket 4"]


def test_batcher_round_admits_no_queued_ticket_while_a_next_sentence_waits():
    eng = FakeEngine(5)
    cb, s = _serving(eng, 3, [(1, [1, 6]), (1, None), (1, None), (1, None)])
    cb._round(s)
    assert eng.log == [("admit", [(0, 0), (1, 1), (2, 2)])] and s.nxt == 3
    cb._leave(s, s.active[1], _ended(s.active[1]))
    assert cb._leave(s, s.active[0], _ended(s.active[0])) is False
    # 4 pages free: the next sentence (6 + 1) waits, and ticket 3 (1 + 1), which the pool would take, is not admitted
    assert cb._round(s) == ([], []) and len(eng.log) == 1 and s.nxt == 3 and s.free == {1}
    eng.pool = 9                                       # pages another user of the engine held come back
    followed, new = cb._round(s)
    assert eng.log[1:] == [("admit", [(0, 0)]), ("admit", [(1, 3)])]
    assert [r.ticket for r in followed] == [0] and [r.ticket for r in new] == [3] and s.nxt == 4


def test_default_config_is_todays_pool():
    c = _lib.vcb_config()
    assert c.kv_pool_bytes == 0
    assert _lib.vcb_config.kv_pool_bytes.offset == 80 and C.sizeof(_lib.vcb_config) == 88   # after 19 int32, 8-aligned


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
def _lm(kv="bf16", weights="bf16", nhead=2, edit=False, seed=3, **opts):
    """tiny LM whose heads put no mass on non-audio tokens; TTS: codebook 0 never ends early either (it runs to its length
    cap); edit: codebook 0 ends spans with eog now and then"""
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny", nhead=nhead)
    sd = synthetic.make_state_dict(cfg, seed=seed)
    for k in range(cfg.n_codebooks):
        for t in (cfg.empty_token, cfg.eog, cfg.audio_pad_token, cfg.eos):
            sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    if edit:
        sd["predict_layer.0.2.bias"][cfg.eog] = 2.5
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    m = m.to("cuda:0").eval()
    m.configure_engine(kv_dtype=kv, weight_dtype=weights, **opts)
    return cfg, m


def _utt(cfg, seed, text_len, total):
    """an utterance whose prompt fills `total` positions (text + T + 1 delayed rows); longer texts allow longer generations"""
    from voicecraft_b200 import synthetic
    x, xl, y = synthetic.synthetic_utterance(cfg, seed, text_len=text_len, prompt_frames=total - text_len - 1)
    return x.cuda(), xl.cuda(), y.cuda()


def _budget(m, pages, **opts):
    """reconfigure m for a pool of `pages` KV pages"""
    pb = _lib.load().vcb_counter(m._engine(), b"kv_page_bytes")
    m.configure_engine(kv_pool_gb=(pages + 0.5) * pb / 1e9, **opts)
    assert _lib.load().vcb_counter(m._engine(), b"kv_pages_total") == pages


def _one(s):
    return (C.c_int32 * 1)(s)


def _poll(lib, eng, slot, stream):
    st = (_lib.vcb_status * 1)()
    _lib.check(lib.vcb_poll(eng, _one(slot), 1, st, stream))
    s = st[0]
    return dict(done=s.done, forced=s.forced, n_steps=s.n_steps, n_spans_done=s.n_spans_done, rng=s.rng_offset)


def _kv_valid(m, eng, slot, seq_len):
    """the K and V bytes of positions [0, seq_len) of a slot in every layer (a page's unwritten tail is not compared)"""
    lib, a = _lib.load(), m.args
    H, hd = a.nhead, a.d_model // a.nhead
    kv = m._eng_opts["kv_dtype"]
    slab = 64 * (hd + 4) if kv == "fp8" else 64 * hd * (4 if kv == "fp32" else 2)
    n_pages = (seq_len + 63) // 64
    out = []
    for layer in range(a.num_decoder_layers):
        kb, vb = (C.c_uint8 * (n_pages * H * slab))(), (C.c_uint8 * (n_pages * H * slab))()
        _lib.check(lib.vcb_debug_kv_pages(eng, layer, slot, 0, n_pages, kb, vb))
        for buf in (kb, vb):
            pages = np.frombuffer(buf, dtype=np.uint8).reshape(n_pages, H, slab)
            for t in range(seq_len):
                p, r = divmod(t, 64)
                if kv == "fp8":
                    out.append(pages[p, :, r * hd:(r + 1) * hd].tobytes())
                    out.append(pages[p, :, 64 * hd + 4 * r:64 * hd + 4 * r + 4].tobytes())
                else:
                    es = slab // (64 * hd)
                    out.append(pages[p, :, r * hd * es:(r + 1) * hd * es].tobytes())
    return out


def _drive(m, cfg, x, y, spans=None, n_steps=90, swap_at=None, filler=None):
    """one utterance in slot 0 (seed 7, its own parameters): vcb_sample, then decode steps while it is not done, the logits
    after every sampling step that was not a forced hand-over.  swap_at(i, status): before decode step i, swap it out,
    prefill `filler` into slot 0 (it takes the freed pages), swap the snapshot into slot 2 and go on there.
    Returns (logits, token rows, KV bytes of the written positions, final status)."""
    from voicecraft_b200.voicecraft import _Prompt, _prefill
    lib = _lib.load()
    eng = m._engine()
    stream = torch.cuda.current_stream().cuda_stream
    K, V = cfg.n_codebooks, m.n_audio_tokens[0]
    sp = m._sampling(silence_tokens=(1388, 1898, 131), **KW)
    p = _Prompt(m, x, y, spans)
    _prefill(eng, [(p, 0, 1, 7, 0, sp)], stream)
    slot, swapped, seq_len, logits = 0, False, p.total, []

    def trace():
        t = torch.empty(K, V, device="cuda")
        _lib.check(lib.vcb_debug_logits(eng, t.data_ptr(), K))
        logits.append(t)
    try:
        _lib.check(lib.vcb_sample(eng, _one(slot), 1, None, None, stream))
        trace()
        for i in range(n_steps):
            st = _poll(lib, eng, slot, stream)
            if st["done"]:
                break
            if swap_at is not None and not swapped and swap_at(i, st, seq_len):
                snap = C.c_void_p()
                _lib.check(lib.vcb_swap_out(eng, slot, C.byref(snap), stream))
                _prefill(eng, [(filler, 0, 1, 99, 0, sp)], stream)
                _lib.check(lib.vcb_swap_in(eng, snap, 2, stream))
                lib.vcb_snapshot_free(snap)
                assert _poll(lib, eng, 2, stream) == st
                slot, swapped = 2, True
            _lib.check(lib.vcb_decode_step(eng, _one(slot), 1, None, None, stream))
            seq_len += 1
            if not st["forced"]:
                trace()
        st = _poll(lib, eng, slot, stream)
        rows = m._read_rows(eng, slot, st["n_steps"], stream)
        kv = _kv_valid(m, eng, slot, seq_len)
    finally:
        for s in (0, 2):
            lib.vcb_release(eng, s, 1)
    assert swap_at is None or swapped, "the swap point was never reached"
    return logits, rows, kv, st


def _same(a, b):
    la, ra, ka, sa = a
    lb, rb, kb, sb = b
    assert sa == sb
    assert len(la) == len(lb)
    for i, (u, v) in enumerate(zip(la, lb)):
        assert torch.equal(u, v), f"sampling step {i}: logits differ"
    assert np.array_equal(ra, rb), "tokens differ"
    assert len(ka) == len(kb) and all(u == v for u, v in zip(ka, kb)), "KV bytes differ"


# ---------------------------------------------------------------------------------------------------------------------
# GPU: engine
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_pages_follow_the_steps_under_a_budget():
    from voicecraft_b200.voicecraft import _Prompt, _prefill
    cfg, m = _lm(max_slots=4, max_seq_len=1024)
    _budget(m, 40)
    lib, eng = _lib.load(), m._engine()
    stream = torch.cuda.current_stream().cuda_stream
    free = lambda: lib.vcb_counter(eng, b"kv_pages_free")
    assert free() == 40
    x, _, y = _utt(cfg, 5, 20, 100)
    p = _Prompt(m, x, y)
    _prefill(eng, [(p, 0, 1, 7, 0)], stream)
    assert 40 - free() == 4 == p.pages(1, 16)              # ceil(100 / 64) = 2, in whole chunks of 4
    sp = m._sampling(silence_tokens=(), **KW)
    _lib.check(lib.vcb_sample(eng, _one(0), 1, None, C.byref(sp), stream))
    for i in range(1, 200):
        _lib.check(lib.vcb_decode_step(eng, _one(0), 1, None, C.byref(sp), stream))
        pos = 100 + i - 1                                  # the position step i writes
        assert 40 - free() == min(16, -(-(pos // 64 + 1) // 4) * 4), i
    # a best-of-N group keeps its full reservation
    _prefill(eng, [(p, 1, 2, 7, 0)], stream)
    assert 40 - free() == 8 + 16 + 15
    for s in (1, 0, 2):
        _lib.check(lib.vcb_release(eng, s, 1))
    assert free() == 40


@pytest.mark.gpu
def test_default_engine_pool_and_counters():
    cfg, m = _lm(max_slots=3, max_seq_len=512)
    lib, eng = _lib.load(), m._engine()
    assert lib.vcb_counter(eng, b"kv_pages_total") == lib.vcb_counter(eng, b"kv_pages_free") == 3 * 8
    a = m.args
    assert lib.vcb_counter(eng, b"kv_page_bytes") == 2 * a.num_decoder_layers * 64 * 2 * a.d_model
    with pytest.raises(ValueError):
        m.configure_engine(kv_pool_gb=0)


@pytest.mark.gpu
def test_refused_step_changes_nothing():
    """two utterances fill an 8-page pool; the step that needs a fifth page each is refused (twice), then the other one
    leaves and the first goes on: its state, later tokens and KV bytes equal an engine that was never refused"""
    from voicecraft_b200.voicecraft import _Prompt, _prefill
    cfg, m = _lm(max_slots=4, max_seq_len=512)
    x, _, y = _utt(cfg, 5, 40, 100)
    x2, _, y2 = _utt(cfg, 6, 40, 100)
    ref = _drive(m, cfg, x, y, n_steps=400)
    _budget(m, 8)
    lib, eng = _lib.load(), m._engine()
    stream = torch.cuda.current_stream().cuda_stream
    p, p2 = _Prompt(m, x, y), _Prompt(m, x2, y2)
    sp = m._sampling(silence_tokens=(1388, 1898, 131), **KW)
    _prefill(eng, [(p, 0, 1, 7, 0, sp), (p2, 1, 1, 8, 0, sp)], stream)
    both = (C.c_int32 * 2)(0, 1)
    _lib.check(lib.vcb_sample(eng, both, 2, None, None, stream))
    steps = 0
    for steps in range(1, 157):                              # writes positions 100 .. 255
        _lib.check(lib.vcb_decode_step(eng, both, 2, None, None, stream))
    assert lib.vcb_counter(eng, b"kv_pages_free") == 0
    before = _poll(lib, eng, 0, stream), _poll(lib, eng, 1, stream)
    assert not before[0]["done"] and not before[1]["done"]
    launches = lib.vcb_counter(eng, b"launches")
    assert lib.vcb_decode_step(eng, both, 2, None, None, stream) == _lib.VCB_ERR_KV_FULL
    assert b"KV pool full" in lib.vcb_last_error() and lib.vcb_counter(eng, b"kv_pages_needed") == 2
    assert lib.vcb_decode_step(eng, _one(0), 1, None, None, stream) == _lib.VCB_ERR_KV_FULL
    assert lib.vcb_counter(eng, b"kv_pages_needed") == 1
    assert lib.vcb_counter(eng, b"launches") == launches and lib.vcb_counter(eng, b"kv_pages_free") == 0
    assert (_poll(lib, eng, 0, stream), _poll(lib, eng, 1, stream)) == before
    _lib.check(lib.vcb_release(eng, 1, 1))
    try:
        for _ in range(steps, 400):
            if _poll(lib, eng, 0, stream)["done"]:
                break
            _lib.check(lib.vcb_decode_step(eng, _one(0), 1, None, None, stream))
        st = _poll(lib, eng, 0, stream)
        assert st["n_steps"] > 160
        rows = m._read_rows(eng, 0, st["n_steps"], stream)
        kv = _kv_valid(m, eng, 0, 100 + st["n_steps"] - 1)    # vcb_sample, then one position per decode step
    finally:
        lib.vcb_release(eng, 0, 1)
    assert st == ref[3] and np.array_equal(rows, ref[1]) and kv == ref[2]


SWAPS = [("bf16", "bf16", 2, {}, "page"), ("bf16", "bf16", 2, {}, "mid"), ("fp32", "bf16", 2, {}, "page"),
         ("fp8", "bf16", 2, {}, "mid"), ("fp8", "bf16", 4, {}, "page"), ("bf16", "int8", 2, {}, "mid"),
         ("bf16", "bf16", 4, {}, "page"), ("bf16", "bf16", 2, {"VCB_MEGA": "1"}, "mid"),
         ("bf16", "bf16", 2, {}, "edit"), ("fp8", "bf16", 4, {}, "edit")]


@pytest.mark.gpu
@pytest.mark.parametrize("kv,weights,nhead,env,where", SWAPS)
def test_swap_continues_bit_for_bit(kv, weights, nhead, env, where, monkeypatch):
    """swapped out at a page boundary (the next step grows the new page list), mid-page, or in a multi-span edit with the
    forced hand-over steps of the next span pending; swapped into another slot on other pages: logits, tokens and KV bytes
    equal the uninterrupted run"""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    cfg, m = _lm(kv, weights, nhead, edit=where == "edit", max_slots=4, max_seq_len=512)
    if where == "edit":
        x, _, y = _utt(cfg, 11, 14, 56)
        spans = [(5, 12), (20, 26), (30, 36)]
        at = lambda i, st, seq: st["forced"] > 0 and st["n_spans_done"] >= 1
    else:
        x, _, y = _utt(cfg, 12, 20, 100)
        spans = None
        at = (lambda i, st, seq: seq == 128) if where == "page" else (lambda i, st, seq: i == 40)
    filler = _utt(cfg, 13, 9, 150)
    from voicecraft_b200.voicecraft import _Prompt
    ref = _drive(m, cfg, x, y, spans)
    got = _drive(m, cfg, x, y, spans, swap_at=at, filler=_Prompt(m, filler[0], filler[2]))
    _same(got, ref)
    if env.get("VCB_MEGA"):
        assert _lib.load().vcb_counter(m._engine(), b"mega_grid") > 0, "the persistent kernel did not run"


def _live():
    gc.collect()
    torch.cuda.synchronize()
    lib = _lib.load()
    return lib.vcb_counter(None, b"live_bytes"), lib.vcb_counter(None, b"live_handles")


@pytest.mark.gpu
def test_snapshot_lifetime_and_rejected_swap_in():
    """a snapshot holds pinned memory until it is freed, also after its engine was destroyed; rejected swap-ins hold
    nothing; the engine's swap staging region is one utterance's pages"""
    from voicecraft_b200.voicecraft import _Prompt, _prefill
    live0 = _live()
    cfg, m = _lm(max_slots=3, max_seq_len=512)
    _budget(m, 9)
    lib, eng = _lib.load(), m._engine()
    stream = torch.cuda.current_stream().cuda_stream
    x, _, y = _utt(cfg, 5, 20, 300)                          # 5 written pages, 8 held
    p = _Prompt(m, x, y)
    snap = C.c_void_p()
    page = lib.vcb_counter(eng, b"kv_page_bytes")
    assert lib.vcb_counter(eng, b"swap_stage_bytes") <= 16
    _prefill(eng, [(p, 0, 1, 7, 0)], stream)                 # the engine's own prefill and swap buffers exist after this
    _lib.check(lib.vcb_swap_out(eng, 0, C.byref(snap), stream))
    _lib.check(lib.vcb_swap_in(eng, snap, 0, stream))
    lib.vcb_snapshot_free(snap)
    _lib.check(lib.vcb_release(eng, 0, 1))
    assert lib.vcb_counter(eng, b"swap_stage_bytes") == 5 * page
    base = _live()
    _prefill(eng, [(p, 0, 1, 7, 0)], stream)
    assert lib.vcb_swap_out(eng, 1, C.byref(snap), stream) != 0             # not open
    _lib.check(lib.vcb_swap_out(eng, 0, C.byref(snap), stream))
    assert lib.vcb_snapshot_pages(snap) == 5 and lib.vcb_counter(eng, b"kv_pages_free") == 9
    held = _live()
    assert held[0] > base[0] and held[1] > base[1]
    _prefill(eng, [(p, 1, 1, 7, 0)], stream)                                # 8 pages: 1 free
    for slot in (1, 5, -1):                                                 # open, out of range
        assert lib.vcb_swap_in(eng, snap, slot, stream) != 0
    assert lib.vcb_swap_in(eng, snap, 0, stream) != 0                       # 5 pages needed, 1 free
    assert b"KV pages" in lib.vcb_last_error()
    _, m2 = _lm(max_slots=1, max_seq_len=512)
    assert lib.vcb_swap_in(m2._engine(), snap, 0, stream) != 0              # another engine's snapshot
    assert b"not a snapshot of this engine" in lib.vcb_last_error()
    m2._drop_engine()
    del m2
    assert _live() == held and lib.vcb_counter(eng, b"kv_pages_free") == 1
    _lib.check(lib.vcb_release(eng, 1, 1))
    _lib.check(lib.vcb_swap_in(eng, snap, 2, stream))                        # still valid after the rejections
    lib.vcb_snapshot_free(snap)
    assert _live() == base
    # a snapshot outliving its engine
    _lib.check(lib.vcb_swap_out(eng, 2, C.byref(snap), stream))
    m._drop_engine()
    assert _live() != live0
    lib.vcb_snapshot_free(snap)
    assert _live() == live0
    # a best-of-N group does not swap
    m.configure_engine(kv_pool_gb=None, max_slots=3)
    eng = m._engine()
    _prefill(eng, [(p, 0, 2, 7, 0)], stream)
    assert lib.vcb_swap_out(eng, 1, C.byref(snap), stream) != 0
    assert b"best-of-N" in lib.vcb_last_error()
    _lib.check(lib.vcb_release(eng, 0, 2))
    lib.vcb_snapshot_free(None)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the batcher under a budget
# ---------------------------------------------------------------------------------------------------------------------
def _queue(cfg, n):
    """long utterances (40 text ids) whose prompts take one page"""
    return [_utt(cfg, 70 + i, 40, 50 + 3 * i) for i in range(n)]


@pytest.mark.gpu
def test_batcher_run_under_a_budget_swaps_and_equals_single_calls():
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, m = _lm(max_slots=4, max_seq_len=512)
    utts, seeds = _queue(cfg, 6), [500 + i for i in range(6)]
    singles = []
    for (x, xl, y), s in zip(utts, seeds):
        torch.manual_seed(s)
        singles.append(m.inference_tts(x, xl, y, **KW))

    def run(cb):
        for (x, _, y), s in zip(utts, seeds):
            cb.submit(x, y, seed=s)
        return cb.run()
    free = ContinuousBatcher(m, max_concurrency=4, poll_every=5, **KW)
    plain = run(free)
    assert free.stats["swap_outs"] == 0
    _budget(m, 12, max_slots=4, max_seq_len=512)
    cb = ContinuousBatcher(m, max_concurrency=4, poll_every=5, **KW)
    got = run(cb)
    assert cb.stats["swap_outs"] >= 2 and cb.stats["swap_ins"] == cb.stats["swap_outs"], cb.stats
    for i in range(6):
        assert torch.equal(got[i][0], singles[i][0]) and torch.equal(got[i][1], singles[i][1]), i
        assert torch.equal(plain[i][0], got[i][0]), i
    lib = _lib.load()
    assert lib.vcb_counter(m._engine(), b"kv_pages_free") == 12
    # a pool that cannot hold one utterance's growth fails loudly
    _budget(m, 5, max_slots=4, max_seq_len=512)
    cb = ContinuousBatcher(m, max_concurrency=4, poll_every=5, **KW)
    with pytest.raises(_lib.VcbError, match="smaller than one utterance"):
        run(cb)
    assert lib.vcb_counter(m._engine(), b"kv_pages_free") == 5


@pytest.mark.gpu
def test_batcher_stream_under_a_budget_swaps_cancels_and_equals_unconstrained():
    """stream() under a budget: every ticket's chunks arrive in order and, concatenated, equal those of an unconstrained
    stream and the decode of its seeded inference_tts; a swapped-out ticket can be cancelled (its snapshot goes)"""
    from oracle import encodec_oracle as eo
    from voicecraft_b200.tokenizer import AudioTokenizer
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, m = _lm(max_slots=4, max_seq_len=512)
    ccfg = eo.default_config()
    tok = AudioTokenizer(device="cuda:0", config=ccfg, state_dict=eo.make_state_dict(ccfg, seed=5))
    utts, seeds = _queue(cfg, 7), [600 + i for i in range(7)]
    singles = []
    for (x, xl, y), s in zip(utts, seeds):
        torch.manual_seed(s)
        singles.append(m.inference_tts(x, xl, y, **KW))

    def stream(cb, on_chunk=None):
        for (x, _, y), s in zip(utts, seeds):
            cb.submit(x, y, seed=s)
        audio, lasts = {}, {}
        for t, w, last in cb.stream(tok, chunk_frames=10):
            assert not lasts.get(t), f"ticket {t}: a chunk after its last"
            audio.setdefault(t, []).append(w)
            lasts[t] = last
            if on_chunk is not None:
                on_chunk(cb)
        return audio, lasts
    plain, _ = stream(ContinuousBatcher(m, max_concurrency=4, poll_every=5, **KW))
    _budget(m, 12, max_slots=4, max_seq_len=512)
    cb = ContinuousBatcher(m, max_concurrency=4, poll_every=5, **KW)
    audio, lasts = stream(cb)
    assert cb.stats["swap_outs"] >= 2 and cb.stats["swap_ins"] == cb.stats["swap_outs"], cb.stats
    for i in range(7):
        res, gen = cb.results[i]
        assert torch.equal(res, singles[i][0]) and torch.equal(gen, singles[i][1]), i
        assert lasts[i] is True and torch.equal(torch.cat(audio[i], -1), torch.cat(plain[i], -1)), i
        assert torch.equal(torch.cat(audio[i], -1), tok.decode_codes(gen)), i
    # cancel the first ticket seen swapped out
    cancelled = []

    def cancel_swapped(cb):
        st = cb._live
        if not cancelled and st.pool.swapped:
            t = st.pool.swapped[0][1].ticket
            assert cb.cancel(t)
            cancelled.append((t, len(audio2.get(t, []))))
    audio2 = {}
    cb = ContinuousBatcher(m, max_concurrency=4, poll_every=5, **KW)
    for (x, _, y), s in zip(utts, seeds):
        cb.submit(x, y, seed=s)
    for t, w, last in cb.stream(tok, chunk_frames=10):
        audio2.setdefault(t, []).append(w)
        cancel_swapped(cb)
    assert cancelled, "no ticket was swapped out"
    t, n = cancelled[0]
    assert len(audio2.get(t, [])) == n and cb.results[t] is None
    for i in range(7):
        if i != t:
            assert torch.equal(cb.results[i][0], singles[i][0]), i
    assert _lib.load().vcb_counter(m._engine(), b"kv_pages_free") == 12
    assert cb.stats["swap_ins"] < cb.stats["swap_outs"]


@pytest.mark.gpu
def test_tts_many_under_a_budget_swaps_and_equals_unconstrained(monkeypatch):
    from voicecraft_b200 import voicecraft as vc
    cfg, m = _lm(max_slots=4, max_seq_len=512)
    utts, seeds = _queue(cfg, 3), [700, 701, 702]
    xs, ys = [u[0] for u in utts], [u[2] for u in utts]
    plain = m.inference_tts_many(xs, ys, seeds=seeds, **KW)
    _budget(m, 14, max_slots=4, max_seq_len=512)
    outs = []
    real = vc._EngineOps.swap_out
    monkeypatch.setattr(vc._EngineOps, "swap_out", lambda self, slot: outs.append(slot) or real(self, slot))
    got = m.inference_tts_many(xs, ys, seeds=seeds, **KW)
    assert len(outs) >= 1
    for i in range(3):
        assert torch.equal(got[i][0], plain[i][0]) and torch.equal(got[i][1], plain[i][1]), i
    assert _lib.load().vcb_counter(m._engine(), b"kv_pages_free") == 14
