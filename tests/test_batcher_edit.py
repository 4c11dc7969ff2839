"""Speech editing in the continuous batcher and as a stream, and per-group sampling parameters.

CPU: the host restatement of an edit's final output frames (edit_final_frames / edit_frame_codes) on synthetic token rows,
and submit()'s argument checks.  GPU (-m gpu): the device gather vcb_poll_frames_ex against that restatement and against
vcb_poll_frames, its error contract, the vcb_prompt.sampling contract, and the batcher (run / stream) and the edit streams
against seeded single calls and whole decodes."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

EOG, EMPTY = 2049, 2048


# ---------------------------------------------------------------------------------------------------------------------
# host restatement (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def _simulate(K, gens, seed):
    """delayed token rows of an edit whose span j generates gens[j] frames: yields (rows so far, status) after every row"""
    rng = np.random.default_rng(seed)
    rows, ends = [], []
    for g in gens:
        for r in range(g + K):
            row = rng.integers(0, 2048, K)
            if r >= g:                       # the end token in codebook 0, then the delayed ends of the others
                row[: r - g] = EMPTY
                row[r - g] = EOG
            rows.append(row)
            if r == g + K - 1:
                ends.append(len(rows))
            yield np.array(rows, dtype=np.int64), SimpleNamespace(n_spans_done=len(ends), span_ends=ends + [0] * (8 - len(ends)))


@pytest.mark.parametrize("T,spans,gens", [
    (20, [(0, 5)], [7]),                             # a span at frame 0
    (20, [(15, 20)], [4]),                           # a span ending at T
    (24, [(3, 6), (6, 10)], [5, 0]),                 # adjacent spans, one generating nothing
    (30, [(0, 4), (9, 12), (25, 30)], [3, 6, 2]),    # three spans, at 0 and at T
    (30, [(2, 4), (8, 12), (15, 21)], [0, 9, 1]),
])
@pytest.mark.parametrize("K", [4, 8])
def test_edit_restatement_grows_and_ends_at_the_result(K, T, spans, gens):
    from voicecraft_b200.voicecraft import VoiceCraft, edit_final_frames, edit_frame_codes
    orig = np.random.default_rng(1).integers(0, 2048, (K, T))
    prev, seen = -1, []
    for rows, st in _simulate(K, gens, seed=T + K):
        f = edit_final_frames(rows, st, spans, T, K, EOG)
        assert f >= prev
        prev = f
        seen.append((f, edit_frame_codes(rows, st, orig, spans, K, EOG, 0, f)))
    # the result as _Prompt.result builds it
    pieces, lo, ends = [], 0, st.span_ends[:len(spans)]
    non_mask = list(zip([0] + [e for _, e in spans], [s for s, _ in spans] + [T]))
    for (s0, s1), hi in zip(non_mask, ends):
        pieces += [orig[:, s0:s1], VoiceCraft._undelay(rows[lo:hi], K)]
        lo = hi
    pieces.append(orig[:, non_mask[-1][0]:non_mask[-1][1]])
    res = np.concatenate(pieces, axis=1)
    assert prev == res.shape[1] == T - sum(e - s for s, e in spans) + sum(gens)
    assert seen[0][0] >= spans[0][0]                 # the leading original piece is final before the first row
    for f, codes in seen:                            # final frames never change
        assert np.array_equal(codes, res[:, :f])
    assert np.array_equal(edit_frame_codes(rows, st, orig, spans, K, EOG, 3, prev - 1), res[:, 3:prev - 1])


def test_submit_rejects_bad_edit_tickets():
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import ContinuousBatcher, VoiceCraft
    cfg = synthetic.make_config("tiny")
    cb = ContinuousBatcher(VoiceCraft(cfg), max_concurrency=4)
    x, _, y = synthetic.synthetic_utterance(cfg, 0, 4, 12)
    with pytest.raises(ValueError):
        cb.submit(x, y, best_of=2, mask_interval=torch.tensor([[[2, 5]]]))
    with pytest.raises(ValueError):
        cb.submit(x, y, mask_interval=torch.tensor([[[0, 1], [2, 3], [4, 5], [6, 7]]]))    # max_n_spans = 3
    with pytest.raises(ValueError):
        cb.submit(x, y, mask_interval=torch.tensor([[2, 5]]))
    for bad in (dict(temperature=0.0), dict(temperature=float("inf")), dict(top_p=float("nan"))):
        with pytest.raises(ValueError):
            cb.submit(x, y, **bad)
    assert cb.queue == []
    assert cb.submit(x, y, mask_interval=torch.tensor([[[2, 5]]]), top_k=5) == 0


# ---------------------------------------------------------------------------------------------------------------------
# helpers (GPU)
# ---------------------------------------------------------------------------------------------------------------------
def _lm(seed=3, empty_bias=None, eog_bias=2.5, **over):
    """tiny LM whose heads put no mass on non-audio tokens, except codebook 0's end tokens (eos for TTS, eog at eog_bias for
    the spans of an edit) and, with empty_bias, codebook 0's empty_token"""
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny", **over)
    sd = synthetic.make_state_dict(cfg, seed=seed)
    for k in range(cfg.n_codebooks):
        for t in (cfg.empty_token, cfg.eog, cfg.audio_pad_token, cfg.eos):
            if not (k == 0 and t == cfg.eos):
                sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    sd["predict_layer.0.2.bias"][cfg.eog] = eog_bias
    if empty_bias is not None:
        sd["predict_layer.0.2.bias"][cfg.empty_token] = empty_bias
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    return cfg, m.to("cuda:0").eval()


def _codec():
    from oracle import encodec_oracle as eo
    from voicecraft_b200.tokenizer import AudioTokenizer
    cfg = eo.default_config()
    return AudioTokenizer(device="cuda:0", config=cfg, state_dict=eo.make_state_dict(cfg, seed=5))


def _utt(cfg, seed, text_len, frames):
    from voicecraft_b200 import synthetic
    x, xl, y = synthetic.synthetic_utterance(cfg, seed, text_len=text_len, prompt_frames=frames)
    return x.cuda(), xl.cuda(), y.cuda()


EDIT_SPANS = [[(0, 4)], [(3, 6), (6, 10)], [(2, 5), (9, 12), (17, 20)], [(10, 13), (15, 18)]]   # T = 20


def _edit_utts(cfg, seed0):
    return [_utt(cfg, seed0 + i, 6 + i, 20) for i in range(len(EDIT_SPANS))]


def _mi(spans):
    return torch.tensor([spans])


def _poll_ex(m, eng, stream, slots, srcs, froms, mf, bins, codes=None, src_null=False):
    from voicecraft_b200 import _lib
    n, K = len(slots), m.args.n_codebooks
    if codes is None:
        codes = torch.full((max(n, 1), K, max(mf, 1)), -7, dtype=torch.int64, device="cuda")
    status, final, bad = (_lib.vcb_status * max(n, 1))(), (C.c_int32 * max(n, 1))(), (C.c_int32 * max(3 * n, 1))()
    src = None if src_null else (_lib.vcb_edit_source * max(n, 1))(*srcs)
    rc = _lib.load().vcb_poll_frames_ex(eng, (C.c_int32 * max(n, 1))(*slots), n, src, (C.c_int32 * max(n, 1))(*froms), mf,
                                        0, bins, codes.data_ptr(), status, final, bad, stream)
    return rc, codes, status, list(final), list(bad)


def _poll_plain(m, eng, stream, slots, froms, mf, bins):
    from voicecraft_b200 import _lib
    n, K = len(slots), m.args.n_codebooks
    codes = torch.full((n, K, mf), -7, dtype=torch.int64, device="cuda")
    status, final, bad = (_lib.vcb_status * n)(), (C.c_int32 * n)(), (C.c_int32 * (3 * n))()
    rc = _lib.load().vcb_poll_frames(eng, (C.c_int32 * n)(*slots), n, (C.c_int32 * n)(*froms), mf, 0, bins,
                                     codes.data_ptr(), status, final, bad, stream)
    return rc, codes, status, list(final), list(bad)


# ---------------------------------------------------------------------------------------------------------------------
# vcb_poll_frames_ex
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("K", [4, 8])
def test_poll_frames_ex_matches_host_restatement(K):
    from voicecraft_b200 import _lib
    from voicecraft_b200.voicecraft import edit_final_frames, edit_frame_codes
    cfg, m = _lm(n_codebooks=K, empty_bias=3.0)      # an empty token now and then: bad codes are reported too
    m.configure_engine(max_slots=8)
    utts = _edit_utts(cfg, 700)
    tts_utts = [_utt(cfg, 760 + i, 4 + i, 10 + 3 * i) for i in range(2)]
    bins, lib = 2048, _lib.load()
    ed = m.open_edit_session([u[0] for u in utts], [u[2] for u in utts], [_mi(s) for s in EDIT_SPANS],
                             seeds=[5 + i for i in range(len(utts))], top_k=40)
    tts = m.open_tts_session([u[0] for u in tts_utts], [u[2] for u in tts_utts], seeds=[50, 51], top_k=40)
    slots = ed.slots + tts.slots
    srcs = [p.source() for p in ed.prompts] + [p.source() for p in tts.prompts]
    nE = len(ed.slots)
    reported = [0] * len(slots)
    checked = n_bad = after_done = 0
    try:
        ed.sample()
        tts.sample()
        while after_done < 2:
            for _ in range(2):
                ed.step()
                tts.step()
            for mf in (3, 64):                       # 3: smaller than every original piece
                for pick in range(3):
                    froms = [(0, r, r // 2)[pick] for r in reported]
                    rc, codes, status, final, bad = _poll_ex(m, ed.eng, ed.stream, slots, srcs, froms, mf, bins)
                    assert rc == 0, lib.vcb_last_error()
                    ref = (_lib.vcb_status * len(slots))()
                    _lib.check(lib.vcb_poll(ed.eng, (C.c_int32 * len(slots))(*slots), len(slots), ref, ed.stream))
                    for i in range(nE):
                        st, p = ref[i], ed.prompts[i]
                        assert (status[i].done, status[i].n_steps, status[i].n_spans_done, status[i].rng_offset,
                                list(status[i].span_ends)) == (st.done, st.n_steps, st.n_spans_done, st.rng_offset,
                                                               list(st.span_ends))
                        rows = m._read_rows(ed.eng, slots[i], st.n_steps, ed.stream)
                        T, orig = p.y0.shape[1], p.y0.cpu().numpy()
                        f = edit_final_frames(rows, st, p.spans, T, K, cfg.eog)
                        nw = min(f - froms[i], mf)
                        want = np.zeros((K, mf), dtype=np.int64)
                        want[:, :nw] = edit_frame_codes(rows, st, orig, p.spans, K, cfg.eog, froms[i], froms[i] + nw)
                        wbad = [-1, -1, -1]
                        for t in range(nw):
                            ks = [k for k in range(K) if not 0 <= want[k, t] < bins]
                            if ks:
                                wbad = [froms[i] + t, ks[0], int(want[ks[0], t])]
                                break
                        assert final[i] == f, (i, final[i], f)
                        assert np.array_equal(codes[i].cpu().numpy(), want), i
                        assert bad[3 * i:3 * i + 3] == wbad, (i, bad[3 * i:3 * i + 3], wbad)
                        if st.done:
                            assert f == T - sum(e - s for s, e in p.spans) + sum(
                                st.span_ends[j] - (st.span_ends[j - 1] if j else 0) - K for j in range(len(p.spans)))
                        checked += nw > 0
                        n_bad += wbad[0] >= 0
                    # the TTS slots of the same call equal vcb_poll_frames bit for bit
                    rc2, codes2, status2, final2, bad2 = _poll_plain(m, ed.eng, ed.stream, tts.slots, froms[nE:], mf, bins)
                    assert rc2 == 0, lib.vcb_last_error()
                    assert final[nE:] == final2 and bad[3 * nE:] == bad2
                    assert torch.equal(codes[nE:], codes2)
                    for j in range(len(tts.slots)):
                        assert bytes(status[nE + j]) == bytes(status2[j])
                    reported = [max(r, f) for r, f in zip(reported, final)]
            if ed.all_done() and tts.all_done():
                after_done += 1
    finally:
        ed.close()
        tts.close()
    assert checked > 30


@pytest.mark.gpu
def test_poll_frames_ex_error_contract():
    from voicecraft_b200 import _lib
    cfg, m = _lm()
    m.configure_engine(max_slots=8)
    lib = _lib.load()
    u = _edit_utts(cfg, 800)
    ed = m.open_edit_session([u[1][0]], [u[1][2]], [_mi(EDIT_SPANS[1])], seeds=[1])
    tts = m.open_tts_session([u[0][0]], [u[0][2]], seeds=[2])
    grp = m._free_slots(2, 8)
    K = cfg.n_codebooks
    x_ids = u[0][0][0].long().contiguous()
    y_tok = torch.zeros(6, K, dtype=torch.int64, device="cuda")
    P = _lib.vcb_prompt(slot=grp, n_copies=2, mode=0, x_len=int(x_ids.shape[0]), text_ids_dev=x_ids.data_ptr(), y_len=6,
                        y_tokens_dev=y_tok.data_ptr(), mask_rows_dev=None, n_more_spans=0)
    _lib.check(lib.vcb_prefill(ed.eng, C.byref(P), 1, ed.stream))
    eng, stream = ed.eng, ed.stream
    try:
        ed.sample()
        tts.sample()
        for _ in range(10):
            ed.step()
            tts.step()
        good = [ed.prompts[0].source(), tts.prompts[0].source()]
        slots = [ed.slots[0], tts.slots[0]]
        rc, _, _, final, _ = _poll_ex(m, eng, stream, slots, good, [0, 0], 8, 2048)
        assert rc == 0 and final[0] >= 3, lib.vcb_last_error()

        def src_with(**kw):
            s = ed.prompts[0].source()
            for k, v in kw.items():
                if k == "spans":
                    for j, (a, b) in enumerate(v):
                        s.spans[j][0], s.spans[j][1] = a, b
                else:
                    setattr(s, k, v)
            return s
        closed = next(s for s in range(8) if s not in ed.slots + tts.slots + [grp, grp + 1])
        T = ed.prompts[0].y0.shape[1]
        cases = [
            (slots, [_lib.vcb_edit_source(), good[1]], [0, 0], 8),             # an edit slot without a source
            (slots, [src_with(orig_dev=None), good[1]], [0, 0], 8),
            (slots, [src_with(n_spans=1), good[1]], [0, 0], 8),                # n_spans differs from the prompt's
            (slots, [src_with(n_spans=3), good[1]], [0, 0], 8),
            (slots, [src_with(spans=[(6, 10), (3, 6)]), good[1]], [0, 0], 8),  # not ascending
            (slots, [src_with(spans=[(3, 7), (6, 10)]), good[1]], [0, 0], 8),  # overlapping
            (slots, [src_with(spans=[(5, 3), (6, 10)]), good[1]], [0, 0], 8),
            (slots, [src_with(spans=[(3, 6), (6, T + 1)]), good[1]], [0, 0], 8),   # outside [0, T]
            (slots, [src_with(spans=[(-1, 6), (6, 10)]), good[1]], [0, 0], 8),
            (slots, [good[0], good[0]], [0, 0], 8),                            # a TTS slot given a source
            ([ed.slots[0], closed], [good[0], good[1]], [0, 0], 8),            # a slot that is not open
            ([ed.slots[0], grp], [good[0], good[1]], [0, 0], 8),               # a best-of-N member
            ([ed.slots[0], grp + 1], [good[0], good[1]], [0, 0], 8),
            (slots, good, [-1, 0], 8),                                         # from < 0
            (slots, good, [final[0] + 1, 0], 8),                               # from beyond the reported final frames
            (slots, good, [0, 0], 0),                                          # max_frames < 1
            ([], [], [], 8),                                                   # n < 1
        ]
        sentinel = torch.full((2, K, 8), -7, dtype=torch.int64, device="cuda")
        for i, (sl, srcs, froms, mf) in enumerate(cases + [(slots, good, [0, 0], 8)]):
            codes = sentinel.clone()
            rc, codes, _, _, _ = _poll_ex(m, eng, stream, sl, srcs, froms, mf, 2048, codes=codes,
                                          src_null=i == len(cases))               # last: src NULL
            assert rc != 0, i
            assert lib.vcb_last_error()
            torch.cuda.synchronize()
            assert torch.equal(codes, sentinel), i
        rc, _, _, _, _ = _poll_ex(m, eng, stream, slots, good, [final[0], 0], 8, 2048)
        assert rc == 0, lib.vcb_last_error()
    finally:
        lib.vcb_release(eng, grp, 2)
        ed.close()
        tts.close()


# ---------------------------------------------------------------------------------------------------------------------
# vcb_prompt.sampling
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_group_sampling_contract():
    from voicecraft_b200 import _lib
    from voicecraft_b200.voicecraft import _Prompt, _prefill
    cfg, m = _lm()
    m.configure_engine(max_slots=4)
    lib = _lib.load()
    x, _, y = _utt(cfg, 5, 4, 10)
    sess = m.open_tts_session([x], [y], seeds=[3], top_k=40)
    eng, stream = sess.eng, sess.stream
    one = (C.c_int32 * 1)(sess.slots[0])
    sess.sample()
    sess.step()
    before = sess.poll()[0].n_steps
    assert lib.vcb_decode_step(eng, one, 1, None, None, stream) != 0          # no parameters of its own
    assert b"sampling" in lib.vcb_last_error()
    assert lib.vcb_sample(eng, one, 1, None, None, stream) != 0
    assert sess.poll()[0].n_steps == before
    p = _Prompt(m, x, y)
    free = m._free_slots(1, 4)
    held = m._sessions[free] = [free]
    try:
        pages = lib.vcb_counter(eng, b"kv_pages_free")
        for bad in (dict(temperature=0.0), dict(temperature=-1.0), dict(temperature=float("nan")),
                    dict(temperature=float("inf")), dict(top_p=float("nan")), dict(n_silence=9), dict(n_silence=-1)):
            sp = m._sampling(40, 1.0, 1.0, 3, [1388])
            for k, v in bad.items():
                setattr(sp, k, v)
            with pytest.raises(_lib.VcbError):
                _prefill(eng, [(p, free, 1, 7, 0, sp)], stream)
            assert lib.vcb_counter(eng, b"kv_pages_free") == pages, bad
        sp = m._sampling(40, 0.9, 0.8, 3, [1388])
        _prefill(eng, [(p, free, 1, 7, 0, sp)], stream)                       # the slot was left free
        mine = (C.c_int32 * 1)(free)
        _lib.check(lib.vcb_sample(eng, mine, 1, None, None, stream))
        _lib.check(lib.vcb_decode_step(eng, mine, 1, None, None, stream))
        both = (C.c_int32 * 2)(sess.slots[0], free)
        assert lib.vcb_decode_step(eng, both, 2, None, None, stream) != 0     # one listed slot has none
        _lib.check(lib.vcb_decode_step(eng, both, 2, None, C.byref(sess.sp), stream))   # sp given: as before
        lib.vcb_release(eng, free, 1)
        _prefill(eng, [(p, free, 1, 7, 0)], stream)                           # the group id dropped its parameters
        _lib.check(lib.vcb_sample(eng, mine, 1, None, C.byref(sess.sp), stream))
        assert lib.vcb_decode_step(eng, mine, 1, None, None, stream) != 0
    finally:
        m._release_slots(held)
        sess.close()


# ---------------------------------------------------------------------------------------------------------------------
# ContinuousBatcher with edit tickets and per-ticket parameters
# ---------------------------------------------------------------------------------------------------------------------
DEFAULTS = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
PARAMS = [dict(top_k=40, top_p=0.9, temperature=1.0, stop_repetition=3), dict(top_k=-100, top_p=0.8, temperature=0.8),
          dict(top_k=5, temperature=1.3, stop_repetition=-1), dict(), dict(top_k=20, top_p=0.95, stop_repetition=2),
          dict(top_k=1)]


def _queue(cfg, n, seed0, best_of_at=None):
    """n tickets alternating TTS and edit, each with its own parameters: (x, x_lens, y, mask_interval or None, seed,
    best_of, params)"""
    out = []
    for i in range(n):
        if i % 2:
            x, xl, y = _utt(cfg, seed0 + i, 6 + i % 3, 20)
            mi = _mi(EDIT_SPANS[(i // 2) % len(EDIT_SPANS)])
        else:
            x, xl, y = _utt(cfg, seed0 + i, 3 + i % 4, 8 + 3 * (i % 4))
            mi = None
        out.append((x, xl, y, mi, 900 + 13 * i, 3 if i == best_of_at else 1, PARAMS[i % len(PARAMS)]))
    return out


def _single(m, q):
    """the seeded single call of a ticket with its parameters (unset ones: the batcher's DEFAULTS)"""
    x, xl, y, mi, seed, best_of, params = q
    kw = dict(DEFAULTS, **params)
    torch.manual_seed(seed)
    if mi is not None:
        return m.inference(x, xl, y, mi.cuda(), **kw), None
    if best_of > 1:
        return m.inference_tts_batch(x, xl, y, batch_size=best_of, **kw)
    return m.inference_tts(x, xl, y, **kw)


def _submit(cb, q):
    x, _, y, mi, seed, best_of, params = q
    return cb.submit(x, y, seed=seed, best_of=best_of, mask_interval=mi, **params)


def _same(a, b):
    return torch.equal(a[0], b[0]) and (a[1] is None if b[1] is None else torch.equal(a[1], b[1]))


@pytest.mark.gpu
def test_batcher_run_mixed_queue_equals_single_calls():
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, m = _lm()
    queue = _queue(cfg, 12, 1000, best_of_at=4)
    singles = [_single(m, q) for q in queue]
    cb = ContinuousBatcher(m, max_concurrency=5, poll_every=3, **DEFAULTS)
    for q in queue:
        _submit(cb, q)
    results = cb.run()
    assert cb.stats["prefills"] >= 3
    for i, (r, s) in enumerate(zip(results, singles)):
        assert _same(r, s), i
    assert not m._sessions


@pytest.mark.gpu
def test_batcher_stream_mixed_queue():
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, m = _lm()
    tok = _codec()
    queue = _queue(cfg, 11, 1100)
    singles = [_single(m, q) for q in queue]
    cb = ContinuousBatcher(m, max_concurrency=4, poll_every=4, **DEFAULTS)
    for q in queue[:9]:
        _submit(cb, q)
    audio, lasts, after = {}, {}, []
    cancel = 7                                     # an edit ticket, cancelled at its first chunk

    for t, w, last in cb.stream(tok, chunk_frames=6):
        if t == cancel and t in audio:
            after.append(t)
        assert not lasts.get(t), t
        audio.setdefault(t, []).append(w)
        lasts[t] = last
        if t == cancel and len(audio[t]) == 1:
            assert cb.cancel(cancel)
            for q in queue[9:]:                    # submit() from inside the loop: one TTS and one edit ticket
                _submit(cb, q)
    assert queue[cancel][3] is not None and not after and cb.results[cancel] is None
    assert cb.errors == {}
    for i in range(11):
        if i == cancel:
            continue
        assert _same(cb.results[i], singles[i]), i
        assert lasts[i] is True, i
        whole = singles[i][0] if queue[i][3] is not None else singles[i][1]
        assert torch.equal(torch.cat(audio[i], -1), tok.decode_codes(whole)), i
    assert not m._sessions and cb.queue == []


@pytest.mark.gpu
def test_batcher_stream_edit_with_a_non_audio_frame_fails_alone():
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, m = _lm(empty_bias=1.5)
    tok = _codec()
    queue = _queue(cfg, 10, 1200)
    singles = [_single(m, q) for q in queue]
    bad = {i for i, s in enumerate(singles) if bool((s[0] >= tok.config.bins).any())}
    assert any(queue[i][3] is not None for i in bad) and len(bad) < 10, bad
    cb = ContinuousBatcher(m, max_concurrency=4, poll_every=4, **DEFAULTS)
    for q in queue:
        _submit(cb, q)
    audio, lasts = {}, {}
    for t, w, last in cb.stream(tok, chunk_frames=6):
        audio.setdefault(t, []).append(w)
        lasts[t] = last
    assert set(cb.errors) == bad
    for i in range(10):
        assert lasts[i] is True
        if i in bad:
            assert cb.results[i] is None and audio[i][-1] is None and "non-audio token" in cb.errors[i]
        else:
            assert _same(cb.results[i], singles[i]), i
            whole = singles[i][0] if queue[i][3] is not None else singles[i][1]
            assert torch.equal(torch.cat(audio[i], -1), tok.decode_codes(whole)), i
    assert not m._sessions


# ---------------------------------------------------------------------------------------------------------------------
# inference_many_stream / inference_stream
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_edit_streams_equal_whole_calls():
    from voicecraft_b200 import _lib
    cfg, m = _lm()
    tok = _codec()
    utts = _edit_utts(cfg, 1300)
    mis = [_mi(s) for s in EDIT_SPANS]
    kw = dict(top_k=30, top_p=0.9, temperature=1.0)
    seeds = [21 + i for i in range(len(utts))]
    many = m.inference_many([u[0] for u in utts], [u[2] for u in utts], mis, seeds=seeds, **kw)
    st = m.inference_many_stream([u[0] for u in utts], [u[2] for u in utts], mis, tok, chunk_frames=5, poll_every=4,
                                 seeds=seeds, **kw)
    audio = {}
    for i, w in st:
        audio.setdefault(i, []).append(w)
    assert len(st.results) == len(many)
    for i, (a, b) in enumerate(zip(st.results, many)):
        assert torch.equal(a, b), i
        assert torch.equal(torch.cat(audio[i], -1), tok.decode_codes(b)), i
    # the single call: result, audio and the device generator's offset as after inference
    gen = torch.cuda.default_generators[0]
    x, xl, y = _utt(cfg, 1350, 6, 40)
    cs = tok.open_stream(max_streams=1)
    lead = max(10, cs.min_frames)
    cs.close()
    mi = torch.tensor([[[lead + 2, lead + 6]]]).cuda()
    torch.manual_seed(77)
    res = m.inference(x, xl, y, mi, **kw)
    off = gen.get_offset()
    torch.manual_seed(77)
    ss = m.inference_stream(x, xl, y, mi, tok, chunk_frames=10, poll_every=4, **kw)
    wavs = list(ss)
    assert torch.equal(ss.result, res) and gen.get_offset() == off
    assert torch.equal(torch.cat(wavs, -1), tok.decode_codes(res))
    assert ss.first_audio_steps <= 4                 # the leading original piece: at the first poll
    assert wavs[0].shape[-1] >= lead * tok.hop
    # streaming edits need the device generators
    m.noise_fn = lambda shape, device: torch.ones(shape, device=device)
    with pytest.raises(_lib.VcbError):
        m.inference_stream(x, xl, y, mi, tok, **kw)
    m.noise_fn = None
    assert not m._sessions
