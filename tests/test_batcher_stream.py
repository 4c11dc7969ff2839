"""Streaming audio out of ContinuousBatcher (ContinuousBatcher.stream), and the device gather under every streaming loop
(vcb_poll_frames).  CPU: the benchmark's --queue arm fails cleanly without a device.  GPU (-m gpu): the gather against
the host restatement (_read_rows + final_frames + frame_codes), its error contract, and the batcher stream against single
seeded inference_tts calls and whole decodes."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
EMPTY_BIAS_MIXED = 1.5        # an empty token in codebook 0 now and then: some generations hold one, others do not


def test_bench_stream_queue_needs_a_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "bench_stream.py"), "--queue", "4", "--batch", "2",
                        "--repeats", "1"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode != 0
    assert not any(line.strip().startswith("{") for line in r.stdout.splitlines())


# ---------------------------------------------------------------------------------------------------------------------
# helpers (GPU)
# ---------------------------------------------------------------------------------------------------------------------
def _lm(seed=3, empty_bias=None, **over):
    """tiny LM whose heads put no mass on non-audio tokens, except codebook 0's end token (and, with empty_bias, codebook
    0's empty_token at that bias)"""
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny", **over)
    sd = synthetic.make_state_dict(cfg, seed=seed)
    for k in range(cfg.n_codebooks):
        for t in (cfg.empty_token, cfg.eog, cfg.audio_pad_token, cfg.eos):
            if not (k == 0 and t == cfg.eos):
                sd[f"predict_layer.{k}.2.bias"][t] = -1e4
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


def _utts(cfg, n, seed0):
    """utterances of different lengths; number 2 caps its generation at 2 * 10 rows, 14 of them prompt (6 frames)"""
    from voicecraft_b200 import synthetic
    out = []
    for i in range(n):
        tl, pf = (2, 14) if i == 2 else (3 + i % 5, 8 + 4 * (i % 4))
        x, xl, y = synthetic.synthetic_utterance(cfg, seed0 + i, text_len=tl, prompt_frames=pf)
        out.append((x.cuda(), xl.cuda(), y.cuda()))
    return out


def _singles(m, utts, seeds):
    out = []
    for (x, xl, y), s in zip(utts, seeds):
        torch.manual_seed(s)
        out.append(m.inference_tts(x, xl, y, **KW))
    return out


def _poll_frames(sess, slots, froms, max_frames, bins, codes=None):
    from voicecraft_b200 import _lib
    n, K = len(slots), sess.K
    if codes is None:
        codes = torch.full((n, K, max_frames), -7, dtype=torch.int64, device=sess.dev)
    status, final, bad = (_lib.vcb_status * max(n, 1))(), (C.c_int32 * max(n, 1))(), (C.c_int32 * max(3 * n, 1))()
    a = sess.model.args
    rc = _lib.load().vcb_poll_frames(sess.eng, (C.c_int32 * max(n, 1))(*slots), n, (C.c_int32 * max(n, 1))(*froms),
                                     max_frames, int(a.n_special) if a.special_first else 0, bins, codes.data_ptr(),
                                     status, final, bad, sess.stream)
    return rc, codes, status, list(final), list(bad)


def _host_restatement(sess, i, n_steps, frm, max_frames, bins):
    """final frames, codes [K, max_frames] and the first bad code (lowest frame, then codebook) from the token rows"""
    from voicecraft_b200.voicecraft import _end_token, final_frames, frame_codes
    K = sess.K
    rows = sess.model._read_rows(sess.eng, sess.slots[i], n_steps, sess.stream)
    f = final_frames(rows, K, _end_token(sess.model.args))
    nw = min(f - frm, max_frames)
    codes = np.zeros((K, max_frames), dtype=np.int64)
    codes[:, :nw] = frame_codes(rows, K, frm, frm + nw)
    bad = [-1, -1, -1]
    for t in range(nw):
        ks = [k for k in range(K) if not 0 <= codes[k, t] < bins]
        if ks:
            bad = [frm + t, ks[0], int(rows[frm + t + ks[0], ks[0]])]
            break
    return f, codes, bad


# ---------------------------------------------------------------------------------------------------------------------
# vcb_poll_frames
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("K,empty_bias", [(4, None), (8, None), (4, 30.0)])
def test_poll_frames_matches_host_restatement(K, empty_bias):
    from voicecraft_b200 import _lib
    cfg, m = _lm(empty_bias=empty_bias, n_codebooks=K)
    utts = _utts(cfg, 5, 500)
    bins = 2048
    sess = m.open_tts_session([u[0] for u in utts], [u[2] for u in utts], seeds=[11 + i for i in range(5)], **KW)
    lib = _lib.load()
    calls = lib.vcb_counter(sess.eng, b"poll_frames")
    reported = [0] * sess.B
    n_bad, n_checked, after_done = 0, 0, 0
    try:
        sess.sample()
        while after_done < 2:
            for _ in range(3):
                sess.step()
            for mf in (5, 64):
                for pick in range(3):        # from = 0, the last reported final frames, and one in between
                    froms = [(0, r, r // 2)[pick] for r in reported]
                    rc, codes, status, final, bad = _poll_frames(sess, sess.slots, froms, mf, bins)
                    assert rc == 0, lib.vcb_last_error()
                    ref = (_lib.vcb_status * sess.B)()
                    _lib.check(lib.vcb_poll(sess.eng, sess.c_slots, sess.B, ref, sess.stream))
                    for i in range(sess.B):
                        assert (status[i].done, status[i].n_steps, status[i].rng_offset, status[i].keep) == \
                               (ref[i].done, ref[i].n_steps, ref[i].rng_offset, ref[i].keep)
                        f, want, wbad = _host_restatement(sess, i, ref[i].n_steps, froms[i], mf, bins)
                        assert final[i] == f, (i, final[i], f)
                        assert np.array_equal(codes[i].cpu().numpy(), want), i
                        assert bad[3 * i:3 * i + 3] == wbad, (i, bad[3 * i:3 * i + 3], wbad)
                        if ref[i].done:
                            assert f == ref[i].n_steps - K
                        n_bad += wbad[0] >= 0
                        n_checked += min(f - froms[i], mf) > 0
                    reported = [max(r, f) for r, f in zip(reported, final)]
            if sess.all_done():
                after_done += 1
    finally:
        sess.close()
    assert n_checked > 20
    assert (n_bad > 0) == (empty_bias is not None)
    assert lib.vcb_counter(sess.eng, b"poll_frames") > calls


@pytest.mark.gpu
def test_poll_frames_error_contract():
    from voicecraft_b200 import _lib
    cfg, m = _lm()
    m.configure_engine(max_slots=8)
    utts = _utts(cfg, 2, 600)
    lib = _lib.load()
    sess = m.open_tts_session([u[0] for u in utts], [u[2] for u in utts], seeds=[1, 2], **KW)
    edit = m.open_edit_session([utts[0][0]], [utts[0][2]], [torch.tensor([[[2, 5]]])])
    grp = m._free_slots(2, 8)
    K = cfg.n_codebooks
    x_ids = utts[0][0][0].long().contiguous()
    y_tok = torch.zeros(6, K, dtype=torch.int64, device="cuda")
    P = _lib.vcb_prompt(slot=grp, n_copies=2, mode=0, x_len=int(x_ids.shape[0]), text_ids_dev=x_ids.data_ptr(), y_len=6,
                        y_tokens_dev=y_tok.data_ptr(), mask_rows_dev=None, n_more_spans=0)
    _lib.check(lib.vcb_prefill(sess.eng, C.byref(P), 1, sess.stream))
    try:
        sess.sample()
        for _ in range(20):
            sess.step()
        rc, _, _, final, _ = _poll_frames(sess, sess.slots, [0, 0], 8, 2048)
        assert rc == 0 and final[0] > 0
        closed = next(s for s in range(8) if s not in sess.slots + edit.slots + [grp, grp + 1])
        sentinel = torch.full((2, K, 8), -7, dtype=torch.int64, device="cuda")
        for slots, froms, mf in (([sess.slots[0], closed], [0, 0], 8),           # a slot that is not open
                                 ([sess.slots[0], edit.slots[0]], [0, 0], 8),    # an edit slot
                                 ([sess.slots[0], grp], [0, 0], 8),              # a best-of-N member
                                 ([sess.slots[0], grp + 1], [0, 0], 8),
                                 (sess.slots, [0, -1], 8),                       # from < 0
                                 (sess.slots, [final[0] + 1, 0], 8),             # from beyond the final frames
                                 (sess.slots, [0, 0], 0),                        # max_frames < 1
                                 ([], [], 8)):                                   # n < 1
            codes = sentinel.clone()
            rc, codes, _, _, _ = _poll_frames(sess, slots, froms, mf, 2048, codes=codes)
            assert rc != 0, (slots, froms, mf)
            assert lib.vcb_last_error()
            torch.cuda.synchronize()
            assert torch.equal(codes, sentinel)
        rc, _, _, _, _ = _poll_frames(sess, sess.slots, [final[0], 0], 8, 2048)     # from = the reported final frames
        assert rc == 0
    finally:
        lib.vcb_release(sess.eng, grp, 2)
        edit.close()
        sess.close()


# ---------------------------------------------------------------------------------------------------------------------
# ContinuousBatcher.stream
# ---------------------------------------------------------------------------------------------------------------------
def _collect(it, on_chunk=None):
    audio, lasts = {}, {}
    for t, w, last in it:
        assert not lasts.get(t), f"ticket {t}: a chunk after its last"
        audio.setdefault(t, []).append(w)
        lasts[t] = last
        if on_chunk is not None:
            on_chunk(t, w, last)
    return audio, lasts


@pytest.mark.gpu
def test_batcher_stream_equals_single_calls_and_whole_decodes():
    from voicecraft_b200 import _lib
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, m = _lm()
    tok = _codec()
    utts = _utts(cfg, 10, 800)
    seeds = [300 + 7 * i for i in range(10)]
    singles = _singles(m, utts, seeds)
    assert 0 < singles[2][1].shape[-1] < 8                     # shorter than the codec's min_frames: decoded whole
    cb = ContinuousBatcher(m, max_concurrency=4, poll_every=3, **KW)
    for (x, _, y), s in zip(utts, seeds):
        cb.submit(x, y, seed=s)
    eng = m._engine()
    calls = _lib.load().vcb_counter(eng, b"poll_frames")
    audio, lasts = _collect(cb.stream(tok, chunk_frames=10))
    assert cb.stats["prefills"] >= 3 and cb.stats["max_active"] == 4
    assert _lib.load().vcb_counter(eng, b"poll_frames") > calls
    for i in range(10):
        res, gen = cb.results[i]
        assert torch.equal(res, singles[i][0]) and torch.equal(gen, singles[i][1]), i
        assert lasts[i] is True, i
        assert torch.equal(torch.cat(audio[i], -1), tok.decode_codes(gen)), i
    assert len(audio[2]) == 1 and cb.errors == {}
    assert not any(s._open for s in m._sessions)
    assert cb.queue == []                                       # the queue is spent, as after run()


@pytest.mark.gpu
def test_batcher_stream_admission_cancel_and_abandon():
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, m = _lm()
    tok = _codec()
    utts = _utts(cfg, 9, 900)
    seeds = [40 + i for i in range(9)]
    singles = _singles(m, utts, seeds)
    cb = ContinuousBatcher(m, max_concurrency=3, poll_every=4, **KW)
    for (x, _, y), s in zip(utts[:6], seeds[:6]):
        cb.submit(x, y, seed=s)
    seen_after_cancel = []

    def on_chunk(t, w, last):
        if t == 0 and len(cb.queue) == 6:                      # from inside the loop: three more tickets ...
            for (x, _, y), s in zip(utts[6:], seeds[6:]):
                cb.submit(x, y, seed=s)
            assert cb.cancel(1) and cb.cancel(5)                # ... one active and one queued ticket cancelled
        elif t in (1, 5) and len(cb.queue) == 9:
            seen_after_cancel.append(t)
    audio, lasts = _collect(cb.stream(tok, chunk_frames=8), on_chunk)
    assert len(cb.results) == 9 and not seen_after_cancel and 5 not in audio
    assert cb.results[1] is None and cb.results[5] is None
    for i in (0, 2, 3, 4, 6, 7, 8):
        res, gen = cb.results[i]
        assert torch.equal(res, singles[i][0]) and torch.equal(gen, singles[i][1]), i
        assert lasts[i] is True
        assert torch.equal(torch.cat(audio[i], -1), tok.decode_codes(gen)), i
    assert cb.stats["max_active"] == 3
    # abandoning the iteration releases every slot and codec stream
    cb = ContinuousBatcher(m, max_concurrency=3, poll_every=4, **KW)
    for (x, _, y), s in zip(utts[:4], seeds[:4]):
        cb.submit(x, y, seed=s)
    for _ in cb.stream(tok, chunk_frames=8):
        break
    assert not any(s._open for s in m._sessions)
    cb.submit(utts[0][0], utts[0][2], seed=seeds[0])
    it = cb.stream(tok)
    it.close()
    assert not any(s._open for s in m._sessions)
    torch.manual_seed(seeds[3])
    res, gen = m.inference_tts(*utts[3], **KW)
    assert torch.equal(res, singles[3][0]) and torch.equal(gen, singles[3][1])


@pytest.mark.gpu
def test_batcher_stream_rejects_a_submit_that_does_not_fit():
    from voicecraft_b200 import _lib, synthetic
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, m = _lm()
    tok = _codec()
    utts = _utts(cfg, 2, 950)
    m.configure_engine(max_seq_len=256)
    cb = ContinuousBatcher(m, max_concurrency=2, poll_every=4, **KW)
    cb.submit(utts[0][0], utts[0][2], seed=1)
    it = cb.stream(tok)
    x, _, y = synthetic.synthetic_utterance(cfg, 1, text_len=40, prompt_frames=8)   # 40 * 10 rows of cap: 256 is too few
    with pytest.raises(_lib.VcbError):
        cb.submit(x, y, seed=2)
    assert len(cb.queue) == 1
    t = cb.submit(utts[1][0], utts[1][2], seed=2)
    audio, lasts = _collect(it)
    assert t == 1 and lasts == {0: True, 1: True}


@pytest.mark.gpu
def test_batcher_stream_non_audio_frame_fails_only_its_ticket():
    from voicecraft_b200 import _lib
    from voicecraft_b200.voicecraft import ContinuousBatcher
    tok = _codec()
    lib = _lib.load()
    eng = tok._engine()
    # every utterance draws an empty token into codebook 0: each ticket fails, and no code reaches the codec
    cfg, m = _lm(empty_bias=30.0)
    utts = _utts(cfg, 3, 60)
    cb = ContinuousBatcher(m, max_concurrency=2, poll_every=4, **KW)
    for i, (x, _, y) in enumerate(utts):
        cb.submit(x, y, seed=i)
    before = (lib.enc_counter(eng, b"stream_decodes"), lib.enc_counter(eng, b"tc_decodes"))
    got = list(cb.stream(tok, chunk_frames=10))
    assert (lib.enc_counter(eng, b"stream_decodes"), lib.enc_counter(eng, b"tc_decodes")) == before
    assert sorted(got, key=lambda g: g[0]) == [(0, None, True), (1, None, True), (2, None, True)]
    for i in range(3):
        assert cb.results[i] is None and "non-audio token" in cb.errors[i]
    assert not any(s._open for s in m._sessions)
    # an empty token now and then: the tickets whose generation holds one fail, the others are untouched
    cfg, m = _lm(empty_bias=EMPTY_BIAS_MIXED)
    utts = _utts(cfg, 10, 70)
    seeds = [i for i in range(10)]
    singles = _singles(m, utts, seeds)
    bad = {i for i, (_, gen) in enumerate(singles) if bool((gen >= tok.config.bins).any())}
    assert 0 < len(bad) < 10, bad
    cb = ContinuousBatcher(m, max_concurrency=4, poll_every=4, **KW)
    for (x, _, y), s in zip(utts, seeds):
        cb.submit(x, y, seed=s)
    audio, lasts = _collect(cb.stream(tok, chunk_frames=10))
    assert set(cb.errors) == bad
    for i in range(10):
        assert lasts[i] is True
        if i in bad:
            assert cb.results[i] is None and audio[i][-1] is None
            assert all(w is not None for w in audio[i][:-1])
        else:
            res, gen = cb.results[i]
            assert torch.equal(res, singles[i][0]) and torch.equal(gen, singles[i][1]), i
            assert torch.equal(torch.cat(audio[i], -1), tok.decode_codes(gen)), i
    assert not any(s._open for s in m._sessions)

