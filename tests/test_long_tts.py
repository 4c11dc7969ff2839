"""Long TTS: the reference's sentence loop (gradio_app.py run, mode "Long TTS") as one request.  CPU: the chain
bookkeeping (_Chain), the pool admission of a long ticket's next sentence, and submit's validation.  GPU (-m gpu):
VoiceCraft.inference_long_tts against the explicit loop of inference_tts / inference_tts_batch (tokens, log-probabilities
and the device generator's offset), long tickets mixed into ContinuousBatcher.run() and stream() (16 kHz and resampled,
submit / cancel during the iteration, an audio= ticket encoded once), and a KV budget that swaps a chain mid-sentence."""
import pytest
import torch

from voicecraft_b200 import _lib
from voicecraft_b200.voicecraft import ContinuousBatcher, KvPoolPolicy, _Chain, place_groups

KW = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
TEXT_LENS = [5, 2, 8, 3, 6]      # one prompt of 14 frames: the 2-id sentence reaches its length cap (20 rows)
PROMPT_FRAMES = 14


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
class _FakeEngine:
    def __init__(self, free):
        self.free = free

    def free_pages(self):
        return self.free


def test_chain_hands_each_sentence_the_offset_its_predecessor_ended_at():
    c = _Chain(["x0", "x1", "x2"], offset=96)
    c.start(["p0", "p1", "p2"])
    assert c.offset == 96 and c.prompt == "p0"
    assert c.ended("r0", "l0", 480) is True and c.offset == 480 and c.prompt == "p1"
    assert c.ended("r1", "l1", 512) is True and c.offset == 512 and c.prompt == "p2"
    assert c.ended("r2", "l2", 900) is False and c.offset == 900
    assert c.results == ["r0", "r1", "r2"] and c.logprobs == ["l0", "l1", "l2"]
    c.start(["p0", "p1", "p2"])                          # a restart begins at the first offset again
    assert c.offset == 96 and c.results == [] and c.prompt == "p0"


def test_next_sentence_keeps_its_slots_ahead_of_the_queue():
    pol = KvPoolPolicy(_FakeEngine(20), budget=True, max_swapped=4, chunk=4)
    pol.swapped = [(0, "older", None)]                   # something is swapped out: nothing new is admitted ...
    assert pol.admit_count([(4, 1)], 1) == 0
    assert pol.admit_count([(4, 1), (4, 1)], 1, held=True) == 2   # ... but a chain's next sentences go on
    assert pol.admit_count([(30, 1)], 1, held=True) == 0           # one that does not fit waits for pages
    with pytest.raises(_lib.VcbError, match="smaller than one utterance"):
        pol.admit_count([(30, 1)], 0, held=True)
    # its slots stay out of the free set between sentences, so queued tickets cannot take them
    free = {0, 2, 3}                                     # slot 1 is held by a long ticket between two sentences
    new, nxt = place_groups(free, [1, 2, 1], 0)
    assert new == [(0, 0), (2, 1)] and nxt == 2 and free == set()


def _model():
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny")
    return cfg, VoiceCraft(cfg)


def test_submit_validates_long_tickets():
    from voicecraft_b200 import synthetic
    cfg, m = _model()
    x, _, y = synthetic.synthetic_utterance(cfg, 1, text_len=4, prompt_frames=8)
    cb = ContinuousBatcher(m, max_concurrency=4)
    with pytest.raises(ValueError, match="at least one sentence"):
        cb.submit([], y)
    with pytest.raises(ValueError, match="edit ticket"):
        cb.submit([x, x], y, mask_interval=torch.tensor([[[2, 5]]]))
    with pytest.raises(ValueError, match="best_of"):
        cb.submit([x, x], y, best_of=5)
    assert cb.queue == []
    assert cb.submit([x, x], y, seed=3) == 0 and cb.submit(x, y) == 1
    assert isinstance(cb.queue[0][0], _Chain) and cb.queue[0][0].xs[1] is x


def test_cancel_mid_chain_needs_a_running_stream():
    cfg, m = _model()
    with pytest.raises(_lib.VcbError, match="running stream"):
        ContinuousBatcher(m, max_concurrency=2).cancel(0)


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
def _lm(eos_bias=5.0, eog_bias=None, seed=3, **over):
    """tiny LM whose heads put no mass on non-audio tokens except codebook 0's eos (at eos_bias: sentences end early
    now and then) and, with eog_bias, codebook 0's eog (the end of an edit's span)"""
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny", **over)
    sd = synthetic.make_state_dict(cfg, seed=seed)
    for k in range(cfg.n_codebooks):
        for t in (cfg.empty_token, cfg.eog, cfg.audio_pad_token, cfg.eos):
            if not (k == 0 and t == cfg.eos):
                sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    sd["predict_layer.0.2.bias"][cfg.eos] = eos_bias
    if eog_bias is not None:
        sd["predict_layer.0.2.bias"][cfg.eog] = eog_bias
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    return cfg, m.to("cuda:0").eval()


def _codec(encoder=False):
    from oracle import encodec_oracle as eo
    from voicecraft_b200.tokenizer import AudioTokenizer
    cfg = eo.default_config()
    return AudioTokenizer(device="cuda:0", config=cfg, state_dict=eo.make_state_dict(cfg, seed=5, encoder=encoder))


def _long(cfg, seed, lens=TEXT_LENS, frames=PROMPT_FRAMES):
    """sentences xs (lengths `lens`) and one prompt y"""
    from voicecraft_b200 import synthetic
    xs = [synthetic.synthetic_utterance(cfg, seed + i, text_len=n, prompt_frames=1)[0].cuda() for i, n in enumerate(lens)]
    y = synthetic.synthetic_utterance(cfg, seed + 100, text_len=1, prompt_frames=frames)[2].cuda()
    return xs, y


def _loop(m, xs, y, best_of=1, seed=None, **params):
    """the reference's Long TTS loop: one inference_tts (inference_tts_batch) per sentence on one generator"""
    if seed is not None:
        torch.manual_seed(seed)
    out = []
    for x in xs:
        xl = torch.tensor([x.shape[1]], device=x.device)
        if best_of == 1:
            out.append(m.inference_tts(x, xl, y, logprobs=True, **params))
        else:
            out.append(m.inference_tts_batch(x, xl, y, batch_size=best_of, logprobs=True, **params))
    return out


def _same(got, want, lps=None):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g[0], w[0]) and torch.equal(g[1], w[1]), i
        lp = g[2] if lps is None else lps[i]
        assert torch.equal(lp.isnan(), w[2].isnan()) and torch.equal(lp.nan_to_num(), w[2].nan_to_num()), i


def _collect(it, on_chunk=None):
    audio, lasts = {}, {}
    for t, w, last in it:
        assert not lasts.get(t), f"ticket {t}: a chunk after its last"
        audio.setdefault(t, []).append(w)
        lasts[t] = last
        if on_chunk is not None:
            on_chunk(t, w, last)
    return audio, lasts


def _gen():
    return torch.cuda.default_generators[0]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: single calls
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("best_of,params", [(1, dict(top_k=40)), (1, dict(top_p=0.8, temperature=0.9)),
                                            (1, dict(top_k=-100, temperature=1.3, stop_repetition=-1)),
                                            (3, dict(top_k=40, top_p=0.9))])
def test_inference_long_tts_equals_the_loop(best_of, params):
    cfg, m = _lm()
    xs, y = _long(cfg, 40)
    torch.manual_seed(1234)
    torch.rand(7, device="cuda")                          # the generator is mid-stream, not at offset 0
    start = _gen().get_offset()
    want = _loop(m, xs, y, best_of, **params)
    end = _gen().get_offset()
    _gen().set_offset(start)
    got = m.inference_long_tts(xs, y, best_of=best_of, logprobs=True, **params)
    assert _gen().get_offset() == end
    _same(got, want)
    # sentence ends: the 2-id text at its length cap, a longer one by its end token well before
    T, K = PROMPT_FRAMES, cfg.n_codebooks
    rows = [T + 1 + g.shape[-1] + K for _, g, _ in want]
    caps = [n * (cfg.encodec_sr // 5) for n in TEXT_LENS]
    assert rows[1] >= caps[1] - K, (rows, caps)
    assert any(r < c - 2 * K for r, c in zip(rows, caps)), (rows, caps)
    assert len({g.shape[-1] for _, g, _ in want}) > 1
    _gen().set_offset(start)
    plain = m.inference_long_tts(xs, y, best_of=best_of, **params)
    assert all(len(r) == 2 and torch.equal(r[1], w[1]) for r, w in zip(plain, want))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the batcher
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_batcher_run_mixes_long_plain_and_edit_tickets():
    from voicecraft_b200 import synthetic
    cfg, m = _lm(eog_bias=2.5)
    longs = [(_long(cfg, 200 + 10 * i, lens=TEXT_LENS[i:] + TEXT_LENS[:i]), 900 + i, b) for i, b in enumerate((1, 2, 1))]
    others = []
    for i in range(5):
        x, _, y = synthetic.synthetic_utterance(cfg, 300 + i, text_len=3 + i, prompt_frames=20)
        mi = torch.tensor([[(4, 9)]]) if i % 2 else None
        others.append((x.cuda(), y.cuda(), 700 + i, mi))
    loops = [_loop(m, xs, y, b, seed=s, **KW) for (xs, y), s, b in longs]

    def run(with_longs):
        cb = ContinuousBatcher(m, max_concurrency=3, poll_every=3, **KW)
        tickets = {}
        for j, (x, y, s, mi) in enumerate(others):
            if with_longs and j < len(longs):
                (xs, ly), ls, b = longs[j]
                tickets[("long", j)] = cb.submit(xs, ly, seed=ls, best_of=b)
            tickets[("other", j)] = cb.submit(x, y, seed=s, mask_interval=mi)
        return cb, tickets, cb.run()
    _, t0, alone = run(False)
    cb, t1, got = run(True)
    assert cb.stats["max_active"] == 3
    for j in range(len(others)):
        a, g = alone[t0[("other", j)]], got[t1[("other", j)]]
        assert torch.equal(a[0], g[0]) and (a[1] is None) == (g[1] is None), j
    for j, want in enumerate(loops):
        t = t1[("long", j)]
        assert len(got[t]) == len(TEXT_LENS)
        _same([r + (lp,) for r, lp in zip(got[t], cb.logprobs[t])], want)


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [None, 48000])
def test_batcher_stream_long_tickets(rate):
    """chunks of a long ticket, in sentence order, equal the cat of its per-sentence decodes (resampled as one signal);
    submit and cancel inside the loop; plain tickets beside it are untouched"""
    from voicecraft_b200 import synthetic
    cfg, m = _lm()
    tok = _codec()
    (xs0, y0), (xs1, y1), (xs2, y2) = [_long(cfg, 400 + 10 * i) for i in range(3)]
    loops = [_loop(m, xs, y, seed=s, **KW) for (xs, y), s in (((xs0, y0), 50), ((xs1, y1), 51))]
    px, _, py = synthetic.synthetic_utterance(cfg, 480, text_len=6, prompt_frames=10)
    torch.manual_seed(52)
    plain = m.inference_tts(px.cuda(), torch.tensor([6]).cuda(), py.cuda(), **KW)
    cb = ContinuousBatcher(m, max_concurrency=2, poll_every=3, **KW)
    assert cb.submit(xs0, y0, seed=50) == 0
    assert cb.submit(px.cuda(), py.cuda(), seed=52) == 1
    state = {}

    def on_chunk(t, w, last):
        if "late" not in state:
            state["late"] = cb.submit(xs1, y1, seed=51)           # a long ticket submitted from inside the loop
            state["cancel"] = cb.submit(xs2, y2, seed=53)
        elif t == state["cancel"] and "cancelled" not in state:  # its first chunk: cancel the rest of its chain
            assert cb.cancel(t)
            state["cancelled"] = len(audio_seen.get(t, []))
        audio_seen.setdefault(t, []).append(w)
    audio_seen = {}
    it = cb.stream(tok, chunk_frames=6, sample_rate=rate)
    too_long = synthetic.synthetic_utterance(cfg, 1, text_len=200, prompt_frames=1)[0].cuda()
    with pytest.raises(ValueError, match="streaming engine"):
        cb.submit([xs0[0], too_long], y0, seed=1)
    audio, lasts = _collect(it, on_chunk)
    for t, want in ((0, loops[0]), (state["late"], loops[1])):
        assert lasts[t] is True and len(cb.results[t]) == len(TEXT_LENS), t
        _same([r + (lp,) for r, lp in zip(cb.results[t], cb.logprobs[t])], want)
        whole = torch.cat([tok.decode([(g, None)]) for _, g, _ in want], -1)
        if rate is not None:
            whole = tok.resample(whole, tok.sample_rate, rate)
        assert torch.equal(torch.cat(audio[t], -1), whole), t
    assert torch.equal(cb.results[1][1], plain[1]) and lasts[1] is True
    c = state["cancel"]
    assert cb.results[c] is None and len(audio[c]) == state["cancelled"] + 1 and not lasts[c]
    assert cb.errors == {} and m._sessions == {}


@pytest.mark.gpu
def test_long_tts_stream_single_call_and_audio_ticket():
    """inference_long_tts_stream equals inference_long_tts and the decode of its sentences; an audio= long ticket equals
    its encode_many ticket and encodes its prompt once for the whole chain"""
    cfg, m = _lm()
    tok = _codec(encoder=True)
    xs, y = _long(cfg, 600)
    torch.manual_seed(77)
    start = _gen().get_offset()
    want = _loop(m, xs, y, **KW)
    end = _gen().get_offset()
    _gen().set_offset(start)
    it = m.inference_long_tts_stream(xs, y, tok, chunk_frames=6, sample_rate=44100, **KW)
    chunks = list(it)
    assert _gen().get_offset() == end
    _same([r + (lp,) for r, lp in zip(it.results, it.logprobs)], want)
    whole = tok.resample(torch.cat([tok.decode([(g, None)]) for _, g, _ in want], -1), tok.sample_rate, 44100)
    assert torch.equal(torch.cat(chunks, -1), whole)
    # audio= ticket: one encode for the chain, the result of its y = encode_many(...) ticket
    audio = 0.3 * torch.randn(1, 9600, generator=torch.Generator().manual_seed(3))
    yenc = tok.encode_many([audio], 48000)[0].transpose(1, 2)
    calls = []
    real = tok.encode_many

    def counted(wavs, sample_rate=None):
        calls.append(len(wavs))
        return real(wavs, sample_rate)
    tok.encode_many = counted
    try:
        outs = []
        for stream in (False, True):
            for with_audio in (True, False):
                cb = ContinuousBatcher(m, max_concurrency=2, poll_every=3, tokenizer=tok, **KW)
                if with_audio:
                    cb.submit(xs, audio=audio, sample_rate=48000, seed=9)
                else:
                    cb.submit(xs, yenc, seed=9)
                n0 = len(calls)
                if stream:
                    audio_out, lasts = _collect(cb.stream(tok, chunk_frames=6))
                    res = cb.results[0]
                    assert lasts[0] is True
                    gens = torch.cat([tok.decode([(g, None)]) for _, g in res], -1)
                    assert torch.equal(torch.cat(audio_out[0], -1), gens)
                else:
                    res = cb.run()[0]
                assert calls[n0:] == ([1] if with_audio else [])
                outs.append(res)
    finally:
        tok.encode_many = real
    for a, b in ((outs[0], outs[1]), (outs[2], outs[3]), (outs[0], outs[2])):
        assert len(a) == len(b) == len(xs)
        for (ra, ga), (rb, gb) in zip(a, b):
            assert torch.equal(ra, rb) and torch.equal(ga, gb)


@pytest.mark.gpu
def test_long_tickets_under_a_kv_budget_swap_mid_chain():
    cfg, m = _lm(eos_bias=-1e4)                          # every sentence runs to its length cap: long, page-hungry
    m.configure_engine(max_slots=4, max_seq_len=512)
    lens = [30, 18, 26]
    longs = [(_long(cfg, 800 + 10 * i, lens=lens[i:] + lens[:i], frames=20), 60 + i) for i in range(4)]
    loops = [_loop(m, xs, y, seed=s, **KW) for (xs, y), s in longs]
    pb = _lib.load().vcb_counter(m._engine(), b"kv_page_bytes")
    m.configure_engine(kv_pool_gb=(12 + 0.5) * pb / 1e9, max_slots=4, max_seq_len=512)
    assert _lib.load().vcb_counter(m._engine(), b"kv_pages_total") == 12
    cb = ContinuousBatcher(m, max_concurrency=4, poll_every=5, **KW)
    for (xs, y), s in longs:
        cb.submit(xs, y, seed=s)
    got = cb.run()
    assert cb.stats["swap_outs"] > 0 and cb.stats["swap_ins"] == cb.stats["swap_outs"], cb.stats
    for t, want in enumerate(loops):
        _same([r + (lp,) for r, lp in zip(got[t], cb.logprobs[t])], want)
    tok = _codec()
    cb = ContinuousBatcher(m, max_concurrency=4, poll_every=5, **KW)
    for (xs, y), s in longs:
        cb.submit(xs, y, seed=s)
    audio, lasts = _collect(cb.stream(tok, chunk_frames=10))
    assert cb.stats["swap_outs"] > 0
    for t, want in enumerate(loops):
        _same([r + (lp,) for r, lp in zip(cb.results[t], cb.logprobs[t])], want)
        assert lasts[t] and torch.equal(torch.cat(audio[t], -1),
                                        torch.cat([tok.decode([(g, None)]) for _, g, _ in want], -1)), t
    assert _lib.load().vcb_counter(m._engine(), b"kv_pages_free") == 12
