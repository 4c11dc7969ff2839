"""Streaming decode: the codec chunk by chunk with carried state (enc_stream_decode / CodecStream), and streaming TTS
generation (inference_tts_stream / inference_tts_many_stream).  CPU: an fp32 streaming restatement of the decoder against
the whole-sequence oracle, and the final-frame rule.  GPU (-m gpu): concatenated chunks bit-identical to one decode."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import encodec_oracle as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SMALL = {
    "small_causal_reflect": (dict(n_filters=8, dimension=32, bins=64, lstm=2), 1),
    "small_constpad": (dict(n_filters=8, dimension=32, bins=64, lstm=1, pad_mode="constant"), 3),
    "two_res_no_lstm": (dict(n_filters=8, dimension=32, bins=64, lstm=0, n_residual_layers=2), 4),
}
MIN_FRAMES = 8


# ---------------------------------------------------------------------------------------------------------------------
# fp32 streaming restatement of the SEANet decoder: every layer keeps its own left context explicitly
# ---------------------------------------------------------------------------------------------------------------------
class _StreamOracle:
    def __init__(self, cfg, sd):
        if not cfg.causal:
            raise ValueError("a non-causal codec cannot stream: its convolutions read frames that do not exist yet")
        self.cfg, self.sd, self.state = cfg, sd, {}

    def conv(self, name, x, dil):
        """causal Conv1d; state = the last (k-1)*dil input columns"""
        w, b = self.sd[name + ".weight"], self.sd[name + ".bias"]
        pad = (w.shape[-1] - 1) * dil
        prev = self.state.get(name)
        if prev is None:                       # first chunk: the decoder's own padding (reflect or zeros)
            y = eo.conv1d(self.cfg, x, w, b, dil)
            full = x
        else:
            full = torch.cat([prev, x], -1)
            y = F.conv1d(full, w, b, dilation=dil)
        if pad:
            self.state[name] = full[..., full.shape[-1] - pad:]
        return y

    def convtr(self, name, x, r):
        """causal ConvTranspose1d (k = 2r, right trim r); state = the previous input column"""
        w, b = self.sd[name + ".weight"], self.sd[name + ".bias"]
        prev = self.state.get(name, torch.zeros_like(x[..., :1]))
        n = x.shape[-1]
        y = F.conv_transpose1d(torch.cat([prev, x], -1), w, b, stride=r)[..., r:(n + 1) * r]
        self.state[name] = x[..., -1:]
        return y

    def lstm(self, x, name, layers):
        """x [T,B,C]; state = (h, c) per layer"""
        inp = x
        for l in range(layers):
            w_ih, w_hh = self.sd[f"{name}.weight_ih_l{l}"], self.sd[f"{name}.weight_hh_l{l}"]
            b = self.sd[f"{name}.bias_ih_l{l}"] + self.sd[f"{name}.bias_hh_l{l}"]
            h, c = self.state.get(f"{name}.{l}", (torch.zeros(x.shape[1], x.shape[2]), torch.zeros(x.shape[1], x.shape[2])))
            pre = F.linear(inp, w_ih)
            outs = []
            for t in range(x.shape[0]):
                i, f, g_, o = (pre[t] + F.linear(h, w_hh) + b).chunk(4, dim=-1)
                c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g_)
                h = torch.sigmoid(o) * torch.tanh(c)
                outs.append(h)
            self.state[f"{name}.{l}"] = (h, c)
            inp = torch.stack(outs, 0)
        return inp + x

    @torch.no_grad()
    def chunk(self, codes):
        cfg = self.cfg
        z = sum(F.embedding(codes[:, q], self.sd[f"vq.{q}.embed"]) for q in range(codes.shape[1]))
        x = z.transpose(1, 2)
        for L in eo.layer_plan(cfg):
            n = L["name"]
            if L["kind"] == "conv":
                x = self.conv(n, F.elu(x) if L["elu_in"] else x, L["dil"])
            elif L["kind"] == "lstm":
                x = self.lstm(x.permute(2, 0, 1), n, L["layers"]).permute(1, 2, 0)
            elif L["kind"] == "convtr":
                x = self.convtr(n, F.elu(x), L["stride"])
            else:
                h = self.conv(n + ".conv1", F.elu(x), L["dil"])
                h = self.conv(n + ".conv2", F.elu(h), 1)
                s = x if L["true_skip"] else self.conv(n + ".shortcut", x, 1)
                x = s + h
        return x


def decode_stream(cfg, sd, codes, schedule):
    """codes [B,K,T], schedule = frames per call (summing to T) -> the concatenated waveform [B,channels,T*hop]"""
    assert sum(schedule) == codes.shape[-1]
    st = _StreamOracle(cfg, sd)
    out, t = [], 0
    for n in schedule:
        out.append(st.chunk(codes[..., t:t + n]))
        t += n
    return torch.cat(out, -1)


@pytest.mark.parametrize("name", sorted(SMALL))
@pytest.mark.parametrize("schedule", [[MIN_FRAMES, 1, 1, 3, 27], [40], [9, 2, 7, 1, 21]])
def test_stream_oracle_matches_whole_decode(name, schedule):
    over, seed = SMALL[name]
    cfg = eo.default_config(**over)
    sd = eo.make_state_dict(cfg, seed=seed)
    codes = torch.randint(0, cfg.bins, (2, cfg.n_q, 40), generator=torch.Generator().manual_seed(seed))
    whole = eo.decode(cfg, sd, codes)
    got = decode_stream(cfg, sd, codes, schedule)
    assert got.shape == whole.shape
    # fp32 convolutions over different lengths round differently: 1e-5 relative to the waveform's peak (|wav| ~ 3)
    assert (got - whole).abs().max().item() < 1e-5 * whole.abs().max().item()


def test_stream_oracle_rejects_non_causal():
    cfg = eo.default_config(n_filters=8, dimension=32, bins=64, lstm=1, causal=False, true_skip=True)
    sd = eo.make_state_dict(cfg, seed=2)
    with pytest.raises(ValueError):
        decode_stream(cfg, sd, torch.zeros(1, cfg.n_q, 10, dtype=torch.long), [10])


# ---------------------------------------------------------------------------------------------------------------------
# GPU: CodecStream
# ---------------------------------------------------------------------------------------------------------------------
def _tok(cfg, sd):
    from voicecraft_b200.tokenizer import AudioTokenizer
    return AudioTokenizer(device="cuda:0", config=cfg, state_dict=sd)


def _run_schedules(tok, codes, schedules):
    """Push every stream's next chunk, all streams of a round in ONE call (ragged lens, zero padding).  schedules[i] is a
    list of frame counts, None = no push that round.  Returns each stream's concatenated audio."""
    n = len(schedules)
    hop = tok.hop
    pos = [0] * n
    audio = [[] for _ in range(n)]
    with tok.open_stream(max_streams=n + 2) as cs:
        for r in range(max(len(s) for s in schedules)):
            rows = [i for i in range(n) if r < len(schedules[i]) and schedules[i][r]]
            lens = [schedules[i][r] for i in rows]
            T = max(lens)
            batch = torch.zeros(len(rows), codes.shape[1], T, dtype=torch.long, device="cuda")
            for j, i in enumerate(rows):
                batch[j, :, :lens[j]] = codes[i, :, pos[i]:pos[i] + lens[j]]
            ids = [i + 2 for i in rows]                      # stream ids need not equal row numbers
            wav = cs.decode(batch, ids=ids, lens=lens)
            for j, i in enumerate(rows):
                audio[i].append(wav[j, :, :lens[j] * hop])
                pos[i] += lens[j]
    assert all(p == codes.shape[-1] for p in pos)
    return [torch.cat(a, -1) for a in audio]


SCHEDULES = [
    [10, 1, 1, 3, 145],                                     # (the first push of a fresh stream needs min_frames <= 10)
    [160],
    [20, 2, 1, 40, 97],
    [None, 10, 1, 1, 148],                                  # fresh in a call with continuing streams
    [10, 7, 5, 3, 1, 134],
]


@pytest.mark.gpu
def test_codec_stream_bit_identical_real_shape():
    cfg = eo.default_config()
    sd = eo.make_state_dict(cfg, seed=5)
    tok = _tok(cfg, sd)
    codes = torch.randint(0, cfg.bins, (5, cfg.n_q, 160), generator=torch.Generator().manual_seed(11)).cuda()
    whole = tok.decode_codes(codes)
    got = _run_schedules(tok, codes, SCHEDULES)
    for i in range(5):
        assert torch.equal(got[i], whole[i]), f"stream {i}: max |diff| {(got[i] - whole[i]).abs().max().item()}"
    ref = eo.decode(cfg, sd, codes[:1].cpu())[0]
    w = got[0].cpu()
    snr = 10 * torch.log10((ref ** 2).sum() / ((w - ref) ** 2).sum()).item()
    assert snr >= 80.0, snr
    from voicecraft_b200 import _lib
    lib = _lib.load()
    assert lib.enc_counter(tok._engine(), b"stream_decodes") == 6
    assert lib.enc_counter(tok._engine(), b"stream_min_frames") == MIN_FRAMES
    assert lib.enc_counter(tok._engine(), b"stream_state_bytes") == 36352      # 35.5 KB per stream at this codec shape


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small_constpad", "two_res_no_lstm", "ws_chunked", "convout_tc", "lstm_wide"])
def test_codec_stream_bit_identical_variants(name, monkeypatch):
    knobs = {"ws_chunked": ("VCB_CODEC_WS_GB", "0.02"),        # a 20 MB workspace: the batch is decoded one utterance at a time
             "convout_tc": ("VCB_CODEC_CONVOUT_TC", "1"),      # the final conv as one 7-tap GEMM
             "lstm_wide": ("VCB_CODEC_LSTM_WIDE", "1")}        # 128-column LSTM step tiles
    if name in knobs:
        monkeypatch.setenv(*knobs[name])
        cfg, seed = eo.default_config(), 6
    else:
        over, seed = SMALL[name]
        cfg = eo.default_config(**over)
    tok = _tok(cfg, eo.make_state_dict(cfg, seed=seed))
    codes = torch.randint(0, cfg.bins, (5, cfg.n_q, 160), generator=torch.Generator().manual_seed(seed)).cuda()
    whole = tok.decode_codes(codes)
    got = _run_schedules(tok, codes, SCHEDULES)
    for i in range(5):
        assert torch.equal(got[i], whole[i]), f"stream {i}: max |diff| {(got[i] - whole[i]).abs().max().item()}"


@pytest.mark.gpu
def test_codec_stream_errors_leave_state_untouched():
    from voicecraft_b200._lib import VcbError
    cfg = eo.default_config(n_filters=8, dimension=32, bins=64, lstm=2)
    tok = _tok(cfg, eo.make_state_dict(cfg, seed=1))
    codes = torch.randint(0, cfg.bins, (2, cfg.n_q, 30), generator=torch.Generator().manual_seed(4)).cuda()
    whole = tok.decode_codes(codes)
    hop = tok.hop
    with tok.open_stream(max_streams=2) as cs:
        assert cs.min_frames == MIN_FRAMES
        with pytest.raises(VcbError):                          # a fresh stream below min_frames
            cs.decode(codes[:, :, :MIN_FRAMES - 1])
        a = cs.decode(codes[:, :, :10])
        bad = codes[:, :, 10:13].clone()
        bad[1, 2, 1] = cfg.bins
        for call in (lambda: cs.decode(codes[:, :, 10:13], ids=[0, 0]),          # duplicate id
                     lambda: cs.decode(codes[:, :, 10:13], ids=[0, 2]),          # out-of-range id
                     lambda: cs.decode(bad),                                     # out-of-range code
                     lambda: cs.decode(codes[:, :, 10:13], lens=[0, 3])):        # empty push
            with pytest.raises(VcbError):
                call()
        b = cs.decode(codes[:, :, 10:30])
        got = torch.cat([a, b], -1)
        assert torch.equal(got, whole)
        cs.reset([1])                                           # stream 1 starts over
        c = cs.decode(codes[1:, :, :12], ids=[1])
        assert torch.equal(c[0], whole[1, :, :12 * hop])


@pytest.mark.gpu
def test_open_stream_fails_without_the_tensor_core_decoder(monkeypatch):
    from voicecraft_b200._lib import VcbError
    cfg = eo.default_config(n_filters=8, dimension=32, bins=64, lstm=1, causal=False, true_skip=True)
    with pytest.raises(VcbError, match="tensor-core"):
        _tok(cfg, eo.make_state_dict(cfg, seed=2)).open_stream()
    monkeypatch.setenv("VCB_CODEC_TC", "0")
    cfg = eo.default_config(n_filters=8, dimension=32, bins=64, lstm=1)
    with pytest.raises(VcbError, match="VCB_CODEC_TC=0"):
        _tok(cfg, eo.make_state_dict(cfg, seed=2)).open_stream()


# ---------------------------------------------------------------------------------------------------------------------
# which frames are final (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def _delayed_rows(K, G, end, empty, seed):
    """delayed rows [G+K, K] of G audio frames followed by the end cascade (as the sampler writes them)"""
    import numpy as np
    g = np.random.default_rng(seed)
    frames = g.integers(0, 2048, size=(K, G))
    rows = np.full((G + K, K), empty, dtype=np.int64)
    for t in range(G):
        for k in range(K):
            rows[t + k, k] = frames[k, t]
    for j in range(K):
        rows[G + j, j] = end
    return rows


@pytest.mark.parametrize("K", [1, 4, 8])
def test_final_frames_are_a_prefix_of_undelay(K):
    import numpy as np
    from voicecraft_b200.voicecraft import VoiceCraft, final_frames, frame_codes
    end, empty = 2051, 2048
    for G in (0, 1, 5, 30):
        rows = _delayed_rows(K, G, end, empty, seed=G + 10 * K)
        full = VoiceCraft._undelay(rows, K)
        assert full.shape == (K, G)
        prev = 0
        for p in range(rows.shape[0] + 1):
            f = final_frames(rows[:p], K, end)
            assert prev <= f <= G                               # frames only become final, never at / after the end
            assert np.array_equal(frame_codes(rows[:p], K, 0, f), full[:, :f])
            prev = f
        assert final_frames(rows, K, end) == G


def test_bench_stream_needs_a_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "bench_stream.py"), "--repeats", "1"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode != 0
    assert not any(line.strip().startswith("{") for line in r.stdout.splitlines())


# ---------------------------------------------------------------------------------------------------------------------
# GPU: streaming generation
# ---------------------------------------------------------------------------------------------------------------------
def _lm(seed=3, favour_empty=False):
    """tiny LM whose heads put no mass on non-audio tokens, except codebook 0's end token (and, with favour_empty, a
    codebook 0 that prefers empty_token)"""
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=seed)
    for k in range(cfg.n_codebooks):
        for t in (cfg.empty_token, cfg.eog, cfg.audio_pad_token, cfg.eos):
            if not (k == 0 and t == cfg.eos):
                sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    if favour_empty:
        sd["predict_layer.0.2.bias"][cfg.empty_token] = 30.0
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    return cfg, m.to("cuda:0").eval()


def _real_codec():
    cfg = eo.default_config()
    return _tok(cfg, eo.make_state_dict(cfg, seed=5))


@pytest.mark.gpu
def test_inference_tts_stream_matches_inference_tts():
    from voicecraft_b200 import synthetic
    cfg, m = _lm()
    tok = _real_codec()
    x, xl, y = synthetic.synthetic_utterance(cfg, 21, text_len=12, prompt_frames=20)
    x, y = x.cuda(), y.cuda()
    gen_dev = torch.cuda.default_generators[0]
    torch.manual_seed(7)
    res, gen = m.inference_tts(x, xl, y, top_k=40)
    off = gen_dev.get_offset()
    torch.manual_seed(7)
    ts = m.inference_tts_stream(x, xl, y, tok, chunk_frames=10, poll_every=4, top_k=40)
    chunks = list(ts)
    assert len(chunks) > 1
    G = gen.shape[-1]
    assert ts.first_audio_steps < G + cfg.n_codebooks            # audio before the last token was sampled
    assert torch.equal(ts.result[0], res) and torch.equal(ts.result[1], gen)
    assert gen_dev.get_offset() == off
    audio = torch.cat(chunks, -1)
    assert torch.equal(audio, tok.decode([(gen, None)]))
    # abandoning the iteration releases the slots: the model keeps working
    torch.manual_seed(7)
    ts = m.inference_tts_stream(x, xl, y, tok, chunk_frames=10, poll_every=4, top_k=40)
    for _ in ts:
        break
    del ts
    torch.manual_seed(7)
    ts = m.inference_tts_stream(x, xl, y, tok, chunk_frames=10, poll_every=4, top_k=40)
    next(iter(ts))
    ts.close()
    torch.manual_seed(7)
    res2, gen2 = m.inference_tts(x, xl, y, top_k=40)
    assert torch.equal(res2, res) and torch.equal(gen2, gen)
    assert not any(s._open for s in m._sessions)


@pytest.mark.gpu
def test_inference_tts_many_stream_matches_many():
    from voicecraft_b200 import synthetic
    cfg, m = _lm()
    tok = _real_codec()
    xs, ys = [], []
    for i in range(6):
        # utterance 2: text of 2 ids caps the generation at 2 * 10 audio rows, 14 of them prompt -> 6 frames (< min_frames)
        x, _, y = synthetic.synthetic_utterance(cfg, 40 + i, text_len=2 if i == 2 else 8, prompt_frames=14 if i == 2 else 16)
        xs.append(x.cuda())
        ys.append(y.cuda())
    seeds = [100 + i for i in range(6)]
    ref = m.inference_tts_many(xs, ys, seeds=seeds, top_k=40)
    ts = m.inference_tts_many_stream(xs, ys, tok, chunk_frames=10, poll_every=4, seeds=seeds, top_k=40)
    audio = {i: [] for i in range(6)}
    for i, w in ts:
        audio[i].append(w)
    assert 0 < ref[2][1].shape[-1] < 8
    for i in range(6):
        assert torch.equal(ts.results[i][0], ref[i][0]) and torch.equal(ts.results[i][1], ref[i][1]), i
        assert torch.equal(torch.cat(audio[i], -1), tok.decode_codes(ref[i][1])), i


@pytest.mark.gpu
def test_non_audio_final_frame_raises_before_the_codec():
    from voicecraft_b200 import _lib, synthetic
    cfg, m = _lm(favour_empty=True)
    tok = _real_codec()
    xs, ys = [], []
    for i in range(2):
        x, _, y = synthetic.synthetic_utterance(cfg, 60 + i, text_len=8, prompt_frames=16)
        xs.append(x.cuda())
        ys.append(y.cuda())
    lib = _lib.load()
    eng = tok._engine()
    before = (lib.enc_counter(eng, b"stream_decodes"), lib.enc_counter(eng, b"tc_decodes"))
    with pytest.raises(_lib.VcbError, match="utterance .*frame .*non-audio"):
        for _ in m.inference_tts_many_stream(xs, ys, tok, chunk_frames=10, poll_every=4, seeds=[1, 2], top_k=40):
            pass
    assert (lib.enc_counter(eng, b"stream_decodes"), lib.enc_counter(eng, b"tc_decodes")) == before
    assert not any(s._open for s in m._sessions)
