"""Resampling (torchaudio's Resample with its defaults) for prompt audio in and streamed audio out.

CPU: the package's filter tables against the SHA-256 of torchaudio's (tests/golden/resample.json), the fp64 oracle
against the reference's convert_audio output (tests/golden/resample.npz), the streaming rule, and the WAV reader.
GPU (-m gpu): enc_resample against the fixtures, enc_resampler_push bit-identical to one-shot, the streams with
sample_rate=, tokenize_audio at any rate and the resampler's lifetime."""
import gc
import hashlib
import json
import os
import struct

import numpy as np
import pytest
import torch

from oracle import resample_oracle as ro

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EPS = 2.0 ** -24


def _meta():
    with open(os.path.join(GOLDEN, "resample.json")) as f:
        return json.load(f)["pairs"]


def _fixture():
    return np.load(os.path.join(GOLDEN, "resample.npz"))


PAIRS = [(p["orig"], p["new"]) for p in _meta()]


def _mono(x):
    """convert_audio's down-mix to the codec's one channel: mean(0, keepdim=True) in fp32"""
    return torch.from_numpy(x).mean(0, keepdim=True).numpy()


# ---------------------------------------------------------------------------------------------------------------------
# CPU: tables, oracle, streaming rule
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pair", _meta(), ids=lambda p: f"{p['orig']}-{p['new']}")
def test_table_is_bit_equal_to_torchaudio(pair):
    from voicecraft_b200.tokenizer import resample_dims, resample_table
    t = resample_table(pair["orig"], pair["new"])
    assert resample_dims(pair["orig"], pair["new"]) == (pair["o"], pair["n"], pair["w"], pair["taps"])
    assert t.dtype == torch.float32 and tuple(t.shape) == (pair["n"], pair["taps"])
    assert hashlib.sha256(t.numpy().tobytes()).hexdigest() == pair["table_sha256"]
    # the oracle's numpy table: the same to the last bit of fp32 or one unit of it
    k = ro.table(pair["orig"], pair["new"])
    assert np.all(np.abs(k.astype(np.float64) - t.numpy()) <= np.spacing(np.abs(t.numpy())))


def test_rate_checks():
    from voicecraft_b200.tokenizer import resample_dims
    for bad in ((0, 16000), (16000, -1)):
        with pytest.raises(ValueError, match="positive"):
            resample_dims(*bad)
    with pytest.raises(ValueError, match="cap"):
        resample_dims(16000, 44099)                     # 44099 phases x 16014 taps: 2.8 GB


@pytest.mark.parametrize("orig,new", PAIRS)
def test_oracle_matches_convert_audio(orig, new):
    """per sample within 32 * 2^-24 * sum |K||x| (torchaudio's fp32 CPU output sits within 7.5 of those units)"""
    g = _fixture()
    for case in ("stereo", "mono", "short"):
        key = f"{orig}_{new}_{case}"
        x, y = g[key + "_x"], g[key + "_y"]
        ref, bound = ro.resample(_mono(x)[0], orig, new)
        assert y.shape == (1, ro.out_length(x.shape[1], orig, new)) == (1, ref.shape[0])
        err = np.abs(y[0].astype(np.float64) - ref)
        assert np.all(err <= 32 * EPS * bound + 1e-30), (key, float((err / (EPS * bound + 1e-30)).max()))


def _schedules(L, o, w, rng):
    """push schedules of L samples: ones, runs shorter than w + o, zeros, random, and all-but-a-flush"""
    short = max(1, (w + o) // 3)
    out = [[1] * L, [short] * (L // short) + [L % short], [L], [L, 0], [0, L], [], ]
    for _ in range(3):
        s, left = [], L
        while left > 0:
            k = int(rng.choice([0, 1, 2, short, w + o - 1, w + o, 3 * o + 1, left]))
            k = min(k, left)
            s.append(k)
            left -= k
        out.append(s)
    return [s for s in out if sum(s) == L]


@pytest.mark.parametrize("orig,new", [(44100, 16000), (16000, 48000), (16000, 44100), (48000, 16000), (8000, 16000)])
def test_stream_oracle_concatenates_to_the_whole(orig, new):
    rng = np.random.default_rng(orig + new)
    o, n, w = ro.dims(orig, new)
    for L in (0, 1, w - 1, w + o, 5 * o + 3, 1000):
        x = rng.standard_normal(L)
        whole, _ = ro.resample(x, orig, new)
        for sched in _schedules(L, o, w, rng):
            st, got, pos = ro.Stream(orig, new), [], 0
            for k in sched:
                got.append(st.push(x[pos:pos + k]))
                pos += k
            got.append(st.push(x[:0], final=True))          # flush with no new input
            y = np.concatenate(got)
            assert y.shape[0] == ro.out_length(L, orig, new)
            assert np.array_equal(y, whole), (L, sched)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the WAV reader
# ---------------------------------------------------------------------------------------------------------------------
def _wav(path, data: bytes, tag, ch, sr, bits, extensible=False, extra_chunk=True):
    block = ch * bits // 8
    if extensible:
        guid_tail = b"\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71"
        fmt = struct.pack("<HHIIHHHHIH", 0xFFFE, ch, sr, sr * block, block, bits, 22, bits, 3, tag) + guid_tail
    else:
        fmt = struct.pack("<HHIIHH", tag, ch, sr, sr * block, block, bits)
    body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt
    if extra_chunk:                                    # a chunk the reader must skip, odd-sized (padded)
        body += b"LIST" + struct.pack("<I", 3) + b"abc\x00"
    body += b"data" + struct.pack("<I", len(data)) + data
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", len(body)) + body)


def _samples(rng, ch, n, bits):
    if bits == "f32":
        return rng.uniform(-1, 1, (n, ch)).astype("<f4")
    lim = {16: 2 ** 15, 24: 2 ** 23, 32: 2 ** 31}[bits]
    return rng.integers(-lim, lim, (n, ch), dtype=np.int64)


def _encode(v, bits):
    if bits == "f32":
        return v.astype("<f4").tobytes()
    if bits == 24:
        u = (v.reshape(-1) & 0xFFFFFF).astype("<u4")
        return np.stack([u & 0xFF, (u >> 8) & 0xFF, (u >> 16) & 0xFF], 1).astype(np.uint8).tobytes()
    return v.astype({16: "<i2", 32: "<i4"}[bits]).tobytes()


@pytest.mark.parametrize("bits", [16, 24, 32, "f32"])
@pytest.mark.parametrize("ch", [1, 2])
@pytest.mark.parametrize("extensible", [False, True])
def test_read_wav_formats(tmp_path, bits, ch, extensible):
    from voicecraft_b200.tokenizer import audio_info, read_wav
    rng = np.random.default_rng(ch * 10 + (0 if bits == "f32" else bits))
    v = _samples(rng, ch, 1001, bits)
    p = tmp_path / "a.wav"
    _wav(p, _encode(v, bits), 3 if bits == "f32" else 1, ch, 44100, 32 if bits == "f32" else bits, extensible)
    x, sr = read_wav(p)
    assert sr == 44100 and x.dtype == np.float32 and x.shape == (ch, 1001)
    want = v.T.astype(np.float32) if bits == "f32" else v.T.astype(np.float32) / np.float32(2.0 ** ({16: 15, 24: 23, 32: 31}[bits]))
    assert np.array_equal(x, want)
    assert audio_info(p) == (44100, 1001, ch) and audio_info(p).num_frames == 1001
    w, _ = read_wav(p, offset=990, num_frames=50)        # a window at the file's rate, clipped at its end
    assert np.array_equal(w, want[:, 990:])
    w, _ = read_wav(p, offset=5, num_frames=-1)          # like the reference: both or neither
    assert w.shape == (ch, 1001)


def test_read_wav_pcm16_is_todays_division(tmp_path):
    from voicecraft_b200.tokenizer import read_wav
    v = np.array([[-32768, 32767, 1, -1, 0]], dtype=np.int64).T
    p = tmp_path / "b.wav"
    _wav(p, _encode(v, 16), 1, 1, 16000, 16, extra_chunk=False)
    x, _ = read_wav(p)
    assert np.array_equal(x, v.astype("<i2").reshape(-1, 1).T.astype(np.float32) / 32768.0)


@pytest.mark.parametrize("tag,bits,match", [(1, 8, "PCM with 8 bits"), (3, 64, "IEEE float with 64 bits"),
                                            (6, 8, "format tag 0x6"), (0x55, 16, "format tag 0x55")])
def test_read_wav_refuses_other_formats(tmp_path, tag, bits, match):
    from voicecraft_b200.tokenizer import audio_info, read_wav
    p = tmp_path / "c.wav"
    _wav(p, bytes(64), tag, 1, 8000, bits)
    for fn in (read_wav, audio_info):
        with pytest.raises(ValueError, match=match):
            fn(p)
    q = tmp_path / "d.wav"
    q.write_bytes(b"RIFX" + bytes(40))
    with pytest.raises(ValueError, match="not a RIFF/WAVE"):
        read_wav(q)


def test_tokenize_audio_refuses_more_than_two_channels(tmp_path):
    from voicecraft_b200.tokenizer import AudioTokenizer, default_codec_config, tokenize_audio
    p = tmp_path / "e.wav"
    _wav(p, bytes(3 * 2 * 10), 1, 3, 16000, 16)
    tok = AudioTokenizer(device="cpu", config=default_codec_config(), state_dict={})
    with pytest.raises(ValueError, match="mono or stereo"):
        tokenize_audio(tok, str(p))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the kernel
# ---------------------------------------------------------------------------------------------------------------------
def _rs(orig, new, streams=0):
    from voicecraft_b200.tokenizer import Resampler
    return Resampler(orig, new, streams, "cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("orig,new", PAIRS)
def test_enc_resample_matches_fixtures(orig, new):
    """within 64 * 2^-24 * sum |K||x| of the reference's output (both sides round); exact lengths; a ragged batch gives
    each row what it gives alone, bit for bit"""
    g = _fixture()
    rs = _rs(orig, new)
    rows, alone = [], []
    for case in ("stereo", "mono", "short"):
        key = f"{orig}_{new}_{case}"
        x, y = _mono(g[key + "_x"]), g[key + "_y"]
        xd = torch.from_numpy(x).cuda()
        got, lens = rs(xd)
        assert lens == [y.shape[1]] and tuple(got.shape) == y.shape
        _, bound = ro.resample(x[0], orig, new)
        err = np.abs(got.cpu().numpy()[0].astype(np.float64) - y[0])
        assert np.all(err <= 64 * EPS * bound + 1e-30), (key, float((err / (EPS * bound + 1e-30)).max()))
        rows.append(x[0])
        alone.append(got[0])
    T = max(r.shape[0] for r in rows) + 5
    batch = torch.full((len(rows), T), float("nan"), device="cuda")         # padding must never be read
    for i, r in enumerate(rows):
        batch[i, :r.shape[0]] = torch.from_numpy(r)
    got, lens = rs(batch, [r.shape[0] for r in rows])
    for i, a in enumerate(alone):
        assert lens[i] == a.shape[0] and torch.equal(got[i, :lens[i]], a), i
    rs.close()


def _push_all(rs, rows, schedules, ids=None):
    """push rows[i] (1-D device tensors) by schedules[i] (sample counts; a trailing flush with no input), all streams of
    a round in one call -> each stream's concatenated output"""
    n = len(rows)
    ids = list(range(n)) if ids is None else ids
    pos, tot, out = [0] * n, [0] * n, [[] for _ in range(n)]
    rounds = max(len(s) for s in schedules) + 1
    for r in range(rounds):
        live = [i for i in range(n) if r <= len(schedules[i])]
        if not live:
            break
        lens = [schedules[i][r] if r < len(schedules[i]) else 0 for i in live]
        fin = [r == len(schedules[i]) for i in live]
        T = max(lens + [1])
        x = torch.full((len(live), T), float("nan"), device="cuda")
        for b, i in enumerate(live):
            x[b, :lens[b]] = rows[i][pos[i]:pos[i] + lens[b]]
            pos[i] += lens[b]
        y, olens = rs.push(x, [ids[i] for i in live], lens, fin)
        for b, i in enumerate(live):                # exactly the outputs whose window is complete, the tail at the end
            tot[i] += olens[b]
            L = pos[i]
            assert tot[i] == (ro.out_length(L, rs.orig_sr, rs.new_sr) if fin[b] else ro.Stream(rs.orig_sr, rs.new_sr).ready(L))
            out[i].append(y[b, :olens[b]].clone())
    return [torch.cat(o) for o in out]


@pytest.mark.gpu
@pytest.mark.parametrize("orig,new", [(44100, 16000), (16000, 48000), (16000, 44100), (16000, 24000), (48000, 16000),
                                      (22050, 16000)])
def test_push_is_bit_identical_to_one_shot(orig, new):
    rng = np.random.default_rng(7)
    o, n, w = ro.dims(orig, new)
    rs1, rs = _rs(orig, new), _rs(orig, new, 12)
    lengths = [0, 1, w - 1, w + o, 5 * o + 3, 4000, 9000]
    rows, scheds = [], []
    for L in lengths:
        x = torch.from_numpy(rng.uniform(-1, 1, L).astype(np.float32)).cuda()
        for s in _schedules(L, o, w, rng)[:4]:
            rows.append(x)
            scheds.append(s)
    ids = list(range(len(rows)))
    for k in range(0, len(rows), 12):
        got = _push_all(rs, rows[k:k + 12], scheds[k:k + 12], ids=list(range(min(12, len(rows) - k))))
        rs.reset(range(12))
        for j, g in enumerate(got):
            whole, lens = rs1(rows[k + j][None])
            assert g.shape[0] == lens[0] == ro.out_length(rows[k + j].numel(), orig, new), (k + j, scheds[k + j])
            assert torch.equal(g, whole[0, :lens[0]]), (ids[k + j], scheds[k + j])
    rs.close()
    rs1.close()


@pytest.mark.gpu
def test_push_errors_leave_streams_untouched():
    from voicecraft_b200 import _lib
    rs1, rs = _rs(44100, 16000), _rs(44100, 16000, 2)
    x = torch.from_numpy(np.random.default_rng(3).uniform(-1, 1, (2, 3000)).astype(np.float32)).cuda()
    a, la = rs.push(x[:, :1000], [0, 1], [1000, 1000])                         # a strided view: copied to rows
    for call in (lambda: rs.push(x[:, 1000:1500], [0, 0], [500, 500]),          # an id twice
                 lambda: rs.push(x[:, 1000:1500], [0, 2], [500, 500]),          # an id outside [0, 2)
                 lambda: rs.push(x[:, 1000:1500], [0, 1], [-1, 500]),           # a negative length
                 lambda: rs.push(x[:, 1000:1500], [0, 1], [501, 500])):         # longer than the input
        with pytest.raises(_lib.VcbError):
            call()
    b, lb = rs.push(x[:, 1000:3000].contiguous(), [0, 1], [2000, 2000], [True, True])
    whole, lw = rs1(x)
    for i in range(2):
        assert torch.equal(torch.cat([a[i, :la[i]], b[i, :lb[i]]]), whole[i])
    with pytest.raises(_lib.VcbError, match="final"):                          # finished: reset first
        rs.push(x[:, :10].contiguous(), [0], [10])
    rs.reset([0])
    c, lc = rs.push(x[:1], [0], [3000], [True])
    assert torch.equal(c[0, :lc[0]], whole[0])
    import ctypes as C
    lib = _lib.load()                                                          # the output capacity is checked
    out_lens = (C.c_int32 * 1)()
    y = torch.empty(1, 4, device="cuda")
    assert lib.enc_resample(rs1._h, x.data_ptr(), (C.c_int32 * 1)(3000), 1, 3000, y.data_ptr(), 4, out_lens, None) != 0
    assert b"output holds 4" in lib.vcb_last_error()
    rs.close()
    rs1.close()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: AudioTokenizer.resample, tokenize_audio
# ---------------------------------------------------------------------------------------------------------------------
def _codec():
    from oracle import encodec_oracle as eo
    from voicecraft_b200.tokenizer import AudioTokenizer
    cfg = eo.default_config()
    return AudioTokenizer(device="cuda:0", config=cfg, state_dict=eo.make_state_dict(cfg, seed=5, encoder=True))


@pytest.mark.gpu
def test_tokenizer_resample_shapes_and_same_rate():
    from voicecraft_b200 import _lib
    tok = _codec()
    lib = _lib.load()
    x = torch.randn(3, 1, 4410, device="cuda")
    n0 = lib.enc_counter(None, b"resample_launches")
    assert tok.resample(x, 16000) is x
    assert tok.resample(x, 48000, 48000) is x
    assert lib.enc_counter(None, b"resample_launches") == n0                   # same rate: no launch
    y = tok.resample(x, 44100)
    assert tuple(y.shape) == (3, 1, 1600)
    z = tok.resample(x, 44100, lens=[4410, 441, 0])
    assert torch.equal(z[0], y[0]) and torch.equal(z[1, :, :160], tok.resample(x[1:2, :, :441], 44100)[0])
    assert not z[1, :, 160:].any() and not z[2].any()


@pytest.mark.gpu
def test_tokenize_audio_any_rate(tmp_path):
    from voicecraft_b200 import _lib
    from voicecraft_b200.tokenizer import tokenize_audio
    tok = _codec()
    lib = _lib.load()
    rng = np.random.default_rng(11)
    # float32 stereo at 44.1 kHz
    v = (0.5 * rng.uniform(-1, 1, (22050, 2))).astype("<f4")
    p = tmp_path / "f.wav"
    _wav(p, v.tobytes(), 3, 2, 44100, 32, extensible=True)
    codes = tokenize_audio(tok, str(p))[0][0]
    mono = torch.from_numpy(v.T.copy()).mean(0, keepdim=True)[None].cuda()
    assert torch.equal(codes, tok.encode_codes(tok.resample(mono, 44100)))
    # 24-bit mono at 48 kHz, a window at the file's rate
    iv = rng.integers(-2 ** 22, 2 ** 22, (24000, 1))
    p = tmp_path / "g.wav"
    _wav(p, _encode(iv, 24), 1, 1, 48000, 24)
    codes = tokenize_audio(tok, str(p), offset=4800, num_frames=9600)[0][0]
    x = torch.from_numpy((iv[4800:14400].T.astype(np.float32) / np.float32(2 ** 23)))[None].cuda()
    assert torch.equal(codes, tok.encode_codes(tok.resample(x, 48000)))
    # at the codec's rate: no resampling launch
    n0 = lib.enc_counter(None, b"resample_launches")
    f = (0.3 * rng.uniform(-1, 1, (8000, 1))).astype("<f4")
    p = tmp_path / "h.wav"
    _wav(p, f.tobytes(), 3, 1, 16000, 32)
    assert torch.equal(tokenize_audio(tok, str(p))[0][0], tok.encode_codes(torch.from_numpy(f.T.copy())[None].cuda()))
    s = rng.integers(-2 ** 15, 2 ** 15, (8000, 1))
    p = tmp_path / "i.wav"
    _wav(p, _encode(s, 16), 1, 1, 16000, 16, extra_chunk=False)
    x = torch.from_numpy(s.astype("<i2").reshape(-1, 1).T.astype(np.float32) / 32768.0)[None]
    assert torch.equal(tokenize_audio(tok, str(p))[0][0], tok.encode_codes(x))
    assert lib.enc_counter(None, b"resample_launches") == n0


# ---------------------------------------------------------------------------------------------------------------------
# GPU: CodecStream and the generation streams with sample_rate=
# ---------------------------------------------------------------------------------------------------------------------
RATES = [48000, 44100, 24000]


@pytest.mark.gpu
@pytest.mark.parametrize("sr", RATES)
def test_codec_stream_resampled_is_bit_identical(sr):
    tok = _codec()
    cfg = tok.config
    codes = torch.randint(0, cfg.bins, (3, cfg.n_q, 60), generator=torch.Generator().manual_seed(sr)).cuda()
    whole = tok.resample(tok.decode_codes(codes), 16000, sr)
    with tok.open_stream(max_streams=3, sample_rate=sr) as cs:
        assert cs.sample_rate == sr
        m = cs.min_frames
        out = [[], [], []]
        w = cs.decode(codes[:, :, :m])
        for b in range(3):
            out[b].append(w[b, :, :cs.out_lens[b]])
        w = cs.decode(codes[[0, 2], :, m:m + 5], ids=[0, 2], final=[True, False])     # stream 0 ends with its push
        for b, i in enumerate([0, 2]):
            out[i].append(w[b, :, :cs.out_lens[b]])
        batch = torch.zeros(2, cfg.n_q, 60 - m, dtype=torch.long, device="cuda")      # ragged: zero padding
        batch[0] = codes[1, :, m:]
        batch[1, :, :5] = codes[2, :, m + 5:m + 10]
        w = cs.decode(batch, ids=[1, 2], lens=[60 - m, 5])
        for b, i in enumerate([1, 2]):
            out[i].append(w[b, :, :cs.out_lens[b]])
        w = cs.flush([1])                                                           # stream 1 ends with no new frame
        out[1].append(w[0, :, :cs.out_lens[0]])
        w = cs.decode(codes[2:, :, m + 10:], ids=[2], final=[True])
        out[2].append(w[0, :, :cs.out_lens[0]])
        got = [torch.cat(o, -1) for o in out]
        assert torch.equal(got[0], tok.resample(tok.decode_codes(codes[:1, :, :m + 5]), 16000, sr)[0])
        assert torch.equal(got[1], whole[1]) and torch.equal(got[2], whole[2])
        cs.reset([0])                                                               # both states start over
        w = cs.decode(codes[:1], ids=[0], final=[True])
        assert torch.equal(w[0, :, :cs.out_lens[0]], whole[0])


def _lm(seed=3, empty_bias=None):
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny")
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


def _utts(cfg, n, seed0):
    """utterance 2 caps its generation at 2 * 10 rows, 14 of them prompt: fewer frames than min_frames"""
    from voicecraft_b200 import synthetic
    out = []
    for i in range(n):
        tl, pf = (2, 14) if i == 2 else (3 + i % 5, 8 + 4 * (i % 4))
        x, xl, y = synthetic.synthetic_utterance(cfg, seed0 + i, text_len=tl, prompt_frames=pf)
        out.append((x.cuda(), xl.cuda(), y.cuda()))
    return out


@pytest.fixture
def flushes(monkeypatch):
    """counts CodecStream.flush calls (an utterance that ended at a poll with no new frame)"""
    from voicecraft_b200.tokenizer import CodecStream
    calls = []
    orig = CodecStream.flush

    def counted(self, ids):
        calls.append(list(ids))
        return orig(self, ids)
    monkeypatch.setattr(CodecStream, "flush", counted)
    return calls


@pytest.mark.gpu
@pytest.mark.parametrize("sr", RATES)
def test_tts_streams_at_a_sample_rate(sr, flushes):
    cfg, m = _lm()
    tok = _codec()
    utts = _utts(cfg, 6, 40)
    xs, ys = [u[0] for u in utts], [u[2] for u in utts]
    seeds = [100 + i for i in range(6)]
    ref = m.inference_tts_many(xs, ys, seeds=seeds, top_k=40)
    assert 0 < ref[2][1].shape[-1] < tok.open_stream(1).min_frames                  # decoded (and resampled) whole
    # chunk_frames=1, poll_every=1: every final frame is pushed at once, so each utterance's last frame arrives one poll
    # before its end and the end comes with no new frame
    for chunk, poll in ((1, 1), (10, 4)):
        ts = m.inference_tts_many_stream(xs, ys, tok, chunk_frames=chunk, poll_every=poll, seeds=seeds, top_k=40,
                                         sample_rate=sr)
        audio = {i: [] for i in range(6)}
        for i, w in ts:
            assert w.shape[-1] > 0
            audio[i].append(w)
        for i in range(6):
            assert torch.equal(ts.results[i][1], ref[i][1]), i
            want = tok.resample(tok.decode_codes(ref[i][1]), 16000, sr)
            assert torch.equal(torch.cat(audio[i], -1), want), (chunk, i)
        if chunk == 1:
            assert flushes, "no utterance ended at a poll without a new frame"
    # the single call
    x, xl, y = utts[0]
    torch.manual_seed(7)
    res, gen = m.inference_tts(x, xl, y, top_k=40)
    torch.manual_seed(7)
    ts = m.inference_tts_stream(x, xl, y, tok, chunk_frames=10, poll_every=4, top_k=40, sample_rate=sr)
    chunks = list(ts)
    assert torch.equal(ts.result[1], gen)
    assert torch.equal(torch.cat(chunks, -1), tok.resample(tok.decode_codes(gen), 16000, sr))
    assert not any(s._open for s in m._sessions)


@pytest.mark.gpu
@pytest.mark.parametrize("sr", RATES)
def test_edit_stream_at_a_sample_rate(sr):
    cfg, m = _lm()
    tok = _codec()
    from voicecraft_b200 import synthetic
    spans = [[(0, 4)], [(3, 6), (6, 10)], [(2, 5), (9, 12), (17, 20)], [(10, 13), (15, 18)]]
    utts = []
    for i in range(len(spans)):
        x, xl, y = synthetic.synthetic_utterance(cfg, 1300 + i, text_len=6 + i, prompt_frames=20)
        utts.append((x.cuda(), y.cuda()))
    mis = [torch.tensor([s]) for s in spans]
    kw = dict(top_k=30, top_p=0.9, temperature=1.0)
    seeds = [21 + i for i in range(len(utts))]
    many = m.inference_many([u[0] for u in utts], [u[1] for u in utts], mis, seeds=seeds, **kw)
    st = m.inference_many_stream([u[0] for u in utts], [u[1] for u in utts], mis, tok, chunk_frames=5, poll_every=4,
                                 seeds=seeds, sample_rate=sr, **kw)
    audio = {}
    for i, w in st:
        audio.setdefault(i, []).append(w)
    for i, b in enumerate(many):
        assert torch.equal(st.results[i], b), i
        assert torch.equal(torch.cat(audio[i], -1), tok.resample(tok.decode_codes(b), 16000, sr)), i


@pytest.mark.gpu
@pytest.mark.parametrize("sr", RATES)
def test_batcher_stream_at_a_sample_rate(sr, flushes):
    """re-admitted slots (10 tickets, 3 slots) and failed tickets (a non-audio token now and then)"""
    from voicecraft_b200.voicecraft import ContinuousBatcher
    kw = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
    cfg, m = _lm(empty_bias=1.5)
    tok = _codec()
    utts = _utts(cfg, 10, 70)
    seeds = list(range(10))
    singles = []
    for (x, xl, y), s in zip(utts, seeds):
        torch.manual_seed(s)
        singles.append(m.inference_tts(x, xl, y, **kw))
    bad = {i for i, (_, gen) in enumerate(singles) if bool((gen >= tok.config.bins).any())}
    assert 0 < len(bad) < 10, bad
    cb = ContinuousBatcher(m, max_concurrency=3, poll_every=1, **kw)
    for (x, _, y), s in zip(utts, seeds):
        cb.submit(x, y, seed=s)
    audio, lasts = {}, {}
    for t, w, last in cb.stream(tok, chunk_frames=1, sample_rate=sr):
        assert not lasts.get(t)
        assert w is None or w.shape[-1] > 0 or last
        audio.setdefault(t, []).append(w)
        lasts[t] = last
    assert set(cb.errors) == bad and cb.stats["prefills"] >= 3
    assert flushes
    for i in range(10):
        assert lasts[i] is True
        if i in bad:
            assert cb.results[i] is None and audio[i][-1] is None
        else:
            gen = cb.results[i][1]
            assert torch.equal(gen, singles[i][1]), i
            assert torch.equal(torch.cat(audio[i], -1), tok.resample(tok.decode_codes(gen), 16000, sr)), i
    assert not any(s._open for s in m._sessions)


@pytest.mark.gpu
def test_codec_rate_streams_launch_no_resampler():
    from voicecraft_b200 import _lib
    cfg, m = _lm()
    tok = _codec()
    utts = _utts(cfg, 3, 40)
    lib = _lib.load()
    n0 = lib.enc_counter(None, b"resample_launches")
    for sr in (None, 16000):
        ts = m.inference_tts_many_stream([u[0] for u in utts], [u[2] for u in utts], tok, chunk_frames=10, poll_every=4,
                                         seeds=[1, 2, 3], top_k=40, sample_rate=sr)
        for _ in ts:
            pass
    assert lib.enc_counter(None, b"resample_launches") == n0


# ---------------------------------------------------------------------------------------------------------------------
# GPU: lifetime
# ---------------------------------------------------------------------------------------------------------------------
def _live():
    from voicecraft_b200 import _lib
    gc.collect()
    torch.cuda.synchronize()
    lib = _lib.load()
    return lib.enc_counter(None, b"live_bytes"), lib.enc_counter(None, b"live_handles")


@pytest.mark.gpu
def test_resampler_lifetime():
    import ctypes as C
    from voicecraft_b200 import _lib
    from voicecraft_b200.tokenizer import resample_table
    lib = _lib.load()
    torch.zeros(1, device="cuda")
    before = _live()
    for orig, new, streams in ((44100, 16000, 4), (16000, 48000, 0), (22050, 16000, 1)):
        rs = _rs(orig, new, streams)
        assert _live() != before
        x = torch.randn(1, 5000, device="cuda")
        rs(x)
        if streams:
            rs.push(x, [0], [5000], [True])
        del x
        rs.close()
        assert _live() == before
    h = C.c_void_p()
    table = resample_table(44100, 16000)
    for args in ((0, 16000), (16000, -5)):                                      # rates <= 0
        assert lib.enc_resampler_create(*args, table.data_ptr(), 1, 0, C.byref(h)) != 0 and not h.value
    assert lib.enc_resampler_create(16000, 44099, table.data_ptr(), 1, 0, C.byref(h)) != 0      # table over the cap
    assert b"cap" in lib.vcb_last_error() and not h.value
    # 2^24 streams of 916 carried samples, twice: 123 GB, more than the device holds -- the table was already allocated
    assert lib.enc_resampler_create(44100, 16000, table.data_ptr(), 1 << 24, 0, C.byref(h)) != 0
    assert b"allocation" in lib.vcb_last_error() and not h.value
    assert _live() == before
