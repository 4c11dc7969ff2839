"""The tensor-core EnCodec encoder (codec_tc.cu, enc_encode_ragged), AudioTokenizer.encode_many and audio tickets in the
ContinuousBatcher.

CPU: the folded-row statement of the strided conv (the GEMM the encoder runs, with the per-utterance right padding written
into the rows past an utterance's end) against the oracle's conv1d(stride=r), and the frame count from samples and rate.
GPU (-m gpu): every tensor the encoder stores, read back under VCB_CODEC_KEEP=1, against the float64 layer applied to the
tensor the encoder stored before it (bound 3 x 2^-16 x the layer's |a||w| sum, the decoder's); the codes against the
nearest codes of the GPU's own latent and against the CUDA-core encoder; ragged batches bit for bit; the C ABI's
rejections and counters; and batcher tickets that carry their prompt as audio.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import codec_ref as cr
from oracle import encodec_oracle as eo
from oracle import resample_oracle as ro

UNIT = 3 * 2.0 ** -16
EPS_ELU = 5e-7


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def folded_strided_conv(x, w, b, r, reflect=True):
    """The encoder's strided conv restated: x [B, C, L] -> [B, Cout, ceil(L/r)].  The plane holds r halo rows (the causal
    left pad, rows 1..r mirrored), the L rows, and ceil(L/r)*r - L rows of right padding reflecting x[L-2], x[L-3], ...
    Folded as rows [.][r*C], output frame t is a 2-tap conv over folded rows t (halo included: rows r t - r .. r t - 1)
    and t + 1, with K = 2 r C: weight tap j < r on the first, tap r + j on the second."""
    B, Cin, L = x.shape
    T = -(-L // r)
    extra = T * r - L
    left = x[:, :, 1:r + 1].flip(-1) if reflect else torch.zeros(B, Cin, r, dtype=x.dtype)
    right = x[:, :, L - 1 - extra:L - 1].flip(-1) if reflect else torch.zeros(B, Cin, extra, dtype=x.dtype)
    plane = torch.cat([left, x, right], dim=-1)                    # [B, C, r + T r]
    rows = plane.transpose(1, 2).reshape(B, T + 1, r * Cin)        # folded rows: row f = plane rows f r .. f r + r - 1
    Wf = w.permute(0, 2, 1).reshape(w.shape[0], 2, r * Cin)        # [Cout][tap half][p * Cin + ci]
    return (torch.einsum("bfk,ok->bof", rows[:, :-1], Wf[:, 0]) + torch.einsum("bfk,ok->bof", rows[:, 1:], Wf[:, 1])
            + b[None, :, None])


@pytest.mark.parametrize("r", [2, 4, 5, 8])
@pytest.mark.parametrize("pad_mode", ["reflect", "constant"])
def test_folded_strided_conv_is_the_oracle_conv(r, pad_mode):
    cfg = eo.default_config(pad_mode=pad_mode)
    g = torch.Generator().manual_seed(r)
    Cin, Cout = 6, 5
    w = torch.randn(Cout, Cin, 2 * r, generator=g, dtype=torch.float64)
    b = torch.randn(Cout, generator=g, dtype=torch.float64)
    for L in range(4 * r, 5 * r):                                  # every length mod r
        x = torch.randn(2, Cin, L, generator=g, dtype=torch.float64)
        want = eo.conv1d(cfg, x, w, b, 1, r)
        got = folded_strided_conv(x, w, b, r, pad_mode == "reflect")
        assert got.shape == want.shape, (L, got.shape, want.shape)
        assert (got - want).abs().max() < 1e-12, L


@pytest.mark.parametrize("rate", [16000, 44100, 48000])
def test_frames_from_samples_and_rate(rate):
    from voicecraft_b200.tokenizer import AudioTokenizer, default_codec_config
    cfg = eo.default_config(n_filters=4, dimension=8, bins=16, lstm=0)
    tok = AudioTokenizer(device="cpu", config=default_codec_config(**vars(cfg)), state_dict={})
    sd = eo.make_state_dict(cfg, seed=1, encoder=True)
    for n in [1, 2, 319, 320, 321, 1921, 2240, 2241, 4410, 4799, 44100, 48001, 160007]:
        m = n if rate == 16000 else ro.out_length(n, rate, 16000)      # the resampled length (torchaudio's)
        T = eo.encode_latent(cfg, sd, torch.full((1, 1, m), 0.1)).shape[-1]
        assert tok.frames(n, rate) == T, (n, rate)


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
def _lib():
    from voicecraft_b200 import _lib
    return _lib


def gpu_tok(cfg, sd):
    from voicecraft_b200.tokenizer import AudioTokenizer
    return AudioTokenizer(device="cuda:0", config=cfg, state_dict=sd)


def counter(tok, name):
    return int(_lib().load().enc_counter(tok._engine(), name.encode()))


def fetch(tok, name):
    """enc_debug_tensor `name` -> (float64 [B, C, halo + T], halo)"""
    lib, dims = _lib().load(), (C.c_int32 * 4)()
    _lib().check(lib.enc_debug_tensor(tok._engine(), name.encode(), None, 0, dims))
    out = np.empty(tuple(dims)[:3], dtype=np.float32)
    _lib().check(lib.enc_debug_tensor(tok._engine(), name.encode(), out.ctypes.data, out.size, dims))
    return torch.from_numpy(out).double(), int(dims[3])


def valid(tok, name, C_real, L):
    """the stored tensor's first L rows of its C_real channels"""
    full, halo = fetch(tok, name)
    return full[:, :C_real, halo:halo + L]


def within(tag, got, ref, bound):
    assert got.shape == ref.shape, (tag, got.shape, ref.shape)
    ratio = ((got - ref).abs() / bound).max().item()
    print(f"RATIO {tag} {ratio:.4f}")
    assert ratio <= 1.0, f"{tag}: error {ratio:.2f} x its bound"


def chain(cfg, n):
    L = [n]
    for r in reversed(cfg.ratios):
        L.append(-(-L[-1] // r))
    return L


def ragged(tok, wavs):
    """enc_encode_ragged over [1, N_i] rows -> (codes [B, K, T_N], frames)"""
    B, N = len(wavs), max(w.shape[-1] for w in wavs)
    x = torch.zeros(B, 1, N, device="cuda:0")
    for b, w in enumerate(wavs):
        x[b, 0, :w.shape[-1]] = w.cuda()
    lens = (C.c_int32 * B)(*[w.shape[-1] for w in wavs])
    frames = (C.c_int32 * B)()
    T = chain(tok.config, N)[-1]
    codes = torch.full((B, tok.config.n_q, T), -7, device="cuda:0", dtype=torch.long)
    _lib().check(_lib().load().enc_encode_ragged(tok._engine(), x.data_ptr(), lens, B, N, codes.data_ptr(), frames,
                                                 torch.cuda.current_stream().cuda_stream))
    return codes.cpu(), list(frames)


def lstm_integrating(cfg, sd, seed):
    g = torch.Generator().manual_seed(seed)
    H = cfg.n_filters * 2 ** len(cfg.ratios)
    for l in range(cfg.lstm):
        b = sd[f"enc.lstm.bias_ih_l{l}"]
        sd[f"enc.lstm.bias_hh_l{l}"].zero_()
        b[:H] = -1.0
        b[H:2 * H] = 4.0 + 2.0 * torch.rand(H, generator=g)
        b[2 * H:3 * H] = 1.5 * (2.0 * torch.randint(0, 2, (H,), generator=g) - 1.0)
        sd[f"enc.lstm.weight_hh_l{l}"] *= 2.0
    return sd


REGIMES = {"plain": lambda cfg, sd, seed: sd, "lstm_integrating": lstm_integrating}


# ---------------------------------------------------------------------------------------------------------------------
# GPU: stage by stage against float64
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("regime", sorted(REGIMES))
@pytest.mark.parametrize("N", [16000, 16001, 32319])
def test_encoder_stages_vs_fp64(regime, N, monkeypatch):
    """Every GEMM output within 3 x 2^-16 x A (A = sum |a||w| + |b| of its own reduction) of the float64 layer applied to
    the tensor the encoder stored before it; the LSTM teacher-forced; the free-running latent per frame as a RATIO of the
    CUDA-core encoder's 1e-4 (|err|_2 <= 1e-4 |ref|_2 per frame)."""
    monkeypatch.setenv("VCB_CODEC_KEEP", "1")
    cfg = eo.default_config()
    sd = REGIMES[regime](cfg, eo.make_state_dict(cfg, seed=21, encoder=True), 21)
    sd64 = cr.double(sd)
    wav = 0.3 * torch.randn(1, 1, N, generator=torch.Generator().manual_seed(N))
    tok = gpu_tok(cfg, sd)
    assert counter(tok, "tc_encoder") == 1
    codes, frames = ragged(tok, [wav[0]])
    L = chain(cfg, N)
    plan = eo.encoder_plan(cfg)
    ch = cfg.n_filters
    # enc.conv_in on the fp32 input
    ref = cr.layer(cfg, sd64, plan[0], {"x": wav.double()})["raw"]
    ab = cr.abs_bound(cfg, sd64, plan[0], {"x": wav.double()})["raw"]
    x = valid(tok, "enc.x0", ch, L[0])
    within("enc.x0", x, ref, UNIT * ab + 1e-30)
    x_elu = valid(tok, "enc.x0.elu", ch, L[0])
    within("enc.x0.elu", x_elu, F.elu(x), EPS_ELU + 2.0 ** -16 * x.abs())
    for s, r in enumerate(reversed(cfg.ratios)):
        Lres = [p for p in plan if p["name"].startswith(f"enc.down{s}.res")]
        for j, P in enumerate(Lres):
            name = P["name"]
            h = valid(tok, name + ".h", ch // cfg.compress, L[s])
            inp = {"x": x, "x_elu": x_elu}
            out = cr.layer(cfg, sd64, P, dict(inp, h_elu=h))
            ab = cr.abs_bound(cfg, sd64, P, dict(inp, h_elu=h))
            within(f"{name}.h", h, cr.layer(cfg, sd64, P, inp)["h"], UNIT * ab["h"] + EPS_ELU)
            if j < len(Lres) - 1:
                x = valid(tok, name, ch, L[s])
                within(name, x, out["raw"], UNIT * ab["raw"])
                x_elu = valid(tok, name + ".elu", ch, L[s])
            else:
                x_elu = valid(tok, name + ".elu", ch, L[s])
                within(name + ".elu", x_elu, F.elu(out["raw"]), UNIT * ab["raw"] + EPS_ELU)
                # the right padding past the utterance's rows: the reflection the strided conv reads
                full, halo = fetch(tok, name + ".elu")
                extra = -(-L[s] // r) * r - L[s]
                for i in range(extra):
                    assert torch.equal(full[:, :, halo + L[s] + i], full[:, :, halo + L[s] - 2 - i]), (name, i)
        P = [p for p in plan if p["name"] == f"enc.down{s}.conv"][0]
        ref = cr.layer(cfg, sd64, P, {"x_elu": x_elu})["raw"]
        ab = cr.abs_bound(cfg, sd64, P, {"x_elu": x_elu})["raw"]
        ch *= 2
        x = valid(tok, P["name"], ch, L[s + 1])
        within(P["name"], x, ref, UNIT * ab)
        if s < len(cfg.ratios) - 1:
            x_elu = valid(tok, P["name"] + ".elu", ch, L[s + 1])
    # LSTM, teacher-forced on the h the encoder stored
    T = L[-1]
    inp = x.permute(2, 0, 1)
    for l in range(cfg.lstm):
        full, halo = fetch(tok, f"enc.hs{l}")
        hs = full[:, :ch, halo:halo + T].permute(2, 0, 1)
        h_ref, _, err_h, _ = cr.lstm_teacher_forced(sd64, "enc.lstm", l, inp, hs, UNIT)
        within(f"enc.hs{l}", hs, h_ref, err_h + 2.0 ** -20)
        inp = hs
    u = valid(tok, "enc.lstm", ch, T)
    h_last = hs.permute(1, 2, 0)
    within("enc.lstm", u, F.elu(h_last + x), EPS_ELU + 2.0 ** -16 * (h_last.abs() + x.abs()))
    P = plan[-1]
    ref = cr.layer(cfg, sd64, P, {"x_elu": u})["raw"]
    ab = cr.abs_bound(cfg, sd64, P, {"x_elu": u})["raw"]
    lat, halo = fetch(tok, "enc.latent")
    assert halo == 0 and lat.shape == (1, cfg.dimension, T) and frames == [T]
    within("enc.latent", lat, ref, UNIT * ab)
    free = eo.encode_latent(cfg, sd64, wav.double())
    ratio = ((lat - free).norm(dim=1) / (1e-4 * free.norm(dim=1))).max().item()
    print(f"RATIO enc_latent_free {regime} N={N} {ratio:.4f}")
    assert ratio <= 1.0, ratio                     # (the codes' bound in the next test takes the latent this close)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [2, 17])
def test_codes_are_nearest_of_the_gpu_latent_and_match_cuda_core(B, monkeypatch):
    """The codes are the nearest codes of the tensor-core latent (4e-5 slack of the fp32 search, as for the CUDA-core
    encoder), and equal encode_codes (the CUDA-core encoder) except in frames whose float64 decision gap at some stage is
    below 4 d (|z| + n_q max|e|) + 8e-5: d = 2e-4 |z| per frame bounds the distance of the two latents (each within 1e-4
    |z| of float64), by which a squared distance moves at most 2 d (|r - e1| + |r - e2|), plus the two searches' slack."""
    monkeypatch.setenv("VCB_CODEC_KEEP", "1")
    cfg = eo.default_config()
    sd = eo.make_state_dict(cfg, seed=13, encoder=True)
    sd64 = cr.double(sd)
    g = torch.Generator().manual_seed(B)
    wavs = [0.3 * torch.randn(1, 4801 + 517 * b, generator=g) for b in range(B)]
    tok = gpu_tok(cfg, sd)
    codes, frames = ragged(tok, wavs)
    lat, _ = fetch(tok, "enc.latent")
    emax = max(sd64[f"vq.{q}.embed"].norm(dim=1).max().item() for q in range(cfg.n_q))
    worst, exempt, checked = 0.0, 0, 0
    for b in range(B):
        T = frames[b]
        z = lat[b:b + 1, :, :T]
        resid = z[0].t()
        for q in range(cfg.n_q):
            emb = sd64[f"vq.{q}.embed"]
            dist = torch.cdist(resid, emb).pow(2)
            idx = codes[b, q, :T]
            worst = max(worst, (dist.gather(1, idx[:, None])[:, 0] - dist.min(dim=1).values).max().item())
            resid = resid - emb[idx]
        assert (codes[b, :, T:] == 0).all()
        cc = tok.encode_codes(wavs[b][None].cuda()).cpu()[0]
        ref = eo.encode_latent(cfg, sd64, wavs[b][None].double())
        _, gaps = eo.rvq_encode(cfg, sd64, ref, return_gaps=True)
        zn = ref[0].norm(dim=0)
        bound = 4 * 2e-4 * zn * (zn + cfg.n_q * emax) + 8e-5
        close = (gaps[0] < bound[None]).any(dim=0)
        differ = (codes[b, :, :T] != cc).any(dim=0)
        assert not (differ & ~close).any(), (b, torch.nonzero(differ & ~close))
        exempt += int(close.sum())
        checked += T
    print(f"RATIO rvq_tc B={B} {worst / 4e-5:.4f} (exempt frames {exempt}/{checked})")
    assert worst <= 4e-5, worst


# ---------------------------------------------------------------------------------------------------------------------
# GPU: ragged batches
# ---------------------------------------------------------------------------------------------------------------------
def _rows(seed, lengths):
    g = torch.Generator().manual_seed(seed)
    return [0.3 * torch.randn(1, n, generator=g) for n in lengths]


LENGTHS = [16000, 16001, 16319, 32000, 9601, 1500, 700, 3, 4799, 2241, 12345, 1921, 5120, 6401, 640, 7999, 30001]


@pytest.mark.gpu
def test_ragged_rows_are_bit_identical_alone_permuted_and_chunked(monkeypatch):
    """Lengths = 0, 1, 319 (mod 320), rows below the tensor-core minimum, B = 1 and 17, and a small workspace limit that
    cuts the batch into several chunks: every row's codes equal its codes alone and in a permuted batch, frames_host is
    the ceil chain, rows below the minimum equal encode_codes of the row alone bit for bit, and the tensor-core work
    follows the rows' lengths (encode_rows)."""
    cfg = eo.default_config()
    sd = eo.make_state_dict(cfg, seed=31, encoder=True)
    wavs = _rows(31, LENGTHS)
    tok = gpu_tok(cfg, sd)
    r0 = counter(tok, "encode_rows")
    codes, frames = ragged(tok, wavs)
    rows_one_chunk = counter(tok, "encode_rows") - r0
    assert frames == [chain(cfg, n)[-1] for n in LENGTHS]
    short = [b for b, n in enumerate(LENGTHS) if n <= 1920]
    assert short == [b for b, n in enumerate(LENGTHS) if n in (1500, 700, 3, 640)]
    for b in range(len(wavs)):
        T = frames[b]
        alone, fa = ragged(tok, [wavs[b]])
        assert fa == [T] and torch.equal(alone[0, :, :T], codes[b, :, :T]), b
        assert (codes[b, :, T:] == 0).all(), b
        if b in short:
            assert torch.equal(codes[b, :, :T], tok.encode_codes(wavs[b][None].cuda()).cpu()[0]), b
    perm = torch.randperm(len(wavs), generator=torch.Generator().manual_seed(5)).tolist()
    pc, pf = ragged(tok, [wavs[p] for p in perm])
    for i, p in enumerate(perm):
        assert pf[i] == frames[p] and torch.equal(pc[i, :, :frames[p]], codes[p, :, :frames[p]]), p
    del tok
    monkeypatch.setenv("VCB_CODEC_WS_GB", "0.2")
    tok = gpu_tok(cfg, sd)
    r0 = counter(tok, "encode_rows")
    cc, cf = ragged(tok, wavs)
    rows_chunked = counter(tok, "encode_rows") - r0
    assert cf == frames and torch.equal(cc, codes)
    # one chunk runs every tensor-core row at the longest length; sorted chunks follow the lengths more closely
    n_tc = len(wavs) - len(short)
    assert rows_one_chunk == n_tc * -(-max(LENGTHS) // 2) * 2
    assert rows_chunked < rows_one_chunk, (rows_chunked, rows_one_chunk)


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [44100, 48000])
def test_encode_many_resamples_like_resampled_rows(rate):
    cfg = eo.default_config()
    tok = gpu_tok(cfg, eo.make_state_dict(cfg, seed=41, encoder=True))
    g = torch.Generator().manual_seed(rate)
    wavs = [0.3 * torch.randn(2 if i % 2 else 1, n, generator=g) for i, n in enumerate([44100, 30011, 99999, 5000, 800])]
    got = tok.encode_many(wavs, rate)
    mono = [w.mean(dim=0, keepdim=True) if w.shape[0] > 1 else w for w in wavs]
    want = tok.encode_many([tok.resample(w[None].cuda(), rate)[0] for w in mono])
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == (1, cfg.n_q, tok.frames(wavs[i].shape[1], rate)) and torch.equal(a, b), i


@pytest.mark.gpu
def test_encode_many_without_tensor_cores_is_encode_codes(monkeypatch):
    monkeypatch.setenv("VCB_CODEC_TC", "0")
    cfg = eo.default_config()
    tok = gpu_tok(cfg, eo.make_state_dict(cfg, seed=43, encoder=True))
    wavs = _rows(43, [16000, 2241, 700, 5000])
    got = tok.encode_many(wavs)
    assert counter(tok, "tc_encoder") == 0 and counter(tok, "tc_encodes") == 0
    for w, a in zip(wavs, got):
        assert torch.equal(a.cpu(), tok.encode_codes(w[None].cuda()).cpu())


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the C ABI
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_abi_rejections_counters_and_lifetime():
    import gc
    gc.collect()
    lib, VcbError = _lib().load(), _lib().VcbError
    live0 = int(lib.enc_counter(None, b"live_bytes"))
    cfg = eo.default_config()
    sd = eo.make_state_dict(cfg, seed=47, encoder=True)
    tok = gpu_tok(cfg, sd)
    eng = tok._engine()
    x = 0.3 * torch.randn(2, 1, 4000, device="cuda:0")
    codes = torch.full((2, cfg.n_q, chain(cfg, 4000)[-1]), -7, device="cuda:0", dtype=torch.long)
    frames = (C.c_int32 * 2)()
    st = torch.cuda.current_stream().cuda_stream
    l0, e0, r0 = counter(tok, "launches"), counter(tok, "tc_encodes"), counter(tok, "encode_rows")
    for B, lens in [(0, [4000, 4000]), (2, [0, 4000]), (2, [4000, 4001]), (2, [-1, 10])]:
        with pytest.raises(VcbError):
            _lib().check(lib.enc_encode_ragged(eng, x.data_ptr(), (C.c_int32 * 2)(*lens), B, 4000, codes.data_ptr(), frames, st))
    torch.cuda.synchronize()
    assert counter(tok, "launches") == l0 and (codes == -7).all()
    assert counter(tok, "tc_encodes") == e0 and counter(tok, "encode_rows") == r0
    dec_only = gpu_tok(cfg, {k: v for k, v in sd.items() if not k.startswith("enc.")})
    with pytest.raises(VcbError, match="encoder weights"):
        _lib().check(lib.enc_encode_ragged(dec_only._engine(), x.data_ptr(), (C.c_int32 * 2)(4000, 4000), 2, 4000,
                                           codes.data_ptr(), frames, st))
    with pytest.raises(VcbError, match="encoder weights"):
        dec_only.encode_many([x[0].cpu()])
    _lib().check(lib.enc_encode_ragged(eng, x.data_ptr(), (C.c_int32 * 2)(4000, 1000), 2, 4000, codes.data_ptr(), frames, st))
    assert counter(tok, "tc_encodes") == e0 + 1 and counter(tok, "encode_rows") == r0 + 4000
    _lib().check(lib.enc_encode_ragged(eng, x.data_ptr(), (C.c_int32 * 2)(1000, 900), 2, 4000, codes.data_ptr(), frames, st))
    assert counter(tok, "tc_encodes") == e0 + 1 and counter(tok, "encode_rows") == r0 + 4000
    torch.cuda.synchronize()
    del tok, dec_only, eng
    gc.collect()
    assert int(lib.enc_counter(None, b"live_bytes")) == live0


# ---------------------------------------------------------------------------------------------------------------------
# GPU: batcher tickets with prompt audio
# ---------------------------------------------------------------------------------------------------------------------
def _lm(seed=3):
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=seed)
    for k in range(cfg.n_codebooks):
        for t in (cfg.empty_token, cfg.eog, cfg.audio_pad_token, cfg.eos):
            if not (k == 0 and t == cfg.eos):
                sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    sd["predict_layer.0.2.bias"][cfg.eog] = 2.5
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    return cfg, m.to("cuda:0").eval()


def _tickets(cfg, seed0):
    """(x, audio, rate, mask_interval, seed): TTS and one edit ticket, prompts of different lengths and rates"""
    from voicecraft_b200 import synthetic
    g = torch.Generator().manual_seed(seed0)
    out = []
    for i, (n, rate) in enumerate([(8000, 16000), (13230, 44100), (9600, 48000), (6400, 16000), (11025, 44100),
                                   (12000, 16000)]):
        x, _, _ = synthetic.synthetic_utterance(cfg, seed0 + i, text_len=4 + i % 3, prompt_frames=8)
        audio = 0.3 * torch.randn(2 if i == 1 else 1, n, generator=g)
        mi = torch.tensor([[(3, 9), (14, 18)]]) if i == 3 else None
        out.append((x.cuda(), audio, rate, mi, 700 + 11 * i))
    return out


def _submit(cb, q, with_audio, tok):
    x, audio, rate, mi, seed = q
    if with_audio:
        return cb.submit(x, audio=audio, sample_rate=rate, seed=seed, mask_interval=mi, top_k=40)
    return cb.submit(x, tok.encode_many([audio], rate)[0].transpose(1, 2), seed=seed, mask_interval=mi, top_k=40)


@pytest.mark.gpu
@pytest.mark.parametrize("pool", [False, True])
def test_batcher_audio_tickets_equal_code_tickets(pool):
    """run() and stream() with a queue of audio and code tickets (different lengths and rates, one edit, one submit(audio=)
    from inside the stream loop; with and without a KV pool budget) are token-identical to the same tickets given
    y = encode_many([audio], rate)[0].transpose(1, 2), and the stream's chunks are equal too."""
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg, m = _lm()
    if pool:                                       # a budget of a few growth chunks: tickets wait and swap
        from voicecraft_b200 import _lib as L
        pb = L.load().vcb_counter(m._engine(), b"kv_page_bytes")
        m.configure_engine(kv_pool_gb=(4 * L.KV_GROW_PAGES + 0.5) * pb / 1e9)
    ccfg = eo.default_config()
    tok = gpu_tok(ccfg, eo.make_state_dict(ccfg, seed=5, encoder=True))
    tickets = _tickets(cfg, 500)
    with pytest.raises(Exception, match="tokenizer"):
        ContinuousBatcher(m, max_concurrency=3).submit(tickets[0][0], audio=tickets[0][1])
    with pytest.raises(ValueError, match="exactly one"):
        ContinuousBatcher(m, max_concurrency=3, tokenizer=tok).submit(tickets[0][0])
    runs = {}
    for with_audio in (True, False):
        cb = ContinuousBatcher(m, max_concurrency=3, poll_every=3, tokenizer=tok)
        for i, q in enumerate(tickets):
            _submit(cb, q, with_audio and i % 2 == 0 or (with_audio and i == 3), tok)
        runs[with_audio] = cb.run()
    for i, (a, b) in enumerate(zip(runs[True], runs[False])):
        assert torch.equal(a[0], b[0]) and (a[1] is None) == (b[1] is None), i
        assert a[1] is None or torch.equal(a[1], b[1]), i
    streams = {}
    for with_audio in (True, False):
        cb = ContinuousBatcher(m, max_concurrency=3, poll_every=3, tokenizer=tok)
        for q in tickets[:-1]:
            _submit(cb, q, with_audio, tok)
        chunks, late = {}, False
        for t, w, last in cb.stream(tok, chunk_frames=5):
            chunks.setdefault(t, []).append(None if w is None else w.cpu())
            if not late:
                late = True
                _submit(cb, tickets[-1], with_audio, tok)
        streams[with_audio] = (chunks, list(cb.results))
    (ca, ra), (cc, rc) = streams[True], streams[False]
    assert sorted(ca) == sorted(cc) == list(range(len(tickets)))
    for t in ca:
        assert len(ca[t]) == len(cc[t]) and all(torch.equal(u, v) for u, v in zip(ca[t], cc[t])), t
        assert torch.equal(ra[t][0], rc[t][0]), t
    assert torch.equal(ra[0][0], runs[False][0][0])
    assert not m._sessions
