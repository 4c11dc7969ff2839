"""EnCodec decode: oracle vs the fixtures produced from the transformers twin (CPU), CUDA path vs oracle (-m gpu)."""
import os

import numpy as np
import pytest
import torch

from oracle import encodec_oracle as eo

CASES = {
    "small_causal_reflect": (dict(n_filters=8, dimension=32, bins=64, lstm=2), 1),
    "small_noncausal_trueskip": (dict(n_filters=8, dimension=32, bins=64, lstm=1, causal=False, true_skip=True), 2),
    "small_constpad": (dict(n_filters=8, dimension=32, bins=64, lstm=1, pad_mode="constant"), 3),
    "mid_default": (dict(n_filters=16, dimension=64, bins=256), 4),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_twin_fixture(name, golden_dir):
    g = np.load(os.path.join(golden_dir, "codec.npz"))
    over, seed = CASES[name]
    cfg = eo.default_config(**over)
    sd = eo.make_state_dict(cfg, seed=seed)
    wav = eo.decode(cfg, sd, torch.from_numpy(g[f"{name}.codes"]))
    ref = g[f"{name}.wav"]
    assert wav.shape == ref.shape
    assert np.abs(wav.numpy() - ref).max() < 2e-5


def test_hop_and_shapes():
    cfg = eo.default_config(n_filters=4, dimension=16, bins=32, lstm=0)
    sd = eo.make_state_dict(cfg, seed=0)
    for T in (1, 7, 8):
        codes = torch.randint(0, 32, (2, 4, T))
        assert eo.decode(cfg, sd, codes).shape == (2, 1, 320 * T)


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_encode_matches_twin_fixture(name, golden_dir):
    """wav -> latent -> codes of the oracle against the transformers twin's encoder + RVQ (codec_encode.npz)."""
    g = np.load(os.path.join(golden_dir, "codec_encode.npz"))
    over, seed = CASES[name]
    cfg = eo.default_config(**over)
    sd = eo.make_state_dict(cfg, seed=seed, encoder=True)
    wav = torch.from_numpy(g[f"{name}.wav"])
    z = eo.encode_latent(cfg, sd, wav)
    assert np.abs(z.numpy() - g[f"{name}.latent"]).max() < 2e-5
    assert np.array_equal(eo.rvq_encode(cfg, sd, z).numpy(), g[f"{name}.codes"])


def test_encoder_decoder_weights_are_independent_of_the_flag():
    cfg = eo.default_config(n_filters=4, dimension=16, bins=32, lstm=1)
    a, b = eo.make_state_dict(cfg, seed=3), eo.make_state_dict(cfg, seed=3, encoder=True)
    assert all(torch.equal(a[k], b[k]) for k in a) and any(k.startswith("enc.") for k in b)


def _gpu_tok(cfg, sd):
    from voicecraft_b200.tokenizer import AudioTokenizer
    return AudioTokenizer(device="cuda:0", config=cfg, state_dict=sd)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_cuda_decode_matches_fixture(name, golden_dir):
    """Tolerance: fp32 kernels vs fp32 twin, |err| <= 2e-4 on O(1) waveforms (different summation order only)."""
    g = np.load(os.path.join(golden_dir, "codec.npz"))
    over, seed = CASES[name]
    cfg = eo.default_config(**over)
    tok = _gpu_tok(cfg, eo.make_state_dict(cfg, seed=seed))
    codes = torch.from_numpy(g[f"{name}.codes"])
    wav = tok.decode_codes(codes.cuda()).cpu().numpy()
    ref = g[f"{name}.wav"]
    assert wav.shape == ref.shape
    assert np.abs(wav - ref).max() < 2e-4, np.abs(wav - ref).max()
    # reference call signature: one utterance, [(codes, None)]
    one = tok.decode([(codes[:1].cuda(), None)])
    assert one.shape == (1, 1, ref.shape[-1]) and np.abs(one.cpu().numpy() - ref[:1]).max() < 2e-4


@pytest.mark.gpu
def test_cuda_decode_full_size_vs_oracle():
    """Real codec shape (n_filters 64, 4x2048, LSTM 2) on 2 x 1 s of tokens; odd T exercises ragged tiles."""
    cfg = eo.default_config()
    sd = eo.make_state_dict(cfg, seed=7)
    codes = torch.randint(0, 2048, (2, 4, 53), generator=torch.Generator().manual_seed(5))
    ref = eo.decode(cfg, sd, codes).numpy()
    wav = _gpu_tok(cfg, sd).decode_codes(codes.cuda()).cpu().numpy()
    assert wav.shape == ref.shape == (2, 1, 53 * 320)
    err = np.abs(wav - ref).max()
    assert err < 5e-4 * max(1.0, np.abs(ref).max()), err


@pytest.mark.gpu
def test_cuda_decode_batch_independence():
    """Property at larger sizes: decoding a batch equals decoding each row alone (bit-exact, same kernels)."""
    cfg = eo.default_config(n_filters=16, dimension=64, bins=256)
    tok = _gpu_tok(cfg, eo.make_state_dict(cfg, seed=9))
    codes = torch.randint(0, 256, (19, 4, 40), generator=torch.Generator().manual_seed(6)).cuda()
    full = tok.decode_codes(codes)
    for b in (0, 7, 18):
        assert torch.equal(full[b:b + 1], tok.decode_codes(codes[b:b + 1]))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_cuda_encode_matches_fixture(name, golden_dir):
    """SURVEY.md section 8f row f1: AudioTokenizer.encode (SEANetEncoder + RVQ) on the GPU against the twin's codes.  Integer
    output: identical, except where the two nearest codes are equidistant to within fp32 noise (decision gap < 1e-4; the
    fixtures' smallest gap is 0.013, so in practice identical) -- and then every later stage of that frame may differ too."""
    g = np.load(os.path.join(golden_dir, "codec_encode.npz"))
    over, seed = CASES[name]
    cfg = eo.default_config(**over)
    tok = _gpu_tok(cfg, eo.make_state_dict(cfg, seed=seed, encoder=True))
    wav = torch.from_numpy(g[f"{name}.wav"])
    codes = tok.encode_codes(wav.cuda()).cpu().numpy()
    ref, gaps = g[f"{name}.codes"], g[f"{name}.gaps"]
    assert codes.shape == ref.shape
    bad = codes != ref
    first_bad = bad.cumsum(axis=1) == 1                       # first differing stage per (b, t)
    assert not (bad & first_bad & (gaps >= 1e-4)).any(), f"{int(bad.sum())} codes differ"
    one = tok.encode(wav[:1].cuda())                          # reference signature: [(codes[1,K,T], None)]
    assert one[0][1] is None and np.array_equal(one[0][0].cpu().numpy(), codes[:1])


@pytest.mark.gpu
def test_cuda_encode_decode_round_trip_full_size():
    """Real codec shape (n_filters 64, 4 x 2048, LSTM 2), 1 s of audio: GPU codes == oracle codes, and decode(encode(wav))
    has the input's length (size-independent property: T frames -> T * hop samples)."""
    cfg = eo.default_config()
    sd = eo.make_state_dict(cfg, seed=11, encoder=True)
    wav = torch.randn(2, 1, 16000, generator=torch.Generator().manual_seed(12)) * 0.3
    ref, gaps = eo.rvq_encode(cfg, sd, eo.encode_latent(cfg, sd, wav), return_gaps=True)
    tok = _gpu_tok(cfg, sd)
    codes = tok.encode_codes(wav.cuda())
    bad = (codes.cpu() != ref)
    assert not (bad & (bad.cumsum(dim=1) == 1) & (gaps >= 1e-4)).any(), f"{int(bad.sum())} codes differ"
    out = tok.decode_codes(codes)
    assert out.shape == (2, 1, 16000)


def _counter(tok, name):
    from voicecraft_b200 import _lib
    return int(_lib.load().enc_counter(tok._engine(), name.encode()))


@pytest.mark.gpu
def test_tensor_core_decoder_runs_the_default_codec():
    """The default 16 kHz codec must decode on the tensor-core path (csrc/codec_tc.cu), not fall back to the CUDA-core kernels.
    Tolerance (stated for the 3-pass bf16 hi/lo product, fp32 accumulation): waveform SNR >= 80 dB against the fp32 oracle
    and max |err| <= 2e-4 of the peak."""
    cfg = eo.default_config()
    sd = eo.make_state_dict(cfg, seed=7)
    codes = torch.randint(0, 2048, (3, 4, 61), generator=torch.Generator().manual_seed(15))
    ref = eo.decode(cfg, sd, codes)
    tok = _gpu_tok(cfg, sd)
    wav = tok.decode_codes(codes.cuda()).cpu()
    assert _counter(tok, "tc_enabled") == 1 and _counter(tok, "tc_decodes") == 1
    snr = 10 * torch.log10((ref ** 2).sum() / ((wav - ref) ** 2).sum()).item()
    assert snr >= 80.0, snr
    assert (wav - ref).abs().max() <= 2e-4 * max(1.0, ref.abs().max().item())
    # shorter than the reflect paddings need: the CUDA-core kernels take over, same answer
    short = tok.decode_codes(codes[:, :, :5].cuda()).cpu()
    assert _counter(tok, "tc_decodes") == 1
    assert (short - eo.decode(cfg, sd, codes[:, :, :5])).abs().max() < 5e-4


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small_causal_reflect", "small_constpad", "mid_default"])
def test_cuda_core_decoder_matches_fixture(name, golden_dir, monkeypatch):
    """VCB_CODEC_TC=0 keeps the round-1 fp32 CUDA-core decoder reachable (it still serves the configurations the tensor-core
    path does not cover); same fixtures, same tolerance."""
    monkeypatch.setenv("VCB_CODEC_TC", "0")
    g = np.load(os.path.join(golden_dir, "codec.npz"))
    over, seed = CASES[name]
    cfg = eo.default_config(**over)
    tok = _gpu_tok(cfg, eo.make_state_dict(cfg, seed=seed))
    wav = tok.decode_codes(torch.from_numpy(g[f"{name}.codes"]).cuda()).cpu().numpy()
    assert _counter(tok, "tc_enabled") == 0
    assert np.abs(wav - g[f"{name}.wav"]).max() < 2e-4


@pytest.mark.gpu
def test_tensor_core_decoder_chunking_is_invisible(monkeypatch):
    """A workspace limit that forces the batch through several chunks must not change a bit of the waveform."""
    cfg = eo.default_config(n_filters=16, dimension=64, bins=256)
    sd = eo.make_state_dict(cfg, seed=9)
    codes = torch.randint(0, 256, (11, 4, 33), generator=torch.Generator().manual_seed(6)).cuda()
    full = _gpu_tok(cfg, sd).decode_codes(codes)
    monkeypatch.setenv("VCB_CODEC_WS_GB", "0.02")
    tok = _gpu_tok(cfg, sd)
    assert torch.equal(tok.decode_codes(codes), full)
    assert _counter(tok, "tc_decodes") == 1


@pytest.mark.gpu
@pytest.mark.parametrize("tc", ["1", "0"])
def test_decoder_variants_two_residual_layers_no_lstm(tc, monkeypatch):
    """Structure variants no fixture covers: two (dilated) residual layers per stage and no LSTM, on the tensor-core path and on
    the CUDA-core kernels, against the oracle (SNR >= 80 dB / 2e-4 of the peak)."""
    monkeypatch.setenv("VCB_CODEC_TC", tc)
    cfg = eo.default_config(n_filters=16, dimension=64, bins=256, n_residual_layers=2, lstm=0)
    sd = eo.make_state_dict(cfg, seed=21)
    codes = torch.randint(0, 256, (3, 4, 29), generator=torch.Generator().manual_seed(22))
    ref = eo.decode(cfg, sd, codes)
    tok = _gpu_tok(cfg, sd)
    wav = tok.decode_codes(codes.cuda()).cpu()
    assert _counter(tok, "tc_enabled") == int(tc)
    snr = 10 * torch.log10((ref ** 2).sum() / ((wav - ref) ** 2).sum()).item()
    assert snr >= 80.0, snr
    assert (wav - ref).abs().max() <= 2e-4 * max(1.0, ref.abs().max().item())


@pytest.mark.gpu
def test_tensor_core_decoder_is_causal_at_full_length():
    """Size-independent property at BASELINE's 16 s length (T = 800 frames, 256 000 samples per utterance): the codec is causal,
    so the waveform of the first 40 frames does not depend on what follows -- bit for bit on the tensor-core path (a row's
    arithmetic does not depend on the tile it falls in) -- and that prefix is checked against the fp32 oracle."""
    cfg = eo.default_config()
    sd = eo.make_state_dict(cfg, seed=31)
    codes = torch.randint(0, 2048, (2, 4, 800), generator=torch.Generator().manual_seed(32))
    tok = _gpu_tok(cfg, sd)
    full = tok.decode_codes(codes.cuda())
    assert full.shape == (2, 1, 800 * 320) and bool(torch.isfinite(full).all())
    head = tok.decode_codes(codes[:, :, :40].cuda())
    assert _counter(tok, "tc_decodes") == 2
    assert torch.equal(full[..., : 40 * 320], head)
    ref = eo.decode(cfg, sd, codes[:, :, :40])
    snr = 10 * torch.log10((ref ** 2).sum() / ((head.cpu() - ref) ** 2).sum()).item()
    assert snr >= 80.0, snr
    # the tail is real signal too (not zeros / garbage): its energy is of the order of the head's
    e_head, e_tail = full[..., : 40 * 320].pow(2).mean().item(), full[..., -40 * 320:].pow(2).mean().item()
    assert 0.05 * e_head < e_tail < 20.0 * e_head, (e_head, e_tail)
