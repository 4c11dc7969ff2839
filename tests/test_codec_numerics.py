"""The EnCodec kernels (csrc/codec_tc.cu, csrc/encodec.cu) stage by stage against float64.

The reference is oracle/encodec_oracle.py run on float64 weights (CPU tests below pin that run to the fp32 one, which the
fixtures pin to the transformers twin).  On the GPU (-m gpu) every tensor the tensor-core decoder stores is read back
under VCB_CODEC_KEEP=1 (same kernels and launches, every tensor in rows of its own) and compared with the float64 layer
applied to the tensor the GPU stored one stage earlier, so each bound holds one stage's arithmetic.

Bounds.  The tensor-core GEMMs multiply bf16 (hi, lo) pairs in three passes (hi*hi, hi*lo, lo*hi) with fp32 accumulation:
    weight and activation as hi + lo: 2^-17 relative each;  the dropped lo*lo: 2^-18;  the output stored as hi + lo: 2^-17;
    fp32 accumulation over K <= 3584 terms: about sqrt(K) 2^-24 < 2^-18
all relative to A = sum |a||w| + |bias| of the output element (codec_ref.abs_bound), not to the output itself: about
2.5 x 2^-16 A, stated as UNIT = 3 x 2^-16.  An ELU'd tensor adds EPS_ELU = 5e-7 absolute (ex2.approx: 2^-22 relative of a
value <= 1, and fp32 rounding).  The CUDA-core kernels (the encoder, VCB_CODEC_TC=0) are plain fp32: FP32_UNIT = 2^-20 of
A per layer (sqrt(K) 2^-24 with K <= 3584, with margin for the order of summation).
The largest observed error of every check is printed as a fraction of its bound (pytest -s / -rP)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import codec_ref as cr
from oracle import encodec_oracle as eo
from test_codec import CASES

UNIT = 3 * 2.0 ** -16
EPS_ELU = 5e-7
FP32_UNIT = 2.0 ** -20

SMALL = dict(n_filters=8, dimension=32, bins=64)
CONFIGS = {
    "default": {},
    "two_res_no_lstm": dict(SMALL, lstm=0, n_residual_layers=2),
    "small_constpad": dict(SMALL, lstm=1, pad_mode="constant"),
}
MIN_T = {"default": 8, "two_res_no_lstm": 10, "small_constpad": 8}


# ---------------------------------------------------------------------------------------------------------------------
# weights.  No trained checkpoint is available offline: the regimes below stand in for what a trained codec does to the
# kernels (cells that integrate, common-mode offsets that cancel, a small waveform after large activations).
# ---------------------------------------------------------------------------------------------------------------------
def lstm_integrating(cfg, sd, seed):
    """Forget-gate bias +4..+6 (time constants of 55..400 steps), input-gate bias -1, a signed bias on the candidate so a
    cell keeps integrating one way, output-gate bias +4 on a third of the units, recurrent weights doubled."""
    g = torch.Generator().manual_seed(seed)
    H = cfg.n_filters * 2 ** len(cfg.ratios)
    for side in ("dec", "enc"):
        for l in range(cfg.lstm):
            if f"{side}.lstm.bias_ih_l{l}" not in sd:
                continue
            b = sd[f"{side}.lstm.bias_ih_l{l}"]
            sd[f"{side}.lstm.bias_hh_l{l}"].zero_()
            b[:H] = -1.0
            b[H:2 * H] = 4.0 + 2.0 * torch.rand(H, generator=g)
            b[2 * H:3 * H] = 1.5 * (2.0 * torch.randint(0, 2, (H,), generator=g) - 1.0)
            b[3 * H:] = torch.where(torch.arange(H) % 3 == 0, 4.0, 0.0) + 0.05 * torch.randn(H, generator=g)
            sd[f"{side}.lstm.weight_hh_l{l}"] *= 2.0
    return sd


def offset(cfg, sd, seed):
    """Every ConvTranspose's bias puts +20 or -20 on each channel of its stage, so the stage's ELU runs both branches at
    scale; the residual block's conv1 (on the ELU'd tensor) and shortcut (on the raw one) are made orthogonal to that
    offset, so the large terms cancel in their sums."""
    g = torch.Generator().manual_seed(seed)
    for i in range(len(cfg.ratios)):
        b = sd[f"dec.up{i}.convtr.bias"]
        v = 20.0 * (2.0 * torch.randint(0, 2, b.shape, generator=g) - 1.0)
        b += v
        for name, e in ((f"dec.up{i}.res0.conv1.weight", F.elu(v)), (f"dec.up{i}.res0.shortcut.weight", v)):
            w = sd[name]
            w -= (w * e[None, :, None]).sum(1, keepdim=True) * e[None, :, None] / (e * e).sum()
    return sd


def tiny_out(cfg, sd, seed):
    """Stage-1 activations of O(10) and a waveform that peaks near 0.02."""
    sd["dec.conv_in.weight"] *= 10.0
    sd["dec.up0.convtr.weight"] *= 3.0
    sd[f"dec.up{len(cfg.ratios) - 1}.convtr.weight"] *= 0.05
    sd["dec.conv_out.weight"] *= 0.1
    sd["dec.conv_out.bias"] *= 0.1
    return sd


REGIMES = {"plain": lambda cfg, sd, seed: sd, "lstm_integrating": lstm_integrating, "offset": offset, "tiny_out": tiny_out}


def weights(cfg, regime, seed, encoder=False):
    return REGIMES[regime](cfg, eo.make_state_dict(cfg, seed=seed, encoder=encoder), seed)


def rand_codes(cfg, B, T, seed):
    return torch.randint(0, cfg.bins, (B, cfg.n_q, T), generator=torch.Generator().manual_seed(seed))


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the float64 run, the intermediates, layer / abs_bound
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_float64_run_matches_fp32_run(name):
    over, seed = CASES[name]
    cfg = eo.default_config(**over)
    sd = eo.make_state_dict(cfg, seed=seed, encoder=True)
    sd64 = cr.double(sd)
    codes = rand_codes(cfg, 2, 21, seed)
    w64, rec = eo.decode(cfg, sd64, codes, return_intermediates=True)
    assert w64.dtype == torch.float64 and all(v.dtype == torch.float64 for v in rec.values())
    assert (w64 - eo.decode(cfg, sd, codes)).abs().max() < 2e-5
    assert rec["wav"] is w64 and list(rec)[-1] == "wav"
    wav = 0.3 * torch.randn(2, cfg.channels, 3205, generator=torch.Generator().manual_seed(seed))
    z64, enc = eo.encode_latent(cfg, sd64, wav.double(), return_intermediates=True)
    z32 = eo.encode_latent(cfg, sd, wav)
    assert z64.dtype == torch.float64 and enc["enc.latent"] is z64 and z64.shape[-1] == math.ceil(3205 / 320)
    assert (z64 - z32).abs().max() < 2e-5
    c64, gaps = eo.rvq_encode(cfg, sd64, z64, return_gaps=True)
    bad = c64 != eo.rvq_encode(cfg, sd, z32)
    assert not (bad & (bad.cumsum(dim=1) == 1) & (gaps >= 1e-4)).any()


@pytest.mark.parametrize("name", sorted(CASES))
def test_layers_chained_reproduce_decode(name):
    """codec_ref.layer over the plan is decode, bit for bit (fp32 and float64), tensor by tensor; abs_bound dominates."""
    over, seed = CASES[name]
    cfg = eo.default_config(**over)
    sd32 = eo.make_state_dict(cfg, seed=seed)
    codes = rand_codes(cfg, 2, 13, seed + 1)
    for sd in (sd32, cr.double(sd32)):
        wav, rec = eo.decode(cfg, sd, codes, return_intermediates=True)
        x = eo.rvq_decode(sd, codes)
        assert torch.equal(x, rec["z"])
        for L in eo.layer_plan(cfg):
            out = cr.layer(cfg, sd, L, {"x": x})
            if L["kind"] != "lstm":
                ab = cr.abs_bound(cfg, sd, L, {"x": x})
                assert (ab["raw"] >= out["raw"].abs() * (1 - 1e-6)).all()
                if L["kind"] == "res":
                    assert (ab["h"] >= out["h"].abs() * (1 - 1e-6)).all()
                    # the block's tail from a given hidden tensor is the same tail
                    assert torch.equal(cr.layer(cfg, sd, L, {"x": x, "x_elu": F.elu(x), "h_elu": out["h"]})["raw"], out["raw"])
            x = out["raw"]
        assert torch.equal(x, wav)


def test_teacher_forced_lstm_is_the_lstm_when_fed_its_own_states():
    cfg = eo.default_config(**SMALL, lstm=2)
    sd = cr.double(weights(cfg, "lstm_integrating", 3))
    x = torch.randn(50, 2, 128, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    states = {}
    eo.lstm(x, sd, "dec.lstm", 2, states)
    h, c, eh, ec = cr.lstm_teacher_forced(sd, "dec.lstm", 1, states["hs0"], states["hs1"], UNIT)
    assert torch.equal(h, states["hs1"]) and torch.equal(c, states["c1"])
    assert (eh > 0).all() and (ec[-1] > ec[0]).all()


def test_hostile_regimes_are_hostile():
    """On the float64 reference: the regimes do what their names say at the sizes the GPU tests use them."""
    cfg = eo.default_config(**SMALL, lstm=2)
    _, rec = eo.decode(cfg, cr.double(weights(cfg, "lstm_integrating", 5)), rand_codes(cfg, 1, 800, 5), return_intermediates=True)
    _assert_integrating(rec)
    cfg = eo.default_config(**SMALL, lstm=1)
    codes = rand_codes(cfg, 1, 16, 6)
    sd = cr.double(weights(cfg, "offset", 6))
    _, rec = eo.decode(cfg, sd, codes, return_intermediates=True)
    _assert_offset_cancels(cfg, sd, rec)


def _assert_integrating(rec):
    for l in (0, 1):
        c = rec[f"c{l}"].abs()
        assert 5.0 <= c[..., -1].median() <= 50.0 and c[..., -1].max() >= 10.0, (c[..., -1].median(), c[..., -1].max())
        assert c[..., -1].median() >= 3.0 * c[..., 7].median()            # still integrating long after step 7
    sat = (rec["hs1"][..., 400:].abs() > 0.95).float().mean().item()       # |h| = o |tanh c| near 1: both saturated
    assert sat >= 0.15, sat


def _assert_offset_cancels(cfg, sd, rec):
    L = [L for L in eo.layer_plan(cfg) if L["name"] == "dec.up0.res0"][0]
    x = rec["x1.raw"]
    assert (x.abs() > 10).float().mean() > 0.9 and (x > 10).any() and (x < -10).any()
    ab = cr.abs_bound(cfg, sd, L, {"x": x})["h"]
    h = eo.conv1d(cfg, F.elu(x), sd[L["name"] + ".conv1.weight"], sd[L["name"] + ".conv1.bias"], L["dil"])
    frac = (ab >= 100 * h.abs()).float().mean().item()
    assert frac >= 0.25, frac                                              # sum |a||w| >= 100 |sum a w| on a quarter of outputs


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
    """enc_debug_tensor `name` -> (float64 [B, C, halo + T], halo), or None where the plan has no such tensor"""
    lib, dims = _lib().load(), (C.c_int32 * 4)()
    if lib.enc_debug_tensor(tok._engine(), name.encode(), None, 0, dims):
        return None
    out = np.empty(tuple(dims)[:3], dtype=np.float32)
    _lib().check(lib.enc_debug_tensor(tok._engine(), name.encode(), out.ctypes.data, out.size, dims))
    return torch.from_numpy(out).double(), int(dims[3])


RATIOS = {}


def within(tag, name, got, ref, bound):
    """|got - ref| <= bound element-wise; the worst ratio is kept for the report"""
    assert got.shape == ref.shape, (tag, name, got.shape, ref.shape)
    ratio = ((got - ref).abs() / bound).max().item()
    RATIOS[tag] = max(RATIOS.get(tag, 0.0), ratio)
    print(f"RATIO {tag} {name} {ratio:.4f}")
    assert ratio <= 1.0, f"{tag} {name}: error {ratio:.2f} x its bound at {np.unravel_index(((got - ref).abs() / bound).argmax().item(), got.shape)}"


def snr_db(got, ref):
    return 10 * torch.log10((ref ** 2).sum() / ((got - ref) ** 2).sum().clamp_min(1e-300)).item()


def wav_bound(cfg, sd64, codes):
    """Waveform bound of a whole decode, free-running: the layers are 1-Lipschitz-ish at these weight scales (gain about
    1.2 each), so the error at the output is at most the sum over the D layers of each one's UNIT x A, taken as
    D x UNIT x the largest A of the final conv, floored at 2^-20."""
    _, rec = eo.decode(cfg, sd64, codes, return_intermediates=True)
    L = eo.layer_plan(cfg)[-1]
    last = [k for k in rec if k.startswith("o") and not k.endswith(".raw")][-1]
    ab = cr.abs_bound(cfg, sd64, L, {"x_elu": rec[last]})["raw"]
    depth = 3 + cfg.lstm + len(cfg.ratios) * (1 + 2 * cfg.n_residual_layers)
    return rec["wav"], depth * UNIT * ab.max().item() + 2.0 ** -20


def check_structure(cfg, name, full, halo, c_real, zero_halo):
    """padded channels are exactly zero; halo rows are zero, or the mirror of rows 1..halo"""
    assert (full[:, c_real:, halo:] == 0).all(), f"{name}: padded channels"
    if name.startswith("h") and not name.startswith("hs") or name.startswith("enc.") and name.endswith(".h"):
        return                                                             # a hidden tensor's halo rows are never written
    for t in range(1, halo + 1):
        want = torch.zeros_like(full[:, :, 0]) if zero_halo else full[:, :, halo + t]
        assert torch.equal(full[:, :, halo - t], want), f"{name}: halo row -{t}"


def stage_checks(tag, cfg, sd64, codes, tok, wav):
    """Every stored tensor against the float64 layer applied to the stored tensor before it."""
    plan = eo.layer_plan(cfg)
    n_stage = len(cfg.ratios)
    G = {}

    def load(name, c_real, zero_halo=False):
        got = fetch(tok, name)
        assert got is not None, name
        full, halo = got
        check_structure(cfg, name, full, halo, c_real, zero_halo or cfg.pad_mode == "constant")
        G[name] = full[:, :c_real, halo:]
        return G[name]

    B, K, T = codes.shape
    z_ref = eo.rvq_decode(sd64, codes)
    z_abs = sum(F.embedding(codes[:, q], sd64[f"vq.{q}.embed"]).abs() for q in range(K)).transpose(1, 2)
    within(tag, "z", load("z", cfg.dimension), z_ref, 2.0 ** -16 * z_abs + 1e-30)
    H = cfg.n_filters * 2 ** n_stage
    L = plan[0]
    ref, ab = cr.layer(cfg, sd64, L, {"x": G["z"]})["raw"], cr.abs_bound(cfg, sd64, L, {"x": G["z"]})["raw"]
    if cfg.lstm:
        within(tag, "x0", load("x0", H), ref, UNIT * ab)
        x = G["x0"].permute(2, 0, 1)
        for l in range(cfg.lstm):
            hs = load(f"hs{l}", H, True).permute(2, 0, 1)
            h, c, eh, ec = cr.lstm_teacher_forced(sd64, "dec.lstm", l, x, hs, UNIT)
            within(tag, f"hs{l}", hs, h, eh)
            got_c = fetch(tok, f"c{l}")[0][:, :, 0]
            within(tag, f"c{l}", got_c, c[-1], ec[-1])
            x = hs
        u0 = G[f"hs{cfg.lstm - 1}"] + G["x0"]
        within(tag, "u0", load("u0", H, True), F.elu(u0), 2.0 ** -16 * (G[f"hs{cfg.lstm - 1}"].abs() + G["x0"].abs()) + EPS_ELU)
    else:
        within(tag, "u0", load("u0", H, True), F.elu(ref), UNIT * ab + EPS_ELU)
    cur, ch, stage = G["u0"], H, 0
    for L in plan[1 + (1 if cfg.lstm else 0):-1]:
        if L["kind"] == "convtr":
            stage += 1
            ch //= 2
            j = 0
            inp = {"x_elu": cur}
            ref, ab = cr.layer(cfg, sd64, L, inp)["raw"], cr.abs_bound(cfg, sd64, L, inp)["raw"]
            within(tag, f"x{stage}.raw", load(f"x{stage}.raw", ch), ref, UNIT * ab)
            within(tag, f"x{stage}.elu", load(f"x{stage}.elu", ch), F.elu(ref), UNIT * ab + EPS_ELU)
            raw, cur = G[f"x{stage}.raw"], G[f"x{stage}.elu"]
        else:
            sj = f"{stage}.{j}"
            inp = {"x": raw, "x_elu": cur}
            ab = cr.abs_bound(cfg, sd64, L, inp)["h"]
            within(tag, f"h{sj}", load(f"h{sj}", L["hidden"]), cr.layer(cfg, sd64, L, inp)["h"], UNIT * ab + EPS_ELU)
            inp["h_elu"] = G[f"h{sj}"]
            ref, ab = cr.layer(cfg, sd64, L, inp)["raw"], cr.abs_bound(cfg, sd64, L, inp)["raw"]
            last = j == cfg.n_residual_layers - 1
            within(tag, f"o{sj}", load(f"o{sj}", ch, last and stage < n_stage), F.elu(ref), UNIT * ab + EPS_ELU)
            cur = G[f"o{sj}"]
            if not last:
                within(tag, f"o{sj}.raw", load(f"o{sj}.raw", ch), ref, UNIT * ab)
                raw = G[f"o{sj}.raw"]
            j += 1
    L = plan[-1]
    inp = {"x_elu": cur}
    within(tag, "wav", wav.double(), cr.layer(cfg, sd64, L, inp)["raw"], UNIT * cr.abs_bound(cfg, sd64, L, inp)["raw"])


def keep_decode(monkeypatch, cfg, sd, codes, env=()):
    """decode with and without VCB_CODEC_KEEP: the same launches, the same waveform bit for bit -> (tokenizer, waveform)"""
    for k, v in env:
        monkeypatch.setenv(k, v)
    monkeypatch.delenv("VCB_CODEC_KEEP", raising=False)
    plain = gpu_tok(cfg, sd)
    n0 = counter(plain, "launches")
    want = plain.decode_codes(codes.cuda()).cpu()
    n_plain = counter(plain, "launches") - n0
    assert counter(plain, "tc_decodes") == 1
    monkeypatch.setenv("VCB_CODEC_KEEP", "1")
    tok = gpu_tok(cfg, sd)
    n0 = counter(tok, "launches")
    wav = tok.decode_codes(codes.cuda()).cpu()
    assert counter(tok, "launches") - n0 == n_plain and counter(tok, "tc_decodes") == 1
    assert torch.equal(wav, want), "VCB_CODEC_KEEP changed the waveform"
    return tok, wav


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the tensor-core decoder, stage by stage
# ---------------------------------------------------------------------------------------------------------------------
def _stage_cases():
    out = []
    for name in CONFIGS:
        m = MIN_T[name]
        if name == "default":        # 75 MMAC per frame in float64, twice (layer and bound): the grid is thinned, every T kept
            grid = [("plain", 1, m), ("plain", 1, m + 1), ("plain", 3, 16), ("plain", 1, 17), ("plain", 1, 53), ("plain", 1, 128),
                    ("plain", 3, 129), ("lstm_integrating", 3, 53), ("offset", 3, 17), ("tiny_out", 1, 53)]
        else:
            # (the offset regime is built for one residual block per stage)
            regimes = ["plain", "tiny_out"] + (["lstm_integrating", "offset"] if CONFIGS[name]["lstm"] else [])
            grid = [(r, B, T) for r in regimes for B in (1, 3) for T in (m, m + 1, 16, 17, 53, 128, 129)
                    if r == "plain" or (B, T) in ((3, 53), (1, 129))]
        out += [pytest.param(name, r, B, T, id=f"{name}-{r}-B{B}-T{T}") for r, B, T in grid]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,regime,B,T", _stage_cases())
def test_decoder_stage_vs_fp64(name, regime, B, T, monkeypatch):
    """Teacher-forced: tensor n against the float64 layer of the GPU's own tensor n-1, |err| <= UNIT x A + EPS_ELU per
    element (the module docstring derives it).  A stage's rows per utterance are T x {1, 8, 40, 160, 320} plus its halo, so the T
    values put some stage's row count on, just below and just above a multiple of the 128-row tile."""
    cfg = eo.default_config(**CONFIGS[name])
    sd = weights(cfg, regime, 40 + T)
    codes = rand_codes(cfg, B, T, 41 + T)
    tok, wav = keep_decode(monkeypatch, cfg, sd, codes)
    stage_checks(f"stage/{name}/{regime}", cfg, cr.double(sd), codes, tok, wav)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["plain", "tiny_out"])
def test_decoder_chain_vs_fp64(regime, monkeypatch):
    """Free-running, default codec, B = 3, T = 61: every stored tensor against the float64 run's tensor of the same name.
    Bound, relative to that tensor's own rms so a late stage cannot hide an early one: a tensor d layers deep carries
    the errors of d layers, each about 2^-16 of an rms-sized value when nothing cancels (A is then a few rms):
    rms(err) <= d x 2^-16 x rms(ref), and no element beyond 16 x that (the LSTM's h under tiny_out, whose gates sit on the
    steep part of the sigmoid with inputs of O(10), has the heaviest tail: 9.7 x on an H100)."""
    cfg = eo.default_config()
    sd = weights(cfg, regime, 7)
    codes = rand_codes(cfg, 3, 61, 15)
    tok, wav = keep_decode(monkeypatch, cfg, sd, codes)
    _, rec = eo.decode(cfg, cr.double(sd), codes, return_intermediates=True)
    depth = 0
    for name, ref in rec.items():
        if name.startswith("c"):
            continue
        depth += 0 if name.endswith(".elu") or name.endswith(".raw") and name.startswith("o") else 1
        got = wav.double() if name == "wav" else fetch(tok, name)
        if name != "wav":
            if got is None:
                continue
            got = got[0][:, :ref.shape[1], got[1]:]
        rms = ref.pow(2).mean().sqrt().item()
        err = got - ref
        lim = depth * 2.0 ** -16 * rms
        r_rms, r_max = err.pow(2).mean().sqrt().item() / lim, err.abs().max().item() / (16 * lim)
        RATIOS[f"chain/{regime}"] = max(RATIOS.get(f"chain/{regime}", 0.0), r_rms, r_max)
        print(f"RATIO chain/{regime} {name} rms {r_rms:.4f} max {r_max:.4f}")
        assert r_rms <= 1.0 and r_max <= 1.0, (name, r_rms, r_max)


@pytest.mark.gpu
@pytest.mark.parametrize("wide", ["0", "1"])
@pytest.mark.parametrize("regime", ["plain", "lstm_integrating"])
def test_lstm_800_steps_vs_fp64(regime, wide, monkeypatch):
    """Default codec, T = 800, B = 2, 64- and 128-column step tiles.  Each step is fed the h the GPU stored for the step
    before while the cell state runs free in float64, so the cell's drift over 800 dependent steps is in the comparison:
    hs0, hs1 at every step against codec_ref.lstm_teacher_forced's bound (the recurrence in its docstring: a gate error
    of UNIT x A per step, carried by the forget gate, so about 1 / (1 - f) steps' worth, not 800), the final cell states
    c0, c1 (the only cell states the decoder keeps) against the same recurrence, and u0."""
    cfg = eo.default_config()
    sd = weights(cfg, regime, 31)
    codes = rand_codes(cfg, 2, 800, 32)
    monkeypatch.setenv("VCB_CODEC_LSTM_WIDE", wide)
    monkeypatch.setenv("VCB_CODEC_KEEP", "1")
    tok = gpu_tok(cfg, sd)
    tok.decode_codes(codes.cuda())
    assert counter(tok, "tc_decodes") == 1
    sd64 = cr.double(sd)
    tag = f"lstm800/{regime}/wide{wide}"
    H = 1024
    x0, halo = fetch(tok, "x0")
    x = x0[:, :, halo:].permute(2, 0, 1)
    rec = {}
    for l in (0, 1):
        full, halo = fetch(tok, f"hs{l}")
        hs = full[:, :H, halo:].permute(2, 0, 1)
        h, c, eh, ec = cr.lstm_teacher_forced(sd64, "dec.lstm", l, x, hs, UNIT)
        rec[f"c{l}"], rec[f"hs{l}"] = c.permute(1, 2, 0), h.permute(1, 2, 0)
        for t in (0, 1, 7, 99, 400, 799):
            within(tag, f"hs{l}[t={t}]", hs[t], h[t], eh[t])
        within(tag, f"hs{l}", hs, h, eh)
        within(tag, f"c{l}", fetch(tok, f"c{l}")[0][:, :, 0], c[-1], ec[-1])
        x = hs
    if regime == "lstm_integrating":
        _assert_integrating(rec)
    u0, halo = fetch(tok, "u0")
    skip = x0[:, :, 0:].permute(2, 0, 1)
    ref = F.elu(x + skip).permute(1, 2, 0)
    # (x0 is added in fp32 and stored as hi + lo, u0 again: two roundings of 2^-17 that are both attained, so this
    # check runs close to its bound by construction)
    within(tag, "u0", u0[:, :H, halo:], ref, 2.0 ** -16 * (x.abs() + skip.abs()).permute(1, 2, 0) + EPS_ELU)


@pytest.mark.gpu
def test_full_length_waveform_vs_fp64():
    """Default codec, B = 1, T = 800: all 256 000 samples against float64, and the worst 320-sample frame, so a bad tile,
    TMA coordinate or halo beyond row 2^15 of a stage shows wherever it is."""
    cfg = eo.default_config()
    sd = weights(cfg, "plain", 31)
    codes = rand_codes(cfg, 1, 800, 33)
    tok = gpu_tok(cfg, sd)
    wav = tok.decode_codes(codes.cuda()).cpu().double()
    assert counter(tok, "tc_decodes") == 1
    ref, bound = wav_bound(cfg, cr.double(sd), codes)
    within("full_length", "wav", wav, ref, torch.full_like(ref, bound))
    frames_err = (wav - ref).pow(2).view(800, 320).sum(1)
    frames_ref = ref.pow(2).view(800, 320).sum(1)
    worst = (10 * torch.log10(frames_ref / frames_err.clamp_min(1e-300))).min().item()
    total = snr_db(wav, ref)
    print(f"RATIO full_length snr {total:.1f} dB worst frame {worst:.1f} dB")
    assert total >= 80.0 and worst >= 70.0, (total, worst)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: batches at the real codec shape, the switch between the decoders, the CUDA-core decoder
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tc,B", [("1", b) for b in (1, 16, 17, 32, 127, 128, 129, 200)] + [("0", b) for b in (16, 17, 33)])
def test_batch_rows_at_real_shape(tc, B, monkeypatch):
    """Default codec, T = 24.  B = 129 is the first batch with a second 128-row tile in every LSTM step and another
    stride of the time-major planes; the CUDA-core decoder (VCB_CODEC_TC=0) takes 16 utterances per chunk, so B = 17 is
    its first second chunk.  Row b of the batch is row b decoded alone, bit for bit, and rows 0 and B-1 meet the float64 bound."""
    monkeypatch.setenv("VCB_CODEC_TC", tc)
    cfg = eo.default_config()
    sd = weights(cfg, "plain", 9)
    codes = rand_codes(cfg, B, 24, 10)
    tok = gpu_tok(cfg, sd)
    full = tok.decode_codes(codes.cuda())
    assert counter(tok, "tc_decodes") == int(tc)
    for b in sorted({0, 15, 16, 127, 128, B - 1}):
        if b < B:
            assert torch.equal(full[b:b + 1], tok.decode_codes(codes[b:b + 1].cuda())), f"row {b} of {B}"
    rows = sorted({0, B - 1})
    ref, bound = wav_bound(cfg, cr.double(sd), codes[rows])
    within(f"batch/tc{tc}", f"B={B}", full[rows].cpu().double(), ref, torch.full_like(ref, bound))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["default", "two_res_no_lstm"])
def test_fallback_boundary(name, monkeypatch):
    """T = 1 .. min_T + 1: the tensor-core decoder runs exactly from stream_min_frames on, both decoders meet the float64
    bound on either side of the switch, and at T = min_T (the reflect halo as long as the signal it mirrors) they agree
    within twice that bound."""
    cfg = eo.default_config(**CONFIGS[name])
    sd = weights(cfg, "plain", 51)
    sd64 = cr.double(sd)
    tok = gpu_tok(cfg, sd)
    tok._engine()                                                          # the knob is read when the engine is built
    monkeypatch.setenv("VCB_CODEC_TC", "0")
    core = gpu_tok(cfg, sd)
    core._engine()
    min_T = counter(tok, "stream_min_frames")
    assert min_T == MIN_T[name] and counter(core, "tc_enabled") == 0
    for T in range(1, min_T + 2):
        codes = rand_codes(cfg, 2, T, 52 + T)
        n0 = counter(tok, "tc_decodes")
        wav = tok.decode_codes(codes.cuda()).cpu().double()
        assert counter(tok, "tc_decodes") - n0 == int(T >= min_T), T
        ref, bound = wav_bound(cfg, sd64, codes)
        within(f"fallback/{name}", f"T={T}", wav, ref, torch.full_like(ref, bound))
        if T >= min_T:
            other = core.decode_codes(codes.cuda()).cpu().double()
            within(f"fallback/{name}", f"T={T} cuda-core", other, ref, torch.full_like(ref, bound))
            assert (other - wav).abs().max().item() <= 2 * bound


@pytest.mark.gpu
@pytest.mark.parametrize("name,regime", [("mid_default", "plain"), ("mid_default", "lstm_integrating"), ("mid_default", "offset"),
                                         ("mid_default", "tiny_out"), ("default", "lstm_integrating"), ("default", "offset"),
                                         ("default", "tiny_out"), ("small_noncausal_trueskip", "plain"),
                                         ("small_noncausal_trueskip", "lstm_integrating")])
def test_cuda_core_decoder_vs_fp64(name, regime, monkeypatch):
    """VCB_CODEC_TC=0 (and the non-causal, identity-skip codec only these kernels serve), T = 37, B = 2, free-running:
    plain fp32 kernels, so the waveform is within the depth x FP32_UNIT x A bound (wav_bound with the fp32 unit)."""
    monkeypatch.setenv("VCB_CODEC_TC", "0")
    cfg = eo.default_config(**(CASES[name][0] if name != "default" else {}))
    sd = weights(cfg, regime, 61)
    codes = rand_codes(cfg, 2, 37, 62)
    tok = gpu_tok(cfg, sd)
    wav = tok.decode_codes(codes.cuda()).cpu().double()
    assert counter(tok, "tc_enabled") == 0
    ref, bound = wav_bound(cfg, cr.double(sd), codes)
    if regime == "offset":
        # the cancelled sums lose A / |sum| of relative accuracy at every stage: the bound is stated on the stage that
        # cancels (x 20 offset over O(1) signal), not on the last conv
        bound *= 20
    within(f"cuda_core/{name}", regime, wav, ref, torch.full_like(ref, bound * FP32_UNIT / UNIT + 2.0 ** -20))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the encoder
# ---------------------------------------------------------------------------------------------------------------------
def _encode(monkeypatch, cfg, sd, wav):
    monkeypatch.setenv("VCB_CODEC_KEEP", "1")
    tok = gpu_tok(cfg, sd)
    codes = tok.encode_codes(wav.cuda()).cpu()
    lat, halo = fetch(tok, "enc.latent")
    assert halo == 0
    return tok, codes, lat


@pytest.mark.gpu
@pytest.mark.parametrize("N,B", [(319, 1), (320, 2), (321, 17), (16000, 1), (16001, 2), (2563, 17), (79999, 1), (160000, 1)])
def test_encoder_latent_vs_fp64(N, B, monkeypatch):
    """The latent the GPU quantises ("enc.latent") against float64, frame by frame: |err|_2 <= 1e-4 |ref|_2 per frame.
    The encoder is 15 fp32 layers of K <= 3584 and an LSTM: sqrt(K) 2^-24 = 3.6e-6 per layer when nothing cancels, about
    5e-5 in all; an encoder wrong by 1e-3, which changes few codes, fails.  N off a multiple of the hop takes the extra
    right padding of every strided conv; B = 17 the second chunk of 16 utterances; frames = ceil-chain of the ratios."""
    cfg = eo.default_config()
    sd = weights(cfg, "plain", 11, encoder=True)
    wav = 0.3 * torch.randn(B, 1, N, generator=torch.Generator().manual_seed(N))
    tok, codes, lat = _encode(monkeypatch, cfg, sd, wav)
    T = N
    for r in reversed(cfg.ratios):
        T = -(-T // r)
    assert lat.shape == (B, cfg.dimension, T) and codes.shape == (B, cfg.n_q, T)
    ref = eo.encode_latent(cfg, cr.double(sd), wav.double())
    ratio = ((lat - ref).norm(dim=1) / (1e-4 * ref.norm(dim=1))).max().item()
    RATIOS["enc_latent"] = max(RATIOS.get("enc_latent", 0.0), ratio)
    print(f"RATIO enc_latent N={N} B={B} {ratio:.4f}")
    assert ratio <= 1.0, ratio
    with pytest.raises(_lib().VcbError, match="no tensor|not active"):
        _lib().check(_lib().load().enc_debug_tensor(tok._engine(), b"enc.nothing", None, 0, (C.c_int32 * 4)()))


@pytest.mark.gpu
@pytest.mark.parametrize("B", [2, 17, 33])
def test_rvq_codes_given_the_gpu_latent(B, monkeypatch):
    """The codes are the nearest codes of the GPU's own latent: at every stage, with the residual the GPU's earlier codes
    leave, no code is closer than the chosen one by more than 4e-5 in squared distance (the scores are 128-term fp32
    sums of magnitude about 16: sqrt(128) 2^-24 x 16 x 2 = 2e-5).  This separates a drifting encoder from a wrong search.
    Codebook 1 holds a duplicated row, so every frame that picks it is an exact tie, and either index is right."""
    cfg = eo.default_config()
    sd = weights(cfg, "plain", 13, encoder=True)
    sd["vq.1.embed"][7] = sd["vq.1.embed"][3]
    wav = 0.3 * torch.randn(B, 1, 4801, generator=torch.Generator().manual_seed(B))
    _, codes, lat = _encode(monkeypatch, cfg, sd, wav)
    sd64 = cr.double(sd)
    resid = lat.transpose(1, 2).reshape(-1, cfg.dimension)
    worst = 0.0
    for q in range(cfg.n_q):
        emb = sd64[f"vq.{q}.embed"]
        dist = torch.cdist(resid, emb).pow(2)
        idx = codes[:, q].reshape(-1)
        assert int(idx.min()) >= 0 and int(idx.max()) < cfg.bins
        worst = max(worst, (dist.gather(1, idx[:, None])[:, 0] - dist.min(dim=1).values).max().item())
        resid = resid - emb[idx]
    print(f"RATIO rvq B={B} {worst / 4e-5:.4f}")
    assert worst <= 4e-5, worst


# ---------------------------------------------------------------------------------------------------------------------
# GPU: stream state with cells that remember
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_stream_state_under_integration():
    """CodecStream pushes of uneven lengths with lstm_integrating weights, bit for bit the one-shot decode: a cell state
    carried wrongly (or not frozen at a stream's last valid step while longer rows of the call go on) does not decay
    away here as it does with forgetting cells."""
    cfg = eo.default_config()
    sd = weights(cfg, "lstm_integrating", 71)
    tok = gpu_tok(cfg, sd)
    m = counter(tok, "stream_min_frames")
    total = [m + 1 + 37 + 9, m + 3 + 1 + 20, m]                           # stream 2 ends after the first call
    codes = [rand_codes(cfg, 1, n, 72 + i)[0] for i, n in enumerate(total)]
    want = [tok.decode_codes(c[None].cuda())[0] for c in codes]
    calls = [([0, 1, 2], [m, m + 3, m]), ([1, 0], [1, 1]), ([0, 1], [37, 20]), ([0], [9])]
    got, pos = [[] for _ in total], [0] * len(total)
    with tok.open_stream(max_streams=3) as cs:
        for ids, lens in calls:
            T = max(lens)
            batch = torch.zeros(len(ids), cfg.n_q, T, dtype=torch.long)
            for r, (i, n) in enumerate(zip(ids, lens)):
                batch[r, :, :n] = codes[i][:, pos[i]:pos[i] + n]
            wav = cs.decode(batch.cuda(), ids=ids, lens=lens)
            for r, (i, n) in enumerate(zip(ids, lens)):
                got[i].append(wav[r, :, :n * 320])
                pos[i] += n
    for i in range(len(total)):
        assert pos[i] == total[i] and torch.equal(torch.cat(got[i], -1), want[i]), f"stream {i}"
