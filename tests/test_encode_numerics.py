"""The tensor-core EnCodec encoder (csrc/codec_tc.cu, enc_encode_ragged) stage by stage against float64, in every
configuration it serves, row by row over ragged multi-row chunks, and in its default workspace.

On the GPU (-m gpu) every tensor the encoder stores is read back under VCB_CODEC_KEEP=1 and compared, for every checked
row of the chunk over that row's own stage lengths, with the float64 layer (oracle/encodec_oracle.py through codec_ref)
applied to the tensor the GPU stored one stage earlier for that row.  Which tensors exist, under which names and with
which halos, is derived from eo.encoder_plan (enc_tensors), not written down for one configuration.  Outside KEEP the
stages share two arenas; that layout is tied to the checked one by requiring the same codes bit for bit.

Bounds.  Every GEMM multiplies bf16 (hi, lo) pairs in three passes with fp32 accumulation.  Relative to
A = sum |a||w| + |bias| of the output element (codec_ref.abs_bound):
    weight and activation as hi + lo: 2^-17 each;  the dropped lo*lo: 2^-18;  the output stored as hi + lo: 2^-17;
    fp32 accumulation over K terms: about sqrt(K) 2^-24.
The encoder's reductions are deeper than the decoder's: enc.conv_in K = 64 (the 7-sample window as one k-block), the
residual blocks K = 3 C and hidden + C, the LSTM 1024 per gate, enc.conv_out 7 x 1024 = 7168, and the strided convs
K = 2 r C, up to 2 x 8 x 512 = 8192 for the last one.  At K = 8192 the accumulation term is sqrt(8192) 2^-24 = 0.35 x 2^-16
(0.23 x 2^-16 at the decoder's K = 3584), so the sum is 1.75 x 2^-16 + 0.35 x 2^-16 = 2.1 x 2^-16 A, still under
UNIT = 3 x 2^-16.  An ELU'd tensor adds EPS_ELU = 5e-7 absolute (ex2.approx and fp32 rounding of a value <= 1); where A
itself is 0 (padding rows) the bound is 1e-30, so those rows must be exact.  An LSTM layer is teacher-forced on the h the
encoder stored (codec_ref.lstm_teacher_forced, plus 2^-20 absolute as in test_encode_tc).
The RVQ search is fp32: a score e.r - |e|^2/2 is a D-term dot product and one more term, wrong by at most about
(D + 2) 2^-24 (sum |e_i r_i| + |e|^2/2), and the residual it is taken of has drifted from the exact one by 2^-24 |r| per
earlier stage; the chosen code's squared distance may exceed the best one's by twice the two scores' errors.
The largest observed error of every check is printed as a fraction of its bound (RATIO lines, pytest -rP).  The weights
are random (no trained checkpoint is available offline): nothing here measures a trained codec's margins."""
import math

import pytest
import torch
import torch.nn.functional as F

import codec_ref as cr
from oracle import encodec_oracle as eo
from test_codec_numerics import SMALL, check_structure, fetch, lstm_integrating, within
from test_encode_tc import chain, ragged, valid

UNIT = 3 * 2.0 ** -16
EPS_ELU = 5e-7

ENC_CONFIGS = {
    "default": {},
    "small_constpad": dict(SMALL, lstm=1, pad_mode="constant"),
    "two_res_no_lstm": dict(SMALL, lstm=0, n_residual_layers=2),
    "small_lstm2": dict(SMALL, lstm=2),
    "three_res": dict(SMALL, n_residual_layers=3),             # intermediate halos of 4 and 8 rows
    "ratios_442": dict(SMALL, ratios=[4, 4, 2]),               # three stages, other fold widths, a 64-unit LSTM
    "small_lstm3": dict(SMALL, lstm=3),                        # layer 2 overwrites layer 0's h plane
}


def config(name):
    return eo.default_config(**ENC_CONFIGS[name])


# ---------------------------------------------------------------------------------------------------------------------
# the plan: tensors, names, halos, lengths
# ---------------------------------------------------------------------------------------------------------------------
def enc_tensors(cfg):
    """The tensors the tensor-core encoder stores, in launch order, derived from eo.encoder_plan.  Per tensor: its debug
    names ("raw" / "elu": None where that form is not stored or not named), stage (0 = samples, one more per strided
    conv), real channels C, halo rows and what they hold ("reflect", "zero", or "unwritten" for a residual block's hidden
    tensor), time-major layout, the plan entry that writes it ("writer"), and the stride of the strided conv that reads it
    past its end ("rpad", 0 if none)."""
    plan = eo.encoder_plan(cfg)
    n, nres, nl, kres = len(cfg.ratios), cfg.n_residual_layers, cfg.lstm, cfg.residual_kernel_size
    ratios = list(reversed(cfg.ratios))
    pad = "reflect" if cfg.pad_mode == "reflect" else "zero"

    def t(raw, elu, stage, C, halo, kind, writer, tm=False, rpad=0):
        return dict(raw=raw, elu=elu, stage=stage, C=C, halo=halo, kind=kind, tm=tm, writer=writer, rpad=rpad)

    def block_input(s, C, name, writer):
        if nres > 0:                                      # read by the first residual block (raw by its shortcut)
            return t(name, name + ".elu", s, C, kres - 1, pad, writer)
        return t(None, name + ".elu", s, C, ratios[s], pad, writer, rpad=ratios[s])     # read by the strided conv only

    out = [t("enc.input", None, 0, cfg.kernel_size, 0, "zero", None)]
    for L in plan:
        name = L["name"]
        s = int(name.split(".")[1][len("down"):]) if name.startswith("enc.down") else n
        if name == "enc.conv_in":
            out.append(block_input(0, L["cout"], "enc.x0", name))
        elif L["kind"] == "res":
            j = int(name.rsplit("res", 1)[1])
            out.append(t(None, name + ".h", s, L["hidden"], out[-1]["halo"], "unwritten", name))
            if j == nres - 1:
                out.append(t(None, name + ".elu", s, L["dim"], ratios[s], pad, name, rpad=ratios[s]))
            else:                                         # the next block's conv1 reads (kres - 1) x its dilation back
                out.append(t(name, name + ".elu", s, L["dim"], (kres - 1) * L["dil"] * cfg.dilation_base, pad, name))
        elif L["kind"] == "conv" and "stride" in L and L["stride"] > 1:
            if s < n - 1:
                out.append(block_input(s + 1, L["cout"], name, name))
            elif nl:
                out.append(t(name, None, n, L["cout"], 0, "zero", name, tm=True))
            else:                                         # straight into enc.conv_out's input
                out.append(t(None, "enc.lstm", n, L["cout"], cfg.last_kernel_size - 1, pad, name))
        elif L["kind"] == "lstm":
            for l in range(min(nl, 2)):
                out.append(t(f"enc.hs{l}", None, n, L["dim"], 1, "zero", name, tm=True))
            out.append(t(None, "enc.lstm", n, L["dim"], cfg.last_kernel_size - 1, pad, name))
    return out


def lstm_checkable(nl):
    """LSTM layers whose input and output h sequences are both still in the two hs planes after the last layer ran
    (layer l writes plane l % 2, so from 3 layers on only the last layer's input and output survive)"""
    return [l for l in range(nl) if l >= nl - 2 and (l == 0 or l - 1 >= nl - 2)]


def hop(cfg):
    return math.prod(cfg.ratios)


def enc_rows(cfg, n):
    """plane rows per utterance of every stage (enc_rows in codec_tc.cu): the stage length rounded up to its stride"""
    L = chain(cfg, n)
    return [-(-L[s] // r) * r for s, r in enumerate(reversed(cfg.ratios))] + [L[-1]]


def tc_accepts(cfg, n):
    """tc_encoder_accepts restated: with reflect padding every stage longer than the padding its convolutions reflect"""
    if n < 1:
        return False
    if cfg.pad_mode != "reflect":
        return True
    L = chain(cfg, n)
    nres = cfg.n_residual_layers
    res_pad = (cfg.residual_kernel_size - 1) * cfg.dilation_base ** (nres - 1) if nres else 0
    if L[0] <= cfg.kernel_size - 1:
        return False
    if any(L[s] <= res_pad or L[s] <= r for s, r in enumerate(reversed(cfg.ratios))):
        return False
    return L[-1] > cfg.last_kernel_size - 1


def min_accepted(cfg):
    n = 1
    while not tc_accepts(cfg, n):
        n += 1
    return n


def fold_lengths(cfg):
    """(below, on, above).  N = hop (T - 1) + 1 takes the maximal right padding, r - 1 rows, at every stage.  The last
    strided conv's input (halo r, r T rows) then has r (T + 1) plane rows per utterance: a multiple of 128 at
    T = 128 / r - 1, one folded row (r plane rows) below and above it at T -/+ 1."""
    r = cfg.ratios[0]
    T = 128 // r - 1
    return [hop(cfg) * (t - 1) + 1 for t in (T - 1, T, T + 1)]


# ---------------------------------------------------------------------------------------------------------------------
# regimes: weights and input.  Each stands in for something a trained codec or real audio does to the kernels.
# ---------------------------------------------------------------------------------------------------------------------
def enc_offset(cfg, sd, seed):
    """Each strided conv but the last puts +20 or -20 on every channel of the next stage (its bias), so that stage's ELU
    runs both branches at scale; the next stage's first residual block has conv1 (on the ELU'd input) and shortcut (on
    the raw one) orthogonal to that offset, so the large terms cancel in their sums."""
    g = torch.Generator().manual_seed(seed)
    for s in range(len(cfg.ratios) - 1):
        b = sd[f"enc.down{s}.conv.bias"]
        v = 20.0 * (2.0 * torch.randint(0, 2, b.shape, generator=g) - 1.0)
        b += v
        for name, e in ((f"enc.down{s + 1}.res0.conv1.weight", F.elu(v)), (f"enc.down{s + 1}.res0.shortcut.weight", v)):
            w = sd[name]
            w -= (w * e[None, :, None]).sum(1, keepdim=True) * e[None, :, None] / (e * e).sum()
    return sd


def plain_wav(n, g):
    return 0.3 * torch.randn(1, n, generator=g)


def quiet_wav(n, g):
    """1e-4 amplitude with two stretches of exact digital silence, one at the start (which the left padding mirrors)"""
    w = 1e-4 * torch.randn(1, n, generator=g)
    w[:, :n // 4] = 0.0
    w[:, n // 2:n // 2 + n // 5] = 0.0
    return w


def loud_wav(n, g):
    """full-scale noise around a 0.5 DC offset, clipped to +-1"""
    return (0.5 + torch.randn(1, n, generator=g)).clamp(-1.0, 1.0)


IDENTITY = lambda cfg, sd, seed: sd                                        # noqa: E731
REGIMES = {"plain": (IDENTITY, plain_wav), "lstm_integrating": (lstm_integrating, plain_wav), "offset": (enc_offset, plain_wav),
           "quiet": (IDENTITY, quiet_wav), "loud": (IDENTITY, loud_wav)}


def enc_weights(cfg, regime, seed):
    sd = eo.make_state_dict(cfg, seed=seed, encoder=True)
    sd["vq.1.embed"][7] = sd["vq.1.embed"][3]          # an exact tie in codebook 1: either index is the nearest code
    return REGIMES[regime][0](cfg, sd, seed)


def enc_wavs(regime, lengths, seed):
    g = torch.Generator().manual_seed(seed)
    return [REGIMES[regime][1](n, g) for n in lengths]


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(ENC_CONFIGS))
def test_tensor_walk_follows_the_plan(name):
    """enc_tensors against eo.encoder_plan: every plan entry but enc.conv_out writes a stored tensor, names are unique,
    a residual block's hidden tensor shares its input's halo, each intermediate block output keeps the halo the next
    block's dilated conv1 reads, every strided conv's input holds r rows of halo and its right padding, and the forms
    without a name are the ones the plan never stores."""
    cfg = config(name)
    plan = eo.encoder_plan(cfg)
    walk = enc_tensors(cfg)
    n, nres, nl = len(cfg.ratios), cfg.n_residual_layers, cfg.lstm
    names = [x for t in walk for x in (t["raw"], t["elu"]) if x is not None]
    assert len(names) == len(set(names))
    assert {t["writer"] for t in walk[1:]} == {L["name"] for L in plan[:-1]}
    assert tc_accepts(cfg, min_accepted(cfg)) and not tc_accepts(cfg, min_accepted(cfg) - 1)
    for L in plan:
        mine = [t for t in walk if t["writer"] == L["name"]]
        if L["kind"] == "res":
            h, o = mine
            assert h["halo"] == walk[walk.index(h) - 1]["halo"] and h["C"] == L["hidden"]
            if not L["name"].endswith(f"res{nres - 1}"):
                nxt = [P for P in plan if P["kind"] == "res" and P["name"].startswith(L["name"][:-1])
                       and int(P["name"].rsplit("res", 1)[1]) == int(L["name"].rsplit("res", 1)[1]) + 1][0]
                assert o["halo"] == (cfg.residual_kernel_size - 1) * nxt["dil"] and o["raw"] == L["name"]
        if "stride" in L and L["stride"] > 1:
            src = walk[walk.index(mine[0]) - 1]
            assert src["rpad"] == src["halo"] == L["stride"] and src["elu"] is not None
    if name == "three_res":
        assert [t["halo"] for t in walk if t["raw"] and ".res" in t["raw"]] == [4, 8] * n
    assert (f"enc.down{n - 1}.conv" in names) == bool(nl)
    assert ("enc.x0" in names) == (nres > 0)
    assert [x for x in names if x.startswith("enc.hs")] == [f"enc.hs{l}" for l in range(min(nl, 2))]
    assert names[-1] == "enc.lstm"
    assert lstm_checkable(nl) == {0: [], 1: [0], 2: [0, 1]}.get(nl, [nl - 1])
    below, on, above = fold_lengths(cfg)
    r = cfg.ratios[0]
    assert tc_accepts(cfg, below)
    for N, rows in ((below, 128 - r), (on, 128), (above, 128 + r)):
        L, R = chain(cfg, N), enc_rows(cfg, N)
        assert all(L[s] % rr == 1 % rr for s, rr in enumerate(reversed(cfg.ratios)))       # maximal right padding
        assert R[n - 1] + r == rows


def test_regimes_do_what_they_say():
    """On the float64 reference, at the sizes the GPU tests use: quiet input is 1e-4 with exact silence, where enc.conv_in
    is its bias exactly; loud input is clipped at full scale around its offset; offset puts +-20 on the next stage and
    its first block cancels it; lstm_integrating cells keep integrating over the frames of a fold_lengths row."""
    cfg = config("small_lstm2")
    n = fold_lengths(cfg)[1]
    q = quiet_wav(n, torch.Generator().manual_seed(1))
    assert q.abs().max() <= 1e-3 and (q == 0).double().mean() >= 0.4 and q[0, -1] != 0
    sd = cr.double(enc_weights(cfg, "plain", 2))
    _, rec = eo.encode_latent(cfg, sd, q[None].double(), return_intermediates=True)
    x = rec["enc.conv_in"][0]
    b = sd["enc.conv_in.bias"][:, None]
    assert torch.equal(x[:, cfg.kernel_size:n // 4], b.expand(-1, n // 4 - cfg.kernel_size))
    assert (x - b).abs().max() <= 1e-3
    ld = loud_wav(n, torch.Generator().manual_seed(3))
    assert ld.abs().max() == 1.0 and (ld.abs() == 1.0).double().mean() >= 0.3 and ld.mean() >= 0.3
    sd = cr.double(enc_weights(cfg, "offset", 4))
    _, rec = eo.encode_latent(cfg, sd, plain_wav(n, torch.Generator().manual_seed(4))[None].double(), return_intermediates=True)
    x = rec["enc.down0.conv"]
    assert (x.abs() > 10).double().mean() > 0.9 and (x > 10).any() and (x < -10).any()
    L = [P for P in eo.encoder_plan(cfg) if P["name"] == "enc.down1.res0"][0]
    ab = cr.abs_bound(cfg, sd, L, {"x": x})["h"]
    h = eo.conv1d(cfg, F.elu(x), sd[L["name"] + ".conv1.weight"], sd[L["name"] + ".conv1.bias"], L["dil"])
    assert (ab >= 100 * h.abs()).double().mean() >= 0.25
    assert rec["enc.down1.res0"].abs().max() < 10                      # the block output is back to O(1)
    sd = cr.double(enc_weights(cfg, "lstm_integrating", 5))
    _, rec = eo.encode_latent(cfg, sd, plain_wav(n, torch.Generator().manual_seed(5))[None].double(), return_intermediates=True)
    states = {}
    eo.lstm(rec[f"enc.down{len(cfg.ratios) - 1}.conv"].permute(2, 0, 1), sd, "enc.lstm", cfg.lstm, states)
    for l in range(cfg.lstm):
        c = states[f"c{l}"].abs()
        assert c[-1].median() >= 3.0 * c[0].median() and c[-1].max() >= 5.0, (l, c[0].median(), c[-1].median(), c[-1].max())


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


def input_window(cfg, w):
    """what enc.input holds for a wav row [N]: channel j at row t = sample t - (k-1) + j, left padding folded in"""
    k = cfg.kernel_size
    x = w.double().reshape(1, 1, -1)
    p = eo._pad1d(x, k - 1, 0, cfg.pad_mode) if cfg.pad_mode == "reflect" else F.pad(x, (k - 1, 0))
    return p[0, 0].unfold(0, k, 1).t()                                     # [k, N]


def chunk_order(cfg, inp, wavs):
    """chunk row -> input row, read from the stored enc.input plane: row j is the wav whose samples it holds (within the
    hi + lo split, 2^-17 relative) up to that wav's length, and zeros after it"""
    k = cfg.kernel_size
    order = []
    for j in range(inp.shape[0]):
        hit = []
        for b, w in enumerate(wavs):
            N = w.shape[-1]
            if N > inp.shape[2]:
                continue
            want = input_window(cfg, w)
            if ((inp[j, :k, :N] - want).abs() <= 2.0 ** -16 * want.abs()).all() and (inp[j, :, N:] == 0).all():
                hit.append(b)
        assert len(hit) == 1, (j, hit)
        order.append(hit[0])
    assert sorted(order) == list(range(len(wavs)))
    return order


def enc_stage_checks(tag, cfg, sd64, wavs, tok, rows=None):
    """Every tensor the encoder stored for chunk rows `rows` (default: all) against the float64 layer applied to the
    tensor it stored one stage earlier for that row, over the row's own stage lengths; the structure of every plane
    (padded channels, halos, right padding); the latent; the codes of the call against the GPU's own latent.
    Needs the chunk's tensors: one enc_encode_ragged call of `wavs` under VCB_CODEC_KEEP=1 that made one chunk."""
    B = len(wavs)
    rows = list(range(B)) if rows is None else rows
    walk = enc_tensors(cfg)
    n, nl = len(cfg.ratios), cfg.lstm
    ratios = list(reversed(cfg.ratios))
    reflect = cfg.pad_mode == "reflect"
    plan = eo.encoder_plan(cfg)
    # (a plane's rows past the chunk's longest utterance, up to the stride, belong to no utterance and are never read by
    # a valid row: the structure is checked up to that utterance's length)
    Lmax = chain(cfg, max(w.shape[-1] for w in wavs))
    got = {}
    for t in walk:
        for form in ("raw", "elu"):
            nm = t[form]
            if nm is None:
                continue
            r = fetch(tok, nm)
            assert r is not None, nm
            full, halo = r
            assert full.shape[0] == B and halo == t["halo"], (nm, full.shape, halo, t)
            check_structure(cfg, nm, full[:, :, :halo + Lmax[t["stage"]]], halo, t["C"], t["kind"] == "zero")
            if nm == "enc.input":
                order = chunk_order(cfg, full, wavs)
            got[nm] = (full[rows], halo)
    # forms the plan does not store are not exposed either
    for nm in ["enc.x0" if cfg.n_residual_layers == 0 else None, f"enc.down{n - 1}.conv" if not nl else None,
               f"enc.hs{min(nl, 2)}", f"enc.down{n - 1}.res{cfg.n_residual_layers - 1}"]:
        assert nm is None or fetch(tok, nm) is None, nm
    lat = valid(tok, "enc.latent", cfg.dimension, chain(cfg, max(w.shape[-1] for w in wavs))[-1])

    for jj, j in enumerate(rows):
        b = order[j]
        Lb = chain(cfg, wavs[b].shape[-1])

        def stored(nm, t):
            full, halo = got[nm]
            return full[jj:jj + 1, :t["C"], halo:halo + Lb[t["stage"]]]

        def check_out(kind, t, ref, ab):
            if t["raw"]:
                within(f"{tag}/{kind}", f"{t['raw']} row {j}", stored(t["raw"], t), ref, UNIT * ab + 1e-30)
            if t["elu"]:
                within(f"{tag}/{kind}", f"{t['elu']} row {j}", stored(t["elu"], t), F.elu(ref), UNIT * ab + EPS_ELU)

        def forms(t):
            return {k: stored(t[f], t) for k, f in (("x", "raw"), ("x_elu", "elu")) if t[f]}

        it = iter(walk[1:])
        cur = None
        for P in plan:
            if P["name"] == "enc.conv_in":
                t = next(it)
                inp = {"x": wavs[b].double().reshape(1, 1, -1)}
                check_out("conv_in", t, cr.layer(cfg, sd64, P, inp)["raw"], cr.abs_bound(cfg, sd64, P, inp)["raw"])
                cur = t
            elif P["kind"] == "res":
                th, to = next(it), next(it)
                inp = forms(cur)
                ab = cr.abs_bound(cfg, sd64, P, inp)["h"]
                within(f"{tag}/res_h", f"{th['elu']} row {j}", stored(th["elu"], th), cr.layer(cfg, sd64, P, inp)["h"],
                       UNIT * ab + EPS_ELU)
                inp["h_elu"] = stored(th["elu"], th)
                check_out("res_out", to, cr.layer(cfg, sd64, P, inp)["raw"], cr.abs_bound(cfg, sd64, P, inp)["raw"])
                cur = to
            elif P["kind"] == "conv" and P["stride"] > 1:
                s, r = cur["stage"], P["stride"]
                # the right padding the strided conv reads past this row's end: rows L-2, L-3, ... or zeros
                full, halo = got[cur["elu"]]
                L = Lb[s]
                for i in range(-(-L // r) * r - L):
                    want = full[jj, :, halo + L - 2 - i] if reflect else torch.zeros_like(full[jj, :, 0])
                    assert torch.equal(full[jj, :, halo + L + i], want), (cur["elu"], j, i)
                t = next(it)
                inp = {"x_elu": stored(cur["elu"], cur)}
                check_out("down", t, cr.layer(cfg, sd64, P, inp)["raw"], cr.abs_bound(cfg, sd64, P, inp)["raw"])
                cur = t
            elif P["kind"] == "lstm":
                hs_t = [next(it) for _ in range(min(nl, 2))]
                u_t = next(it)
                x0 = stored(cur["raw"], cur).permute(2, 0, 1)                   # [T, 1, H]
                plane = {l: hs_t[l & 1] for l in range(nl)}
                for l in lstm_checkable(nl):
                    x_in = x0 if l == 0 else stored(plane[l - 1]["raw"], plane[l - 1]).permute(2, 0, 1)
                    hs = stored(plane[l]["raw"], plane[l]).permute(2, 0, 1)
                    h_ref, _, err_h, _ = cr.lstm_teacher_forced(sd64, "enc.lstm", l, x_in, hs, UNIT)
                    within(f"{tag}/lstm_h", f"layer {l} row {j}", hs, h_ref, err_h + 2.0 ** -20)
                h_last = stored(plane[nl - 1]["raw"], plane[nl - 1])
                x0 = x0.permute(1, 2, 0)
                within(f"{tag}/lstm_u", f"enc.lstm row {j}", stored(u_t["elu"], u_t), F.elu(h_last + x0),
                       EPS_ELU + 2.0 ** -16 * (h_last.abs() + x0.abs()))
                cur = u_t
            else:                                                                  # enc.conv_out -> the fp32 latent
                inp = {"x_elu": stored(cur["elu"], cur)}
                ref, ab = cr.layer(cfg, sd64, P, inp)["raw"], cr.abs_bound(cfg, sd64, P, inp)["raw"]
                within(f"{tag}/latent", f"row {j}", lat[b:b + 1, :, :Lb[-1]], ref, UNIT * ab + 1e-30)
        assert next(it, None) is None
    return order, lat


def nearest_codes(tag, cfg, sd64, lat, codes, frames):
    """The codes are the nearest codes of the GPU's own latent at every RVQ stage, each frame and code within the fp32
    search's slack (module docstring): |score error| <= (D + 2) 2^-24 (sum |e_i r_i| + |e|^2 / 2) + sum |e_i| drift_i,
    where drift bounds how far the search's fp32 residual is from the exact residual of the same codes."""
    D = cfg.dimension
    for b in range(codes.shape[0]):
        T = frames[b]
        r = lat[b, :, :T].t()
        drift = torch.zeros_like(r)
        gaps, slacks = [], []
        for q in range(cfg.n_q):
            emb = sd64[f"vq.{q}.embed"]
            idx = codes[b, q, :T]
            assert int(idx.min()) >= 0 and int(idx.max()) < cfg.bins
            dist = r.pow(2).sum(1, keepdim=True) - 2 * r @ emb.t() + emb.pow(2).sum(1)[None]
            best = dist.argmin(dim=1)

            def err(i):
                e = emb[i]
                return (D + 2) * 2.0 ** -24 * ((e * r).abs().sum(1) + e.pow(2).sum(1) / 2) + (e.abs() * drift).sum(1)
            gaps.append(dist.gather(1, idx[:, None])[:, 0] - dist.gather(1, best[:, None])[:, 0])
            slacks.append(2 * (err(idx) + err(best)))
            r = r - emb[idx]
            drift = drift + 2.0 ** -24 * r.abs()
        within(f"{tag}/rvq", f"row {b}", torch.stack(gaps).clamp_min(0), torch.zeros(cfg.n_q, T, dtype=torch.float64),
               torch.stack(slacks))
        assert (codes[b, :, T:] == 0).all(), b


# ---------------------------------------------------------------------------------------------------------------------
# GPU: every configuration stage by stage
# ---------------------------------------------------------------------------------------------------------------------
def _enc_cases():
    """Per configuration: a mixed chunk of three rows (the fold boundary, a middle length, the shortest accepted row),
    one folded row below and above the boundary, with constant padding the shortest rows, and every regime that applies
    on a mixed chunk.  The fp64 cost follows the samples checked, so the lengths stay near the fold boundary."""
    out = []
    for name in ENC_CONFIGS:
        cfg = config(name)
        below, on, above = fold_lengths(cfg)
        nmin = min_accepted(cfg)
        mid = (on + nmin) // 2 + 1
        grid = [("plain", "mixed", [on, mid, nmin]), ("plain", "below", [below]), ("plain", "above", [above, nmin + 1])]
        if cfg.pad_mode != "reflect":
            h = hop(cfg)
            grid += [("plain", "shortest", [1, 2, 3, 7, h - 1, h, h + 1]), ("plain", "one_sample", [1])]
        regimes = (["lstm_integrating"] if cfg.lstm else []) + ["offset", "quiet", "loud"]
        grid += [(r, "mixed", [on, mid]) for r in regimes]
        out += [pytest.param(name, r, lens, id=f"{name}-{r}-{what}") for r, what, lens in grid]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,regime,lens", _enc_cases())
def test_encoder_stage_vs_fp64(name, regime, lens, monkeypatch):
    """One chunk of rows with distinct lengths under VCB_CODEC_KEEP=1: every stored tensor of every row against float64
    (enc_stage_checks), the chunk rows in longest-first order, and the codes nearest of the GPU's latent.  A longer,
    loud call runs first, so the checked chunk lies in a workspace full of another chunk's data: a row, halo or padding
    the encoder does not write shows."""
    monkeypatch.setenv("VCB_CODEC_KEEP", "1")
    cfg = config(name)
    seed = 100 + len(lens) + lens[0] % 97
    sd = enc_weights(cfg, regime, seed)
    sd64 = cr.double(sd)
    wavs = enc_wavs(regime, lens, seed)
    tok = gpu_tok(cfg, sd)
    assert counter(tok, "tc_encoder") == 1, name
    N = max(max(lens), min_accepted(cfg))
    ragged(tok, enc_wavs("loud", [N + 2 * hop(cfg) + 3, N + hop(cfg)], seed + 1))
    r0 = counter(tok, "encode_rows")
    codes, frames = ragged(tok, wavs)
    assert counter(tok, "encode_rows") - r0 == len(lens) * enc_rows(cfg, max(lens))[0], "not one tensor-core chunk"
    assert frames == [chain(cfg, N)[-1] for N in lens]
    tag = f"enc/{name}/{regime}"
    order, lat = enc_stage_checks(tag, cfg, sd64, wavs, tok)
    assert order == sorted(range(len(lens)), key=lambda b: -lens[b])
    nearest_codes(tag, cfg, sd64, lat, codes, frames)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [129, 200])
def test_batch_rows_at_real_shape(B, monkeypatch):
    """Default codec, B short rows of distinct lengths just above the 1 920-sample minimum, in mixed order: the LSTM steps
    take a second 128-row tile (Bcap = 256).  Every row's codes and latent equal the row encoded alone, bit for bit, and
    chunk rows 0, 127, 128 and B-1 meet the float64 bounds stage by stage."""
    monkeypatch.setenv("VCB_CODEC_KEEP", "1")
    cfg = eo.default_config()
    sd = enc_weights(cfg, "plain", 81)
    sd64 = cr.double(sd)
    nmin = min_accepted(cfg)
    assert nmin == 1921
    lens = [nmin + 7 * i for i in range(B)]
    lens = [lens[p] for p in torch.randperm(B, generator=torch.Generator().manual_seed(B)).tolist()]
    wavs = enc_wavs("plain", lens, 82)
    tok = gpu_tok(cfg, sd)
    r0 = counter(tok, "encode_rows")
    codes, frames = ragged(tok, wavs)
    assert counter(tok, "encode_rows") - r0 == B * enc_rows(cfg, max(lens))[0]
    _, lat = enc_stage_checks(f"enc/batch{B}", cfg, sd64, wavs, tok, rows=[0, 127, 128, B - 1])
    nearest_codes(f"enc/batch{B}", cfg, sd64, lat, codes, frames)
    for b in range(B):
        alone, fa = ragged(tok, [wavs[b]])
        T = frames[b]
        assert fa == [T] and torch.equal(alone[0, :, :T], codes[b, :, :T]), b
        la = valid(tok, "enc.latent", cfg.dimension, T)
        assert torch.equal(la[0], lat[b, :, :T]), b


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ENC_CONFIGS))
def test_acceptance_boundary(name):
    """The longest length the tensor-core encoder declines and the shortest it takes (encode_rows counts the rows it
    ran), as tc_accepts states them; with constant padding a single sample is taken."""
    cfg = config(name)
    tok = gpu_tok(cfg, enc_weights(cfg, "plain", 91))
    assert counter(tok, "tc_encoder") == 1
    nmin = min_accepted(cfg)
    assert (nmin == 1) == (cfg.pad_mode != "reflect")
    for N in (nmin - 1, nmin):
        if N < 1:
            continue
        r0 = counter(tok, "encode_rows")
        codes, frames = ragged(tok, enc_wavs("plain", [N], N))
        assert frames == [chain(cfg, N)[-1]] and (codes >= 0).all()
        assert counter(tok, "encode_rows") - r0 == (enc_rows(cfg, N)[0] if N == nmin else 0), N


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ENC_CONFIGS))
def test_default_workspace_matches_keep(name, monkeypatch):
    """One ragged batch encoded four ways: with and without VCB_CODEC_KEEP (rows of their own for every tensor, the
    layout the stage checks read, against the two arenas the stages share), each in one chunk and with a workspace
    limit so small that every row is a chunk of its own.  The codes agree bit for bit, and KEEP launches the same."""
    cfg = config(name)
    sd = enc_weights(cfg, "plain", 95)
    below, on, above = fold_lengths(cfg)
    nmin = min_accepted(cfg)
    lens = [on, nmin, above, (on + nmin) // 2, below + 5]
    wavs = enc_wavs("plain", lens, 96)
    runs = {}
    for keep in ("0", "1"):
        for ws in (None, "1e-6"):
            monkeypatch.setenv("VCB_CODEC_KEEP", keep)
            if ws is None:
                monkeypatch.delenv("VCB_CODEC_WS_GB", raising=False)
            else:
                monkeypatch.setenv("VCB_CODEC_WS_GB", ws)
            tok = gpu_tok(cfg, sd)
            assert counter(tok, "tc_encoder") == 1
            l0, r0 = counter(tok, "launches"), counter(tok, "encode_rows")
            codes, frames = ragged(tok, wavs)
            runs[keep, ws] = (codes, frames, counter(tok, "launches") - l0, counter(tok, "encode_rows") - r0)
            del tok
    want = runs["1", None]
    assert want[3] == len(lens) * enc_rows(cfg, max(lens))[0]
    for (keep, ws), (codes, frames, launches, nrows) in runs.items():
        assert frames == want[1] and torch.equal(codes, want[0]), (keep, ws)
        assert launches == runs["1", ws][2], (keep, ws, launches, runs["1", ws][2])
        assert nrows == (want[3] if ws is None else sum(enc_rows(cfg, N)[0] for N in lens)), (keep, ws)
