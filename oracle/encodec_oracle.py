"""TEST INFRASTRUCTURE ONLY -- torch-CPU fp32 restatement of EnCodec token -> waveform decode (and, for SURVEY.md
section 8f row f1, of the waveform -> token encode: SEANetEncoder + ResidualVectorQuantizer.encode, data/tokenizer.py:127-129).

The reference calls ``audiocraft`` (facebookresearch/audiocraft @ c5157b5bf14bf83449c17ea1eeb66c19fb4bc7f0,
un-vendored, NOT installable offline) at data/tokenizer.py:109-110 (model load) and :131-133
(``self.codec.decode(frames)``).  This module restates that dependency's published algorithm:

  EncodecModel.decode            = quantizer.decode(codes) -> decoder(latent)            (audiocraft models/encodec.py)
  ResidualVectorQuantizer.decode = sum_k codebook_k[codes[:, k, :]]                       (quantization/core_vq.py)
  SEANetDecoder                  = conv k7 -> LSTM(n layers, + skip) -> n x [ELU, ConvTranspose1d(k=2r, stride r),
                                   ResBlock(ELU, conv k3 dil d, ELU, conv k1, + skip)] -> ELU -> conv k7
                                                                                         (modules/seanet.py, conv.py, lstm.py)
  StreamableConv1d padding       = causal: left pad (k-1)*dil ; else split ; 'reflect' or 'constant'
  StreamableConvTranspose1d trim = causal: trim right ceil(pad * trim_right_ratio); else split

PARITY UNPINNED BY THE REFERENCE: the reference has no test or golden vector at this boundary and audiocraft
cannot be imported here.  The restatement is pinned instead against the structurally identical, importable
``transformers.models.encodec.modeling_encodec.EncodecModel`` (same layer algebra; tests/golden/make_golden_codec.py
runs it in the build container and commits input/output fixtures).  Weight-norm is folded by the caller
(w = g * v / ||v||), as audiocraft does at load for inference.
"""
import math
from types import SimpleNamespace

import torch
import torch.nn.functional as F


def default_config(**over):
    """16 kHz / 50 Hz / 4 x 2048 codec the reference uses (README.md:198, config.py:51; SURVEY.md section 7 hard parts)."""
    c = dict(n_q=4, bins=2048, dimension=128, n_filters=64, ratios=[8, 5, 4, 2], kernel_size=7, last_kernel_size=7,
             residual_kernel_size=3, dilation_base=2, n_residual_layers=1, compress=2, lstm=2, causal=True,
             pad_mode="reflect", true_skip=False, trim_right_ratio=1.0, channels=1, sample_rate=16000)
    c.update(over)
    return SimpleNamespace(**c)


def layer_plan(cfg):
    """The decoder as a flat list of layer descriptors (names are the state-dict prefixes this repo uses)."""
    plan = []
    mult = 2 ** len(cfg.ratios)
    ch = mult * cfg.n_filters
    plan.append(dict(kind="conv", name="dec.conv_in", cin=cfg.dimension, cout=ch, k=cfg.kernel_size, dil=1, elu_in=False))
    if cfg.lstm:
        plan.append(dict(kind="lstm", name="dec.lstm", dim=ch, layers=cfg.lstm))
    for i, r in enumerate(cfg.ratios):
        plan.append(dict(kind="convtr", name=f"dec.up{i}.convtr", cin=ch, cout=ch // 2, k=2 * r, stride=r, elu_in=True))
        ch //= 2
        for j in range(cfg.n_residual_layers):
            hidden = ch // cfg.compress
            plan.append(dict(kind="res", name=f"dec.up{i}.res{j}", dim=ch, hidden=hidden, k=cfg.residual_kernel_size,
                             dil=cfg.dilation_base ** j, true_skip=cfg.true_skip))
    plan.append(dict(kind="conv", name="dec.conv_out", cin=cfg.n_filters, cout=cfg.channels, k=cfg.last_kernel_size, dil=1,
                     elu_in=True))
    return plan


def weight_shapes(cfg):
    """name -> shape of every tensor the decoder + quantizer need (folded weights, PyTorch layouts)."""
    shp = {}
    for q in range(cfg.n_q):
        shp[f"vq.{q}.embed"] = (cfg.bins, cfg.dimension)
    for L in layer_plan(cfg):
        n = L["name"]
        if L["kind"] == "conv":
            shp[n + ".weight"] = (L["cout"], L["cin"], L["k"])
            shp[n + ".bias"] = (L["cout"],)
        elif L["kind"] == "convtr":
            shp[n + ".weight"] = (L["cin"], L["cout"], L["k"])
            shp[n + ".bias"] = (L["cout"],)
        elif L["kind"] == "lstm":
            for l in range(L["layers"]):
                shp[f"{n}.weight_ih_l{l}"] = (4 * L["dim"], L["dim"])
                shp[f"{n}.weight_hh_l{l}"] = (4 * L["dim"], L["dim"])
                shp[f"{n}.bias_ih_l{l}"] = (4 * L["dim"],)
                shp[f"{n}.bias_hh_l{l}"] = (4 * L["dim"],)
        else:
            shp[n + ".conv1.weight"] = (L["hidden"], L["dim"], L["k"])
            shp[n + ".conv1.bias"] = (L["hidden"],)
            shp[n + ".conv2.weight"] = (L["dim"], L["hidden"], 1)
            shp[n + ".conv2.bias"] = (L["dim"],)
            if not L["true_skip"]:
                shp[n + ".shortcut.weight"] = (L["dim"], L["dim"], 1)
                shp[n + ".shortcut.bias"] = (L["dim"],)
    return shp


def encoder_plan(cfg):
    """SEANetEncoder (audiocraft modules/seanet.py): conv k7 -> per ratio (reversed) [ResBlock x n, ELU, Conv1d(k=2r, stride r)]
    -> LSTM + skip -> ELU -> conv k7 (-> dimension)."""
    plan = [dict(kind="conv", name="enc.conv_in", cin=cfg.channels, cout=cfg.n_filters, k=cfg.kernel_size, stride=1, elu_in=False)]
    ch = cfg.n_filters
    for i, r in enumerate(reversed(cfg.ratios)):
        for j in range(cfg.n_residual_layers):
            plan.append(dict(kind="res", name=f"enc.down{i}.res{j}", dim=ch, hidden=ch // cfg.compress,
                             k=cfg.residual_kernel_size, dil=cfg.dilation_base ** j, true_skip=cfg.true_skip))
        plan.append(dict(kind="conv", name=f"enc.down{i}.conv", cin=ch, cout=2 * ch, k=2 * r, stride=r, elu_in=True))
        ch *= 2
    if cfg.lstm:
        plan.append(dict(kind="lstm", name="enc.lstm", dim=ch, layers=cfg.lstm))
    plan.append(dict(kind="conv", name="enc.conv_out", cin=ch, cout=cfg.dimension, k=cfg.last_kernel_size, stride=1, elu_in=True))
    return plan


def encoder_weight_shapes(cfg):
    shp = {}
    for L in encoder_plan(cfg):
        n = L["name"]
        if L["kind"] == "conv":
            shp[n + ".weight"] = (L["cout"], L["cin"], L["k"])
            shp[n + ".bias"] = (L["cout"],)
        elif L["kind"] == "lstm":
            for l in range(L["layers"]):
                shp[f"{n}.weight_ih_l{l}"] = (4 * L["dim"], L["dim"])
                shp[f"{n}.weight_hh_l{l}"] = (4 * L["dim"], L["dim"])
                shp[f"{n}.bias_ih_l{l}"] = (4 * L["dim"],)
                shp[f"{n}.bias_hh_l{l}"] = (4 * L["dim"],)
        else:
            shp[n + ".conv1.weight"] = (L["hidden"], L["dim"], L["k"])
            shp[n + ".conv1.bias"] = (L["hidden"],)
            shp[n + ".conv2.weight"] = (L["dim"], L["hidden"], 1)
            shp[n + ".conv2.bias"] = (L["dim"],)
            if not L["true_skip"]:
                shp[n + ".shortcut.weight"] = (L["dim"], L["dim"], 1)
                shp[n + ".shortcut.bias"] = (L["dim"],)
    return shp


def make_state_dict(cfg, seed=0, encoder=False):
    """Deterministic random weights (CPU generator) scaled so activations stay O(1) through the stack.  The encoder's
    weights (encoder=True) are drawn AFTER the decoder's, so decoder fixtures do not depend on the flag."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd = {}
    shapes = dict(weight_shapes(cfg))
    if encoder:
        shapes.update(encoder_weight_shapes(cfg))
    for name, shape in shapes.items():
        if name.endswith("embed"):
            sd[name] = torch.randn(*shape, generator=g) * 0.5
        elif name.endswith("bias") or "bias_" in name:
            sd[name] = torch.randn(*shape, generator=g) * 0.05
        elif "lstm" in name:
            sd[name] = torch.randn(*shape, generator=g) * (0.7 / math.sqrt(shape[1]))
        else:
            fan_in = shape[1] * shape[2] if ".convtr." not in name else shape[0] * shape[2] / 2
            sd[name] = torch.randn(*shape, generator=g) * (1.2 / math.sqrt(fan_in))
    return sd


def _pad1d(x, left, right, mode):
    """audiocraft conv.py pad1d: reflect padding with the small-input guard."""
    if mode != "reflect":
        return F.pad(x, (left, right), "constant", 0.0)
    length = x.shape[-1]
    max_pad = max(left, right)
    extra = 0
    if length <= max_pad:
        extra = max_pad - length + 1
        x = F.pad(x, (0, extra))
    y = F.pad(x, (left, right), "reflect")
    return y[..., : y.shape[-1] - extra]


def conv1d(cfg, x, w, b, dil=1, stride=1):
    """StreamableConv1d (audiocraft modules/conv.py): pad (k_eff - stride) in total -- causal: all on the left -- plus the
    extra right padding that completes the last window (get_extra_padding_for_conv1d), then a plain conv."""
    k = (w.shape[-1] - 1) * dil + 1
    total = k - stride
    length = x.shape[-1]
    n_frames = (length - k + total) / stride + 1
    extra = (math.ceil(n_frames) - 1) * stride + (k - total) - length
    if cfg.causal:
        x = _pad1d(x, total, extra, cfg.pad_mode)
    else:
        right = total // 2
        x = _pad1d(x, total - right, right + extra, cfg.pad_mode)
    return F.conv1d(x, w, b, dilation=dil, stride=stride)


def convtr1d(cfg, x, w, b, stride):
    """StreamableConvTranspose1d: full transposed conv, then trim the fixed padding (k - stride)."""
    k = w.shape[-1]
    total = k - stride
    y = F.conv_transpose1d(x, w, b, stride=stride)
    if cfg.causal:
        right = math.ceil(total * cfg.trim_right_ratio)
    else:
        right = total // 2
    left = total - right
    return y[..., left: y.shape[-1] - right]


def lstm_cell(pre_t, h, c, w_hh, b):
    """One LSTM step: pre_t = W_ih x_t [B,4C], (h, c) of the previous step -> (h, c); gate order i,f,g,o (torch.nn.LSTM)."""
    gates = pre_t + F.linear(h, w_hh) + b
    i, f, g_, o = gates.chunk(4, dim=-1)
    c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g_)
    h = torch.sigmoid(o) * torch.tanh(c)
    return h, c


def lstm(x, sd, name, layers, states=None):
    """StreamableLSTM with skip: y = LSTM(x) + x over [T,B,C], in the dtype of x.  `states` (a dict) receives every layer's
    h and c sequences, [T,B,C], as hs{l} and c{l}."""
    T, B, C = x.shape
    inp = x
    for l in range(layers):
        w_ih, w_hh = sd[f"{name}.weight_ih_l{l}"], sd[f"{name}.weight_hh_l{l}"]
        b = sd[f"{name}.bias_ih_l{l}"] + sd[f"{name}.bias_hh_l{l}"]
        h = torch.zeros(B, C, dtype=x.dtype)
        c = torch.zeros(B, C, dtype=x.dtype)
        outs, cells = [], []
        pre = F.linear(inp, w_ih)                                   # [T,B,4C]
        for t in range(T):
            h, c = lstm_cell(pre[t], h, c, w_hh, b)
            outs.append(h)
            cells.append(c)
        inp = torch.stack(outs, dim=0)
        if states is not None:
            states[f"hs{l}"] = inp
            states[f"c{l}"] = torch.stack(cells, dim=0)
    return inp + x


def apply_layer(cfg, sd, L, inputs):
    """One entry of layer_plan / encoder_plan.  inputs["x"] is the layer's input [B,C,T].  Where the layer applies ELU first,
    inputs["x_elu"] replaces ELU(x) if given (then a layer that reads nothing else needs no "x"), and inputs["h_elu"] the
    ELU'd hidden tensor of a residual block: a caller that holds these tensors as another implementation stored them checks
    that implementation one layer at a time.  -> {"raw": output}, plus "h" (a block's ELU'd hidden tensor) or the LSTM's
    hs{l} / c{l} sequences [B,C,T]."""
    n, x = L["name"], inputs.get("x")

    def elu(key, v):
        return inputs[key] if key in inputs else F.elu(v)
    if L["kind"] == "conv":
        a = elu("x_elu", x) if L["elu_in"] else x
        return {"raw": conv1d(cfg, a, sd[n + ".weight"], sd[n + ".bias"], L.get("dil", 1), L.get("stride", 1))}
    if L["kind"] == "lstm":
        states = {}
        y = lstm(x.permute(2, 0, 1), sd, n, L["layers"], states)
        return dict({k: v.permute(1, 2, 0) for k, v in states.items()}, raw=y.permute(1, 2, 0))
    if L["kind"] == "convtr":
        return {"raw": convtr1d(cfg, elu("x_elu", x), sd[n + ".weight"], sd[n + ".bias"], L["stride"])}
    h = conv1d(cfg, elu("x_elu", x), sd[n + ".conv1.weight"], sd[n + ".conv1.bias"], L["dil"])
    he = elu("h_elu", h)
    h = conv1d(cfg, he, sd[n + ".conv2.weight"], sd[n + ".conv2.bias"], 1)
    s = x if L["true_skip"] else conv1d(cfg, x, sd[n + ".shortcut.weight"], sd[n + ".shortcut.bias"], 1)
    return {"h": he, "raw": s + h}


def rvq_decode(sd, codes):
    """codes [B,K,T] -> latent [B,D,T]: the sum of the codebook rows, in the codebooks' dtype."""
    B, K, T = codes.shape
    emb0 = sd["vq.0.embed"]
    z = torch.zeros(B, T, emb0.shape[1], dtype=emb0.dtype)
    for q in range(K):
        z = z + F.embedding(codes[:, q], sd[f"vq.{q}.embed"])
    return z.transpose(1, 2)


@torch.no_grad()
def decode(cfg, sd, codes, return_intermediates=False):
    """codes [B,K,T] int64 -> waveform [B,channels,T*hop], in the dtype of the weights (sd.double(): a float64 run).
    With return_intermediates also a dict of every tensor the CUDA decoder exposes, under its enc_debug_tensor name, each
    [B,C,T_stage]: z, x0, hs{l}, c{l} (the cell state after every step), u0, x{i}.raw, x{i}.elu, h{i}.{j}, o{i}.{j}.raw,
    o{i}.{j}, wav."""
    x = rvq_decode(sd, codes)
    rec = {"z": x}
    for L in layer_plan(cfg):
        n = L["name"]
        out = apply_layer(cfg, sd, L, {"x": x})
        x = out["raw"]
        if n == "dec.conv_in":
            rec["x0"] = x
            if not cfg.lstm:
                rec["u0"] = F.elu(x)
        elif L["kind"] == "lstm":
            rec.update({k: v for k, v in out.items() if k != "raw"})
            rec["u0"] = F.elu(x)
        elif L["kind"] == "convtr":
            stage = n[len("dec.up"):].split(".")[0]
            stage = str(int(stage) + 1)
            rec[f"x{stage}.raw"], rec[f"x{stage}.elu"] = x, F.elu(x)
        elif L["kind"] == "res":
            sj = stage + "." + n.rsplit("res", 1)[1]
            rec[f"h{sj}"], rec[f"o{sj}.raw"], rec[f"o{sj}"] = out["h"], x, F.elu(x)
    rec["wav"] = x
    return (x, rec) if return_intermediates else x


@torch.no_grad()
def encode_latent(cfg, sd, wav, return_intermediates=False):
    """wav [B,channels,N] -> latent [B,dimension,T], in the dtype of wav and the weights.  With return_intermediates also
    {layer name: output} of every encoder_plan entry, and the latent as "enc.latent"."""
    x = wav
    rec = {}
    for L in encoder_plan(cfg):
        x = rec[L["name"]] = apply_layer(cfg, sd, L, {"x": x})["raw"]
    rec["enc.latent"] = x
    return (x, rec) if return_intermediates else x


@torch.no_grad()
def rvq_encode(cfg, sd, z, return_gaps=False):
    """ResidualVectorQuantizer.encode (audiocraft quantization/core_vq.py): per stage, nearest code in Euclidean distance
    (dist = -(|x|^2 - 2 x.e + |e|^2), arg max), then subtract it.  z [B,D,T] -> codes [B,K,T] (+ per decision, the gap
    between the two best distances: a fp32 implementation may legitimately differ only where it is ~1e-6 relative)."""
    B, D, T = z.shape
    resid = z.transpose(1, 2).reshape(B * T, D)
    codes, gaps = [], []
    for q in range(cfg.n_q):
        emb = sd[f"vq.{q}.embed"]
        dist = -(resid.pow(2).sum(1, keepdim=True) - 2 * resid @ emb.t() + emb.pow(2).sum(1)[None])
        top2 = dist.topk(2, dim=-1)
        idx = top2.indices[:, 0]
        gaps.append((top2.values[:, 0] - top2.values[:, 1]).view(B, T))
        codes.append(idx.view(B, T))
        resid = resid - F.embedding(idx, emb)
    codes = torch.stack(codes, dim=1)
    return (codes, torch.stack(gaps, dim=1)) if return_gaps else codes


@torch.no_grad()
def encode(cfg, sd, wav):
    """wav [B,channels,N] fp32 -> codes [B,K,T] int64   (EncodecModel.encode)."""
    return rvq_encode(cfg, sd, encode_latent(cfg, sd, wav))


# ----------------------------------------------------------------------------------------------------------------
# bridge to the transformers twin (used only by tests/golden/make_golden_codec.py in the build container)
# ----------------------------------------------------------------------------------------------------------------
def to_hf_model(cfg, sd):
    """Build transformers' EncodecModel with the same folded weights (weight_norm g := ||v||, so w == v)."""
    from transformers import EncodecConfig, EncodecModel
    hc = EncodecConfig(sampling_rate=cfg.sample_rate, audio_channels=cfg.channels, upsampling_ratios=list(cfg.ratios),
                       codebook_size=cfg.bins, codebook_dim=cfg.dimension, hidden_size=cfg.dimension,
                       num_filters=cfg.n_filters, num_lstm_layers=cfg.lstm, num_residual_layers=cfg.n_residual_layers,
                       residual_kernel_size=cfg.residual_kernel_size, dilation_growth_rate=cfg.dilation_base,
                       compress=cfg.compress, kernel_size=cfg.kernel_size, last_kernel_size=cfg.last_kernel_size,
                       use_causal_conv=cfg.causal, pad_mode=cfg.pad_mode, use_conv_shortcut=not cfg.true_skip,
                       trim_right_ratio=cfg.trim_right_ratio, norm_type="weight_norm", normalize=False,
                       target_bandwidths=[cfg.n_q * math.log2(cfg.bins) * (cfg.sample_rate / math.prod(cfg.ratios)) / 1000])
    m = EncodecModel(hc).eval()

    def set_conv(mod, w, b):
        conv = mod.conv
        p = conv.parametrizations.weight
        with torch.no_grad():
            p.original1.copy_(w)
            p.original0.copy_(w.flatten(1).norm(dim=1).view(-1, 1, 1))
            conv.bias.copy_(b)
    with torch.no_grad():
        for q in range(cfg.n_q):
            m.quantizer.layers[q].codebook.embed.copy_(sd[f"vq.{q}.embed"])
        layers = list(m.decoder.layers)
        idx = 0
        for L in layer_plan(cfg):
            n = L["name"]
            if L["kind"] in ("conv", "convtr"):
                while not hasattr(layers[idx], "conv"):
                    idx += 1
                set_conv(layers[idx], sd[n + ".weight"], sd[n + ".bias"])
                idx += 1
            elif L["kind"] == "lstm":
                while not hasattr(layers[idx], "lstm"):
                    idx += 1
                for l in range(L["layers"]):
                    for part in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                        getattr(layers[idx].lstm, f"{part}_l{l}").copy_(sd[f"{n}.{part}_l{l}"])
                idx += 1
            else:
                while not hasattr(layers[idx], "block"):
                    idx += 1
                blk = layers[idx]
                set_conv(blk.block[1], sd[n + ".conv1.weight"], sd[n + ".conv1.bias"])
                set_conv(blk.block[3], sd[n + ".conv2.weight"], sd[n + ".conv2.bias"])
                if not L["true_skip"]:
                    set_conv(blk.shortcut, sd[n + ".shortcut.weight"], sd[n + ".shortcut.bias"])
                idx += 1
        if "enc.conv_in.weight" in sd:
            layers = list(m.encoder.layers)
            idx = 0
            for L in encoder_plan(cfg):
                n = L["name"]
                if L["kind"] == "conv":
                    while not hasattr(layers[idx], "conv"):
                        idx += 1
                    set_conv(layers[idx], sd[n + ".weight"], sd[n + ".bias"])
                    idx += 1
                elif L["kind"] == "lstm":
                    while not hasattr(layers[idx], "lstm"):
                        idx += 1
                    for l in range(L["layers"]):
                        for part in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                            getattr(layers[idx].lstm, f"{part}_l{l}").copy_(sd[f"{n}.{part}_l{l}"])
                    idx += 1
                else:
                    while not hasattr(layers[idx], "block"):
                        idx += 1
                    blk = layers[idx]
                    set_conv(blk.block[1], sd[n + ".conv1.weight"], sd[n + ".conv1.bias"])
                    set_conv(blk.block[3], sd[n + ".conv2.weight"], sd[n + ".conv2.bias"])
                    if not L["true_skip"]:
                        set_conv(blk.shortcut, sd[n + ".shortcut.weight"], sd[n + ".shortcut.bias"])
                    idx += 1
    return m
