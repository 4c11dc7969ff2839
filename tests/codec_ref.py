"""Test helper: one EnCodec layer at a time, in float64, on top of oracle/encodec_oracle.py (no second statement of any
operation).  A CUDA decoder is checked stage by stage by giving `layer` the tensors that decoder itself stored for the
previous stage (bf16 hi + lo, exact in float64): the difference to its next tensor then holds that stage's arithmetic
only, and `abs_bound` is what such an error is proportional to."""
import torch
import torch.nn.functional as F

from oracle import encodec_oracle as eo


def double(sd):
    return {k: v.double() for k, v in sd.items()}


def layer(cfg, sd, L, inputs):
    """One entry L of eo.layer_plan(cfg) / eo.encoder_plan(cfg) on `inputs` (see eo.apply_layer for its keys and result)."""
    return eo.apply_layer(cfg, sd, L, inputs)


def abs_bound(cfg, sd, L, inputs):
    """The same layer with |input|, |weight|, |bias|: per output element the sum of |a||w| over its reduction, |bias|
    included.  A product computed from rounded parts of a and w, summed in finite precision, is wrong by a multiple of the
    rounding unit times this sum, however much the true sum cancels.  Keys as `layer`; "h" bounds a residual block's hidden
    tensor before its ELU (ELU is 1-Lipschitz, so also after).  The LSTM's bound depends on its running state: see
    lstm_teacher_forced."""
    assert L["kind"] != "lstm"
    inp = dict(inputs)
    if "x_elu" not in inp and (L["kind"] != "conv" or L["elu_in"]):
        inp["x_elu"] = F.elu(inp["x"])
    if L["kind"] == "res" and "h_elu" not in inp:
        inp["h_elu"] = layer(cfg, sd, L, inp)["h"]
    a_sd = {k: v.abs() for k, v in sd.items() if k.startswith(L["name"] + ".")}
    out = eo.apply_layer(cfg, a_sd, L, {k: v.abs() for k, v in inp.items()})
    if L["kind"] == "res":
        # the hidden tensor's bound is conv1 alone: with a non-negative input the block's ELU is the identity
        out["h"] = eo.conv1d(cfg, inp["x_elu"].abs(), a_sd[L["name"] + ".conv1.weight"], a_sd[L["name"] + ".conv1.bias"], L["dil"])
    return out


def lstm_teacher_forced(sd, name, l, x, h_stored, unit):
    """Layer l of LSTM `name` over x [T,B,C], each step fed the h the implementation under test stored for the step before
    (h_stored [T,B,C]; h_{-1} = 0), with the cell state running free in float64 (an implementation need not store it).
    -> (h, c, err_h, err_c), each [T,B,C]: the reference states, and the error an implementation may have whose gate
    pre-activations are wrong by `unit` x (|W_ih||x| + |W_hh||h| + |b|) and whose stored h is rounded to 2^-17:
        |dc_t| <= f_t |dc_{t-1}| + |c_{t-1}| df/4 + di/4 + dg + 2^-22 |c_t|      (sigmoid' <= 1/4, tanh' <= 1, |tanh| <= 1)
        |dh_t| <= do/4 + |dc_t| + 2^-16 |h_t|
    The f_t |dc_{t-1}| term is why the error is a sum over the steps the cell remembers, not over all steps."""
    w_ih, w_hh = sd[f"{name}.weight_ih_l{l}"], sd[f"{name}.weight_hh_l{l}"]
    b = sd[f"{name}.bias_ih_l{l}"] + sd[f"{name}.bias_hh_l{l}"]
    T, B, C = x.shape
    pre = F.linear(x, w_ih)
    pre_abs = F.linear(x.abs(), w_ih.abs()) + b.abs()
    c = torch.zeros(B, C, dtype=x.dtype)
    dc = torch.zeros(B, C, dtype=x.dtype)
    hs, cs, ehs, ecs = [], [], [], []
    for t in range(T):
        h_prev = h_stored[t - 1] if t > 0 else torch.zeros(B, C, dtype=x.dtype)
        d_i, d_f, d_g, d_o = (unit * (pre_abs[t] + F.linear(h_prev.abs(), w_hh.abs()))).chunk(4, dim=-1)
        f = torch.sigmoid((pre[t] + F.linear(h_prev, w_hh) + b).chunk(4, dim=-1)[1])
        c_prev = c
        h, c = eo.lstm_cell(pre[t], h_prev, c, w_hh, b)
        dc = f * dc + c_prev.abs() * d_f / 4 + d_i / 4 + d_g + 2.0 ** -22 * c.abs()
        hs.append(h)
        cs.append(c)
        ecs.append(dc)
        ehs.append(d_o / 4 + dc + 2.0 ** -16 * h.abs())
    return torch.stack(hs), torch.stack(cs), torch.stack(ehs), torch.stack(ecs)
