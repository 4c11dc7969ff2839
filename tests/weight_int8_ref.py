"""Torch restatement of the int8 weight policy (weight_dtype="int8", DESIGN.md section 2.2).

For each output feature m (a row of W, fp32 as loaded): e = the smallest integer >= -126 with max|W[m,:]| <= 127 * 2^e, and
q = round-half-even(W / 2^e), which lies in [-127, 127].  Dividing by a power of two is exact wherever the quotient is a
normal number, so torch on the CPU reproduces the engine's bytes; W_deq = q * 2^e is a bf16 value exactly.
"""
import torch

SUFFIXES = ("self_attn.in_proj_weight", "self_attn.out_proj.weight", "linear1.weight", "linear2.weight")


def quantize_rows(W):
    """fp32 [N, K] -> (q int8 [N, K], e int32 [N])"""
    W = W.float()
    amax = W.abs().amax(dim=1)
    m, p = torch.frexp(amax)                       # amax = m * 2^p, m in [0.5, 1)
    e = torch.where(m <= 127.0 / 128.0, p - 7, p - 6)
    e = torch.where(amax > 0, e, torch.full_like(e, -126)).clamp(min=-126).to(torch.int32)
    q = torch.round(W / torch.pow(2.0, e.double()).float().unsqueeze(1))
    return q.to(torch.int8), e


def dequantize_rows(q, e):
    return q.float() * torch.pow(2.0, e.double()).float().unsqueeze(1)


def quantized_keys(sd):
    """the reference state-dict keys of every matrix the decode GEMM streams"""
    return [k for k in sd if (k.startswith("decoder.layers.") and k.endswith(SUFFIXES)) or
            (k.startswith("predict_layer.") and (k.endswith(".0.weight") or k.endswith(".2.weight")))]


def dequantize_state_dict(sd):
    """sd with every quantized matrix replaced by q * 2^e"""
    out = dict(sd)
    for k in quantized_keys(sd):
        out[k] = dequantize_rows(*quantize_rows(sd[k]))
    return out
