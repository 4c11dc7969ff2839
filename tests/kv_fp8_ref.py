"""The fp8 KV policy restated with torch on the CPU (DESIGN.md section 2.2): the quantizer the QKV epilogues run, the
engine's slab layout, and the CPU oracle with K / V stored under that policy."""
import torch
import torch.nn.functional as F

from oracle import lm_oracle

PAGE = 64


def kv_fp8_exponent(amax):
    """smallest integer e with amax <= 448 * 2^e, clamped to e >= -126 (an all-zero row gets -126)"""
    m, k = torch.frexp(amax.float())                      # amax = m * 2^k, m in [0.5, 1); 448 = 0.875 * 2^9
    e = torch.where(m <= 0.875, k - 9, k - 8)
    e = torch.where(amax == 0, torch.full_like(e, -126), e)
    return torch.clamp(e, min=-126)


def quantize_kv_fp8(x):
    """x [..., hd] fp32 -> (e4m3 [..., hd], fp32 scale 2^e [...]): x / 2^e rounded to e4m3 (nearest even)"""
    x = x.float()
    scale = torch.ldexp(torch.ones(()), kv_fp8_exponent(x.abs().amax(-1)).float())
    return (x / scale[..., None]).to(torch.float8_e4m3fn), scale


def dequantize_kv_fp8(q, scale):
    return q.float() * scale[..., None]


def to_slabs(pool):
    """fp32 pool [pages][H][64][hd] -> the engine's fp8 slabs [pages][H][64 * hd bytes, then 64 fp32 scales] (uint8), and
    the dequantized pool"""
    q, s = quantize_kv_fp8(pool)
    n, H = pool.shape[:2]
    slabs = torch.cat([q.view(torch.uint8).reshape(n, H, -1), s.contiguous().view(torch.uint8).reshape(n, H, -1)], -1)
    return slabs.contiguous(), dequantize_kv_fp8(q, s)


def split_slabs(raw, H, hd):
    """raw slab bytes [pages][H][slab] (vcb_debug_kv_pages) -> (e4m3 bytes [pages][H][64][hd], scales [pages][H][64])"""
    raw = torch.as_tensor(raw).view(torch.uint8).reshape(-1, H, PAGE * (hd + 4))
    q = raw[..., :PAGE * hd].reshape(-1, H, PAGE, hd)
    s = raw[..., PAGE * hd:].contiguous().view(torch.float32).reshape(-1, H, PAGE)
    return q, s


class OracleLMFp8(lm_oracle.OracleLM):
    """OracleLM whose K / V go through quantize_kv_fp8 per (token, head) where kv_round_bf16 would round them to bf16.
    oracle/ stays as the reference pinned it, so _mha is restated here with the storage step as `store_kv`; with
    store_kv the identity it must compute exactly what OracleLM._mha does (test_kv_fp8.py checks that)."""

    def __init__(self, cfg, state_dict):
        super().__init__(cfg, state_dict, kv_round_bf16=False)

    @staticmethod
    def store_kv(x):
        """x [T, B, H, hd] -> what the cache holds"""
        return dequantize_kv_fp8(*quantize_kv_fp8(x))

    def _mha(self, l, h, mask4, past_kv):
        c = self.c
        D, H = c.d_model, c.nhead
        hd = D // H
        pre = f"decoder.layers.{l}.self_attn."
        q_in = h.transpose(1, 0)
        T, B, _ = q_in.shape
        proj = F.linear(q_in, self.sd[pre + "in_proj_weight"], self.sd[pre + "in_proj_bias"])
        proj = proj.unflatten(-1, (3, D)).unsqueeze(0).transpose(0, -2).squeeze(-2).contiguous()
        q, k, v = proj[0], proj[1], proj[2]
        k = self.store_kv(k.reshape(T, B, H, hd)).reshape(T, B, D)
        v = self.store_kv(v.reshape(T, B, H, hd)).reshape(T, B, D)
        q = q.view(T, B * H, hd).transpose(0, 1).view(B, H, T, hd)
        k = k.view(T, B * H, hd).transpose(0, 1).view(B, H, T, hd)
        v = v.view(T, B * H, hd).transpose(0, 1).view(B, H, T, hd)
        present = torch.stack([k, v], dim=0)
        if past_kv is not None:
            k = torch.cat([past_kv[0], k], dim=-2)
            v = torch.cat([past_kv[1], v], dim=-2)
        o = F.scaled_dot_product_attention(q, k, v, mask4, 0.0, is_causal=False)
        o = o.permute(2, 0, 1, 3).contiguous().view(B * T, D)
        o = F.linear(o, self.sd[pre + "out_proj.weight"], self.sd[pre + "out_proj.bias"])
        return o.view(T, B, D).transpose(1, 0), present
