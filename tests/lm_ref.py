"""Test helper: the codec LM one stage at a time in float64 over a reference-format state_dict, as tests/codec_ref.py does
for EnCodec.  A CUDA pass is checked stage by stage by giving a stage the tensors the pass itself stored before it (fp32
rows, bf16 hi + lo planes: exact in float64), so the difference to the tensor it stores next holds that stage's arithmetic
only.  `*_abs` is the same stage on |input|, |weight|, |bias|: per output element A = sum |a||w| + |b|, what the rounding
error of a product of rounded parts summed in finite precision is proportional to, however much the true sum cancels.

The embeddings are restated in float32 in the kernels' order instead (sum over codebooks ascending, alpha * pe rounded
before the add, as eager torch does it): the device result is exact against them.

The stages chained reproduce oracle/lm_oracle.py (test_lm_numerics.py::test_stages_chained_reproduce_oracle), which the
golden fixtures pin to the reference implementation."""
import math

import torch
import torch.nn.functional as F

EPS = 1e-5


def double(sd):
    return {k: v.double() for k, v in sd.items() if v.is_floating_point()}


def _lin(x, w, b):
    return x @ w.t() + b


def _lin_abs(x, w, b):
    return x.abs() @ w.abs().t() + b.abs()


# ---- embeddings (float32, the kernels' order) ------------------------------------------------------------------------
def audio_embedding(sd, toks):
    """sum_k E_k[toks[..., k]], k ascending, in float32: toks [..., K] int64"""
    acc = None
    for k in range(toks.shape[-1]):
        e = F.embedding(toks[..., k], sd[f"audio_embedding.{k}.word_embeddings.weight"].float())
        acc = e if acc is None else acc + e
    return acc


def prompt_rows(sd, pe, x_ids, y_tok, mask_rows=None):
    """embed_rows_kernel: the prefill rows [x_len + y_len, d] of one prompt.  Text row i: E_text[id] + alpha_t * PE[i];
    audio row j: sum_k E_k[y_tok[j, k]] (or mask_embedding[mask_rows[j]] where mask_rows[j] >= 0) + alpha_a * PE[j]"""
    alpha_t = sd["text_positional_embedding.alpha"].float()
    alpha_a = sd["audio_positional_embedding.alpha"].float()
    xl, yl = x_ids.shape[0], y_tok.shape[0]
    text = F.embedding(x_ids, sd["text_embedding.word_embeddings.weight"].float()) + alpha_t * pe[:xl]
    audio = audio_embedding(sd, y_tok)
    if mask_rows is not None:
        m = mask_rows >= 0
        audio[m] = sd["mask_embedding"].float()[mask_rows[m].long()]
    return torch.cat([text, audio + alpha_a * pe[:yl]])


def next_input(sd, pe, toks, j):
    """the sampler's next-input embedding of an audio row at index j: sum_k E_k[toks[k]] + alpha_a * PE[j]"""
    return audio_embedding(sd, toks) + sd["audio_positional_embedding.alpha"].float() * pe[j]


# ---- transformer stages (float64) ------------------------------------------------------------------------------------
def layer_norm(x, g, b):
    return F.layer_norm(x, (x.shape[-1],), g, b, EPS)


def ln_parts(x):
    """(mean, rstd) of each row"""
    mean = x.mean(-1, keepdim=True)
    return mean, 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + EPS)


def _p(l):
    return f"decoder.layers.{l}."


def ln1(sd, l, x):
    return layer_norm(x, sd[_p(l) + "norm1.weight"], sd[_p(l) + "norm1.bias"])


def ln2(sd, l, x):
    return layer_norm(x, sd[_p(l) + "norm2.weight"], sd[_p(l) + "norm2.bias"])


def final_ln(sd, x):
    return layer_norm(x, sd["decoder.norm.weight"], sd["decoder.norm.bias"])


def qkv(sd, l, h):
    """h [rows, d] (LN1 output) -> [rows, 3d]: q | k | v"""
    return _lin(h, sd[_p(l) + "self_attn.in_proj_weight"], sd[_p(l) + "self_attn.in_proj_bias"])


def qkv_abs(sd, l, h):
    return _lin_abs(h, sd[_p(l) + "self_attn.in_proj_weight"], sd[_p(l) + "self_attn.in_proj_bias"])


def attention(q, K, V):
    """one row: q [H, hd], K / V [T, H, hd] (keys 0..pos) -> [H * hd]"""
    hd = q.shape[-1]
    s = torch.einsum("hd,thd->ht", q, K) / math.sqrt(hd)
    return torch.einsum("ht,thd->hd", torch.softmax(s, -1), V).reshape(-1)


def out_proj(sd, l, a, x):
    """residual rows after the attention block: x + a W_o^T + b_o"""
    return x + _lin(a, sd[_p(l) + "self_attn.out_proj.weight"], sd[_p(l) + "self_attn.out_proj.bias"])


def out_proj_abs(sd, l, a):
    return _lin_abs(a, sd[_p(l) + "self_attn.out_proj.weight"], sd[_p(l) + "self_attn.out_proj.bias"])


def ffn1(sd, l, h):
    """ReLU(h W_1^T + b_1), h the LN2 output"""
    return torch.relu(_lin(h, sd[_p(l) + "linear1.weight"], sd[_p(l) + "linear1.bias"]))


def ffn1_abs(sd, l, h):
    return _lin_abs(h, sd[_p(l) + "linear1.weight"], sd[_p(l) + "linear1.bias"])


def ffn2(sd, l, f, x):
    return x + _lin(f, sd[_p(l) + "linear2.weight"], sd[_p(l) + "linear2.bias"])


def ffn2_abs(sd, l, f):
    return _lin_abs(f, sd[_p(l) + "linear2.weight"], sd[_p(l) + "linear2.bias"])


def _h1(sd, K):
    w = torch.cat([sd[f"predict_layer.{k}.0.weight"] for k in range(K)])
    b = torch.cat([sd[f"predict_layer.{k}.0.bias"] for k in range(K)])
    return w, b


def heads1(sd, K, h):
    """GELU (erf) of the K stacked predict_layer.{k}.0 on the final-LN output h -> [rows, K * Hh]"""
    return F.gelu(_lin(h, *_h1(sd, K)))


def heads1_pre(sd, K, h):
    """heads1 before the GELU"""
    return _lin(h, *_h1(sd, K))


def heads1_abs(sd, K, h):
    return _lin_abs(h, *_h1(sd, K))


def heads2(sd, K, g):
    """predict_layer.{k}.2 on codebook k's slice of heads1's output g [rows, K * Hh] -> logits [rows, K, V]"""
    Hh = g.shape[-1] // K
    return torch.stack([_lin(g[:, k * Hh:(k + 1) * Hh], sd[f"predict_layer.{k}.2.weight"], sd[f"predict_layer.{k}.2.bias"])
                        for k in range(K)], 1)


def heads2_abs(sd, K, g):
    Hh = g.shape[-1] // K
    return torch.stack([_lin_abs(g[:, k * Hh:(k + 1) * Hh], sd[f"predict_layer.{k}.2.weight"],
                                 sd[f"predict_layer.{k}.2.bias"]) for k in range(K)], 1)


def fold_abs(W, gamma, beta, b, x):
    """The folded LayerNorm's bound for y = LN(x; gamma, beta) W^T + b computed as rstd (W (gamma x) - mean W gamma) + b':
    per output rstd sum_k |w_k gamma_k| (|x_k| + |mean|) + |W| |beta| + |b| -- the operand is gamma * x (hi / lo), and the
    mean is subtracted after the product, so the error scales with |x| + |mean| rather than with |x - mean|."""
    mean, rstd = ln_parts(x)
    return rstd * ((x.abs() + mean.abs()) @ (W * gamma).abs().t()) + beta.abs() @ W.abs().t() + b.abs()


def layer_weights(sd, l, which):
    """(W, gamma, beta, b) of the GEMM a LayerNorm is folded into: "qkv" (LN1) or "ffn1" (LN2)"""
    if which == "qkv":
        return (sd[_p(l) + "self_attn.in_proj_weight"], sd[_p(l) + "norm1.weight"], sd[_p(l) + "norm1.bias"],
                sd[_p(l) + "self_attn.in_proj_bias"])
    return sd[_p(l) + "linear1.weight"], sd[_p(l) + "norm2.weight"], sd[_p(l) + "norm2.bias"], sd[_p(l) + "linear1.bias"]


def heads_weights(sd, K):
    w, b = _h1(sd, K)
    return w, sd["decoder.norm.weight"], sd["decoder.norm.bias"], b


# ---- the stages chained: a whole sequence with a causal mask (the CPU check against the oracle) ----------------------
def forward(sd, cfg, x):
    """x [T, d] embedding rows of one utterance -> (logits [T, K, V], [(K, V) [T, H, hd]] per layer)"""
    H, L, K = cfg.nhead, cfg.num_decoder_layers, cfg.n_codebooks
    T, d = x.shape
    hd = d // H
    kv = []
    for l in range(L):
        p = qkv(sd, l, ln1(sd, l, x))
        q, k, v = (t.reshape(T, H, hd) for t in p.split(d, -1))
        kv.append((k, v))
        a = torch.stack([attention(q[t], k[:t + 1], v[:t + 1]) for t in range(T)])
        x = out_proj(sd, l, a, x)
        x = ffn2(sd, l, ffn1(sd, l, ln2(sd, l, x)), x)
    return heads2(sd, K, heads1(sd, K, final_ln(sd, x))), kv
