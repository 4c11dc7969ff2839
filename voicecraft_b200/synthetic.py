"""Synthetic configs / random-init checkpoints in the reference's state_dict format.

There is no network in the build or GPU environment, so tests and bench.py use random-init
weights of the reference architecture (key names / shapes: reference models/voicecraft.py:106-195,
z_scripts/e830M.sh:21-60).  Generation is on the CPU generator so the same seed gives the same
checkpoint in the build container (where the golden fixtures are produced from the real reference)
and on the GPU box.
"""
from argparse import Namespace

import torch

# Reference argparse defaults that the model reads (config.py:50-84) + e830M.sh overrides.
_BASE = dict(
    n_codebooks=4, text_vocab_size=100, text_pad_token=100, audio_vocab_size="2048", empty_token=2048,
    eog=2049, audio_pad_token=2050, eos=2051, n_special=4, reduced_eog=1, special_first=0,
    encodec_sr=50, max_n_spans=3, shuffle_mask_embedding=0, audio_embedding_dim=2048,
    text_embedding_dropout=0.1, audio_embedding_dropout=0.0, text_positional_embedding_dropout=0.1,
    audio_positional_embedding_dropout=0.1, trm_dropout=0.1,
)

CONFIGS = {
    # name: (d_model, nhead, layers)
    "tiny": (256, 2, 2),          # head_dim 128, CPU-oracle friendly
    "small": (512, 4, 4),
    "330M": (1024, 16, 24),       # head_dim 64 stand-in (SURVEY.md section 0.5)
    "830M": (2048, 16, 16),       # z_scripts/e830M.sh:34-37
}


def make_config(name="830M", **overrides):
    d, h, l = CONFIGS[name]
    cfg = dict(_BASE)
    cfg.update(d_model=d, audio_embedding_dim=d, nhead=h, num_decoder_layers=l)
    cfg.update(overrides)
    if cfg.get("eos", -1) is None or cfg["eos"] <= 0:
        cfg["eos"] = -1
        if "n_special" not in overrides:
            cfg["n_special"] = 3
    return Namespace(**cfg)


GEMM_WEIGHT_SUFFIXES = ("in_proj_weight", "out_proj.weight", "linear1.weight", "linear2.weight",
                        ".0.weight", ".2.weight")


def is_gemm_weight(key):
    return key.startswith(("decoder.layers.", "predict_layer.")) and key.endswith(GEMM_WEIGHT_SUFFIXES)


def make_state_dict(cfg, seed=0, bf16_exact=True, logit_scale=2.0, dtype=torch.float32):
    """Random checkpoint with the reference's keys.  ``bf16_exact`` rounds the GEMM matrices to
    bf16-representable fp32 values, so an fp32 reference run and the bf16-weight H100 path see
    identical weights."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    K, D, H, L = cfg.n_codebooks, cfg.d_model, cfg.nhead, cfg.num_decoder_layers
    V = int(eval(cfg.audio_vocab_size) if isinstance(cfg.audio_vocab_size, str) else cfg.audio_vocab_size)
    NV = V + cfg.n_special

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g, dtype=torch.float32) * std

    sd = {}
    sd["eog"] = torch.full((K, 1), cfg.eog, dtype=torch.long)
    if cfg.eos > 0:
        sd["eos"] = torch.full((K, 1), cfg.eos, dtype=torch.long)
    sd["mask_embedding"] = rn(cfg.max_n_spans, D)
    sd["text_embedding.word_embeddings.weight"] = rn(cfg.text_vocab_size + 1, D)
    for k in range(K):
        sd[f"audio_embedding.{k}.word_embeddings.weight"] = rn(NV, D, std=0.7)
    sd["text_positional_embedding.alpha"] = torch.tensor([1.25])
    sd["audio_positional_embedding.alpha"] = torch.tensor([0.75])
    for l in range(L):
        p = f"decoder.layers.{l}."
        sd[p + "self_attn.in_proj_weight"] = rn(3 * D, D, std=D ** -0.5)
        sd[p + "self_attn.in_proj_bias"] = rn(3 * D, std=0.05)
        sd[p + "self_attn.out_proj.weight"] = rn(D, D, std=0.5 * D ** -0.5)
        sd[p + "self_attn.out_proj.bias"] = rn(D, std=0.05)
        sd[p + "linear1.weight"] = rn(4 * D, D, std=D ** -0.5)
        sd[p + "linear1.bias"] = rn(4 * D, std=0.05)
        sd[p + "linear2.weight"] = rn(D, 4 * D, std=0.5 * (4 * D) ** -0.5)
        sd[p + "linear2.bias"] = rn(D, std=0.05)
        for n in ("norm1", "norm2"):
            sd[p + n + ".weight"] = 1.0 + rn(D, std=0.1)
            sd[p + n + ".bias"] = rn(D, std=0.05)
    sd["decoder.norm.weight"] = 1.0 + rn(D, std=0.1)
    sd["decoder.norm.bias"] = rn(D, std=0.05)
    for k in range(K):
        sd[f"predict_layer.{k}.0.weight"] = rn(V // 2, D, std=D ** -0.5)
        sd[f"predict_layer.{k}.0.bias"] = rn(V // 2, std=0.05)
        sd[f"predict_layer.{k}.2.weight"] = rn(NV, V // 2, std=logit_scale * (V // 2) ** -0.5)
        sd[f"predict_layer.{k}.2.bias"] = rn(NV, std=0.1)
    if bf16_exact:
        for key in sd:
            if is_gemm_weight(key):
                sd[key] = sd[key].to(torch.bfloat16).to(torch.float32)
    if dtype != torch.float32:
        sd = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}
    return sd


def synthetic_utterance(cfg, seed, text_len, prompt_frames):
    """Random phoneme ids / codec codes shaped like the reference's inputs (SURVEY.md section 8d)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    V = int(eval(cfg.audio_vocab_size) if isinstance(cfg.audio_vocab_size, str) else cfg.audio_vocab_size)
    x = torch.randint(0, cfg.text_vocab_size, (1, text_len), generator=g)
    y = torch.randint(0, V, (1, prompt_frames, cfg.n_codebooks), generator=g)
    return x, torch.tensor([text_len]), y
