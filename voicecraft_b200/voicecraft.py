"""H100-native drop-in for the inference surface of the reference's ``models/voicecraft.py``.

Same constructor (``VoiceCraft(args)`` / ``VoiceCraft(config=dict)``), same ``state_dict`` keys, same
``inference_tts`` / ``inference_tts_batch`` / ``inference`` signatures and return shapes
(reference models/voicecraft.py:97-121, 561-573, 908-920, 1156-1169).  The module only *holds* the
parameters; every inference call goes through libvcb200.so (hand-written sm_90a kernels: paged-KV
attention, wgmma GEMMs, fused sampler).  There is no PyTorch / CPU fallback: without the extension or
without an H100 (sm_90) GPU the calls raise.

Random numbers: the reference samples with ``torch.multinomial(softmax(l), 1)``, which ATen evaluates as
``argmax(softmax(l) / q)`` with ``q = empty_like(p).exponential_(1)`` from the device's global generator.
The fused sampler kernel generates exactly that ``q`` itself: every utterance (or best-of-N group) owns the
Philox stream of a torch CUDA generator at (seed, offset) and consumes, per sampling step, what the reference's
draw of shape ``[n*K, V]`` consumes.  ``inference_tts`` / ``inference_tts_batch`` / ``inference`` take the
stream of the model device's default generator and leave it advanced as the reference would; batched sessions
give every utterance its own seed, so row *i* of a batch equals the single call of utterance *i* under that
seed.  ``noise_fn`` replaces the generator (tests feed CPU-generator noise to compare with the CPU oracle).

Sampling controls the reference lacks, accepted wherever ``top_k`` is and off by default (see sampling_controls):
``ras_window`` / ``ras_tau`` turn on repetition-aware sampling, ``min_frames`` / ``max_frames`` bound each generation's
length in frames.

Out of scope (training): ``forward`` and ``prepare_mask_intervals`` raise NotImplementedError.
"""
import copy
import ctypes as C
import logging
import math
import os
import time
from argparse import Namespace
from types import SimpleNamespace
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .alignment import Alignment, head_masks
from .codebooks_patterns import DelayedPatternProvider

try:  # same mixin as the reference (voicecraft.py:23, 89-95); optional so the hot path has no hard dependency
    from huggingface_hub import PyTorchModelHubMixin
    _HubBase = (PyTorchModelHubMixin,)
    _HUB_KW = dict(library_name="voicecraft", repo_url="https://github.com/jasonppy/VoiceCraft", tags=["text-to-speech"])
except Exception:  # pragma: no cover
    _HubBase = ()
    _HUB_KW = {}

# configure_engine(kv_dtype=...) -> vcb_config.kv_dtype (VCB_KV_* of include/vcb200.h)
KV_DTYPES = {"bf16": 0, "fp32": 1, "fp8": 2}
# configure_engine(weight_dtype=...) -> vcb_config.weight_dtype (VCB_W_* of include/vcb200.h)
WEIGHT_DTYPES = {"bf16": 0, "int8": 1}


def sampling_controls(ras_window=0, ras_tau=0.1, min_frames=0, max_frames=None):
    """The vcb_sampling fields (ras_window, ras_threshold, min_frames, max_frames) of the sampling controls the
    reference lacks (include/vcb200.h, DESIGN.md section 2.2); the defaults change nothing.

    ras_window = W in [0, 256], ras_tau = tau in (0, 1]: repetition-aware sampling (VALL-E 2) for W > 0.  A drawn token
    that already occurs >= ceil(tau * W) times (computed in float64) among the last W tokens of its codebook in the
    current generation is redrawn from the full tempered distribution, without top-k / top-p.  Every sampling step then
    consumes two noise draws of the generator, so the utterance must sample from the device generator: caller noise
    (model.noise_fn, noise_fns) is rejected.
    min_frames >= 0: the end token cannot come before that many frames of the TTS output or of each edit span.
    max_frames None or >= 1: the end token is forced at that many frames, as the reference's length cap forces it.
    Raises ValueError on a value outside these ranges and on min_frames > max_frames."""
    def whole(v, name):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
            raise ValueError(f"{name} must be an integer, got {v!r}")
        return int(v)
    W, lo = whole(ras_window, "ras_window"), whole(min_frames, "min_frames")
    if not 0 <= W <= 256:
        raise ValueError(f"ras_window must lie in [0, 256], got {W}")
    tau = float(ras_tau)
    if not 0.0 < tau <= 1.0:
        raise ValueError(f"ras_tau must lie in (0, 1], got {ras_tau!r}")
    if lo < 0:
        raise ValueError(f"min_frames must be >= 0, got {lo}")
    hi = 0
    if max_frames is not None:
        hi = whole(max_frames, "max_frames")
        if hi < 1:
            raise ValueError(f"max_frames must be None or >= 1, got {hi}")
        if lo > hi:
            raise ValueError(f"min_frames={lo} exceeds max_frames={hi}")
    return W, (math.ceil(tau * W) if W else 0), lo, hi


def _no_host_noise_under_ras(ras_window, host_noise):
    """repetition-aware sampling draws its second noise plane from the utterance's own device generator"""
    if ras_window > 0 and host_noise:
        raise ValueError("ras_window > 0 samples from the device generator: caller noise (model.noise_fn / noise_fns) "
                         "cannot drive its second draw")


def sine_pe(length: int, dim: int) -> torch.Tensor:
    """Sinusoidal table of SinePositionalEmbedding.extend_pe (embedding.py:67-92), fp32 [length, dim]."""
    import math
    pe = torch.zeros(length, dim)
    position = torch.arange(0, length, dtype=torch.float32).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * -(math.log(10000.0) / dim))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe


# ---------------------------------------------------------------------------------------------------------
# parameter containers with the reference's attribute names (so state_dict keys match, SURVEY.md section 8b)
# ---------------------------------------------------------------------------------------------------------
class _TokenEmbedding(nn.Module):
    def __init__(self, dim, vocab):
        super().__init__()
        self.word_embeddings = nn.Embedding(vocab, dim)


class _Alpha(nn.Module):
    def __init__(self):
        super().__init__()
        self.alpha = nn.Parameter(torch.ones(1))


class _OutProj(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(d, d))
        self.bias = nn.Parameter(torch.zeros(d))
        nn.init.xavier_uniform_(self.weight)


class _SelfAttn(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.empty(3 * d, d))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * d))
        self.out_proj = _OutProj(d)
        nn.init.xavier_uniform_(self.in_proj_weight)


class _Layer(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.self_attn = _SelfAttn(d)
        self.linear1 = nn.Linear(d, 4 * d)
        self.linear2 = nn.Linear(4 * d, d)
        self.norm1 = nn.LayerNorm(d, eps=1e-5)
        self.norm2 = nn.LayerNorm(d, eps=1e-5)


class _Decoder(nn.Module):
    def __init__(self, d, n_layers):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(d) for _ in range(n_layers)])
        self.norm = nn.LayerNorm(d, eps=1e-5)


class VoiceCraft(nn.Module, *_HubBase, **_HUB_KW):
    def __new__(cls, args: Optional[Namespace] = None, config: Optional[Dict] = None, **kwargs):
        if args is not None:
            if config is not None:
                raise ValueError("Cannot provide both `args` and `config`.")
            config = vars(args)
        if _HubBase:
            return super().__new__(cls, args=args, config=config, **kwargs)
        return super().__new__(cls)

    def __init__(self, args: Optional[Namespace] = None, config: Optional[Dict] = None):
        super().__init__()
        if args is None:
            if config is None:
                raise ValueError("Either `args` or `config` must be provided.")
            args = Namespace(**config)
        a = self.args = copy.copy(args)
        self.pattern = DelayedPatternProvider(n_q=a.n_codebooks)
        if not getattr(a, "special_first", False):
            a.special_first = 0
        if not getattr(a, "n_special", False):
            a.n_special = 3
        a.eos = getattr(a, "eos", -1)
        K, d = a.n_codebooks, a.d_model
        self.eog = nn.Parameter(torch.full((K, 1), a.eog, dtype=torch.long), requires_grad=False)
        if a.eos > 0:
            assert a.eos != a.audio_pad_token and a.eos != a.empty_token, a.eos
            self.eos = nn.Parameter(torch.full((K, 1), a.eos, dtype=torch.long), requires_grad=False)
        if isinstance(a.audio_vocab_size, str):
            a.audio_vocab_size = eval(a.audio_vocab_size)
        self.n_text_tokens = a.text_vocab_size + 1
        assert a.text_pad_token == a.text_vocab_size
        self.n_audio_tokens = [a.audio_vocab_size + a.n_special] * K
        assert a.audio_vocab_size == a.empty_token, a.empty_token
        assert a.eog == a.audio_vocab_size + 1, a.eog
        assert a.audio_pad_token == a.audio_vocab_size + 2, a.audio_pad_token
        assert getattr(a, "audio_embedding_dim", d) == d, "audio_embedding_dim must equal d_model (summed embeddings)"

        self.text_embedding = _TokenEmbedding(d, self.n_text_tokens)
        self.audio_embedding = nn.ModuleList([_TokenEmbedding(d, self.n_audio_tokens[k]) for k in range(K)])
        self.mask_embedding = nn.Parameter(torch.randn(a.max_n_spans, d), requires_grad=True)
        self.text_positional_embedding = _Alpha()
        self.audio_positional_embedding = _Alpha()
        self.decoder = _Decoder(d, a.num_decoder_layers)
        self.predict_layer = nn.ModuleList([
            nn.Sequential(nn.Linear(d, a.audio_vocab_size // 2), nn.GELU(),
                          nn.Linear(a.audio_vocab_size // 2, self.n_audio_tokens[k])) for k in range(K)])

        # engine configuration (see configure_engine)
        self._eng = None
        self._eng_key = None
        self._eng_opts = dict(max_slots=8, max_seq_len=2048, max_new_tokens=4096, kv_dtype="bf16", weight_dtype="bf16",
                              kv_pool_gb=None, align_text_cap=0)
        self.noise_fn = None          # optional: callable(shape, device) -> fp32 Exp(1) tensor on `device`
        self.poll_every = 4           # inference_tts*: poll the done flag every N steps (device generator only)
        self._sessions = {}           # first slot -> slot list of every group held by a call, session or batcher (the engine
                                      # is not rebuilt under them); read and written by _free_slots / _take_slots / _release_slots
        self.last_stats = {}
        self.trace_logits = None      # set to a list to collect the raw logits [n*K, V] of every sampling step

    # ------------------------------------------------------------------------------------------------
    # training surface: out of scope for this build (SURVEY.md section 8f)
    # ------------------------------------------------------------------------------------------------
    def forward(self, batch):
        raise NotImplementedError("training forward is out of scope of the H100 decode engine "
                                  "(reference models/voicecraft.py:472-559)")

    def prepare_mask_intervals(self, y_lens):
        raise NotImplementedError("training-only helper (reference models/voicecraft.py:198-237)")

    # ------------------------------------------------------------------------------------------------
    # engine management
    # ------------------------------------------------------------------------------------------------
    def configure_engine(self, **opts):
        """max_slots, max_seq_len, max_new_tokens, kv_dtype ('bf16' default | 'fp32' | 'fp8': e4m3 with a power-of-two
        scale per token and head, half the cache bytes of bf16; INTEGRATION.md), weight_dtype ('bf16' default | 'int8': the
        GEMM weights as int8 with a power-of-two scale per output feature, half the weight bytes; INTEGRATION.md),
        kv_pool_gb (None default: every slot can reach max_seq_len; a number: a KV page pool of that many GB (1e9 bytes),
        taken as utterances grow; the batcher and sessions swap utterances to host memory when it runs out;
        INTEGRATION.md), align_text_cap (0 default: no alignment; n: calls may ask for alignment= of texts up to n tokens,
        and the first one allocates a log of max_slots * max_seq_len * n fp32; INTEGRATION.md).
        Rebuilds lazily."""
        for k in opts:
            if k not in self._eng_opts:
                raise KeyError(k)
        if "kv_dtype" in opts and opts["kv_dtype"] not in KV_DTYPES:
            raise ValueError(f"kv_dtype {opts['kv_dtype']!r}: one of {sorted(KV_DTYPES)}")
        if "weight_dtype" in opts and opts["weight_dtype"] not in WEIGHT_DTYPES:
            raise ValueError(f"weight_dtype {opts['weight_dtype']!r}: one of {sorted(WEIGHT_DTYPES)}")
        if opts.get("kv_pool_gb") is not None and not opts["kv_pool_gb"] > 0:
            raise ValueError(f"kv_pool_gb {opts['kv_pool_gb']!r}: None or a positive number of GB")
        cap = opts.get("align_text_cap", 0)
        if not isinstance(cap, (int, np.integer)) or not 0 <= cap <= _lib.ALIGN_MAX_TEXT:
            raise ValueError(f"align_text_cap {cap!r}: an int in [0, {_lib.ALIGN_MAX_TEXT}]")
        self._eng_opts.update(opts)
        self._drop_engine()

    def _drop_engine(self):
        if getattr(self, "_eng", None) is not None:
            held = getattr(self, "_sessions", {})
            if held:
                raise _lib.VcbError(f"{len(held)} DecodeSession(s) still hold slots of this engine: close them before "
                                    "reconfiguring / moving / reloading the model")
            _lib.load().vcb_destroy(self._eng)
        self._eng = None
        self._eng_key = None

    def _free_slots(self, n, eng_slots):
        """first of n consecutive engine slots that no group holds"""
        used = {s for slots in self._sessions.values() for s in slots}
        for base in range(0, eng_slots - n + 1):
            if not any((base + i) in used for i in range(n)):
                return base
        raise _lib.VcbError("no free engine slots")

    def _take_slots(self, n, need_seq=0):
        """Hold n consecutive free engine slots: (engine, slot list).  Single calls, sessions and batchers share one engine;
        it grows first when it is too small for the slots already held plus n, or for `need_seq` positions, but not while
        anything is held.  Give the slots back with _release_slots."""
        o = self._eng_opts
        held = sum(len(s) for s in self._sessions.values())
        if held + n > o["max_slots"] or need_seq > o["max_seq_len"]:
            if held:
                raise _lib.VcbError(f"engine too small (max_slots={o['max_slots']}, max_seq_len={o['max_seq_len']}) and "
                                    f"{held} slot(s) are held by open DecodeSessions: close them or configure_engine() first")
            o["max_slots"] = max(o["max_slots"], n)
            o["max_seq_len"] = max(o["max_seq_len"], (need_seq + 255) // 256 * 256)
            self._drop_engine()
        eng = self._engine()
        base = self._free_slots(n, o["max_slots"])
        slots = self._sessions[base] = list(range(base, base + n))
        return eng, slots

    def _release_slots(self, held, starts=None, n_copies=1, keep_held=False):
        """vcb_release the groups of n_copies slots that begin at `starts` (default: all of `held`, a list _take_slots
        returned; releasing a slot that is not open does nothing), then give `held` back unless keep_held.  Does nothing
        once `held` was given back."""
        if self._sessions.get(held[0]) is not held:
            return
        for s in held[::n_copies] if starts is None else starts:
            _lib.load().vcb_release(self._eng, s, n_copies)
        if not keep_held:
            del self._sessions[held[0]]

    def __del__(self):
        try:
            self._sessions.clear()
            self._drop_engine()
        except Exception:
            pass

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        state_dict = {k: v for k, v in state_dict.items() if not k.startswith("accuracy_metrics")}
        out = super().load_state_dict(state_dict, strict=strict, **kw)
        self._drop_engine()
        return out

    def _apply(self, fn, *a, **kw):
        out = super()._apply(fn, *a, **kw)
        if hasattr(self, "_eng"):
            self._drop_engine()
        return out

    def _engine(self):
        dev = self.mask_embedding.device
        if dev.type != "cuda":
            raise _lib.VcbError("VoiceCraft (H100) has no CPU path: move the model to a CUDA device (`.to('cuda')`)")
        o = self._eng_opts
        key = (dev.index or 0, tuple(sorted(o.items())))
        if self._eng is not None and self._eng_key == key:
            return self._eng
        self._drop_engine()
        lib = _lib.load()
        a = self.args
        cfg = _lib.vcb_config(
            d_model=a.d_model, nhead=a.nhead, num_layers=a.num_decoder_layers, n_codebooks=a.n_codebooks,
            audio_vocab_size=a.audio_vocab_size, n_special=a.n_special, text_vocab_rows=self.n_text_tokens,
            empty_token=a.empty_token, eog=a.eog, audio_pad_token=a.audio_pad_token, eos=a.eos if a.eos > 0 else -1,
            encodec_sr=int(a.encodec_sr), max_n_spans=a.max_n_spans, max_slots=o["max_slots"],
            max_seq_len=o["max_seq_len"], max_new_tokens=o["max_new_tokens"],
            kv_dtype=KV_DTYPES[o["kv_dtype"]], device=dev.index or 0, weight_dtype=WEIGHT_DTYPES[o["weight_dtype"]],
            kv_pool_bytes=0 if o["kv_pool_gb"] is None else int(o["kv_pool_gb"] * 1e9), align_text_cap=int(o["align_text_cap"]))
        h = C.c_void_p()
        _lib.check(lib.vcb_create(C.byref(cfg), C.byref(h)))
        try:
            with torch.cuda.device(dev):
                for k, v in self.state_dict().items():
                    if not v.is_floating_point():
                        continue
                    t = v.detach().to(device=dev, dtype=torch.float32).contiguous()
                    shape = (C.c_int64 * max(t.dim(), 1))(*t.shape) if t.dim() else (C.c_int64 * 1)(1)
                    _lib.check(lib.vcb_load_weight(h, k.encode(), t.data_ptr(), shape, max(t.dim(), 1), 1))
                pe = sine_pe(max(4000, o["max_seq_len"]), a.d_model).to(dev)
                _lib.check(lib.vcb_load_pe(h, pe.data_ptr(), pe.shape[0], 1))
                _lib.check(lib.vcb_finalize_weights(h))
        except Exception:
            lib.vcb_destroy(h)
            raise
        self._eng, self._eng_key = h, key
        return h

    # ------------------------------------------------------------------------------------------------
    # helpers
    # ------------------------------------------------------------------------------------------------
    def _sampling(self, top_k, top_p, temperature, stop_repetition, silence_tokens, ras_window=0, ras_tau=0.1,
                  min_frames=0, max_frames=None):
        W, c, lo, hi = sampling_controls(ras_window, ras_tau, min_frames, max_frames)
        sp = _lib.vcb_sampling(top_k=int(top_k), top_p=float(top_p), temperature=float(temperature),
                               stop_repetition=int(stop_repetition), n_silence=min(len(silence_tokens), 8),
                               ras_window=W, ras_threshold=c, min_frames=lo, max_frames=hi)
        for i, t in enumerate(list(silence_tokens)[:8]):
            sp.silence_tokens[i] = int(t)
        return sp

    @staticmethod
    def _rng_threads(dev, numel):
        """threads of ATen's distribution_nullary_kernel for a draw of `numel` elements (calc_execution_policy)"""
        p = torch.cuda.get_device_properties(dev)
        grid = min((numel + 255) // 256, p.multi_processor_count * (p.max_threads_per_multi_processor // 256))
        return 256 * grid

    def _check_ids(self, x_ids, y_tok):
        """the reference raises on an out-of-range id (nn.Embedding / F.embedding); the kernels index raw tables"""
        if x_ids.numel() and (int(x_ids.min()) < 0 or int(x_ids.max()) >= self.n_text_tokens):
            raise IndexError(f"text id out of range [0, {self.n_text_tokens})")
        if y_tok.numel() and (int(y_tok.min()) < 0 or int(y_tok.max()) >= self.n_audio_tokens[0]):
            raise IndexError(f"audio token out of range [0, {self.n_audio_tokens[0]})")

    def _draw_noise(self, buf):
        """caller-provided Exp(1) noise with the call shape of the reference's multinomial draw"""
        q = self.noise_fn(tuple(buf.shape), buf.device)
        buf.copy_(q.to(device=buf.device, dtype=torch.float32))
        return buf

    def shift(self, rearranged_y):
        """Delay every segment with the codebook pattern (reference voicecraft.py:254-262)."""
        shifted_y, patterns = [], []
        for segs in rearranged_y:
            pats = [self.pattern.get_pattern(s.shape[1]) for s in segs]
            out = [p.build_pattern_sequence(z=s.unsqueeze(0).contiguous(), special_token=self.args.empty_token,
                                            keep_only_valid_steps=False) for p, s in zip(pats, segs)]
            shifted_y.append([o[0].squeeze(0) for o in out])
            patterns.append(pats)
        return shifted_y, patterns

    def _read_rows(self, eng, slot, n_steps, stream):
        K = self.args.n_codebooks
        buf = (C.c_int32 * (n_steps * K))()
        _lib.check(_lib.load().vcb_read_tokens(eng, slot, buf, n_steps, stream))
        return np.frombuffer(buf, dtype=np.int32).reshape(n_steps, K).astype(np.int64)

    def _read_lp(self, eng, slot, n_steps, stream):
        """log-probability rows [n_steps, K] fp32 of the slot's delayed token rows (vcb_read_logprobs)"""
        K = self.args.n_codebooks
        buf = (C.c_float * (n_steps * K))()
        _lib.check(_lib.load().vcb_read_logprobs(eng, slot, buf, n_steps, stream))
        return np.frombuffer(buf, dtype=np.float32).reshape(n_steps, K).copy()

    @staticmethod
    def _undelay(rows: np.ndarray, K: int) -> np.ndarray:
        """rows [n,K] (delayed, as sampled) -> [K, n-K]   (reference voicecraft.py:1126-1137).  For a finished
        generation n-K == final_frames(rows, K, end): the frames before the end token."""
        n = rows.shape[0]
        return np.stack([rows[k: n - (K - k), k] for k in range(K)], axis=0)

    # ------------------------------------------------------------------------------------------------
    # inference_tts  (reference voicecraft.py:908-1153)
    # ------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def inference_tts(self, x: torch.Tensor, x_lens: torch.Tensor, y: torch.Tensor, top_k: int = -100,
                      top_p: float = 1.0, temperature: float = 1.0, stop_repetition: int = 3, kvcache: int = 1,
                      silence_tokens: List[int] = [1388, 1898, 131], *kargs, logprobs: bool = False,
                      ras_window: int = 0, ras_tau: float = 0.1, min_frames: int = 0,
                      max_frames: Optional[int] = None, alignment=None):
        """logprobs=True: returns (res, gen, lp), lp [1,K,G] fp32 the log-probability of each frame of gen under the
        model's raw distribution (vcb_read_logprobs).  ras_window, ras_tau, min_frames, max_frames: see
        sampling_controls.  alignment (None: off; True: every head of every layer, L * H probes per row; {layer: [heads]}):
        the result also ends with an Alignment of res (voicecraft_b200/alignment.py); needs
        configure_engine(align_text_cap >= the text's tokens).  Tokens are those of a call without it."""
        sp = self._sampling(top_k, top_p, temperature, stop_repetition, silence_tokens, ras_window, ras_tau, min_frames,
                            max_frames)
        return self._tts_impl(x, x_lens, y, sp, silence_tokens, 1, logprobs, alignment)

    @torch.no_grad()
    def inference_tts_batch(self, x: torch.Tensor, x_lens: torch.Tensor, y: torch.Tensor, top_k: int = -100,
                            top_p: float = 1.0, temperature: float = 1.0, stop_repetition: int = 3, kvcache: int = 1,
                            batch_size: int = 5, silence_tokens: List[int] = [1388, 1898, 131], *kargs,
                            logprobs: bool = False, ras_window: int = 0, ras_tau: float = 0.1, min_frames: int = 0,
                            max_frames: Optional[int] = None, alignment=None):
        """Best-of-N: the first sample to end wins (reference voicecraft.py:1156-1439).  logprobs=True: returns
        (res, gen, lp) as inference_tts does, lp the kept copy's; alignment: likewise, the kept copy's Alignment."""
        sp = self._sampling(top_k, top_p, temperature, stop_repetition, silence_tokens, ras_window, ras_tau, min_frames,
                            max_frames)
        return self._tts_impl(x, x_lens, y, sp, silence_tokens, batch_size, logprobs, alignment)

    def _tts_impl(self, x, x_lens, y, sp, silence_tokens, n_copies, logprobs, alignment=None):
        assert x.ndim == 2, x.shape
        assert x_lens.ndim == 1, x_lens.shape
        assert y.ndim == 3, y.shape
        assert y.shape[0] == 1 and y.shape[2] == self.args.n_codebooks, y.transpose(2, 1).shape
        logging.info(f"silence tokens: {silence_tokens}, note that if you are not using the pretrained encodec "
                     f"6f79c6a8, make sure you specified it yourself, rather than using the default")
        sess = DecodeSession(self, [x], [y], sp, n_copies=n_copies, alignment=alignment)
        try:
            out, = sess._run_single(logprobs)
        finally:
            sess.close()
        keep = sess._kept(0, sess.status)
        self.last_stats = dict(steps=int(sess.status[keep].n_steps), keep=int(keep))
        return out

    # ------------------------------------------------------------------------------------------------
    # speech editing  (reference voicecraft.py:561-906)
    # ------------------------------------------------------------------------------------------------
    def _edit_prompt(self, y, spans):
        """Segment / placeholder layout of voicecraft.py:239-320, 615-683 as integer index tables.

        y [K,T] (device).  Returns (tokens [T',K] int64 device, mask_rows int32 [T'], more_mask_rows, non_mask)."""
        a = self.args
        K, T = y.shape
        M = len(spans)
        reduced_eog = getattr(a, "reduced_eog", 0)
        starts = [s for s, _ in spans] + [T]
        ends = [0] + [e for _, e in spans]
        non_mask = list(zip(ends, starts))
        # (source interval, end token or None) for every segment, non-masked first then masked
        segs = []
        for i, (s0, s1) in enumerate(non_mask):
            last = i == len(non_mask) - 1
            if a.eos > 0:
                assert reduced_eog
                tail = a.eos if last else None
            elif reduced_eog:
                tail = a.eog if last else None
            else:
                tail = a.eog
            segs.append((s0, s1, tail))
        for (s0, s1) in spans:
            segs.append((s0, s1, a.eog))
        assert not getattr(a, "shuffle_mask_embedding", 0), "shuffle_mask_embedding is a training-time option"
        vals = list(range(a.max_n_spans))[:M]
        mask_val = vals + vals
        # column table: src[k, c] >= 0 -> y[k, src]; otherwise -(token+1)
        cols_src = []
        mask_rows = []
        for j, (s0, s1, tail) in enumerate(segs):
            n_src = (s1 - s0) + (1 if tail is not None else 0)
            blk = np.full((K, n_src + K), -(a.empty_token + 1), dtype=np.int64)
            for k in range(K):
                blk[k, 1 + k: 1 + k + (s1 - s0)] = np.arange(s0, s1)
                if tail is not None:
                    blk[k, 1 + k + (s1 - s0)] = -(tail + 1)
            cols_src.append(blk)
            mask_rows += [-1] * blk.shape[1]
            if j < len(segs) - 1:
                cols_src.append(np.full((K, 1), -(a.eog + 1), dtype=np.int64))    # placeholder column (:264-288)
                mask_rows.append(mask_val[j])
        src = np.concatenate(cols_src, axis=1)
        # cut right after placeholder M plus the first (all-empty) column of the first masked segment (:672-679)
        ph = [i for i, m in enumerate(mask_rows) if m >= 0]
        cut = ph[M] + 2
        src, mask_rows = src[:, :cut], mask_rows[:cut]
        src_t = torch.from_numpy(src).to(y.device)
        tok = torch.where(src_t >= 0, torch.gather(y, 1, src_t.clamp(min=0)), -(src_t + 1))
        return (tok.transpose(1, 0).contiguous(), torch.tensor(mask_rows, dtype=torch.int32, device=y.device),
                mask_val[M + 1:], non_mask)

    @torch.no_grad()
    def inference(self, x: torch.Tensor, x_lens: torch.Tensor, y: torch.Tensor, mask_interval: torch.Tensor,
                  top_k: int = -100, top_p: float = 1.0, temperature: float = 1.0, stop_repetition: int = -1,
                  kvcache: int = 1, silence_tokens: List[int] = [1388, 1898, 131], *, logprobs: bool = False,
                  ras_window: int = 0, ras_tau: float = 0.1, min_frames: int = 0,
                  max_frames: Optional[int] = None):
        """logprobs=True: returns (res, lp), lp [1,K,T'] fp32 aligned with res: the log-probability of each generated
        frame under the model's raw distribution (vcb_read_logprobs), NaN on the frames copied from y.  ras_window,
        ras_tau, min_frames, max_frames: see sampling_controls; the length bounds hold per masked span"""
        assert x.ndim == 2, x.shape
        assert x_lens.ndim == 1, x_lens.shape
        assert y.ndim == 3, y.shape
        assert y.shape[0] == 1 and y.shape[2] == self.args.n_codebooks, y.transpose(2, 1).shape
        assert mask_interval.shape == torch.Size((1, mask_interval.shape[1], 2)), mask_interval
        logging.info(f"silence tokens: {silence_tokens}, note that if you are not using the pretrained encodec "
                     f"6f79c6a8, make sure you specified it yourself, rather than using the default")
        sess = DecodeSession(self, [x], [y], self._sampling(top_k, top_p, temperature, stop_repetition, silence_tokens,
                                                            ras_window, ras_tau, min_frames, max_frames),
                             mask_intervals=[mask_interval], n_copies=1)
        try:
            out, = sess._run_single(logprobs)
        finally:
            sess.close()
        self.last_stats = dict(steps=int(sess.status[0].n_steps))
        return (out[0], out[2]) if logprobs else out[0]

    # ------------------------------------------------------------------------------------------------
    # driver-level batching of INDEPENDENT utterances (SURVEY.md section 8f row f2; BASELINE config 2).
    # Not a reference API: the reference decodes one utterance per call.  Each utterance keeps its own
    # state machine; one Exp(1) draw of shape [B*K, V] per step feeds all of them.
    # ------------------------------------------------------------------------------------------------
    def open_edit_session(self, xs, ys, mask_intervals, top_k=-100, top_p=1.0, temperature=1.0, stop_repetition=-1,
                          silence_tokens=(1388, 1898, 131), seeds=None, noise_fns=None, ras_window=0, ras_tau=0.1,
                          min_frames=0, max_frames=None):
        """Independent speech-editing utterances decoded as one batch (BASELINE config 3).  mask_intervals: list of
        [1,M,2] tensors.  Returns a DecodeSession; results() gives the edited [1,K,T'] per utterance.  ras_window,
        ras_tau, min_frames, max_frames: see sampling_controls."""
        return DecodeSession(self, xs, ys, self._sampling(top_k, top_p, temperature, stop_repetition, silence_tokens,
                                                          ras_window, ras_tau, min_frames, max_frames),
                             mask_intervals=mask_intervals, seeds=seeds, noise_fns=noise_fns)

    @torch.no_grad()
    def inference_many(self, xs, ys, mask_intervals, poll_every: int = 4, logprobs: bool = False, **kw):
        """Batched counterpart of `inference` (speech editing) for independent utterances; logprobs=True: a list of
        (res, lp) as inference(..., logprobs=True) returns them."""
        out = self.open_edit_session(xs, ys, mask_intervals, **kw)._run_many(poll_every, logprobs)
        return [(r[0], r[2]) if logprobs else r[0] for r in out]

    def open_tts_session(self, xs, ys, top_k=-100, top_p=1.0, temperature=1.0, stop_repetition=3,
                         silence_tokens=(1388, 1898, 131), seeds=None, noise_fns=None, best_of=1, ras_window=0,
                         ras_tau=0.1, min_frames=0, max_frames=None, alignment=None):
        """xs: list of [1,L] int64, ys: list of [1,T,K] int64 (any device).  Prefills every utterance (one packed,
        chunked pass) and returns a DecodeSession whose .step() runs one decode step for all of them.

        seeds: one generator seed per utterance -- utterance i samples from the Philox stream of a torch CUDA generator
        seeded with seeds[i] (offset 0), i.e. its tokens equal ``torch.manual_seed(seeds[i]); inference_tts(x_i, ., y_i)``.
        Default: the device generator's current seed + i at its current offset (the global generator is left untouched).
        noise_fns: instead, one callable(shape=[best_of*K,V], device) per utterance (tests: CPU-generator noise for the
        oracle).
        best_of: each utterance is sampled best_of times and keeps the copy that ends first, what
        ``inference_tts_batch(x_i, ., y_i, batch_size=best_of)`` returns under the same seed.  The copies share one
        prefill and the KV pages of the prompt's full pages.
        ras_window, ras_tau, min_frames, max_frames: see sampling_controls.
        alignment: as inference_tts's, for every utterance; results() then ends each tuple with its Alignment."""
        return DecodeSession(self, xs, ys, self._sampling(top_k, top_p, temperature, stop_repetition, silence_tokens,
                                                          ras_window, ras_tau, min_frames, max_frames),
                             seeds=seeds, noise_fns=noise_fns, best_of=best_of, alignment=alignment)

    @torch.no_grad()
    def inference_tts_many(self, xs, ys, poll_every: int = 8, logprobs: bool = False, **kw):
        """Returns a list of (res [1,K,T+G], gen [1,K,G]) like inference_tts (inference_tts_batch with best_of > 1), one
        per utterance; logprobs=True: (res, gen, lp) as inference_tts(..., logprobs=True) returns them; alignment= (see
        open_tts_session): each tuple ends with the utterance's Alignment."""
        return self.open_tts_session(xs, ys, **kw)._run_many(poll_every, logprobs)

    # ------------------------------------------------------------------------------------------------
    # streaming: audio while the tokens are generated (TtsStream)
    # ------------------------------------------------------------------------------------------------
    # Every stream takes sample_rate=: chunks at that rate instead of the codec's, resampled on the device as they are
    # decoded (CodecStream); concatenated they equal tokenizer.resample(<the codec-rate audio>, codec rate, sample_rate).
    def inference_tts_many_stream(self, xs, ys, tokenizer, chunk_frames: int = 25, poll_every: int = 8, seeds=None,
                                  sample_rate: int = None, **kw):
        """inference_tts_many with the audio handed out while it is generated: iterates (i, wav [1, channels, n*hop]),
        utterance i's chunks in order; concatenated they equal ``tokenizer.decode_codes(gen_i)``.  Afterwards
        ``.results`` equals what inference_tts_many returns.  `seeds` and alignment= as in open_tts_session; with
        alignment, ``.alignments`` holds utterance i's Alignment."""
        _no_stream_best_of(kw.get("best_of", 1))
        sess = self.open_tts_session(xs, ys, seeds=seeds, **kw)
        return TtsStream(sess, tokenizer, chunk_frames, poll_every, sample_rate)

    def inference_tts_stream(self, x: torch.Tensor, x_lens: torch.Tensor, y: torch.Tensor, tokenizer, chunk_frames: int = 25,
                             poll_every: int = 8, top_k: int = -100, top_p: float = 1.0, temperature: float = 1.0,
                             stop_repetition: int = 3, silence_tokens: List[int] = [1388, 1898, 131],
                             sample_rate: int = None, ras_window: int = 0, ras_tau: float = 0.1, min_frames: int = 0,
                             max_frames: Optional[int] = None, alignment=None):
        """inference_tts with the audio handed out while it is generated: iterates wav chunks [1, channels, n*hop] whose
        concatenation equals ``tokenizer.decode([(gen, None)])``.  Afterwards ``.result`` is (res, gen), what inference_tts
        returns: the utterance samples from the device generator's stream at its current offset and leaves it advanced by
        the steps it ran, as inference_tts does.  alignment=: ``.alignment`` is then the Alignment inference_tts returns."""
        assert x.ndim == 2 and x.shape[0] == 1 and x_lens.ndim == 1 and y.ndim == 3 and y.shape[0] == 1, (x.shape, y.shape)
        sess = DecodeSession(self, [x], [y], self._sampling(top_k, top_p, temperature, stop_repetition, silence_tokens,
                                                            ras_window, ras_tau, min_frames, max_frames),
                             n_copies=1, alignment=alignment)
        return _SingleTtsStream(sess, tokenizer, chunk_frames, poll_every, sample_rate)

    def inference_many_stream(self, xs, ys, mask_intervals, tokenizer, chunk_frames: int = 25, poll_every: int = 8,
                              seeds=None, sample_rate: int = None, **kw):
        """inference_many with the audio handed out while it is generated: iterates (i, wav [1, channels, n*hop]),
        utterance i's chunks in order; concatenated they equal ``tokenizer.decode_codes(res_i)``, the whole edited
        utterance.  The frames before the first masked span are final at once, so they are the first chunk.  Afterwards
        ``.results`` equals what inference_many returns.  `seeds` as in open_tts_session; the device generators only."""
        sess = self.open_edit_session(xs, ys, mask_intervals, seeds=seeds, **kw)
        return TtsStream(sess, tokenizer, chunk_frames, poll_every, sample_rate)

    def inference_stream(self, x: torch.Tensor, x_lens: torch.Tensor, y: torch.Tensor, mask_interval: torch.Tensor, tokenizer,
                         chunk_frames: int = 25, poll_every: int = 8, top_k: int = -100, top_p: float = 1.0,
                         temperature: float = 1.0, stop_repetition: int = -1, kvcache: int = 1,
                         silence_tokens: List[int] = [1388, 1898, 131], sample_rate: int = None,
                         ras_window: int = 0, ras_tau: float = 0.1, min_frames: int = 0,
                         max_frames: Optional[int] = None):
        """inference (speech editing) with the audio handed out while it is generated: iterates wav chunks
        [1, channels, n*hop] whose concatenation equals ``tokenizer.decode_codes(res)``, the whole edited utterance.
        Afterwards ``.result`` is res, what inference returns, and the device generator is left where inference leaves
        it.  The device generator only (model.noise_fn must be None)."""
        assert x.ndim == 2 and x.shape[0] == 1 and x_lens.ndim == 1 and y.ndim == 3 and y.shape[0] == 1, (x.shape, y.shape)
        assert mask_interval.shape == torch.Size((1, mask_interval.shape[1], 2)), mask_interval
        sess = DecodeSession(self, [x], [y], self._sampling(top_k, top_p, temperature, stop_repetition, silence_tokens,
                                                            ras_window, ras_tau, min_frames, max_frames),
                             mask_intervals=[mask_interval], n_copies=1)
        return _SingleTtsStream(sess, tokenizer, chunk_frames, poll_every, sample_rate)

    # ------------------------------------------------------------------------------------------------
    # Long TTS  (reference gradio_app.py run, mode "Long TTS"): one prompt, one sentence after another
    # ------------------------------------------------------------------------------------------------
    def _long_ticket(self, xs, y, best_of, top_k, top_p, temperature, stop_repetition, silence_tokens, ras_window, ras_tau,
                     min_frames, max_frames, alignment=None):
        """a one-ticket ContinuousBatcher holding xs as a long ticket on the device generator's stream at its current
        offset, and the ticket's _Chain"""
        _no_host_noise_under_ras(sampling_controls(ras_window, ras_tau, min_frames, max_frames)[0],
                                 self.noise_fn is not None)
        if self.noise_fn is not None:
            raise _lib.VcbError("Long TTS samples from the device generator (model.noise_fn must be None)")
        gen = torch.cuda.default_generators[self.mask_embedding.device.index or 0]
        cb = ContinuousBatcher(self, max_concurrency=_check_best_of(best_of), top_k=top_k, top_p=top_p,
                               temperature=temperature, stop_repetition=stop_repetition, silence_tokens=silence_tokens,
                               ras_window=ras_window, ras_tau=ras_tau, min_frames=min_frames, max_frames=max_frames)
        chain = _Chain(list(xs), int(gen.get_offset()))
        cb.submit(chain, y, seed=int(gen.initial_seed()), best_of=best_of, alignment=alignment)
        return cb, chain, gen

    @torch.no_grad()
    def inference_long_tts(self, xs, y: torch.Tensor, best_of: int = 1, logprobs: bool = False, top_k: int = -100,
                           top_p: float = 1.0, temperature: float = 1.0, stop_repetition: int = 3, kvcache: int = 1,
                           silence_tokens: List[int] = [1388, 1898, 131], ras_window: int = 0, ras_tau: float = 0.1,
                           min_frames: int = 0, max_frames: Optional[int] = None, alignment=None):
        """The reference's Long TTS loop as one call: xs a list of [1,L_i] text-token tensors, one per sentence, all
        prompted by y [1,T,K].  Returns one (res, gen) per sentence ((res, gen, lp) with logprobs=True, and the sentence's
        Alignment last with alignment=, as inference_tts returns them), equal to
        ``[inference_tts(x_i, ., y, ...) for x_i in xs]`` (inference_tts_batch(..., batch_size=best_of) with best_of > 1),
        and leaves the device generator where that loop leaves it: sentence i+1 samples from where sentence i ended.
        Runs as one long ticket of a ContinuousBatcher (submit with a list of x); the device generator only.
        ras_window, ras_tau, min_frames, max_frames: see sampling_controls; they apply to every sentence."""
        cb, chain, gen = self._long_ticket(xs, y, best_of, top_k, top_p, temperature, stop_repetition, silence_tokens,
                                           ras_window, ras_tau, min_frames, max_frames, alignment)
        out = cb.run()[0]
        gen.set_offset(chain.offset)
        self.last_stats = dict(steps=cb.stats["steps"])
        if logprobs:
            out = [r + (lp,) for r, lp in zip(out, cb.logprobs[0])]
        if cb.alignments[0] is not None:
            out = [r + (al,) for r, al in zip(out, cb.alignments[0])]
        return out

    def inference_long_tts_stream(self, xs, y: torch.Tensor, tokenizer, chunk_frames: int = 25, sample_rate: int = None,
                                  top_k: int = -100, top_p: float = 1.0, temperature: float = 1.0,
                                  stop_repetition: int = 3, kvcache: int = 1, silence_tokens: List[int] = [1388, 1898, 131],
                                  ras_window: int = 0, ras_tau: float = 0.1, min_frames: int = 0,
                                  max_frames: Optional[int] = None, alignment=None):
        """inference_long_tts with the audio handed out while it is generated: iterates wav chunks [1, channels, n], the
        sentences in order; concatenated they equal ``torch.cat([tokenizer.decode([(gen_i, None)]) for gen_i in gens],
        -1)`` (each sentence decoded from a fresh codec state), and with sample_rate the tokenizer.resample of that
        concatenation.  Afterwards ``.results`` is what inference_long_tts returns, ``.logprobs`` its lp per sentence,
        ``.alignments`` (with alignment=) its Alignment per sentence,
        and the device generator is left where inference_long_tts leaves it.  best_of = 1 only: the kept copy of a
        best-of-N sentence is known only when its group ends."""
        cb, chain, gen = self._long_ticket(xs, y, 1, top_k, top_p, temperature, stop_repetition, silence_tokens,
                                           ras_window, ras_tau, min_frames, max_frames, alignment)
        return LongTtsStream(cb, chain, gen, tokenizer, chunk_frames, sample_rate)


def _check_best_of(best_of) -> int:
    if isinstance(best_of, bool) or int(best_of) != best_of or best_of < 1:
        raise ValueError(f"best_of must be an integer >= 1, got {best_of!r}")
    return int(best_of)


def _no_stream_best_of(best_of):
    """best-of-N keeps the copy that ends first, so which copy's audio to hand out is known only when the group ends"""
    if _check_best_of(best_of) > 1:
        raise ValueError(f"best_of={best_of}: streaming hands out audio while it is generated, but the kept copy of a "
                         "best-of-N utterance is known only when its group ends; use inference_tts_many / run() instead")


def _end_token(a) -> int:
    """the token that ends a TTS generation in codebook 0 (reference voicecraft.py:1034-1045)"""
    return a.eos if a.eos > 0 else a.eog


def final_frames(rows: np.ndarray, K: int, end: int) -> int:
    """How many leading frames of the delayed token rows [n,K] are final: frame t is final once rows up to t+K-1 exist
    (its last codebook has been sampled) and rows[t, 0] is not the end token.  Frames are final in order, so the answer
    only grows as rows are added; for a finished generation it is n-K (what _undelay returns)."""
    m = max(0, rows.shape[0] - K + 1)
    hit = np.flatnonzero(rows[:m, 0] == end)
    return int(hit[0]) if hit.size else m


def frame_codes(rows: np.ndarray, K: int, t0: int, t1: int) -> np.ndarray:
    """frames [t0, t1) of the delayed rows, un-delayed: [K, t1-t0] with [k, t] = rows[t + k, k]"""
    return np.stack([rows[t0 + k: t1 + k, k] for k in range(K)], axis=0)


def _edit_pieces(rows, status, spans, T, K, eog):
    """The final pieces of an edit's output y0[:, 0:s1] ++ G1 ++ y0[:, e1:s2] ++ ... ++ GM ++ y0[:, eM:T], in order:
    (0, first y0 column, frames) for an original piece, (1, first token row, frames) for a generated span.  With
    d = n_spans_done: original pieces 0..d, the spans before d, and span d's frames that final_frames makes final."""
    M = len(spans)
    d = min(int(status.n_spans_done), M)
    out, r0 = [], 0
    for j in range(M + 1):
        c0 = 0 if j == 0 else spans[j - 1][1]
        out.append((0, c0, (T if j == M else spans[j][0]) - c0))
        if j == M:
            break
        if j == d:
            out.append((1, r0, final_frames(rows[r0:], K, eog)))
            break
        end = int(status.span_ends[j])
        out.append((1, r0, max(0, end - r0 - K)))
        r0 = end
    return out


def edit_final_frames(rows: np.ndarray, status, spans, T: int, K: int, eog: int) -> int:
    """How many leading frames of an edit's output (_Prompt.result) are final, from its delayed token rows [n,K] and its
    vcb_status: the original pieces up to n_spans_done, the spans generated before it, and the final frames of the span
    being generated, by final_frames' rule on the rows since it began (end token eog).  Only grows as rows are added;
    once every span is done it is the output's length."""
    return sum(n for _, _, n in _edit_pieces(rows, status, spans, T, K, eog))


def edit_frame_codes(rows: np.ndarray, status, orig: np.ndarray, spans, K: int, eog: int, t0: int, t1: int) -> np.ndarray:
    """output frames [t0, t1) of an edit (t1 <= edit_final_frames): [K, t1-t0], each from the original codes orig [K,T]
    or un-delayed from the token rows"""
    out, f = [np.zeros((K, 0), dtype=np.int64)], 0
    for kind, src, n in _edit_pieces(rows, status, spans, orig.shape[1], K, eog):
        a, b = max(t0, f), min(t1, f + n)
        if a < b:
            u0, u1 = src + a - f, src + b - f
            out.append(orig[:, u0:u1] if kind == 0 else frame_codes(rows[src:], K, a - f, b - f))
        f += n
    return np.concatenate(out, axis=1).astype(np.int64)


def _check_capacity(status):
    """a slot that ran out of max_new_tokens / max_seq_len stops with done == 2"""
    if any(s.done == 2 for s in status):
        raise _lib.VcbError("decode stopped: engine capacity (max_new_tokens / max_seq_len) exhausted; "
                            "raise it with configure_engine()")


class _Prompt:
    """One utterance's prompt, held on the model's device: the TTS layout (the prompt delayed by the codebook pattern,
    reference voicecraft.py:961-967) or, given `spans`, the speech-editing layout (VoiceCraft._edit_prompt).  `need_seq`
    bounds the engine positions its generation can reach, with max_frames > 0 (vcb_sampling.max_frames) that bound's.
    Raises ValueError on more than 8 spans; the caller checks the id ranges (VoiceCraft._check_ids) before it takes a
    slot."""

    def __init__(self, model, x, y, spans=None, max_frames=0):
        a = model.args
        K, dev = a.n_codebooks, model.mask_embedding.device
        self.model, self.spans = model, spans
        x = x.to(dev, non_blocking=True)
        y = y.to(dev, non_blocking=True)
        if a.special_first:
            y = y + int(a.n_special)
        self.y0 = y.transpose(2, 1)[0].long().contiguous()                       # [1,T,K] -> [K,T]
        self.x_ids = x[0].long().contiguous()
        x_len = int(self.x_ids.shape[0])
        if spans is None:
            shifted, _ = model.shift([[self.y0]])
            prompt = shifted[0][0][:, : -(K - 1)] if K > 1 else shifted[0][0]     # voicecraft.py:967
            self.y_tok = prompt.transpose(1, 0).contiguous()                      # [T+1, K]
            self.mask_rows, self.more_vals = None, []
            cap, extra = x_len * (int(a.encodec_sr) // 5), K
        else:
            if len(spans) > min(8, int(a.max_n_spans)):
                raise ValueError(f"{len(spans)} masked spans: at most min(8, max_n_spans={a.max_n_spans}) per utterance")
            self.y_tok, self.mask_rows, self.more_vals, self.non_mask = model._edit_prompt(self.y0, spans)
            cap, extra = x_len * 10, (K + 3) * (len(spans) + 1)
        rows = int(self.y_tok.shape[0])
        if max_frames > 0:
            # the forced end token comes at max_frames steps of a generation: the TTS output or, for an edit, each span,
            # whose K - 1 closing steps and hand-over columns `extra` already counts.  The reference's cap still holds.
            cap = min(cap, rows + max_frames * (1 if spans is None else len(spans)))
        self.need_seq = x_len + max(rows, cap + 1) + extra + 8
        self.total = x_len + int(self.y_tok.shape[0])           # positions the prefill writes
        self.align = None                                       # vcb_prompt.align_heads (ctypes uint32 array) or None

    def pages(self, n_copies, max_pages):
        """KV pages vcb_prefill takes for it: a one-copy prompt its positions' pages in whole growth chunks, a best-of-N
        group its full reservation"""
        if n_copies == 1:
            g = _lib.KV_GROW_PAGES
            return min(max_pages, ((self.total + 63) // 64 + g - 1) // g * g)
        return max_pages + (n_copies - 1) * (max_pages - self.total // 64)

    def fill(self, slot, n_copies, seed=None, offset=0, sp=None):
        """its vcb_prompt in slots slot .. slot+n_copies-1, sampling from the Philox stream of a torch CUDA generator at
        (seed, offset); seed None: host noise.  sp: the group's own vcb_sampling (vcb_decode_step with sp NULL)"""
        P = _lib.vcb_prompt(slot=slot, n_copies=n_copies, mode=0 if self.spans is None else 1,
                            x_len=int(self.x_ids.shape[0]), text_ids_dev=self.x_ids.data_ptr(),
                            y_len=int(self.y_tok.shape[0]), y_tokens_dev=self.y_tok.data_ptr(),
                            mask_rows_dev=None if self.mask_rows is None else self.mask_rows.data_ptr(),
                            n_more_spans=len(self.more_vals))
        for i, v in enumerate(self.more_vals):
            P.more_mask_rows[i] = int(v)
        if sp is not None:
            P.sampling = C.pointer(sp)
        if self.align is not None:
            P.align_heads = self.align
        if seed is not None:
            m = self.model
            P.rng_seed = int(seed) & 0xFFFFFFFFFFFFFFFF
            P.rng_offset = int(offset)
            # the group's draw per sampling step is [n_copies*K, V], as the reference's multinomial
            P.rng_threads = m._rng_threads(self.y0.device, n_copies * m.args.n_codebooks * m.n_audio_tokens[0])
        return P

    def source(self):
        """its vcb_edit_source for vcb_poll_frames_ex: y0 and the spans of an edit, zeros for TTS"""
        src = _lib.vcb_edit_source()
        if self.spans is not None:
            src.orig_dev, src.T, src.n_spans = self.y0.data_ptr(), int(self.y0.shape[1]), len(self.spans)
            for j, (s0, s1) in enumerate(self.spans):
                src.spans[j][0], src.spans[j][1] = s0, s1
        return src

    def result(self, rows, st, lp_rows=None):
        """(res [1,K,T+G], gen [1,K,G]) as inference_tts returns them, or (res, None) with res as inference returns it,
        from the utterance's delayed token rows [n,K] and its vcb_status.  A TTS utterance that is not done (a truncated
        session) keeps its final frames only: the still-delayed tail is dropped.
        lp_rows: the log-probability rows [n,K] of those tokens (vcb_read_logprobs); the result then also holds lp, fp32
        on the model's device, un-delayed as the codes: [1,K,G] aligned with gen, or [1,K,T'] aligned with an edit's res,
        NaN on the frames copied from the original."""
        a = self.model.args
        K, dev = a.n_codebooks, self.y0.device
        gen, lp = None, None
        if self.spans is None:
            n = rows.shape[0] - K if st.done else final_frames(rows, K, _end_token(a))
            gen = torch.from_numpy(frame_codes(rows, K, 0, n)).to(dev)
            res = torch.cat([self.y0, gen], dim=1).unsqueeze(0)
            expected = self.y0.shape[1] + n
            assert res.shape == torch.Size((1, K, expected)), f"res.shape: {res.shape}, expected_y_len: {expected}"
            if lp_rows is not None:
                lp = frame_codes(lp_rows, K, 0, n)
        else:
            assert st.done, "edit session results() needs finished utterances"
            ends = [st.span_ends[j] for j in range(st.n_spans_done)]
            assert len(ends) == len(self.spans), f"len(generated): {len(ends)}, num_mask: {len(self.spans)}"
            pieces, lps, lo = [], [], 0
            for (s0, s1), hi in zip(self.non_mask, ends):
                pieces.append(self.y0[:, s0:s1])
                pieces.append(torch.from_numpy(VoiceCraft._undelay(rows[lo:hi], K)).to(dev))
                if lp_rows is not None:
                    lps += [np.full((K, s1 - s0), np.nan, np.float32), VoiceCraft._undelay(lp_rows[lo:hi], K)]
                lo = hi
            s0, s1 = self.non_mask[-1]
            pieces.append(self.y0[:, s0:s1])
            res = torch.cat(pieces, dim=1).unsqueeze(0)
            if lp_rows is not None:
                lp = np.concatenate(lps + [np.full((K, s1 - s0), np.nan, np.float32)], axis=1)
        if a.special_first:
            res = res - int(a.n_special)
            gen = None if gen is None else gen - int(a.n_special)
        out = res, None if gen is None else gen.unsqueeze(0)
        return out if lp_rows is None else out + (torch.from_numpy(lp).unsqueeze(0).to(dev),)


def _align_heads(model, alignment, xs, edit=False):
    """alignment= of a call as the vcb_prompt.align_heads of its prompts (a ctypes uint32 array, or None: off), checked
    against the texts xs ([1,L] tensors) and the engine's align_text_cap; raises ValueError"""
    masks = head_masks(alignment, model.args.num_decoder_layers, model.args.nhead)
    if masks is None:
        return None
    if edit:
        raise ValueError("alignment: speech edits are not supported (TTS results only)")
    cap = model._eng_opts["align_text_cap"]
    longest = max(int(x.shape[-1]) for x in xs)
    if longest > cap:
        raise ValueError(f"alignment of a {longest}-token text needs configure_engine(align_text_cap >= {longest}) "
                         f"(align_text_cap is {cap})")
    return (C.c_uint32 * len(masks))(*[int(v) for v in masks])


def _read_alignment(model, eng, slot, prompt, frames, stream):
    """the Alignment of the first `frames` frames of the result in `slot` (prefilled from `prompt` with align_heads):
    frame t is the row at position x_len + t (voicecraft_b200/alignment.py)"""
    x_len = int(prompt.x_ids.shape[0])
    buf = np.empty((frames, x_len), dtype=np.float32)
    _lib.check(_lib.load().vcb_read_alignment(eng, slot, buf.ctypes.data_as(C.POINTER(C.c_float)), x_len, frames, stream))
    soft = torch.from_numpy(buf).to(prompt.y0.device)
    return Alignment.from_soft(soft, model.args.encodec_sr, prompt.x_ids)


def _prefill(eng, prompts, stream):
    """one packed prefill of [(_Prompt, slot, n_copies, seed, offset[, sp])] (see _Prompt.fill); a failed prefill holds
    nothing"""
    P = (_lib.vcb_prompt * len(prompts))()
    for j, (p, *where) in enumerate(prompts):
        P[j] = p.fill(*where)
    _lib.check(_lib.load().vcb_prefill(eng, P, len(prompts), stream))


class _AudioStream:
    """The iterator of a streaming loop (TtsStream, BatcherStream).  Its state `st` is held by the loop's generator
    `_run(st)`, not by the iterator, so dropping the iterator closes it at once (no reference cycle).  Closing it early
    (break, close(), garbage collection) runs `_finish(st)`, which releases the engine slots and the codec streams."""

    def _start(self, st, n_streams):
        """open n_streams codec streams and the codec's CUDA stream on st.dev, then the loop"""
        self._st, self._it = st, None
        st.codec = st.push = None
        try:
            st.codec = st.tok.open_stream(max_streams=n_streams, sample_rate=st.sample_rate)
            st.cstream = torch.cuda.Stream(device=st.dev)
        except Exception:
            self.close()
            raise
        self._it = self._run(st)

    @staticmethod
    def _close_codec(st):
        if st.codec is not None:
            st.codec.close()
            st.codec = None

    @property
    def push_host_seconds(self):
        """host time spent in the push steps so far, outside the device waits"""
        return self._st.push.host_s if self._st.push is not None else 0.0

    def __iter__(self):
        return self

    def __next__(self):
        return next(self._it)

    def close(self):
        st = getattr(self, "_st", None)
        if st is None:
            return
        if self._it is not None:
            self._it.close()
        self._finish(st)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class TtsStream(_AudioStream):
    """Audio of a DecodeSession while it generates (VoiceCraft.inference_tts_stream / inference_tts_many_stream).

    Iterating runs the session: every `poll_every` steps it polls, reads the token rows and sends each utterance's newly
    final frames to the codec (a CodecStream on a second CUDA stream) -- all utterances with enough new frames in one call.
    The next decode steps are enqueued before the chunk's waveform is waited for.  A chunk is the waveform of those frames,
    bit-identical to the same samples of ``decode_codes`` of the utterance's whole generation.  An utterance's first
    chunk waits for max(chunk_frames, min_frames) frames; one that ends with fewer than min_frames frames is decoded in one
    ``decode_codes`` call.  Yields (i, wav [1, channels, n*hop]).  After the iteration, ``results`` holds what
    ``DecodeSession.results()`` returns.  Closing it early (break, close(), garbage collection) releases the session's
    engine slots and the codec streams."""

    def __init__(self, sess: "DecodeSession", tokenizer, chunk_frames: int = 25, poll_every: int = 8, sample_rate=None):
        if chunk_frames < 1 or poll_every < 1:
            raise ValueError("chunk_frames and poll_every must be >= 1")
        if sess.n_copies > 1:
            sess.close()
            _no_stream_best_of(sess.n_copies)
        if sess.edit and sess._host_noise:
            sess.close()
            raise _lib.VcbError("streaming an edit needs the device generators (model.noise_fn / noise_fns must be None): "
                                "the polls do not follow the forced hand-over steps, so host noise would be drawn for them")
        self._start(SimpleNamespace(sess=sess, dev=sess.dev, tok=tokenizer, chunk_frames=int(chunk_frames),
                                    poll_every=int(poll_every), results=None, logprobs=None, alignments=None,
                                    first_audio_steps=None,
                                    sample_rate=sample_rate), sess.B)

    @property
    def results(self):
        return self._st.results

    @property
    def logprobs(self):
        """after the iteration: utterance i's lp, as DecodeSession.results(logprobs=True) returns it"""
        return self._st.logprobs

    @property
    def alignments(self):
        """after the iteration, for a session opened with alignment=: utterance i's Alignment (else None)"""
        return self._st.alignments

    @property
    def first_audio_steps(self):
        """session steps sampled when the poll that gathered the first chunk ran"""
        return self._st.first_audio_steps

    @property
    def sess(self):
        return self._st.sess

    @staticmethod
    def _finish(st):
        _AudioStream._close_codec(st)
        st.sess.close()

    @staticmethod
    @torch.no_grad()
    def _run(st):
        sess = st.sess
        try:
            with torch.cuda.device(sess.dev):
                push = _PushStep(sess.model, sess.eng, sess.stream, st.tok, st.codec, st.cstream, st.chunk_frames,
                                 st.poll_every, strict=True)
                st.push = push
                live = [_Utterance(s, i, f"utterance {i}", src=p.source()) for i, (s, p) in
                        enumerate(zip(sess.slots, sess.prompts))]
                sess.sample()
                while sess.steps % st.poll_every:
                    sess.step()
                while True:
                    def advance(status):             # the next steps are queued while the codec works
                        if not all(s.done for s in status):
                            for _ in range(st.poll_every):
                                sess.step()
                    polled = sess.steps
                    status, out, _ = push([r for r in live if not r.closed], advance)
                    done = all(s.done for s in status)
                    for r, w in out:
                        if w is None:
                            continue
                        if st.first_audio_steps is None:
                            st.first_audio_steps = polled
                        yield r.cid, w
                    if done and all(r.closed for r in live):
                        break
                out = sess.results(logprobs=True)
                st.results = [(o[0], o[1]) for o in out]
                st.logprobs = [o[2] for o in out]
                st.alignments = [o[3] for o in out] if sess.align else None
                if sess.edit:                        # what inference_many / inference return: res alone
                    st.results = [res for res, _ in st.results]
        finally:
            TtsStream._finish(st)


class _Utterance:
    """An utterance of a streaming loop: engine slot, codec stream id, its vcb_edit_source (_Prompt.source), frames sent
    to the codec (pushed), all of its audio handed out (closed), its vcb_status at the last poll.  A sentence of a long
    ticket shares its codec stream id, and so its resampler stream, with the ticket's other sentences: `more` marks one
    that a later sentence follows (its resampler stream is not finished with it), `carry` one that an earlier sentence
    preceded (its resampler stream may hold that sentence's pending samples)."""
    __slots__ = ("slot", "cid", "label", "ticket", "src", "pushed", "closed", "status", "more", "carry")

    def __init__(self, slot, cid, label, ticket=None, src=None, more=False, carry=False):
        self.slot, self.cid, self.label, self.ticket = slot, cid, label, ticket
        self.src = _lib.vcb_edit_source() if src is None else src
        self.pushed, self.closed, self.status = 0, False, None
        self.more, self.carry = more, carry


class _PushStep:
    """One poll of a streaming loop (TtsStream, ContinuousBatcher.stream).  vcb_poll_frames_ex gathers the live
    utterances' newly final frames (of an edit: of its whole output, original pieces included) on the device behind one wait; those with enough new frames go to the codec in one ragged call on
    a second CUDA stream; the caller's next decode steps are enqueued; then the waveform is waited for.

    An utterance (_Utterance) has its first chunk waits for max(chunk_frames, min_frames) frames, later ones for chunk_frames,
    the last one takes what is left; one that ends with fewer than min_frames frames is decoded whole (decode_codes).
    Resampled (a codec stream with its own sample_rate), an utterance's last push is marked final; one that ends at a
    poll with no new frame has its resampler tail flushed, and one decoded whole is resampled in one call.  A chunk that
    resamples to no sample is not handed out unless it closes its utterance.
    A chunk holding a non-audio code fails its utterance before any of its codes reach the codec: `strict` raises
    VcbError before the codec is called at all."""

    def __init__(self, model, eng, stream, tokenizer, codec, cstream, chunk_frames, poll_every, strict):
        a = model.args
        self.lib, self.eng, self.stream, self.tok, self.codec, self.cstream = _lib.load(), eng, stream, tokenizer, codec, cstream
        self.dev, self.K, self.strict = model.mask_embedding.device, a.n_codebooks, strict
        self.chunk_frames, self.first = chunk_frames, max(chunk_frames, codec.min_frames)
        self.resampled = codec.sample_rate != tokenizer.sample_rate
        # new frames at one poll: fewer than a chunk's threshold were left over, plus at most one per row sampled since the
        # last poll (a newly admitted utterance: its first sample and poll_every steps)
        self.max_frames = self.first + poll_every + 1
        self.offset = int(a.n_special) if a.special_first else 0
        self.host_s = 0.0                    # host time in the step, outside the three device waits

    def __call__(self, live, advance):
        """live: utterances that are not closed.  advance(status) enqueues the next decode steps.  Returns (status, out,
        failed): out lists (utterance, wav [1, channels, n*hop], or None when it closes with no new frames) in `live`
        order; failed maps a failed utterance to its message.  Raises VcbError when a slot ran out of engine capacity."""
        t_in = time.perf_counter()
        n, mf, lib = len(live), self.max_frames, self.lib
        codes = torch.empty((n, self.K, mf), dtype=torch.int64, device=self.dev)     # fresh: the codec stream reads it
        status, final, bad = (_lib.vcb_status * n)(), (C.c_int32 * n)(), (C.c_int32 * (3 * n))()
        t0 = time.perf_counter()
        _lib.check(lib.vcb_poll_frames_ex(self.eng, (C.c_int32 * n)(*[r.slot for r in live]), n,
                                          (_lib.vcb_edit_source * n)(*[r.src for r in live]),
                                          (C.c_int32 * n)(*[r.pushed for r in live]), mf, self.offset,
                                          int(self.tok.config.bins), codes.data_ptr(), status, final, bad, self.stream))
        waited = time.perf_counter() - t0
        _check_capacity(status)
        push, whole, failed, flush = {}, {}, {}, []
        for j, r in enumerate(live):
            fin, f = bool(status[j].done), int(final[j])
            new = f - r.pushed
            if r.pushed == 0 and fin and f < self.codec.min_frames:
                if f == 0 and r.carry and not r.more and self.resampled:     # the earlier sentences' tail is pending
                    flush.append(j)
                whole[j] = f
            elif new > 0 and (fin or new >= (self.first if r.pushed == 0 else self.chunk_frames)):
                push[j] = min(new, mf)
            else:
                r.closed = fin and r.pushed == f
                if r.closed and r.pushed > 0 and self.resampled and not r.more:  # its last push was not final: the tail
                    flush.append(j)                                               # is pending
                continue
            if bad[3 * j] >= 0:
                failed[r] = (f"{r.label}: frame {bad[3 * j]} holds the non-audio token {bad[3 * j + 2]} in codebook "
                             f"{bad[3 * j + 1]}; it has no waveform")
                push.pop(j, None)
                whole.pop(j, None)
                r.closed = True
                continue
            r.pushed += push[j] if j in push else f
            r.closed = fin and r.pushed == f
        if failed and self.strict:
            raise _lib.VcbError(next(iter(failed.values())))
        wav, tail, wavs = None, None, {}
        wav_lens = tail_lens = None
        if push or any(whole.values()) or flush:     # the codec works on its own CUDA stream ...
            with torch.cuda.stream(self.cstream):
                codes.record_stream(self.cstream)
                if push:
                    rows = list(push)
                    wav = self.codec.decode(codes[rows, :, :max(push.values())], ids=[live[j].cid for j in rows],
                                            lens=list(push.values()),
                                            final=[live[j].closed and not live[j].more for j in rows]
                                            if self.resampled else None)
                    wav_lens = self.codec.out_lens
                if flush:
                    tail = self.codec.flush([live[j].cid for j in flush])
                    tail_lens = self.codec.out_lens
                for j, f in whole.items():
                    r = live[j]
                    if f == 0:
                        continue
                    w = self.tok.decode_codes(codes[j:j + 1, :, :f])
                    if self.resampled and (r.more or r.carry):     # a long ticket's resampler runs across its sentences
                        w = self.codec.push_audio(w, [r.cid], [not r.more])
                        n_out = self.codec.out_lens[0]
                        if n_out == 0:
                            continue
                        w = w[:, :, :n_out]
                    elif self.resampled:
                        w = self.tok.resample(w, self.tok.sample_rate, self.codec.sample_rate)
                    wavs[j] = w
            ev = torch.cuda.Event()
            ev.record(self.cstream)
        t1 = time.perf_counter()
        advance(status)                      # ... while the next steps are already queued on the LM's
        t2 = time.perf_counter()
        out = []
        if wav is not None or tail is not None or wavs:
            ev.synchronize()
            cur = torch.cuda.current_stream(self.dev)
            for out_wav, rows, lens in ((wav, list(push), wav_lens), (tail, flush, tail_lens)):
                if out_wav is None:
                    continue
                out_wav.record_stream(cur)
                for b, j in enumerate(rows):
                    if lens[b] > 0:
                        wavs[j] = out_wav[b:b + 1, :, :lens[b]]
            for w in wavs.values():
                w.record_stream(cur)
        t3 = time.perf_counter()
        for j, r in enumerate(live):
            if j in wavs:
                out.append((r, wavs[j]))
            elif r.closed and r not in failed:
                out.append((r, None))
        self.host_s += (time.perf_counter() - t_in) - waited - (t2 - t1) - (t3 - t2)
        return status, out, failed


class _SingleTtsStream(TtsStream):
    """TtsStream of one utterance (inference_tts_stream): yields the wav chunks alone; ``result`` = (res, gen)"""

    def __next__(self):
        return next(self._it)[1]

    @property
    def result(self):
        return None if self.results is None else self.results[0]

    @property
    def logprobs(self):
        """after the iteration: the lp that inference_tts / inference return with logprobs=True"""
        lps = TtsStream.logprobs.fget(self)
        return None if lps is None else lps[0]

    @property
    def alignment(self):
        """after the iteration: the Alignment inference_tts returns with alignment= (None without it)"""
        als = TtsStream.alignments.fget(self)
        return None if als is None else als[0]


class LongTtsStream:
    """Iterator of VoiceCraft.inference_long_tts_stream: the wav chunks of its one long ticket (a BatcherStream), in
    sentence order.  A sentence holding a non-audio frame raises VcbError.  Closing it early releases the engine slots
    and the codec streams, and leaves the device generator where it was."""

    def __init__(self, cb, chain, gen, tokenizer, chunk_frames, sample_rate):
        self._cb, self._chain, self._gen = cb, chain, gen
        self.results = self.logprobs = self.alignments = None
        self._it = cb.stream(tokenizer, chunk_frames, sample_rate)

    def __iter__(self):
        return self

    def __next__(self):
        try:
            _, w, _ = next(self._it)
        except StopIteration:
            cb = self._cb
            if cb.results and cb.results[0] is not None:
                self.results, self.logprobs, self.alignments = cb.results[0], cb.logprobs[0], cb.alignments[0]
                self._gen.set_offset(self._chain.offset)
            raise
        if w is None:
            self.close()
            raise _lib.VcbError(self._cb.errors[0])
        return w

    def close(self):
        self._it.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class DecodeSession:
    """A batch of independent utterances resident in the engine, one random stream each, and one slot each or, best-of-N,
    one group of consecutive slots each."""

    def __init__(self, model: "VoiceCraft", xs, ys, sp, mask_intervals=None, seeds=None, noise_fns=None, *, best_of=1,
                 n_copies=None, alignment=None):
        """best_of: each utterance is sampled in best_of slots and keeps the copy that ends first (inference_tts_batch).
        n_copies (the single calls inference_tts, inference_tts_batch, inference and inference_tts_stream): best_of, and
        the one utterance samples from the device generator's stream at its current offset, and results() leaves the
        generator advanced as the single call does."""
        K = model.args.n_codebooks
        dev = model.mask_embedding.device
        self.model, self.sp, self.dev, self.K = model, sp, dev, K
        self.B, self.V, self.n_copies = len(xs), model.n_audio_tokens[0], _check_best_of(n_copies or best_of)
        self.lib = _lib.load()
        self.edit = mask_intervals is not None
        if seeds is not None and len(seeds) != self.B:
            raise ValueError("seeds: one per utterance")
        if noise_fns is not None and len(noise_fns) != self.B:
            raise ValueError("noise_fns: one per utterance")
        _no_host_noise_under_ras(sp.ras_window, noise_fns is not None or model.noise_fn is not None)
        self.prompts = []
        for i, (x, y) in enumerate(zip(xs, ys)):
            assert x.ndim == 2 and y.ndim == 3 and y.shape[2] == K
            spans = [(int(s), int(e)) for s, e in mask_intervals[i][0].tolist()] if self.edit else None
            self.prompts.append(_Prompt(model, x, y, spans, sp.max_frames))
        # one range check for the whole batch (the reference's embedding lookups raise on a bad id)
        model._check_ids(torch.cat([p.x_ids for p in self.prompts]), torch.cat([p.y_tok.reshape(-1) for p in self.prompts]))
        c_masks = _align_heads(model, alignment, xs, self.edit)
        self.align = c_masks is not None
        for p in self.prompts:
            p.align = c_masks
        self.eng, self.slots = model._take_slots(self.B * self.n_copies, max(p.need_seq for p in self.prompts))
        try:
            n = len(self.slots)
            # random streams: caller noise (model.noise_fn: one [B*K,V] draw per step; noise_fns: one [K,V] draw per
            # utterance and step) or, by default, one Philox stream per utterance generated inside the sampler kernel
            self._noise_fns = noise_fns
            self._host_noise = noise_fns is not None or model.noise_fn is not None
            self._buf = torch.empty((n * K, self.V), device=dev, dtype=torch.float32) if self._host_noise else None
            gen = torch.cuda.default_generators[dev.index or 0]
            seed0, off0 = int(gen.initial_seed()), int(gen.get_offset())
            self._gen = gen if n_copies is not None and not self._host_noise else None
            # (seed, offset) per utterance; a single call's (seed0, off0) is the device generator's own stream
            streams = [(None, 0) if self._host_noise else (seeds[i], 0) if seeds is not None else (seed0 + i, off0)
                       for i in range(self.B)]
            self.c_slots = (C.c_int32 * n)(*self.slots)
            self.status = (_lib.vcb_status * n)()
            self.steps = 0
            with torch.cuda.device(dev):
                self.stream = torch.cuda.current_stream().cuda_stream
                _prefill(self.eng, [(p, self.slots[i * self.n_copies], self.n_copies, *streams[i])
                                    for i, p in enumerate(self.prompts)], self.stream)
        except BaseException:
            self.close()                     # a failed prefill holds nothing: give the slots back
            raise

    def _noise(self, draw=True):
        """the host noise buffer (None: the device streams), refilled unless draw is False"""
        if not self._host_noise:
            return None
        if draw and self._noise_fns is not None:
            R = self.n_copies * self.K             # an utterance's rows: member-major, as its group draws them
            for i, fn in enumerate(self._noise_fns):
                self._buf[i * R:(i + 1) * R].copy_(fn((R, self.V), self.dev).to(device=self.dev, dtype=torch.float32))
        elif draw:
            self.model._draw_noise(self._buf)
        return self._buf.data_ptr()

    def _launch(self, fn, noise):
        _lib.check(fn(self.eng, self.c_slots, len(self.slots), noise, C.byref(self.sp), self.stream))
        self.steps += 1

    def sample(self):
        """first sampling step (on the prefill's last hidden states)"""
        self._launch(self.lib.vcb_sample, self._noise())

    def step(self):
        # edit sessions: forced hand-over steps of individual utterances ignore their noise rows / consume no draw
        self._launch(self.lib.vcb_decode_step, self._noise())

    def poll(self):
        _lib.check(self.lib.vcb_poll(self.eng, self.c_slots, len(self.slots), self.status, self.stream))
        return self.status

    def all_done(self):
        st = self.poll()
        _check_capacity(st)
        return all(s.done for s in st)

    def _run_many(self, poll_every, logprobs=False):
        """inference_many / inference_tts_many: sample and step until every utterance is done, polling every
        `poll_every` steps; returns results(logprobs) and closes the session"""
        try:
            self.sample()
            if self.model._eng_opts["kv_pool_gb"] is not None and self.n_copies == 1 and not self._host_noise:
                return self._run_pooled(poll_every, logprobs)
            while True:
                if self.steps % poll_every == 0 and self.all_done():
                    break
                self.step()
            return self.results(logprobs)
        finally:
            self.close()

    def _run_pooled(self, poll_every, logprobs=False):
        """_run_many's loop under a KV budget (KvPoolPolicy), returning the results: a refused step swaps the youngest
        utterance out; a finished one is read and leaves its slot and pages at once; swapped-out utterances come back,
        oldest first, into the session's freed slots"""
        pool = KvPoolPolicy(_EngineOps(self.eng, self.stream, self.sp), True, self.B)
        free, done, results = set(), [False] * self.B, [None] * self.B
        try:
            while True:
                out = {t[1] for t in pool.swapped}
                for i, slot in pool.resume(free, sum(1 for i in range(self.B) if not done[i] and i not in out)):
                    # a slot the session holds; self.slots may now list a slot twice (a finished utterance's, reused)
                    # and miss a freed one, which is harmless: every open slot is listed, index 0 (the oldest) is never
                    # a victim, so _release_slots still finds the session, and releasing a closed slot does nothing
                    self.slots[i] = slot
                out = {t[1] for t in pool.swapped}
                live = [(i, self.slots[i], i, True) for i in range(self.B) if not done[i] and i not in out]
                if not live:
                    break
                for _ in range(poll_every):
                    live, gone = pool.step(live)
                    free.update(slot for _, slot in gone)
                    self.steps += 1
                st = (_lib.vcb_status * len(live))()
                _lib.check(self.lib.vcb_poll(self.eng, (C.c_int32 * len(live))(*[u[1] for u in live]), len(live), st,
                                             self.stream))
                _check_capacity(st)
                for (i, slot, _, _), s in zip(live, st):
                    if s.done:
                        results[i] = self._result(i, slot, s, logprobs)
                        _lib.check(self.lib.vcb_release(self.eng, slot, 1))
                        done[i] = True
                        free.add(slot)
        finally:
            pool.close()
            self.c_slots = (C.c_int32 * len(self.slots))(*self.slots)
        return results

    def _run_single(self, logprobs=False):
        """The loop of a single call; returns results().  The done flag is polled every model.poll_every steps: a finished
        group ignores further steps and consumes nothing, so the device generator still ends exactly where the reference's
        would.  Edits, host noise and trace_logits poll every step; a forced hand-over step then draws no host noise and
        appends no trace."""
        m = self.model
        every = 1 if (self.edit or self._host_noise or m.trace_logits is not None) else max(1, int(m.poll_every))
        with torch.cuda.device(self.dev):
            self.sample()
            self._trace()
            while True:
                if self.steps % every == 0 and self.all_done():
                    break
                forced = every == 1 and any(s.forced for s in self.status)
                self._launch(self.lib.vcb_decode_step, self._noise(draw=not forced))
                if not forced:
                    self._trace()
            return self._results(self.status, logprobs)

    def _trace(self):
        """append the raw logits [n*K, V] of the last sampling step to model.trace_logits (when it is a list)"""
        if self.model.trace_logits is not None:
            rows = len(self.slots) * self.K
            t = torch.empty(rows, self.V, device=self.dev, dtype=torch.float32)
            _lib.check(self.lib.vcb_debug_logits(self.eng, t.data_ptr(), rows))
            self.model.trace_logits.append(t)

    def raw_tokens(self, i):
        """delayed token rows [n_steps, K] of utterance i (host numpy); best-of-N: of its kept copy once the group has
        decided, of its first copy before"""
        st = self.poll()
        j = i * self.n_copies
        if self.n_copies > 1 and st[j].keep >= 0:
            j += st[j].keep
        return self.model._read_rows(self.eng, self.slots[j], st[j].n_steps, self.stream)

    def results(self, logprobs=False):
        """one (res, gen) per utterance as inference_tts returns it ((res, None) for an edit); logprobs=True: (res, gen,
        lp) with lp as inference_tts(..., logprobs=True) / inference(..., logprobs=True) return it"""
        return self._results(self.poll(), logprobs)

    def _kept(self, i, st):
        """index in `st` of utterance i's result: the copy of its best-of-N group that ended first, or its slot"""
        j = i * self.n_copies
        return j + (st[j].keep if self.n_copies > 1 else 0)

    def _result(self, i, slot, st, logprobs):
        """utterance i's result from its slot (its kept copy's) and vcb_status; with alignment, its Alignment last"""
        m = self.model
        lp = m._read_lp(self.eng, slot, st.n_steps, self.stream) if logprobs else None
        out = self.prompts[i].result(m._read_rows(self.eng, slot, st.n_steps, self.stream), st, lp)
        return out + (self._alignment(i, slot, out[0].shape[-1]),) if self.align else out

    def _alignment(self, i, slot, frames):
        return _read_alignment(self.model, self.eng, slot, self.prompts[i], frames, self.stream)

    def _results(self, st, logprobs=False):
        out = []
        for i in range(len(self.prompts)):
            j = self._kept(i, st)
            out.append(self._result(i, self.slots[j], st[j], logprobs))
        if self._gen is not None:
            self._gen.set_offset(int(st[0].rng_offset))
        return out

    def close(self):
        self.model._release_slots(self.slots, n_copies=self.n_copies)


def place_groups(free, sizes, nxt):
    """Admission of ContinuousBatcher: tickets nxt, nxt+1, ... in order, ticket t needing sizes[t] consecutive slots
    (its best-of-N group).  Each takes the lowest run of that many consecutive slots in the set `free`; the first ticket
    that finds none stops the admission, so a later ticket never overtakes it.  Removes the taken slots from `free` and
    returns ([(first slot, ticket)], the next ticket to admit)."""
    new = []
    while nxt < len(sizes):
        n = sizes[nxt]
        base = next((s for s in sorted(free) if all(s + c in free for c in range(n))), None)
        if base is None:
            break
        free.difference_update(range(base, base + n))
        new.append((base, nxt))
        nxt += 1
    return new, nxt


class _Chain:
    """The sentences of a long ticket (ContinuousBatcher.submit with a list of x): they run one after another on the
    ticket's slot(s), sentence i+1 sampling from the ticket's Philox stream at the offset where sentence i ended, as the
    reference's Long TTS loop calls inference_tts once per sentence on one generator.  `offset` is where the next sentence
    starts (first: 0, or the device generator's offset for VoiceCraft.inference_long_tts), and once the chain is done where
    its stream ended; `results` / `logprobs` hold the finished sentences'."""

    def __init__(self, xs, offset=0):
        self.xs, self.offset0 = list(xs), int(offset)
        self.start([])

    def start(self, prompts):
        """(re)start the chain with one _Prompt per sentence"""
        self.prompts, self.offset, self.results, self.logprobs, self.alignments = prompts, self.offset0, [], [], []

    @property
    def need_seq(self):
        return max(p.need_seq for p in self.prompts)

    @property
    def prompt(self):
        """the prompt of the sentence to run now"""
        return self.prompts[len(self.results)]

    def ended(self, result, lp, offset, al=None) -> bool:
        """the sentence running now ended with `result`, `lp`, `al` (its Alignment or None), its stream at `offset`
        (vcb_status.rng_offset of its slot, its group's first): True when another sentence follows"""
        self.results.append(result)
        self.logprobs.append(lp)
        self.alignments.append(al)
        self.offset = int(offset)
        return len(self.results) < len(self.prompts)


class _Ticket:
    """A ContinuousBatcher ticket: `prompt` the _Prompt that runs now (placeholder codes until _encode replaces them),
    `seed`, `best_of`, `sp` its vcb_sampling, `pending` (x, audio, sample_rate) of audio not encoded yet, `chain` a
    long ticket's _Chain and `align` its vcb_prompt.align_heads (None: no alignment), which every prompt it runs carries."""
    __slots__ = ("prompt", "seed", "best_of", "sp", "pending", "chain", "align")

    def __init__(self, prompt, seed, best_of, sp, pending=None, chain=None, align=None):
        self.prompt, self.seed, self.best_of, self.sp, self.pending, self.chain = prompt, seed, best_of, sp, pending, chain
        self.align = align

    @property
    def need_seq(self):
        """engine positions the ticket can reach: a long ticket's longest sentence's"""
        return self.prompt.need_seq if self.chain is None else self.chain.need_seq

    def pages(self, max_pages):
        """KV pages the prefill of its prompt takes for its group of best_of copies"""
        return self.prompt.pages(self.best_of, max_pages)


_TOO_SMALL = ("KV pool smaller than one utterance (kv_pool_gb; pages held by other open sessions or batchers of this model "
              "count against it)")


class KvPoolPolicy:
    """How the batcher and sessions share a KV page pool (DESIGN.md section 7).  `ops` is the engine (_EngineOps; the tests pass a fake):
    free_pages(), step(slots) -> 0 or VCB_ERR_KV_FULL, swap_out(slot) -> snapshot, swap_in(snapshot, slot),
    snapshot_pages(snapshot), free(snapshot).  An utterance is (key, slot, age, single): age orders admissions (oldest
    first), single marks a one-copy utterance (a best-of-N group keeps its full reservation and never swaps).
      admission  strict FIFO; while anything is swapped out, nothing new; otherwise a ticket needs its prompt pages plus one
                 growth chunk per active slot free (budget only: the default pool always covers max_slots full slots).
                 The next sentence of a long ticket keeps its slots and goes first, swapped-out utterances or not
      victim     a refused step swaps out the youngest single utterance it lists and is retried without it
      resume     swapped-out utterances come back, oldest first, when their pages plus a chunk per active slot are free
      bound      at most max_swapped utterances are out at once
    The pages it counts are the engine's free pages: every open session and batcher of the model shares that engine, so
    pages another one holds count against this one's pool."""

    def __init__(self, ops, budget, max_swapped, chunk=_lib.KV_GROW_PAGES):
        self.ops, self.budget, self.max_swapped, self.chunk = ops, bool(budget), int(max_swapped), int(chunk)
        self.swapped = []                 # [(age, key, snapshot)], oldest first
        self.swap_outs = self.swap_ins = 0

    def admit_count(self, needs, n_active, held=False):
        """how many of the queued tickets `needs` [(pages, slots)] (FIFO order) the pool takes now next to n_active slots.
        held: they already hold their slots (the next sentences of long tickets), so swapped-out utterances, which wait
        for free slots, do not hold them back"""
        if self.swapped and not held:
            return 0
        if not self.budget:
            return len(needs)
        free, k = self.ops.free_pages(), 0
        for pages, n in needs:
            if free < pages + self.chunk * n_active:
                if n_active == 0:
                    raise _lib.VcbError(f"{_TOO_SMALL}: its prompt needs {pages} pages, {free} are free")
                break
            free, n_active, k = free - pages, n_active + n, k + 1
        return k

    def resume(self, free_slots, n_active):
        """swap utterances back in, oldest first, each into the lowest slot of the set free_slots; [(key, slot)]"""
        back = []
        while self.swapped and free_slots:
            age, key, snap = self.swapped[0]
            pages, free = self.ops.snapshot_pages(snap), self.ops.free_pages()
            if free < pages + self.chunk * (n_active + 1) and not (n_active == 0 and free >= pages):
                if n_active == 0:
                    raise _lib.VcbError(f"{_TOO_SMALL}: it holds {pages} pages, {free} are free")
                break
            slot = min(free_slots)
            self.ops.swap_in(snap, slot)
            free_slots.discard(slot)
            self.ops.free(snap)
            self.swapped.pop(0)
            self.swap_ins += 1
            n_active += 1
            back.append((key, slot))
        return back

    def step(self, live, leaving=False):
        """one decode step of the utterances `live` [(key, slot, age, single)]; a refused step swaps out the youngest single
        one and is retried.  Returns (the utterances that stepped, [(key, slot)] swapped out).
        leaving: utterances outside `live` hold pages they give back before the caller's next round (finished ones that are
        not released yet).  A refused step that no victim can resolve then does not raise: it returns (None, swapped out
        so far) and the caller steps no further this round."""
        out = []
        while live:
            if self.ops.step([u[1] for u in live]) == 0:
                return live, out
            singles = [u for u in live if u[3]]
            if len(live) == 1 or not singles:
                if leaving:
                    return None, out
                raise _lib.VcbError(f"{_TOO_SMALL}: a step of it alone does not fit")
            if len(self.swapped) >= self.max_swapped:
                raise _lib.VcbError(f"KV pool too small: {len(self.swapped)} utterances are swapped out already")
            victim = max(singles, key=lambda u: u[2])
            snap = self.ops.swap_out(victim[1])
            self.swapped.append((victim[2], victim[0], snap))
            self.swapped.sort(key=lambda t: t[0])
            self.swap_outs += 1
            live = [u for u in live if u is not victim]
            out.append((victim[0], victim[1]))
        return live, out

    def drop(self, key):
        """forget a swapped-out utterance (a cancelled ticket): frees its snapshot; False if it is not swapped out"""
        for i, (_, k, snap) in enumerate(self.swapped):
            if k is key:
                self.ops.free(snap)
                del self.swapped[i]
                return True
        return False

    def close(self):
        """frees every snapshot still held"""
        for _, _, snap in self.swapped:
            self.ops.free(snap)
        self.swapped = []


class _EngineOps:
    """KvPoolPolicy's view of an engine: decode steps with device noise and the sampling parameters `sp` (None: each
    group's own)"""

    def __init__(self, eng, stream, sp=None):
        self.eng, self.stream, self.lib = eng, stream, _lib.load()
        self.sp = None if sp is None else C.byref(sp)

    def free_pages(self):
        return self.lib.vcb_counter(self.eng, b"kv_pages_free")

    def step(self, slots):
        rc = self.lib.vcb_decode_step(self.eng, (C.c_int32 * len(slots))(*slots), len(slots), None, self.sp, self.stream)
        if rc != _lib.VCB_ERR_KV_FULL:
            _lib.check(rc)
        return rc

    def swap_out(self, slot):
        snap = C.c_void_p()
        _lib.check(self.lib.vcb_swap_out(self.eng, slot, C.byref(snap), self.stream))
        return snap

    def swap_in(self, snap, slot):
        _lib.check(self.lib.vcb_swap_in(self.eng, snap, slot, self.stream))

    def snapshot_pages(self, snap):
        return self.lib.vcb_snapshot_pages(snap)

    def free(self, snap):
        self.lib.vcb_snapshot_free(snap)


class ContinuousBatcher:
    """Continuous batching of independent TTS and speech-editing utterances (SURVEY.md section 8f, row f2).

    The reference synthesises one utterance per call in a Python loop (inference_tts_scale.py:43-105; the sentence loop of
    gradio_app.py:248-313).  Here up to `max_concurrency` utterances decode together; the moment one finishes, its tokens
    are read, its slot and KV pages are released and the next queued utterance is prefilled into the free slot while the
    others keep decoding.  Every utterance owns its random stream (`seed`) and its sampling parameters (the constructor's,
    or those given to submit()), so its result is exactly what ``torch.manual_seed(seed); model.inference_tts(x, x_lens,
    y, **params)`` -- or, for an edit ticket, ``model.inference(x, x_lens, y, mask_interval, **params)`` -- returns,
    whatever it was batched with.  run() returns the token lists once the queue has drained; stream() hands out every
    utterance's audio while it is generated and takes submit() / cancel() during the iteration.  A best-of-N ticket
    (submit(..., best_of=N), run() only) decodes as a group on N consecutive slots; max_concurrency counts slots.  A long
    ticket (submit with a list of sentences) is the reference's Long TTS loop: its sentences run one after another on its
    slots, each from where the previous one's random stream ended.
    """

    def __init__(self, model: "VoiceCraft", max_concurrency=32, poll_every=8, top_k=-100, top_p=1.0, temperature=1.0,
                 stop_repetition=3, silence_tokens=(1388, 1898, 131), tokenizer=None, ras_window=0, ras_tau=0.1,
                 min_frames=0, max_frames=None, alignment=None):
        """ras_window, ras_tau, min_frames, max_frames: the tickets' default sampling controls (sampling_controls).
        alignment: the TTS tickets' default alignment= (as inference_tts takes it); alignments[ticket] then holds the
        ticket's Alignment next to results / logprobs (a long ticket's: one per sentence), None for a ticket without"""
        sampling_controls(ras_window, ras_tau, min_frames, max_frames)
        if alignment is not None:
            head_masks(alignment, model.args.num_decoder_layers, model.args.nhead)
        self.alignment = alignment
        self.model, self.B, self.poll_every = model, int(max_concurrency), max(1, int(poll_every))
        self.tokenizer = tokenizer         # encodes the prompt audio of submit(audio=...) tickets
        self.defaults = dict(top_k=top_k, top_p=top_p, temperature=temperature, stop_repetition=stop_repetition,
                             silence_tokens=silence_tokens, ras_window=ras_window, ras_tau=ras_tau, min_frames=min_frames,
                             max_frames=max_frames)
        self.queue = []
        self.stats = dict(steps=0, prefills=0, max_active=0, swap_outs=0, swap_ins=0)
        self.results, self.errors = [], {}
        self.logprobs = []                 # lp of results[ticket] (as inference_tts / inference return it), None with it
        self.alignments = []               # Alignment of results[ticket] (a list for a long ticket), None without
        self._live = None                  # the running stream()'s state

    def submit(self, x, y=None, seed=None, best_of=1, mask_interval=None, top_k=None, top_p=None, temperature=None,
               stop_repetition=None, silence_tokens=None, audio=None, sample_rate=None, ras_window=None, ras_tau=None,
               min_frames=None, max_frames=None, alignment=None):
        """x [1,L] int64, y [1,T,K] int64 (host or device).  Returns the ticket (index into run()'s result list / results).
        audio [channels, N] (instead of y): the prompt as audio at sample_rate (default: the codec's), encoded by the
        constructor's tokenizer when the ticket is admitted, together with the other audio tickets admitted with it
        (AudioTokenizer.encode_many; in stream() on the codec's CUDA stream).  The ticket then returns exactly what it
        returns given ``y = tokenizer.encode_many([audio], sample_rate)[0].transpose(1, 2)``; an edit ticket's mask_interval
        is in frames of that encoding.  Its size is known from the sample count, so admission never waits for the encoder.
        best_of: run() samples the utterance best_of times on consecutive slots and keeps the copy that ends first, as
        ``torch.manual_seed(seed); inference_tts_batch(x, ., y, batch_size=best_of)`` does; the copies count against
        max_concurrency.  stream() serves only best_of = 1.
        mask_interval [1,M,2]: a speech-editing ticket (best_of = 1, at most min(8, max_n_spans) spans); its result is
        (res, None) with res what ``inference(x, ., y, mask_interval, ...)`` returns.
        top_k, top_p, temperature, stop_repetition, silence_tokens, ras_window, ras_tau, min_frames, max_frames: this
        ticket's sampling parameters (sampling_controls for the last four); None takes the constructor's value (not
        inference's or inference_tts' own defaults).  A ticket with max_frames needs, and is admitted against, the
        positions and KV pages that bound lets it reach.
        While a stream() runs, the utterance is admitted at one of its next polls; one that does not fit the engine it
        sized raises VcbError and is not queued.

        x a list of [1,L_i] tensors, one per sentence: a long ticket, the reference's Long TTS mode (gradio_app.py run):
        one prompt (y or audio, encoded once, at admission), one set of sampling parameters, and its result a list with
        one (res, gen) per sentence (logprobs[ticket] likewise) equal to ``torch.manual_seed(seed); [inference_tts(x_i, .,
        y) for x_i in x]`` (inference_tts_batch(..., batch_size=best_of) with best_of > 1).  Its sentences run one after
        another on the ticket's slot(s): when one ends, the next is prefilled there at the next poll, from the offset its
        predecessor's stream ended at, ahead of every queued ticket.  In stream() (best_of = 1) its chunks come in
        sentence order, each sentence decoded from a fresh codec state as the reference decodes each gen_i, and resampled
        across sentence boundaries by one resampler stream, so they equal ``resample(torch.cat([decode_codes(gen_i)],
        -1))``; last=True marks the final sentence's last chunk; cancel() drops the rest of the chain; a sentence that
        fails fails the ticket and errors[ticket] names it.  Raises ValueError on an empty list, on a list with
        mask_interval and, while a stream() runs, on a sentence that does not fit its engine.
        alignment: as inference_tts's; None takes the constructor's value, False is off.  An edit ticket refuses one (the
        constructor's default does not apply to edits), as does a text longer than align_text_cap (ValueError)."""
        if (y is None) == (audio is None):
            raise ValueError("submit takes exactly one of y (codes) and audio")
        if isinstance(x, (list, tuple)):
            x = _Chain(x)
        if isinstance(x, _Chain):
            if not x.xs:
                raise ValueError("a long ticket needs at least one sentence")
            if mask_interval is not None:
                raise ValueError("a list of sentences is a long TTS ticket; an edit ticket (mask_interval) takes one x")
        pending = None
        if audio is not None:
            tok = self.tokenizer
            if tok is None or not tok.has_encoder:
                raise _lib.VcbError("submit(audio=...) needs ContinuousBatcher(..., tokenizer=) with encoder weights (enc.*)")
            audio = torch.as_tensor(audio)
            if audio.ndim != 2 or audio.shape[1] < 1:
                raise ValueError(f"audio must be [channels, samples], got {tuple(audio.shape)}")
            # placeholder codes of the encoded length: the prompt's layout, positions and pages are those of the real ones
            y = torch.zeros(1, tok.frames(int(audio.shape[1]), sample_rate), int(self.model.args.n_codebooks), dtype=torch.long)
            pending = (x, audio, sample_rate)
        best_of = _check_best_of(best_of)
        if best_of > self.B:
            raise ValueError(f"best_of={best_of} copies do not fit max_concurrency={self.B} slots")
        spans = None
        if mask_interval is not None:
            mi = torch.as_tensor(mask_interval)
            if mi.ndim != 3 or mi.shape[0] != 1 or mi.shape[2] != 2:
                raise ValueError(f"mask_interval must be [1, M, 2], got {tuple(mi.shape)}")
            if best_of != 1:
                raise ValueError(f"best_of={best_of}: an edit ticket takes best_of=1")
            spans = [(int(a), int(b)) for a, b in mi[0].tolist()]
            if len(spans) > min(8, int(self.model.args.max_n_spans)):
                raise ValueError(f"{len(spans)} masked spans: at most min(8, max_n_spans={self.model.args.max_n_spans})")
        given = dict(top_k=top_k, top_p=top_p, temperature=temperature, stop_repetition=stop_repetition,
                     silence_tokens=silence_tokens, ras_window=ras_window, ras_tau=ras_tau, min_frames=min_frames,
                     max_frames=max_frames)
        params = {k: self.defaults[k] if v is None else v for k, v in given.items()}
        if not (math.isfinite(params["temperature"]) and params["temperature"] > 0) or math.isnan(params["top_p"]):
            raise ValueError(f"temperature must be finite and > 0 and top_p a number, got {params}")
        sp = self.model._sampling(**params)
        _no_host_noise_under_ras(sp.ras_window, self.model.noise_fn is not None)
        if alignment is None and spans is None:
            alignment = self.alignment
        align = _align_heads(self.model, alignment, x.xs if isinstance(x, _Chain) else [x], spans is not None)
        st = self._live
        if st is not None:
            _no_stream_best_of(best_of)
            job = self._job(x, y, seed, 1, spans, sp, pending, align)
            if job.chain is not None and job.chain.need_seq > st.max_seq:
                raise ValueError(f"a sentence needs {job.chain.need_seq} positions, the streaming engine holds {st.max_seq}: "
                                 "configure_engine(max_seq_len=...) before stream()")
            if job.prompt.need_seq > st.max_seq:
                raise _lib.VcbError(f"utterance needs {job.prompt.need_seq} positions, the streaming engine holds "
                                    f"{st.max_seq}: configure_engine(max_seq_len=...) before stream()")
            st.jobs.append(job)
            self.results.append(None)
            self.logprobs.append(None)
            self.alignments.append(None)
        self.queue.append((x, y, seed, best_of, spans, sp, pending, align))
        return len(self.queue) - 1

    def cancel(self, ticket) -> bool:
        """stream(): a queued ticket is never admitted, an active one's slot is released at the next poll and nothing
        more is yielded for it; results[ticket] stays None.  False if the ticket already handed out its last chunk."""
        st = self._live
        if st is None or not 0 <= ticket < len(st.jobs):
            raise _lib.VcbError(f"no ticket {ticket} in a running stream()")
        if ticket in st.ended:
            return False
        st.cancelled.add(ticket)
        return True

    def _job(self, x, y, seed, best_of, spans, sp, pending=None, align=None):
        """the _Ticket of submit's arguments; raises IndexError on an out-of-range id.  A long ticket's chain (x, a
        _Chain) gets the prompts of its sentences."""
        if not isinstance(x, _Chain):
            p = _Prompt(self.model, x, y, spans, sp.max_frames)
            self.model._check_ids(p.x_ids, p.y_tok)
            p.align = align
            return _Ticket(p, seed, best_of, sp, pending, align=align)
        x.start([_Prompt(self.model, xi, y, None, sp.max_frames) for xi in x.xs])
        for p in x.prompts:
            p.align = align
        self.model._check_ids(torch.cat([p.x_ids for p in x.prompts]), x.prompts[0].y_tok)
        return _Ticket(x.prompt, seed, best_of, sp, pending, x, align)

    def _open(self, s, ops):
        """The state of run() / stream(), `s`, holds eng, slots, jobs, results, cancelled and cstream (the codec's CUDA
        stream; None in run()).  Adds: every slot `free`, nothing `active` (first slot -> _Utterance) or in `follow`
        (utterances whose next sentence waits in their slots), `nxt` the first queued ticket, and the `pool` policy over
        `ops` (_EngineOps) on its CUDA `stream`."""
        o = self.model._eng_opts
        s.stream, s.max_pages = ops.stream, (o["max_seq_len"] + 63) // 64
        s.free, s.active, s.follow, s.nxt = set(s.slots), {}, [], 0
        s.pool = KvPoolPolicy(ops, o["kv_pool_gb"] is not None, self.B)

    def _close(self, s):
        """frees the pool's snapshots, adds its swap counts to stats and releases every slot"""
        if s.pool is not None:
            s.pool.close()
            self.stats["swap_outs"] += s.pool.swap_outs
            self.stats["swap_ins"] += s.pool.swap_ins
        self.model._release_slots(s.slots)    # every slot: releasing one that is not open does nothing
        self.queue = []

    def _leave(self, s, r, kept=None):
        """r leaves `active` and its slots are released.  kept: (slot, vcb_status) of its kept copy when it finished
        (r.status: its group's first slot's): results[ticket] is then (res, gen) as inference_tts returns them ((res,
        None) of an edit, res as inference returns it), logprobs[ticket] its lp, and a long ticket's the lists of its
        sentences' once the last one ends; until then its next sentence (the ticket's prompt now, its stream starting at
        r.status.rng_offset) keeps the slots in `follow`.  Otherwise they go back to `free` and it returns True."""
        m, t, job = self.model, r.ticket, s.jobs[r.ticket]
        follows = False
        if kept is not None:
            slot, st = kept
            res, gen, lp = job.prompt.result(m._read_rows(s.eng, slot, st.n_steps, s.stream), st,
                                             m._read_lp(s.eng, slot, st.n_steps, s.stream))
            al = None if job.align is None else _read_alignment(m, s.eng, slot, job.prompt, res.shape[-1], s.stream)
            if job.chain is None:
                s.results[t], self.logprobs[t] = (res, gen), lp
                if al is not None:
                    self.alignments[t] = al
            elif job.chain.ended((res, gen), lp, r.status.rng_offset, al):
                job.prompt, follows = job.chain.prompt, True
            else:
                s.results[t], self.logprobs[t] = job.chain.results, job.chain.logprobs
                if job.align is not None:
                    self.alignments[t] = job.chain.alignments
        m._release_slots(s.slots, [r.slot], n_copies=job.best_of, keep_held=True)
        del s.active[r.slot]
        if follows:
            s.follow.append(r)
        else:
            s.free.update(range(r.slot, r.slot + job.best_of))
        return not follows

    def _round(self, s):
        """The admissions of a round: the next sentences of long tickets first, into the slots they kept; while none
        waits, swapped-out utterances come back, then the next queued tickets that are not cancelled, at most one per free
        slot, as many as the pool takes, placed by place_groups.  Returns (the next sentences' utterances, the new
        tickets'), both now in `active`."""
        jobs, pool = s.jobs, s.pool

        def needs(ts):
            return [(jobs[t].pages(s.max_pages), jobs[t].best_of) for t in ts]

        def n_active():
            return sum(jobs[r.ticket].best_of for r in s.active.values())

        def admit(new, cids):
            if new:
                self._admit(s, new)
            for (slot, t), cid in zip(new, cids):
                chain = jobs[t].chain
                i = 0 if chain is None else len(chain.results)
                s.active[slot] = _Utterance(slot, cid, f"ticket {t}" + ("" if chain is None else f" sentence {i}"),
                                            ticket=t, src=jobs[t].prompt.source(), carry=i > 0,
                                            more=chain is not None and i + 1 < len(chain.prompts))
            return [s.active[slot] for slot, _ in new]

        k = pool.admit_count(needs([r.ticket for r in s.follow]), n_active(), held=True) if s.follow else 0
        followed = admit([(r.slot, r.ticket) for r in s.follow[:k]], [r.cid for r in s.follow[:k]])
        s.follow, new = s.follow[k:], []
        if not s.follow:
            for r, slot in pool.resume(s.free, n_active()):
                r.slot = slot
                s.active[slot] = r
            cands, t = [], s.nxt
            while len(cands) < len(s.free) and t < len(jobs):
                if t not in s.cancelled:
                    cands.append(t)
                t += 1
            k = pool.admit_count(needs(cands), n_active())
            placed, i = place_groups(s.free, [jobs[c].best_of for c in cands[:k]], 0)
            s.nxt = t if i == len(cands) else cands[i]
            new = admit([(slot, cands[j]) for slot, j in placed], [None] * len(placed))
        self.stats["max_active"] = max(self.stats["max_active"], n_active())
        return followed, new

    def _steps(self, s, live, leaving=False):
        """Up to poll_every decode steps of the utterances `live` (KvPoolPolicy.step: one swapped out leaves `active`, its
        slot goes back to `free`; with `leaving`, a step no swap can fit ends the poll early).  Returns the steps taken."""
        go = [(r, r.slot + c, r.ticket, s.jobs[r.ticket].best_of == 1)
              for r in live for c in range(s.jobs[r.ticket].best_of)]
        n = 0
        for _ in range(self.poll_every if go else 0):
            go, out = s.pool.step(go, leaving)
            for r, slot in out:
                del s.active[slot]
                s.free.add(slot)
            if go is None:
                break
            n += 1
        return n

    def _encode(self, jobs, cstream=None):
        """the prompt audio of the audio tickets among `jobs`, in one encode_many call, and their prompts rebuilt from
        the codes.  cstream: encode there (the codec's stream, whose workspace the encoder
        shares) and make the current stream wait for it."""
        todo = [j for j in jobs if j.pending is not None]
        if not todo:
            return
        tok, cur = self.tokenizer, torch.cuda.current_stream()
        if cstream is not None:
            cstream.wait_stream(cur)
        with torch.cuda.stream(cstream if cstream is not None else cur):
            codes = tok.encode_many([j.pending[1] for j in todo], [j.pending[2] for j in todo])
        if cstream is not None:
            cur.wait_stream(cstream)
            for c in codes:
                c.record_stream(cur)
        for j, c in zip(todo, codes):
            y = c.transpose(1, 2)
            if j.chain is None:
                real = _Prompt(self.model, j.pending[0], y, j.prompt.spans, j.sp.max_frames)
                real.align = j.align
            else:                                # every sentence of a long ticket: one encode for the chain
                j.chain.start([_Prompt(self.model, xi, y, None, j.sp.max_frames) for xi in j.chain.xs])
                for p in j.chain.prompts:
                    p.align = j.align
                real = j.chain.prompt
            assert real.need_seq == j.prompt.need_seq and real.total == j.prompt.total
            j.prompt, j.pending = real, None

    def _admit(self, s, new):
        """one packed prefill + the first sampling step of the newcomers [(first slot, ticket)], each with its ticket's
        sampling parameters (every sampling call of the batcher passes sp = NULL); the audio tickets among them are
        encoded first (_encode).  A long ticket's sentence starts at its chain's offset, any other ticket at 0."""
        m, lib, jobs = self.model, _lib.load(), s.jobs
        self._encode([jobs[t] for _, t in new], s.cstream)
        seed0 = int(torch.cuda.default_generators[m.mask_embedding.device.index or 0].initial_seed())
        _prefill(s.eng, [(jobs[t].prompt, slot, jobs[t].best_of, seed0 + t if jobs[t].seed is None else jobs[t].seed,
                          0 if jobs[t].chain is None else jobs[t].chain.offset, jobs[t].sp) for slot, t in new], s.stream)
        rows = [slot + c for slot, t in new for c in range(jobs[t].best_of)]
        c_new = (C.c_int32 * len(rows))(*rows)
        _lib.check(lib.vcb_sample(s.eng, c_new, len(rows), None, None, s.stream))
        self.stats["prefills"] += 1

    @torch.no_grad()
    def run(self):
        m = self.model
        if m.noise_fn is not None:
            raise _lib.VcbError("ContinuousBatcher uses the per-utterance device generators (model.noise_fn must be None)")
        if self._live is not None:
            raise _lib.VcbError("a stream() of this ContinuousBatcher is running")
        dev, lib = m.mask_embedding.device, _lib.load()
        jobs = [self._job(*q) for q in self.queue]
        n_slots = min(self.B, max(1, sum(j.best_of for j in jobs)))
        eng, slots = m._take_slots(n_slots, max([j.need_seq for j in jobs], default=0))
        s = SimpleNamespace(eng=eng, slots=slots, jobs=jobs, results=[None] * len(jobs), cancelled=set(), cstream=None,
                            pool=None)
        self.logprobs = [None] * len(jobs)
        self.alignments = [None] * len(jobs)
        try:
            with torch.cuda.device(dev):
                self._open(s, _EngineOps(eng, torch.cuda.current_stream().cuda_stream))
                steps = 0
                while True:
                    self._round(s)
                    if not s.active and not s.follow:
                        break
                    steps += self._steps(s, [s.active[k] for k in sorted(s.active)])
                    # ---- poll; the utterances that ended leave (a best-of-N group's result is its kept copy's)
                    order = [k + c for k in sorted(s.active) for c in range(jobs[s.active[k].ticket].best_of)]
                    c_slots = (C.c_int32 * len(order))(*order)
                    status = (_lib.vcb_status * len(order))()
                    _lib.check(lib.vcb_poll(eng, c_slots, len(order), status, s.stream))
                    _check_capacity(status)
                    by_slot = dict(zip(order, status))
                    for slot, r in list(s.active.items()):
                        st = r.status = by_slot[slot]
                        if st.done:
                            kept = slot + (st.keep if jobs[r.ticket].best_of > 1 else 0)
                            self._leave(s, r, (kept, by_slot[kept]))
                self.stats["steps"] = steps
        finally:
            self._close(s)
        return s.results

    def stream(self, tokenizer, chunk_frames: int = 25, sample_rate: int = None) -> "BatcherStream":
        """run() with every utterance's audio handed out while it is generated: iterates (ticket, wav [1, channels, n*hop],
        last).  A ticket's chunks, concatenated, equal ``tokenizer.decode_codes(gen)`` (an edit ticket's:
        ``decode_codes(res)``, the whole edited utterance, whose frames before the first masked span are its first chunk);
        its last chunk has last=True
        (an utterance that generated no frame yields one empty wav).  submit() and cancel() may be called from the loop
        body.  Afterwards ``results[ticket]`` is (res, gen) as run() returns it, None for a cancelled or failed ticket;
        ``errors[ticket]`` says why a ticket failed (a final frame holding a non-audio token: it yields (ticket, None,
        True) and the others go on).  The engine gets `max_concurrency` slots, each with its own codec stream id.
        sample_rate: chunks at that rate, resampled on the device as they are decoded; concatenated they equal
        ``tokenizer.resample(<the codec-rate audio>, codec rate, sample_rate)``."""
        return BatcherStream(self, tokenizer, chunk_frames, sample_rate)


class BatcherStream(_AudioStream):
    """Iterator of ContinuousBatcher.stream().  Closing it early (break, close(), garbage collection) releases the
    batcher's engine slots and the codec streams."""

    def __init__(self, cb: ContinuousBatcher, tokenizer, chunk_frames: int = 25, sample_rate=None):
        m = cb.model
        if m.noise_fn is not None:
            raise _lib.VcbError("ContinuousBatcher uses the per-utterance device generators (model.noise_fn must be None)")
        if cb._live is not None:
            raise _lib.VcbError("a stream() of this ContinuousBatcher is already running")
        if chunk_frames < 1:
            raise ValueError("chunk_frames must be >= 1")
        jobs = [cb._job(*q) for q in cb.queue]
        eng, slots = m._take_slots(cb.B, max([j.need_seq for j in jobs], default=0))
        # a queued best-of-N ticket fails (its kept copy is known only when its group ends); the others are served
        refused = {t for t, j in enumerate(jobs) if j.best_of > 1}
        st = SimpleNamespace(cb=cb, eng=eng, slots=slots, max_seq=m._eng_opts["max_seq_len"], jobs=jobs,
                             results=[None] * len(jobs), cancelled=set(refused), ended=set(refused),
                             refused=sorted(refused), tok=tokenizer, chunk_frames=int(chunk_frames),
                             dev=m.mask_embedding.device, sample_rate=sample_rate, pool=None)
        cb.results, cb.logprobs, cb.alignments, cb._live = st.results, [None] * len(jobs), [None] * len(jobs), st
        cb.errors = {t: f"best_of={jobs[t].best_of}: stream() serves only best_of=1 tickets" for t in refused}
        # a codec stream id belongs to a ticket from its admission to its end: at most max_concurrency are active and, under
        # a KV budget, at most as many more are swapped out
        self._start(st, 2 * cb.B if m._eng_opts["kv_pool_gb"] is not None else cb.B)

    @staticmethod
    def _finish(st):
        cb = st.cb
        if cb._live is not st:
            return
        cb._close(st)
        _AudioStream._close_codec(st)
        cb._live = None

    @staticmethod
    @torch.no_grad()
    def _run(st):
        cb, m = st.cb, st.cb.model
        ids = list(range(st.codec.max_streams))          # free codec stream ids
        try:
            with torch.cuda.device(st.dev):
                cb._open(st, _EngineOps(st.eng, torch.cuda.current_stream().cuda_stream))
                push = st.push = _PushStep(m, st.eng, st.stream, st.tok, st.codec, st.cstream, st.chunk_frames,
                                           cb.poll_every, strict=False)
                empty = torch.zeros(1, st.tok.channels, 0, device=st.dev)
                for t in st.refused:
                    yield t, None, True
                while True:
                    # ---- finished, failed and cancelled utterances leave; a next sentence keeps the codec stream id
                    for r in list(st.active.values()):
                        if r.closed or r.ticket in st.cancelled:
                            done = r.closed and r.ticket not in cb.errors
                            if cb._leave(st, r, (r.slot, r.status) if done else None):
                                ids.append(r.cid)
                    for r in [r for r in st.follow if r.ticket in st.cancelled]:    # no next sentence of a cancelled ticket
                        st.follow.remove(r)
                        st.free.add(r.slot)
                        ids.append(r.cid)
                    for _, r, _ in list(st.pool.swapped):    # a cancelled ticket that is swapped out: its snapshot goes
                        if r.ticket in st.cancelled and st.pool.drop(r):
                            ids.append(r.cid)
                    followed, new = cb._round(st)
                    # a next sentence starts from a fresh codec state, its resampler stream carried on; a new ticket
                    # takes a codec stream id of its own
                    if followed:
                        st.codec.reset([r.cid for r in followed], resampler=False)
                    if new:
                        for r in new:
                            r.cid = ids.pop(0)
                        st.codec.reset([r.cid for r in new])
                    if not st.active and not st.follow:
                        break
                    live = [st.active[s] for s in sorted(st.active)]

                    def advance(status):
                        go = [r for r, s in zip(live, status) if not s.done and not r.closed]
                        # finished tickets keep their slot and pages until the top of the next round releases them: while
                        # any does, a step that swapping cannot fit waits for those pages instead of failing
                        cb.stats["steps"] += cb._steps(st, go, len(go) < len(live))
                    status, out, failed = push(live, advance)
                    wavs = dict(out)
                    for r, s in zip(live, status):
                        r.status = s
                        if r in failed:
                            cb.errors[r.ticket] = failed[r]
                        if r.closed and (not r.more or r in failed):
                            st.ended.add(r.ticket)
                    for r in live:
                        if r.ticket in st.cancelled and (not r.closed or r.more):
                            continue
                        if r in failed:
                            yield r.ticket, None, True
                        elif r in wavs:
                            w, last = wavs[r], r.closed and not r.more
                            if w is not None or last:     # a sentence that ends with no new audio yields nothing
                                yield r.ticket, (empty if w is None else w), last
        finally:
            BatcherStream._finish(st)
