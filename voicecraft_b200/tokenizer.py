"""Drop-in for the reference's ``data/tokenizer.py::AudioTokenizer`` (:101-133).

``AudioTokenizer(signature=path, device=...)`` mirrors the reference constructor; ``decode(frames)`` takes the
reference's ``[(codes[1,K,T], None)]`` and returns the waveform ``[1, channels, T*hop]``; ``encode(wav[1,C,N])`` returns the
reference's ``[(codes[1,K,T], None)]`` (:127-129).  Instead of audiocraft's ``CompressionSolver.model_from_checkpoint`` +
``EncodecModel.decode / encode`` (:109-110, :128, :133) the weights are handed to libvcb200.so, which runs RVQ and the
SEANet decoder / encoder as sm_90a kernels.  No PyTorch / CPU fallback.  The text tokenizer (espeak) is out of scope.
"""
import ctypes as C
import functools
import math
import struct
from collections import namedtuple
from types import SimpleNamespace
from typing import Any

import torch

from . import _lib, _codec_lib


def default_codec_config(**over):
    """Hyper-parameters of the reference's 16 kHz / 50 Hz / 4 x 2048 EnCodec (README.md:198, config.py:51)."""
    c = dict(n_q=4, bins=2048, dimension=128, n_filters=64, ratios=[8, 5, 4, 2], kernel_size=7, last_kernel_size=7,
             residual_kernel_size=3, dilation_base=2, n_residual_layers=1, compress=2, lstm=2, causal=True,
             pad_mode="reflect", true_skip=False, trim_right_ratio=1.0, channels=1, sample_rate=16000)
    c.update(over)
    return SimpleNamespace(**c)


def fold_weight_norm(g: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """w = g * v / ||v|| over all dims but 0 (torch.nn.utils.weight_norm, dim=0)."""
    return v * (g / v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1))))


def state_dict_from_audiocraft(sd: dict, cfg) -> dict:
    """Map an audiocraft EncodecModel state_dict (decoder.model.{i}.*, quantizer.vq.layers.{q}._codebook.embed) to the
    flat names libvcb200 uses.  [memory]-level key layout of audiocraft@c5157b5 (SURVEY.md section 0.8): verify against
    the real checkpoint when one is available."""
    out = {}
    for q in range(cfg.n_q):
        out[f"vq.{q}.embed"] = sd[f"quantizer.vq.layers.{q}._codebook.embed"]

    def conv(prefix):
        if prefix + ".weight" in sd:
            return sd[prefix + ".weight"], sd[prefix + ".bias"]
        return fold_weight_norm(sd[prefix + ".weight_g"], sd[prefix + ".weight_v"]), sd[prefix + ".bias"]
    idx = 0
    out["dec.conv_in.weight"], out["dec.conv_in.bias"] = conv(f"decoder.model.{idx}.conv.conv")
    idx += 1
    if cfg.lstm:
        for l in range(cfg.lstm):
            for part in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                out[f"dec.lstm.{part}_l{l}"] = sd[f"decoder.model.{idx}.lstm.{part}_l{l}"]
        idx += 1
    for i, _ in enumerate(cfg.ratios):
        idx += 1                                         # ELU
        out[f"dec.up{i}.convtr.weight"], out[f"dec.up{i}.convtr.bias"] = conv(f"decoder.model.{idx}.convtr.convtr")
        idx += 1
        for j in range(cfg.n_residual_layers):
            p = f"decoder.model.{idx}"
            out[f"dec.up{i}.res{j}.conv1.weight"], out[f"dec.up{i}.res{j}.conv1.bias"] = conv(p + ".block.1.conv.conv")
            out[f"dec.up{i}.res{j}.conv2.weight"], out[f"dec.up{i}.res{j}.conv2.bias"] = conv(p + ".block.3.conv.conv")
            if not cfg.true_skip:
                out[f"dec.up{i}.res{j}.shortcut.weight"], out[f"dec.up{i}.res{j}.shortcut.bias"] = conv(p + ".shortcut.conv.conv")
            idx += 1
    idx += 1                                             # ELU
    out["dec.conv_out.weight"], out["dec.conv_out.bias"] = conv(f"decoder.model.{idx}.conv.conv")
    if "encoder.model.0.conv.conv.weight" in sd or "encoder.model.0.conv.conv.weight_g" in sd:
        # SEANetEncoder: conv, per ratio (reversed) [ResBlock x n, ELU, strided conv], LSTM, ELU, conv
        idx = 0
        out["enc.conv_in.weight"], out["enc.conv_in.bias"] = conv(f"encoder.model.{idx}.conv.conv")
        idx += 1
        for i, _ in enumerate(cfg.ratios):
            for j in range(cfg.n_residual_layers):
                p = f"encoder.model.{idx}"
                out[f"enc.down{i}.res{j}.conv1.weight"], out[f"enc.down{i}.res{j}.conv1.bias"] = conv(p + ".block.1.conv.conv")
                out[f"enc.down{i}.res{j}.conv2.weight"], out[f"enc.down{i}.res{j}.conv2.bias"] = conv(p + ".block.3.conv.conv")
                if not cfg.true_skip:
                    out[f"enc.down{i}.res{j}.shortcut.weight"], out[f"enc.down{i}.res{j}.shortcut.bias"] = conv(p + ".shortcut.conv.conv")
                idx += 1
            idx += 1                                     # ELU
            out[f"enc.down{i}.conv.weight"], out[f"enc.down{i}.conv.bias"] = conv(f"encoder.model.{idx}.conv.conv")
            idx += 1
        if cfg.lstm:
            for l in range(cfg.lstm):
                for part in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                    out[f"enc.lstm.{part}_l{l}"] = sd[f"encoder.model.{idx}.lstm.{part}_l{l}"]
            idx += 1
        idx += 1                                         # ELU
        out["enc.conv_out.weight"], out["enc.conv_out.bias"] = conv(f"encoder.model.{idx}.conv.conv")
    return out


RESAMPLE_TABLE_CAP = 16 << 20          # bytes of filter table a resampler may hold (44.1 kHz -> 16 kHz needs 296 KB)


def resample_dims(orig_sr: int, new_sr: int):
    """(o, n, w, taps) of torchaudio's Resample(orig_sr, new_sr) with its defaults: the rates over their gcd, the filter
    half-width w = ceil(6 o / (0.99 min(o, n))) and the 2w + o taps of each of the n phases.  Raises ValueError for a
    rate <= 0 and for a pair whose table would exceed RESAMPLE_TABLE_CAP (16000 -> 44099 Hz would need gigabytes)."""
    if int(orig_sr) != orig_sr or int(new_sr) != new_sr or orig_sr <= 0 or new_sr <= 0:
        raise ValueError(f"resample: sample rates must be positive integers, got {orig_sr} -> {new_sr}")
    g = math.gcd(int(orig_sr), int(new_sr))
    o, n = int(orig_sr) // g, int(new_sr) // g
    w = math.ceil(6 * o / (min(o, n) * 0.99))
    taps = 2 * w + o
    if n * taps * 4 > RESAMPLE_TABLE_CAP:
        raise ValueError(f"resample: {orig_sr} -> {new_sr} Hz needs a filter table of {n} phases x {taps} taps "
                         f"({n * taps * 4} bytes), over the {RESAMPLE_TABLE_CAP}-byte cap")
    return o, n, w, taps


@functools.lru_cache(maxsize=None)
def _sinc_table(o: int, n: int) -> torch.Tensor:
    w = resample_dims(o, n)[2]
    base = min(o, n) * 0.99
    # tap positions in fp64; the phase offsets -p/n in fp32 (torchaudio divides an integer arange in the default dtype),
    # promoted to fp64 by the addition.  A clean fp64 -p/n moves some taps of 44.1k <-> 16k by up to 1.3e-5.
    pos = torch.arange(-w, w + o, dtype=torch.float64)[None, None] / o
    t = torch.arange(0, -n, -1, dtype=torch.float32)[:, None, None] / n + pos
    t *= base
    t = t.clamp_(-6, 6)
    window = torch.cos(t * math.pi / 6 / 2) ** 2          # Hann window over the 6 zero crossings
    t *= math.pi
    k = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    k *= window * (base / o)
    return k.to(torch.float32).reshape(n, 2 * w + o).contiguous()


def resample_table(orig_sr: int, new_sr: int) -> torch.Tensor:
    """The filter table of torchaudio.transforms.Resample(orig_sr, new_sr) (sinc_interp_hann, lowpass_filter_width 6,
    rolloff 0.99): fp32 [n][2w + o] on the CPU, built with the same torch ops in fp64 and rounded once, so it is
    bit-equal to torchaudio's (functional._get_sinc_resample_kernel).  Cached per reduced (o, n)."""
    o, n, _, _ = resample_dims(orig_sr, new_sr)
    return _sinc_table(o, n)


class Resampler:
    """Owner of one enc_resampler (torchaudio's Resample(orig_sr, new_sr) on the device): one-shot over ragged rows
    (``__call__``) and, for up to `max_streams` streams, chunk by chunk with carried state (``push``)."""

    def __init__(self, orig_sr: int, new_sr: int, max_streams: int = 0, device=None):
        self.orig_sr, self.new_sr = int(orig_sr), int(new_sr)
        self.o, self.n, self.w, self.taps = resample_dims(orig_sr, new_sr)
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.type != "cuda":
            raise _lib.VcbError("the resampler runs on a CUDA device only")
        self._lib = _lib.load()
        self._h = None
        table = resample_table(orig_sr, new_sr)
        h = C.c_void_p()
        _lib.check(self._lib.enc_resampler_create(self.orig_sr, self.new_sr, table.data_ptr(), int(max_streams),
                                                  self.device.index or 0, C.byref(h)))
        self._h = h
        self.max_streams = int(max_streams)

    def _out(self, rows, cap):
        return torch.empty(max(rows, 1), max(cap, 1), device=self.device, dtype=torch.float32)

    @torch.no_grad()
    def __call__(self, x: torch.Tensor, lens=None):
        """x [R, T] fp32 (device) -> (y [R, cap], out_lens): row r's first out_lens[r] = ceil(n lens[r] / o) samples
        are the resampled first lens[r] (default T) samples of x[r]; cap = max(out_lens).  Current CUDA stream."""
        x = x.to(self.device, dtype=torch.float32).contiguous()
        R, T = x.shape
        lens = [T] * R if lens is None else [int(v) for v in lens]
        cap = max([-(-v * self.n // self.o) for v in lens], default=0)
        y, out_lens = self._out(R, cap), (C.c_int32 * max(R, 1))()
        _lib.check(self._lib.enc_resample(self._h, x.data_ptr(), (C.c_int32 * max(R, 1))(*lens), R, T, y.data_ptr(), cap,
                                          out_lens, torch.cuda.current_stream(self.device).cuda_stream))
        return y[:R, :cap], list(out_lens)[:R]

    @torch.no_grad()
    def push(self, x, ids, lens, final=None):
        """Row r continues stream ids[r] with the first lens[r] samples of x [R, T] (x may be None when every length is
        0); final[r] also emits the stream's tail.  Returns (y [R, cap], out_lens) as __call__ does."""
        R = len(ids)
        x = None if x is None else x.to(self.device, dtype=torch.float32).contiguous()
        T = 0 if x is None else int(x.shape[1])
        most = max([int(v) for v in lens], default=0)
        cap = (self.n * (most + self.w + 2 * self.o)) // self.o + self.n + 1   # >= what any row can emit
        y, out_lens = self._out(R, cap), (C.c_int32 * max(R, 1))()
        fin = None if final is None else (C.c_int32 * max(R, 1))(*[int(bool(f)) for f in final])
        _lib.check(self._lib.enc_resampler_push(self._h, (C.c_int32 * max(R, 1))(*ids), (C.c_int32 * max(R, 1))(*lens), fin, R,
                                                0 if x is None else x.data_ptr(), T, y.data_ptr(), cap, out_lens,
                                                torch.cuda.current_stream(self.device).cuda_stream))
        out_lens = list(out_lens)[:R]
        return y[:R, :max(out_lens, default=0)], out_lens

    def reset(self, ids):
        ids = [int(i) for i in ids]
        _lib.check(self._lib.enc_resampler_reset(self._h, (C.c_int32 * max(len(ids), 1))(*ids), len(ids)))

    def close(self):
        if self._h is not None:
            self._lib.enc_resampler_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class AudioTokenizer:
    """EnCodec audio (decode direction)."""

    def __init__(self, device: Any = None, signature=None, config=None, state_dict=None):
        if not device:
            device = torch.device("cuda:0") if torch.cuda.is_available() else torch.device("cpu")
        self._device = torch.device(device)
        if state_dict is None:
            if signature is None:
                raise ValueError("AudioTokenizer needs a checkpoint `signature` or (`config`, `state_dict`)")
            pkg = torch.load(signature, map_location="cpu", weights_only=False)     # audiocraft checkpoint: best_state + xp.cfg
            sd = pkg["best_state"]["model"] if "best_state" in pkg else pkg
            xp = pkg.get("xp.cfg") if isinstance(pkg, dict) else None
            config = config or default_codec_config()
            if xp is not None:
                s = xp["seanet"]
                config = default_codec_config(n_filters=int(s["n_filters"]), ratios=list(s["ratios"]), lstm=int(s["lstm"]),
                                              causal=bool(s["causal"]), pad_mode=str(s["pad_mode"]),
                                              true_skip=bool(s["true_skip"]), dimension=int(s["dimension"]),
                                              n_q=int(xp["rvq"]["n_q"]), bins=int(xp["rvq"]["bins"]),
                                              sample_rate=int(xp["sample_rate"]), channels=int(xp["channels"]))
            state_dict = state_dict_from_audiocraft(sd, config)
        self.config = config or default_codec_config()
        self.sample_rate = self.config.sample_rate
        self.channels = self.config.channels
        self._sd = {k: v.detach().float() for k, v in state_dict.items()}
        self._eng = None
        self._resamplers = {}
        self.hop = 1
        for r in self.config.ratios:
            self.hop *= int(r)

    @property
    def device(self):
        return self._device

    def _engine(self):
        if self._eng is not None:
            return self._eng
        if self._device.type != "cuda":
            raise _lib.VcbError("AudioTokenizer (H100) has no CPU path: construct it with a CUDA device")
        lib = _lib.load()
        c = self.config
        cfg = _codec_lib.enc_config(n_q=c.n_q, bins=c.bins, dimension=c.dimension, n_filters=c.n_filters,
                                    n_ratios=len(c.ratios), kernel_size=c.kernel_size, last_kernel_size=c.last_kernel_size,
                                    residual_kernel_size=c.residual_kernel_size, dilation_base=c.dilation_base,
                                    n_residual_layers=c.n_residual_layers, compress=c.compress, lstm=c.lstm,
                                    causal=int(c.causal), pad_reflect=int(c.pad_mode == "reflect"),
                                    true_skip=int(c.true_skip), channels=c.channels,
                                    trim_right_ratio=float(c.trim_right_ratio), device=self._device.index or 0)
        for i, r in enumerate(c.ratios):
            cfg.ratios[i] = int(r)
        h = C.c_void_p()
        _lib.check(lib.enc_create(C.byref(cfg), C.byref(h)))
        try:
            with torch.cuda.device(self._device):
                for k, v in self._sd.items():
                    t = v.to(self._device).contiguous()
                    shape = (C.c_int64 * t.dim())(*t.shape)
                    _lib.check(lib.enc_load_weight(h, k.encode(), t.data_ptr(), shape, t.dim(), 1))
                _lib.check(lib.enc_finalize(h))
        except Exception:
            lib.enc_destroy(h)
            raise
        self._eng = h
        return h

    def __del__(self):
        try:
            for r in self._resamplers.values():
                r.close()
            if self._eng is not None:
                _lib.load().enc_destroy(self._eng)
        except Exception:
            pass

    @torch.no_grad()
    def resample(self, wav: torch.Tensor, orig_sr: int, new_sr: int = None, lens=None) -> torch.Tensor:
        """torchaudio.transforms.Resample(orig_sr, new_sr)(wav) on the device (enc_resample): wav [B, C, N] ->
        [B, C, N'], N' = ceil(n N / o); new_sr defaults to the codec's rate.  With lens, row b holds lens[b] samples and
        gives ceil(n lens[b] / o) samples, the rest of its row is zero.  Equal rates return wav itself."""
        new_sr = self.sample_rate if new_sr is None else int(new_sr)
        assert wav.ndim == 3, wav.shape
        if int(orig_sr) == new_sr:
            return wav
        key = (int(orig_sr), new_sr)
        if key not in self._resamplers:
            self._resamplers[key] = Resampler(orig_sr, new_sr, 0, self._device)
        rs = self._resamplers[key]
        B, Ch, N = wav.shape
        x = wav.to(self._device, dtype=torch.float32).contiguous().view(B * Ch, N)
        rows = None if lens is None else [int(lens[b]) for b in range(B) for _ in range(Ch)]
        with torch.cuda.device(self._device):
            y, out_lens = rs(x, rows)
        if lens is not None:
            y.masked_fill_(torch.arange(y.shape[1], device=y.device)[None, :] >=
                           torch.tensor(out_lens, device=y.device)[:, None], 0.0)
        return y.reshape(B, Ch, y.shape[1])

    @torch.no_grad()
    def encode_codes(self, wav: torch.Tensor) -> torch.Tensor:
        """wav [B,channels,N] fp32 -> codes [B,K,T] int64, T = N down-sampled by every ratio (rounded up)."""
        assert wav.ndim == 3 and wav.shape[1] == self.channels, wav.shape
        if "enc.conv_in.weight" not in self._sd:
            raise _lib.VcbError("this AudioTokenizer was built without encoder weights (enc.*)")
        eng = self._engine()
        wav = wav.to(self._device, dtype=torch.float32).contiguous()
        B, _, N = wav.shape
        T = N
        for r in reversed(list(self.config.ratios)):
            T = (T + int(r) - 1) // int(r)
        codes = torch.empty(B, self.config.n_q, T, device=self._device, dtype=torch.long)
        with torch.cuda.device(self._device):
            _lib.check(_lib.load().enc_encode(eng, wav.data_ptr(), codes.data_ptr(), B, N, torch.cuda.current_stream().cuda_stream))
        return codes

    def encode(self, wav: torch.Tensor):
        """Reference signature (data/tokenizer.py:127-129): wav [1,C,N] -> [(codes[1,K,T], None)]."""
        return [(self.encode_codes(wav), None)]

    def frames(self, n_samples: int, sample_rate: int = None) -> int:
        """Code frames of a prompt of n_samples at sample_rate (default: the codec's): resampled to the codec's rate
        (ceil(n N / o)), then down-sampled by every ratio, rounded up at each."""
        n = int(n_samples)
        if sample_rate is not None and int(sample_rate) != self.sample_rate:
            o, r = resample_dims(int(sample_rate), self.sample_rate)[:2]
            n = -(-r * n // o)
        for r in reversed(list(self.config.ratios)):
            n = -(-n // int(r))
        return n

    @property
    def has_encoder(self) -> bool:
        return "enc.conv_in.weight" in self._sd

    @torch.no_grad()
    def encode_many(self, wavs, sample_rate: int = None):
        """Prompts of different lengths in one call: wavs, a list of [channels_i, N_i] tensors at sample_rate (default: the
        codec's; a list gives each its own rate) -> list of codes [1, K, T_i].  Each is mixed to the codec's channel count as convert_audio does
        (mix_channels), resampled on the device when the rate differs (one ragged enc_resample), and all are encoded by one
        enc_encode_ragged: the tensor-core encoder for the rows it covers, each other row alone on the CUDA-core encoder.
        A row's codes do not depend on the rows it is batched with.  Runs on the current CUDA stream."""
        if not self.has_encoder:
            raise _lib.VcbError("this AudioTokenizer was built without encoder weights (enc.*)")
        if len(wavs) == 0:
            return []
        B = len(wavs)
        rates = list(sample_rate) if isinstance(sample_rate, (list, tuple)) else [sample_rate] * B
        rates = [self.sample_rate if r is None else int(r) for r in rates]
        rows = [mix_channels(torch.as_tensor(w).to(self._device, dtype=torch.float32), self.channels, f"prompt {i}")
                for i, w in enumerate(wavs)]
        if min(int(w.shape[1]) for w in rows) < 1:
            raise _lib.VcbError("encode_many: an empty prompt")
        for sr in sorted(set(rates) - {self.sample_rate}):           # one ragged resample per rate
            idx = [i for i in range(B) if rates[i] == sr]
            lens = [int(rows[i].shape[1]) for i in idx]
            x = torch.zeros(len(idx), self.channels, max(lens), device=self._device, dtype=torch.float32)
            for j, i in enumerate(idx):
                x[j, :, :lens[j]] = rows[i]
            o, n = resample_dims(sr, self.sample_rate)[:2]
            y = self.resample(x, sr, lens=lens)
            for j, i in enumerate(idx):
                rows[i] = y[j, :, :-(-n * lens[j] // o)]
        lens = [int(w.shape[1]) for w in rows]
        N = max(lens)
        wav = torch.zeros(B, self.channels, N, device=self._device, dtype=torch.float32)
        for b, w in enumerate(rows):
            wav[b, :, :lens[b]] = w
        TN = self.frames(N)
        codes = torch.empty(B, self.config.n_q, TN, device=self._device, dtype=torch.long)
        frames = (C.c_int32 * B)()
        eng = self._engine()
        with torch.cuda.device(self._device):
            _lib.check(_lib.load().enc_encode_ragged(eng, wav.data_ptr(), (C.c_int32 * B)(*lens), B, N, codes.data_ptr(), frames,
                                                     torch.cuda.current_stream().cuda_stream))
        return [codes[b:b + 1, :, :frames[b]] for b in range(B)]

    @torch.no_grad()
    def decode_codes(self, codes: torch.Tensor) -> torch.Tensor:
        """codes [B,K,T] int64 -> wav [B,channels,T*hop] fp32 (batched entry point used by bench.py)."""
        assert codes.ndim == 3 and codes.shape[1] == self.config.n_q, codes.shape
        eng = self._engine()
        codes = codes.to(self._device).long().contiguous()
        B, _, T = codes.shape
        wav = torch.empty(B, self.channels, T * self.hop, device=self._device, dtype=torch.float32)
        with torch.cuda.device(self._device):
            _lib.check(_lib.load().enc_decode(eng, codes.data_ptr(), wav.data_ptr(), B, T,
                                              torch.cuda.current_stream().cuda_stream))
        return wav

    def decode(self, frames) -> torch.Tensor:
        """Reference signature: frames = [(codes[1,K,T], None)] (data/tokenizer.py:131-133)."""
        return self.decode_codes(frames[0][0])

    def open_stream(self, max_streams: int = 1, sample_rate: int = None) -> "CodecStream":
        """Incremental decode of up to `max_streams` utterances (enc_stream_decode), resampled to `sample_rate` when
        one other than the codec's is given: see CodecStream."""
        return CodecStream(self, max_streams, sample_rate)


class CodecStream:
    """Waveform of a growing code sequence, chunk by chunk.  Stream i's chunks, concatenated, are bit-identical to
    ``decode_codes`` of its whole sequence: the causal decoder carries every layer's left context and the LSTM state from
    one chunk to the next.  A stream's first chunk needs at least ``min_frames`` frames.  Runs only on the tensor-core
    decoder; opening one on a codec it does not cover raises VcbError.  Use it from one CUDA stream at a time.

    With a `sample_rate` other than the codec's, every chunk also goes through a streaming resampler on the same CUDA
    stream (enc_resampler_push, one resampler stream per codec stream and channel): stream i's chunks, concatenated, are
    then bit-identical to ``tokenizer.resample(decode_codes(codes_i), codec rate, sample_rate)``, provided its last
    chunk is marked final (``decode(..., final=)``, or ``flush`` when the utterance ends with no new frame).  A chunk
    holds the samples whose resampling window has fully arrived, so chunk lengths vary; ``out_lens`` gives them."""

    def __init__(self, tokenizer: AudioTokenizer, max_streams: int = 1, sample_rate: int = None):
        self._tok = tokenizer
        self._lib = _lib.load()
        self._h, self._rs = None, None
        eng = tokenizer._engine()
        h = C.c_void_p()
        with torch.cuda.device(tokenizer.device):
            _lib.check(self._lib.enc_stream_create(eng, int(max_streams), C.byref(h)))
        self._h = h
        self.max_streams = int(max_streams)
        self.min_frames = int(self._lib.enc_counter(eng, b"stream_min_frames"))
        self.sample_rate = tokenizer.sample_rate if sample_rate is None else int(sample_rate)
        self.out_lens = []                     # samples per row of the last decode / flush
        if self.sample_rate != tokenizer.sample_rate:
            try:
                self._rs = Resampler(tokenizer.sample_rate, self.sample_rate, self.max_streams * tokenizer.channels,
                                     tokenizer.device)
            except Exception:
                self.close()
                raise

    def _rows(self, ids):
        ch = self._tok.channels
        return [i * ch + c for i in ids for c in range(ch)]

    def _resampled(self, x, ids, lens, final):
        """push rows of x [B*channels, N] through the resampler -> wav [B, channels, n]; out_lens per utterance"""
        ch = self._tok.channels
        rep = (lambda v: [u for u in v for _ in range(ch)])
        with torch.cuda.device(self._tok.device):
            y, out_lens = self._rs.push(x, self._rows(ids), rep(lens), None if final is None else rep(final))
        self.out_lens = out_lens[::ch]
        return y.reshape(len(ids), ch, y.shape[1])

    @torch.no_grad()
    def decode(self, codes: torch.Tensor, ids=None, lens=None, final=None) -> torch.Tensor:
        """codes [B,K,T] -> wav [B,channels,N].  Row b continues stream ids[b] (default b) by its next lens[b] frames
        (default T); samples [0, out_lens[b]) of row b are that audio, later samples are unspecified.  At the codec's
        rate out_lens[b] = lens[b]*hop and N = T*hop; resampled, final[b] (default False) marks stream ids[b]'s last
        chunk, which also emits the resampler's tail.  Every code, padding included, must lie in [0, bins).  Runs on the
        current CUDA stream."""
        if self._h is None:
            raise _lib.VcbError("CodecStream is closed")
        assert codes.ndim == 3 and codes.shape[1] == self._tok.config.n_q, codes.shape
        B, _, T = codes.shape
        ids = list(range(B)) if ids is None else [int(i) for i in ids]
        lens = [T] * B if lens is None else [int(n) for n in lens]
        if len(ids) != B or len(lens) != B or (final is not None and len(final) != B):
            raise ValueError(f"CodecStream.decode: {B} rows, {len(ids)} ids, {len(lens)} lens")
        codes = codes.to(self._tok.device).long().contiguous()
        wav = torch.empty(B, self._tok.channels, T * self._tok.hop, device=self._tok.device, dtype=torch.float32)
        with torch.cuda.device(self._tok.device):
            _lib.check(self._lib.enc_stream_decode(self._tok._engine(), self._h, (C.c_int32 * B)(*ids), (C.c_int32 * B)(*lens), B,
                                                   codes.data_ptr(), T, wav.data_ptr(), torch.cuda.current_stream().cuda_stream))
        if self._rs is None:
            self.out_lens = [n * self._tok.hop for n in lens]
            return wav
        hop = self._tok.hop
        return self._resampled(wav.view(B * self._tok.channels, T * hop), ids, [n * hop for n in lens], final)

    @torch.no_grad()
    def flush(self, ids) -> torch.Tensor:
        """Resampled streams only: end the listed streams with no new frames, emitting the resampler's tail of each ->
        wav [len(ids), channels, n], row b's first out_lens[b] samples.  For an utterance whose last decode was not
        marked final."""
        if self._rs is None:
            raise _lib.VcbError("CodecStream.flush: this stream runs at the codec's rate; there is nothing to flush")
        ids = [int(i) for i in ids]
        return self._resampled(None, ids, [0] * len(ids), [True] * len(ids))

    @torch.no_grad()
    def push_audio(self, wav: torch.Tensor, ids, final=None) -> torch.Tensor:
        """Resampled streams only: continue the listed streams' resamplers with codec-rate audio decoded elsewhere,
        wav [B, channels, N] -> wav [B, channels, n], row b's first out_lens[b] samples; final[b] as in decode."""
        if self._rs is None:
            raise _lib.VcbError("CodecStream.push_audio: this stream runs at the codec's rate; there is nothing to resample")
        B, ch, N = wav.shape
        return self._resampled(wav.reshape(B * ch, N), [int(i) for i in ids], [N] * B, final)

    def reset(self, ids, resampler: bool = True):
        """The listed streams start over at frame 0 (and, unless resampler is False, with an empty resampler)."""
        ids = [int(i) for i in ids]
        _lib.check(self._lib.enc_stream_reset(self._h, (C.c_int32 * max(len(ids), 1))(*ids), len(ids)))
        if self._rs is not None and resampler:
            self._rs.reset(self._rows(ids))

    def close(self):
        if self._rs is not None:
            self._rs.close()
            self._rs = None
        if self._h is not None:
            self._lib.enc_stream_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def save_wav(path, wav: torch.Tensor, sample_rate: int):
    """Write a decoded waveform ([1, C, N] / [C, N] / [N] float in [-1, 1]) as 16-bit PCM -- the serialisation step of the
    reference's drivers (torchaudio.save at inference_tts_scale.py:191) without the torchaudio dependency."""
    import wave
    w = wav.detach().float().cpu()
    while w.dim() > 2:
        w = w[0]
    if w.dim() == 1:
        w = w.unsqueeze(0)
    pcm = (w.clamp(-1.0, 1.0) * 32767.0).round().to(torch.int16).t().contiguous().numpy()     # [N, C] interleaved
    with wave.open(str(path), "wb") as f:
        f.setnchannels(int(w.shape[0]))
        f.setsampwidth(2)
        f.setframerate(int(sample_rate))
        f.writeframes(pcm.tobytes())


AudioInfo = namedtuple("AudioInfo", "sample_rate num_frames num_channels")

# (format tag, bits per sample) -> (numpy dtype of a sample, divisor to [-1, 1)): torchaudio.load's scaling
_WAV_FORMATS = {(1, 16): ("<i2", 32768.0), (1, 24): (None, 8388608.0), (1, 32): ("<i4", 2147483648.0), (3, 32): ("<f4", None)}


def _wav_layout(f, path):
    """RIFF/WAVE header of the open file f -> (format tag, channels, rate, bits, offset and bytes of the data chunk).
    WAVE_FORMAT_EXTENSIBLE (0xFFFE) is reported as its sub-format's tag."""
    head = f.read(12)
    if len(head) < 12 or head[:4] != b"RIFF" or head[8:12] != b"WAVE":
        raise ValueError(f"{path}: not a RIFF/WAVE file")
    fmt = None
    while True:
        chunk = f.read(8)
        if len(chunk) < 8:
            raise ValueError(f"{path}: no data chunk")
        cid, size = chunk[:4], struct.unpack("<I", chunk[4:])[0]
        if cid == b"fmt ":
            fmt = f.read(size)
            if size & 1:
                f.seek(1, 1)
        elif cid == b"data":
            if fmt is None or len(fmt) < 16:
                raise ValueError(f"{path}: data chunk before a complete fmt chunk")
            tag, ch, sr, _, _, bits = struct.unpack("<HHIIHH", fmt[:16])
            if tag == 0xFFFE:
                if len(fmt) < 26:
                    raise ValueError(f"{path}: WAVE_FORMAT_EXTENSIBLE without a sub-format")
                tag = struct.unpack("<H", fmt[24:26])[0]
            start = f.tell()
            f.seek(0, 2)
            return tag, ch, sr, bits, start, min(size, f.tell() - start)     # a streamed file may leave size unset
        else:
            f.seek(size + (size & 1), 1)


def _wav_frame_bytes(tag, ch, bits, path):
    if (tag, bits) not in _WAV_FORMATS or ch < 1:
        kind = {1: "PCM", 3: "IEEE float"}.get(tag, f"format tag {tag:#x}")
        raise ValueError(f"{path}: {kind} with {bits} bits per sample and {ch} channels is not supported "
                         "(PCM 16/24/32-bit or 32-bit float WAV)")
    return ch * bits // 8


def audio_info(path) -> AudioInfo:
    """(sample_rate, num_frames, num_channels) of a WAV file: what the reference's drivers read with torchaudio.info to
    place prompt_end_frame (tts_demo.py:177-181)."""
    with open(path, "rb") as f:
        tag, ch, sr, bits, _, size = _wav_layout(f, path)
    return AudioInfo(sr, size // _wav_frame_bytes(tag, ch, bits, path), ch)


def read_wav(path, offset: int = -1, num_frames: int = -1):
    """WAV PCM 16/24/32-bit or IEEE float 32-bit (plain or WAVE_FORMAT_EXTENSIBLE) -> (float32 ndarray [C, N], rate),
    scaled as torchaudio.load scales it (integers over 2^15, 2^23, 2^31).  With offset and num_frames both given, the
    frames [offset, offset + num_frames) at the file's rate, as torchaudio.load(frame_offset=, num_frames=) reads them."""
    import numpy as np
    with open(path, "rb") as f:
        tag, ch, sr, bits, start, size = _wav_layout(f, path)
        fb = _wav_frame_bytes(tag, ch, bits, path)
        n = size // fb
        first = 0
        if offset != -1 and num_frames != -1:
            first = min(int(offset), n)
            n = min(int(num_frames), n - first)
        f.seek(start + first * fb)
        raw = f.read(n * fb)
    dtype, scale = _WAV_FORMATS[(tag, bits)]
    if dtype is None:                                        # 24-bit: three little-endian bytes, sign-extended
        b = np.frombuffer(raw, dtype=np.uint8).reshape(-1, 3).astype(np.int32)
        x = ((b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)) << 8) >> 8
    else:
        x = np.frombuffer(raw, dtype=dtype)
    x = x.reshape(-1, ch).T
    pcm = x.astype(np.float32) if scale is None else x.astype(np.float32) / scale
    return np.ascontiguousarray(pcm), sr


def mix_channels(wav: torch.Tensor, channels: int, what="audio") -> torch.Tensor:
    """[C, N] -> [channels, N] as convert_audio (data/tokenizer.py:85-95) mixes: mono or stereo in; the mean over the
    channels for a mono codec or a multi-channel input, else the single channel broadcast."""
    if wav.ndim != 2 or wav.shape[0] not in (1, 2):
        raise ValueError(f"{what}: audio must be [channels, samples], mono or stereo; got shape {tuple(wav.shape)}")
    if wav.shape[0] != channels:
        wav = wav.mean(dim=0, keepdim=True).expand(channels, -1) if channels == 1 or wav.shape[0] > 1 \
            else wav.expand(channels, -1)
    return wav


def tokenize_audio(tokenizer: AudioTokenizer, audio_path: str, offset=-1, num_frames=-1):
    """The reference's helper (data/tokenizer.py:137-149) without the torchaudio dependency: load a WAV file (read_wav;
    optionally the window of `num_frames` frames from `offset` at the file's rate), mix it to the codec's channel count
    and resample it to the codec's rate as convert_audio does (:85-97; AudioTokenizer.resample on the device), encode."""
    pcm, sr = read_wav(audio_path, offset, num_frames)
    wav = mix_channels(torch.from_numpy(pcm), tokenizer.channels, audio_path).unsqueeze(0)
    with torch.no_grad():
        if sr != tokenizer.sample_rate:
            wav = tokenizer.resample(wav.to(tokenizer.device), sr)
        return tokenizer.encode(wav)


def tokenize_audio_many(tokenizer: AudioTokenizer, paths, offsets=None, num_frames=None):
    """tokenize_audio over several WAV files in one encode: each file read (read_wav, optionally the window of
    num_frames[i] frames from offsets[i] at its own rate), mixed to the codec's channels, resampled per rate on the device
    and encoded with AudioTokenizer.encode_many -> list of codes [1, K, T_i].  Files at one rate are resampled together."""
    n = len(paths)
    offsets = [-1] * n if offsets is None else list(offsets)
    num_frames = [-1] * n if num_frames is None else list(num_frames)
    pcms = [read_wav(p, o, f) for p, o, f in zip(paths, offsets, num_frames)]
    out = [None] * n
    for sr in sorted({sr for _, sr in pcms}):
        idx = [i for i in range(n) if pcms[i][1] == sr]
        for i, codes in zip(idx, tokenizer.encode_many([torch.from_numpy(pcms[i][0]) for i in idx], sr)):
            out[i] = codes
    return out
