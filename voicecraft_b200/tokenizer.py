"""Drop-in for the reference's ``data/tokenizer.py::AudioTokenizer`` (:101-133).

``AudioTokenizer(signature=path, device=...)`` mirrors the reference constructor; ``decode(frames)`` takes the
reference's ``[(codes[1,K,T], None)]`` and returns the waveform ``[1, channels, T*hop]``; ``encode(wav[1,C,N])`` returns the
reference's ``[(codes[1,K,T], None)]`` (:127-129).  Instead of audiocraft's ``CompressionSolver.model_from_checkpoint`` +
``EncodecModel.decode / encode`` (:109-110, :128, :133) the weights are handed to libvcb200.so, which runs RVQ and the
SEANet decoder / encoder as sm_90a kernels.  No PyTorch / CPU fallback.  The text tokenizer (espeak) is out of scope.
"""
import ctypes as C
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
            if self._eng is not None:
                _lib.load().enc_destroy(self._eng)
        except Exception:
            pass

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

    def open_stream(self, max_streams: int = 1) -> "CodecStream":
        """Incremental decode of up to `max_streams` utterances (enc_stream_decode): see CodecStream."""
        return CodecStream(self, max_streams)


class CodecStream:
    """Waveform of a growing code sequence, chunk by chunk.  Stream i's chunks, concatenated, are bit-identical to
    ``decode_codes`` of its whole sequence: the causal decoder carries every layer's left context and the LSTM state from
    one chunk to the next.  A stream's first chunk needs at least ``min_frames`` frames.  Runs only on the tensor-core
    decoder; opening one on a codec it does not cover raises VcbError.  Use it from one CUDA stream at a time."""

    def __init__(self, tokenizer: AudioTokenizer, max_streams: int = 1):
        self._tok = tokenizer
        self._lib = _lib.load()
        eng = tokenizer._engine()
        h = C.c_void_p()
        with torch.cuda.device(tokenizer.device):
            _lib.check(self._lib.enc_stream_create(eng, int(max_streams), C.byref(h)))
        self._h = h
        self.max_streams = int(max_streams)
        self.min_frames = int(self._lib.enc_counter(eng, b"stream_min_frames"))

    @torch.no_grad()
    def decode(self, codes: torch.Tensor, ids=None, lens=None) -> torch.Tensor:
        """codes [B,K,T] -> wav [B,channels,T*hop].  Row b continues stream ids[b] (default b) by its next lens[b] frames
        (default T); samples [0, lens[b]*hop) of row b are that audio, later samples are unspecified.  Every code, padding
        included, must lie in [0, bins).  Runs on the current CUDA stream."""
        if self._h is None:
            raise _lib.VcbError("CodecStream is closed")
        assert codes.ndim == 3 and codes.shape[1] == self._tok.config.n_q, codes.shape
        B, _, T = codes.shape
        ids = list(range(B)) if ids is None else [int(i) for i in ids]
        lens = [T] * B if lens is None else [int(n) for n in lens]
        if len(ids) != B or len(lens) != B:
            raise ValueError(f"CodecStream.decode: {B} rows, {len(ids)} ids, {len(lens)} lens")
        codes = codes.to(self._tok.device).long().contiguous()
        wav = torch.empty(B, self._tok.channels, T * self._tok.hop, device=self._tok.device, dtype=torch.float32)
        with torch.cuda.device(self._tok.device):
            _lib.check(self._lib.enc_stream_decode(self._tok._engine(), self._h, (C.c_int32 * B)(*ids), (C.c_int32 * B)(*lens), B,
                                                   codes.data_ptr(), T, wav.data_ptr(), torch.cuda.current_stream().cuda_stream))
        return wav

    def reset(self, ids):
        """The listed streams start over at frame 0."""
        ids = [int(i) for i in ids]
        _lib.check(self._lib.enc_stream_reset(self._h, (C.c_int32 * max(len(ids), 1))(*ids), len(ids)))

    def close(self):
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


def tokenize_audio(tokenizer: AudioTokenizer, audio_path: str, offset=-1, num_frames=-1):
    """The reference's helper (data/tokenizer.py:137-149) for 16-bit PCM WAV files, without the torchaudio dependency:
    load (optionally a window of `num_frames` samples from `offset`), mix to the codec's channel count, encode.
    A file at another sample rate is rejected (the reference resamples with torchaudio; do that before calling)."""
    import wave
    import numpy as np
    with wave.open(str(audio_path), "rb") as f:
        sr, ch, n, width = f.getframerate(), f.getnchannels(), f.getnframes(), f.getsampwidth()
        if width != 2:
            raise ValueError("tokenize_audio: 16-bit PCM WAV expected")
        if offset != -1 and num_frames != -1:
            f.setpos(min(int(offset), n))
            n = min(int(num_frames), n - f.tell())
        pcm = np.frombuffer(f.readframes(n), dtype="<i2").reshape(-1, ch).T.astype(np.float32) / 32768.0
    if sr != tokenizer.sample_rate:
        raise ValueError(f"tokenize_audio: file is {sr} Hz, the codec runs at {tokenizer.sample_rate} Hz (resample first)")
    wav = torch.from_numpy(np.ascontiguousarray(pcm))
    if wav.shape[0] != tokenizer.channels:                    # convert_audio (:77-99): down-mix / broadcast
        wav = wav.mean(dim=0, keepdim=True).expand(tokenizer.channels, -1) if tokenizer.channels == 1 or wav.shape[0] > 1 \
            else wav.expand(tokenizer.channels, -1)
    with torch.no_grad():
        return tokenizer.encode(wav.unsqueeze(0))
