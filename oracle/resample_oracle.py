"""fp64 numpy restatement of torchaudio.transforms.Resample(orig, new) with its defaults (sinc_interp_hann,
lowpass_filter_width 6, rolloff 0.99) and of the streaming rule of enc_resampler_push.

Restates torchaudio/functional/functional.py:
  _get_sinc_resample_kernel   -> table()    (n phases x 2w + o taps, fp64, rounded once to fp32)
  _apply_sinc_resample_kernel -> resample() (pad w left / w + o right, stride-o correlation, ceil(n L / o) samples)
The reference's convert_audio (data/tokenizer.py:85-97) calls them through Resample(sr, target_sr).
"""
import math

import numpy as np


def dims(orig, new):
    """(o, n, w): the rates over their gcd and the filter half-width"""
    g = math.gcd(int(orig), int(new))
    o, n = int(orig) // g, int(new) // g
    return o, n, math.ceil(6 * o / (min(o, n) * 0.99))


def table(orig, new):
    """fp32 [n][2w + o].  The phase offsets -p/n are computed in fp32, as torchaudio computes them (an integer arange
    divided in the default dtype), before the fp64 tap positions are added."""
    o, n, w = dims(orig, new)
    base = min(o, n) * 0.99
    pos = np.arange(-w, w + o, dtype=np.float64) / o
    phase = (np.arange(0, -n, -1, dtype=np.float32) / np.float32(n)).astype(np.float64)
    t = np.clip((phase[:, None] + pos[None, :]) * base, -6.0, 6.0)
    window = np.cos(t * math.pi / 6 / 2) ** 2
    t = t * math.pi
    with np.errstate(invalid="ignore", divide="ignore"):
        k = np.where(t == 0, 1.0, np.sin(t) / t)
    return (k * (window * (base / o))).astype(np.float32)


def out_length(L, orig, new):
    o, n, _ = dims(orig, new)
    return -(-int(L) * n // o)


def resample(x, orig, new, K=None):
    """x [L] -> (y [ceil(n L / o)] fp64, bound [same]): y[b*n + p] = sum_i K[p][i] x[b*o + i - w] in fp64 with the fp32
    table, and bound = sum_i |K[p][i]| |x[b*o + i - w]|, the scale of the rounding error of any fp32 evaluation."""
    o, n, w = dims(orig, new)
    K = (table(orig, new) if K is None else K).astype(np.float64)
    x = np.asarray(x, dtype=np.float64)
    L = x.shape[0]
    xp = np.concatenate([np.zeros(w), x, np.zeros(w + o)])
    blocks = L // o + 1
    win = np.lib.stride_tricks.sliding_window_view(xp, 2 * w + o)[::o][:blocks]      # [blocks][taps]
    y, bound = np.zeros((blocks, n)), np.zeros((blocks, n))
    for i in range(2 * w + o):                 # taps in order, elementwise: a sample's sum does not depend on L
        y += win[:, i:i + 1] * K[None, :, i]
        bound += np.abs(win[:, i:i + 1]) * np.abs(K[None, :, i])
    y, bound = y.reshape(-1), bound.reshape(-1)
    m = out_length(L, orig, new)
    return y[:m], bound[:m]


class Stream:
    """The streaming rule of enc_resampler_push for one stream.  After L input samples, block b (outputs b*n .. b*n + n-1)
    is emitted once its whole window has arrived, b*o + w + o <= L; the final push also emits the zero-padded tail up to
    ceil(n L / o).  Emitted samples are computed from the input received so far only."""

    def __init__(self, orig, new):
        self.orig, self.new = orig, new
        self.o, self.n, self.w = dims(orig, new)
        self.K = table(orig, new)
        self.x = np.zeros(0)
        self.emitted = 0
        self.done = False

    def ready(self, L):
        return 0 if L < self.w + self.o else ((L - self.w - self.o) // self.o + 1) * self.n

    def push(self, chunk, final=False):
        assert not self.done, "push after the final push"
        self.x = np.concatenate([self.x, np.asarray(chunk, dtype=np.float64)])
        L = self.x.shape[0]
        total = out_length(L, self.orig, self.new) if final else self.ready(L)
        if not final:                          # every emitted window lies inside the input received so far
            last_block = total // self.n - 1
            assert last_block < 0 or last_block * self.o + self.w + self.o <= L
        y, _ = resample(self.x, self.orig, self.new, self.K)
        if not final:
            y = y[:total]
        out = y[self.emitted:total]
        self.emitted, self.done = total, final
        return out
