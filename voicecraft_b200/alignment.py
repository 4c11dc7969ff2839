"""Text-speech alignment of a TTS result from the codec LM's own attention (DESIGN.md section 4.6, INTEGRATION.md).

Frame <-> row mapping.  The TTS prompt is the delayed pattern of the T prompt frames with its last K-1 columns dropped
(reference voicecraft.py:961-967): column c (engine position x_len + c) holds codebook k of frame c - 1 - k, so the row at
position x_len + c is the one whose logits give (or, in the prompt, would give) codebook 0 of frame c.  Generation continues
the same arithmetic: the first sample reads the row at x_len + T (codebook 0 of frame T, the first generated one) and step
i's row at x_len + T + i gives sampled row i, whose codebook 0 is frame T + i (un-delayed as voicecraft.py:1126-1137 does).
So frame t of `res` is the row at position x_len + t, prompt frames and generated frames alike.

Head choice is a parameter: which heads of a trained VoiceCraft checkpoint align well, and how accurate the resulting word
timings are, has not been measured.
"""
import csv
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

AlignSpec = Union[None, bool, Dict[int, Sequence[int]]]


def head_masks(alignment: AlignSpec, n_layers: int, n_heads: int) -> Optional[np.ndarray]:
    """The alignment= argument as vcb_prompt.align_heads: [n_layers] uint32 head bitmasks, or None (off).
    True: every head of every layer; {layer: [heads]}: those heads."""
    if alignment is None or alignment is False:
        return None
    if n_heads > 32:
        raise ValueError(f"alignment: at most 32 heads per layer are addressable (the model has {n_heads})")
    m = np.zeros(n_layers, dtype=np.uint32)
    if alignment is True:
        m[:] = (1 << n_heads) - 1
        return m
    if not isinstance(alignment, dict) or not alignment:
        raise ValueError("alignment: None, True, or a non-empty {layer: [heads]} dict")
    for layer, heads in alignment.items():
        if not (isinstance(layer, (int, np.integer)) and 0 <= int(layer) < n_layers):
            raise ValueError(f"alignment: layer {layer!r} outside [0, {n_layers})")
        heads = list(heads)
        if not heads:
            raise ValueError(f"alignment: layer {layer} lists no head")
        for h in heads:
            if not (isinstance(h, (int, np.integer)) and 0 <= int(h) < n_heads):
                raise ValueError(f"alignment: head {h!r} of layer {layer} outside [0, {n_heads})")
            m[int(layer)] |= np.uint32(1 << int(h))
    return m


def monotonic_durations(logp: torch.Tensor) -> torch.Tensor:
    """vcb_align_monotonic on a CUDA tensor logp [T, X] fp32: durations [X] int32 on its device (T >= X)."""
    from . import _lib
    T, X = logp.shape
    logp = logp.to(torch.float32).contiguous()
    out = torch.empty(X, dtype=torch.int32, device=logp.device)
    with torch.cuda.device(logp.device):
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(_lib.load().vcb_align_monotonic(logp.data_ptr(), T, X, out.data_ptr(), st))
    return out


class Alignment:
    """soft [T, x_len] fp32: row t is frame t of `res` (prompt frames included); its mean attention weight over the
    selected heads on each text token.  durations [x_len] int32: frames per token from the device monotonic alignment
    search on log(soft) (None when the result has fewer frames than text tokens).  encodec_sr: frames per second.
    text_ids [x_len]: the text tokens (words() splits at the separator among them)."""

    def __init__(self, soft: torch.Tensor, durations: Optional[torch.Tensor], encodec_sr: float, text_ids=None):
        self.soft, self.durations, self.encodec_sr = soft, durations, float(encodec_sr)
        self.text_ids = None if text_ids is None else np.asarray(torch.as_tensor(text_ids).cpu()).reshape(-1)

    @classmethod
    def from_soft(cls, soft: torch.Tensor, encodec_sr: float, text_ids=None) -> "Alignment":
        T, X = soft.shape
        dur = None
        if T >= X and soft.is_cuda:
            # log 0 = -inf is a valid input: such a cell is never preferred over a finite one
            dur = monotonic_durations(torch.log(soft))
        return cls(soft, dur, encodec_sr, text_ids)

    def token_frames(self) -> List[Tuple[int, int]]:
        """[start, end) frames of each text token"""
        if self.durations is None:
            raise ValueError("no durations: the result has fewer frames than text tokens")
        ends = np.cumsum(self.durations.cpu().numpy().astype(np.int64))
        return [(int(e - d), int(e)) for d, e in zip(self.durations.cpu().numpy(), ends)]

    def words(self, sep_id: int) -> List[Tuple[int, int, float, float]]:
        """Tokens grouped into words at the separator token `sep_id` (the reference phonemizer's word separator '_',
        data/tokenizer.py:40): (first_token, last_token, start_s, end_s) per word, separators excluded."""
        frames = self.token_frames()
        if self.text_ids is None:
            raise ValueError("words(): the alignment carries no text ids")
        out, cur = [], []
        for i in range(len(frames)):
            if int(self.text_ids[i]) == sep_id:
                if cur:
                    out.append(cur)
                cur = []
            else:
                cur.append(i)
        if cur:
            out.append(cur)
        sr = self.encodec_sr
        return [(w[0], w[-1], frames[w[0]][0] / sr, frames[w[-1]][1] / sr) for w in out]

    def to_mfa_csv(self, path: str, labels: Sequence[str], sep_id: int) -> None:
        """Write words(sep_id) in the reference's MFA layout `Begin,End,Label,Type,Speaker` (demo/temp/mfa_alignments,
        read by inference_speech_editing_scale.py:get_mask_interval), one label per word."""
        words = self.words(sep_id)
        if len(labels) != len(words):
            raise ValueError(f"{len(labels)} labels for {len(words)} words")
        with open(path, "w", newline="") as f:
            w = csv.writer(f, lineterminator="\n")
            w.writerow(["Begin", "End", "Label", "Type", "Speaker"])
            for (_, _, s, e), lab in zip(words, labels):
                w.writerow([f"{s:.3f}", f"{e:.3f}", lab, "words", "temp"])
