"""Generate tests/golden/resample.{npz,json} by running the REAL reference's convert_audio (data/tokenizer.py:85-97,
imported from /root/reference), i.e. torchaudio.transforms.Resample after the mono down-mix.

Run in the build container only (the GPU box has neither /root/reference nor torchaudio):
    python tests/golden/make_golden_resample.py

For every rate pair it writes seeded mono and stereo inputs (float32, 0.1-0.2 s, plus one row shorter than the filter
half-width) and what convert_audio makes of them at the codec's 1 channel, and to resample.json the SHA-256 of
torchaudio's filter table bytes (fp32 [n][2w + o]) per pair, so the tables themselves need not be stored.
"""
import hashlib
import json
import math
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"

PAIRS = [(8000, 16000), (22050, 16000), (24000, 16000), (32000, 16000), (44100, 16000), (48000, 16000),
         (16000, 8000), (16000, 22050), (16000, 24000), (16000, 44100), (16000, 48000)]


def import_convert_audio():
    """data/tokenizer.py imports phonemizer for its TextTokenizer; convert_audio does not use it, so stub it.  The stub
    needs Punctuation.default_marks() and Separator(...): default arguments call them when the module is imported."""
    sys.path.insert(0, REF)
    mods = {name: types.ModuleType(name) for name in (
        "phonemizer", "phonemizer.backend", "phonemizer.backend.espeak", "phonemizer.backend.espeak.language_switch",
        "phonemizer.backend.espeak.words_mismatch", "phonemizer.punctuation", "phonemizer.separator")}

    class Punctuation:
        @staticmethod
        def default_marks():
            return ';:,.!?¡¿—…"«»“”'

    class Separator:
        def __init__(self, **kw):
            self.__dict__.update(kw)
    mods["phonemizer.backend"].EspeakBackend = object
    mods["phonemizer.backend.espeak.language_switch"].LanguageSwitch = str
    mods["phonemizer.backend.espeak.words_mismatch"].WordMismatch = str
    mods["phonemizer.punctuation"].Punctuation = Punctuation
    mods["phonemizer.separator"].Separator = Separator
    sys.modules.update(mods)
    from data.tokenizer import convert_audio
    return convert_audio


def signal(rng, channels, length, sr):
    """a few tones, a chirp and noise, peak below 1"""
    t = np.arange(length) / sr
    out = []
    for _ in range(channels):
        x = sum(rng.uniform(0.05, 0.25) * np.sin(2 * np.pi * rng.uniform(50, sr / 2) * t + rng.uniform(0, 6.3))
                for _ in range(4))
        x = x + 0.1 * np.sin(2 * np.pi * (100 + rng.uniform(1, 3) * sr / 4 * t) * t) + 0.05 * rng.standard_normal(length)
        out.append(x)
    return np.clip(np.stack(out), -0.99, 0.99).astype(np.float32)


def main():
    from torchaudio.functional.functional import _get_sinc_resample_kernel
    convert_audio = import_convert_audio()
    rng = np.random.default_rng(20261016)
    arrays, meta = {}, {"pairs": []}
    for orig, new in PAIRS:
        g = math.gcd(orig, new)
        o, n = orig // g, new // g
        kernel, w = _get_sinc_resample_kernel(orig, new, g)
        digest = hashlib.sha256(kernel.to(torch.float32).contiguous().numpy().tobytes()).hexdigest()
        cases = []
        # lengths: not multiples of o; one shorter than w
        for name, ch, length in (("stereo", 2, int(0.2 * orig) + 7), ("mono", 1, int(0.1 * orig) + o // 2 + 3),
                                 ("short", 1, max(1, w - 2))):
            if length % o == 0:
                length += 1
            x = signal(rng, ch, length, orig)
            y = convert_audio(torch.from_numpy(x), orig, new, 1).numpy().astype(np.float32)
            key = f"{orig}_{new}_{name}"
            arrays[key + "_x"], arrays[key + "_y"] = x, y
            cases.append(key)
        meta["pairs"].append(dict(orig=orig, new=new, o=o, n=n, w=int(w), taps=int(kernel.shape[-1]),
                                  table_sha256=digest, cases=cases))
        print(f"{orig} -> {new}: {n} phases x {kernel.shape[-1]} taps, cases {cases}")
    np.savez(os.path.join(HERE, "resample.npz"), **arrays)
    with open(os.path.join(HERE, "resample.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print("size", os.path.getsize(os.path.join(HERE, "resample.npz")))


if __name__ == "__main__":
    main()
