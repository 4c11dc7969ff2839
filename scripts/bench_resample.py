"""Device time of the resampler (enc_resample / enc_resampler_push), one JSON line.

- Prompt audio in: AudioTokenizer.resample of 32 prompts of 10 s at 44.1 kHz and at 48 kHz to 16 kHz, next to
  encode_codes of the resampled batch (the step it precedes in tokenize_audio).
- Streamed audio out: one push of a 25-frame chunk (8000 samples at 16 kHz) to 48 kHz and to 44.1 kHz, for 1 and for
  32 streams in one call.
CUDA events around `--iters` calls after a warm-up; the card's name and power limit are read in the same run.
usage: bench_resample.py [--prompts 32] [--seconds 10] [--iters 20]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402


def gpu_identity(index):
    out = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        import pynvml
        pynvml.nvmlInit()
        out["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(index)) / 1000.0
    except Exception as e:  # pragma: no cover
        out["error"] = repr(e)
    return out


def timed_ms(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--prompts", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resample.py needs a CUDA device")
    from oracle import encodec_oracle as eo
    from voicecraft_b200.tokenizer import AudioTokenizer, Resampler, resample_dims
    cfg = eo.default_config()
    tok = AudioTokenizer(device="cuda:0", config=cfg, state_dict=eo.make_state_dict(cfg, seed=0, encoder=True))
    g = torch.Generator(device="cuda:0").manual_seed(0)
    out = {"gpu": gpu_identity(0), "prompts": a.prompts, "seconds": a.seconds, "iters": a.iters}
    for sr in (44100, 48000):
        wav = torch.rand(a.prompts, 1, int(a.seconds * sr), device="cuda:0", generator=g) * 2 - 1
        ms = timed_ms(lambda: tok.resample(wav, sr), a.iters)
        y = tok.resample(wav, sr)
        enc = timed_ms(lambda: tok.encode_codes(y), max(2, a.iters // 5))
        o, n, w, taps = resample_dims(sr, 16000)
        fma = a.prompts * y.shape[-1] * taps
        out[f"in_{sr}"] = {"resample_ms": round(ms, 4), "encode_codes_ms": round(enc, 3), "taps": taps,
                           "gfma_per_s": round(fma / ms / 1e6, 1), "audio_s_per_s": round(a.prompts * a.seconds / ms * 1e3)}
    chunk = 25 * tok.hop
    for sr in (48000, 44100):
        for B in (1, 32):
            rs = Resampler(16000, sr, B, "cuda:0")
            x = torch.rand(B, chunk, device="cuda:0", generator=g) * 2 - 1
            ids, lens = list(range(B)), [chunk] * B
            ms = timed_ms(lambda: rs.push(x, ids, lens), a.iters)
            out[f"out_{sr}_b{B}"] = {"push_ms_per_25_frame_chunk": round(ms, 4)}
            rs.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
