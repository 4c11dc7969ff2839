"""Cost of text-speech alignment at the 830M bench shape (B = 32 utterances, text 80 tokens, 150 prompt frames), bf16 and
fp8 KV, one JSON line per measurement with the card, its power limit and SM clock:
  step     decode-step time (CUDA events around `--steps` steps after `--warmup`) with alignment off, one head, one
           layer's heads and every head of every layer;
  prefill  the packed prefill of the 32 prompts, alignment off and every head;
  probe    the probe's own time per step (profile class 5, which holds only the probe in a step: the step's other class-5
           launch is step_prep, subtracted with the off run's class 5), its bytes (K read twice per text key, once per other
           context key, per selected head and row) and achieved bandwidth;
  mas      vcb_align_monotonic at T = 800 and 4096 (X = 80), CUDA events over 20 calls.

usage: bench_align.py [--warmup 10] [--steps 50]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--warmup", type=int, default=10)
ap.add_argument("--steps", type=int, default=50)
args = ap.parse_args()
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import bench  # noqa: E402
from voicecraft_b200 import _lib  # noqa: E402
from voicecraft_b200.alignment import monotonic_durations  # noqa: E402
from voicecraft_b200.voicecraft import VoiceCraft  # noqa: E402

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
B = 32


class A:
    model, batch, codebooks, text_len, prompt = "830M", B, 4, 80, 150


cfg, sd, utts = bench.make_model_inputs(A)
lib = _lib.load()
L, H, hd = cfg.num_decoder_layers, cfg.nhead, cfg.d_model // cfg.nhead
xs, ys = [u[0].cuda() for u in utts[:B]], [u[2].cuda() for u in utts[:B]]
x_len = int(xs[0].shape[1])


def emit(**kw):
    print(json.dumps(dict(card=card, **kw)), flush=True)


def run(m, kv, name, align):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record()
    sess = m.open_tts_session(xs, ys, top_k=40, seeds=list(range(B)), alignment=align)
    ev[1].record()
    try:
        sess.sample()
        for _ in range(args.warmup):
            sess.step()
        lib.vcb_set_option(sess.eng, b"profile", 1)
        ev[2].record()
        for _ in range(args.steps):
            sess.step()
        ev[3].record()
        torch.cuda.synchronize()
        ms, cnt = (C.c_double * 7)(), (C.c_int64 * 7)()
        _lib.check(lib.vcb_profile_read(sess.eng, ms, cnt, 7))
        lib.vcb_set_option(sess.eng, b"profile", 0)
        ctx = sess.prompts[0].total + args.warmup + args.steps // 2          # mean context of the timed steps
    finally:
        sess.close()
    return dict(kv=kv, alignment=name, prefill_ms=ev[0].elapsed_time(ev[1]),
                step_ms=ev[2].elapsed_time(ev[3]) / args.steps, misc_ms=ms[5] / args.steps, misc_launches=cnt[5] / args.steps,
                ctx=ctx)


for kv in ("bf16", "fp8"):
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    m.configure_engine(kv_dtype=kv, max_slots=B, max_seq_len=1024, max_new_tokens=args.warmup + args.steps + 8,
                       align_text_cap=x_len)
    run(m, kv, "warm-up", None)
    off = run(m, kv, "off", None)
    emit(what="step", **off)
    kv_elem = {"bf16": 2, "fp8": 1}[kv]
    for name, align, heads in (("one head", {L // 2: [0]}, 1), ("one layer", {L // 2: list(range(H))}, H),
                               ("all heads", True, L * H)):
        r = run(m, kv, name, align)
        probe_ms = r["misc_ms"] - off["misc_ms"]
        # per selected head and row: every context key once (max and sum), the text keys again; fp8 adds a 4-byte scale
        per_key = hd * kv_elem + (4 if kv == "fp8" else 0)
        nbytes = B * heads * (r["ctx"] + x_len) * per_key
        emit(what="step", probe_ms=probe_ms, probe_bytes=nbytes,
             probe_gbs=nbytes / (probe_ms * 1e-3) / 1e9 if probe_ms > 0 else None, **r)
    del m
    torch.cuda.empty_cache()

for T in (800, 4096):
    lp = torch.log(torch.softmax(torch.randn(T, x_len, device="cuda"), -1))
    monotonic_durations(lp)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        monotonic_durations(lp)
    e1.record()
    torch.cuda.synchronize()
    emit(what="mas", T=T, X=x_len, ms=e0.elapsed_time(e1) / 20)
