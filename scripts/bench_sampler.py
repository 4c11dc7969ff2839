"""sampler_kernel time per decode step at 830M (profile class 4: one CUDA event pair around each sampler launch), B = 32
and 64 utterances, top-k 40, one device Philox stream per utterance, contexts from 231 on.  Prints one JSON line per batch
with the card, its power limit and SM clock.  --root: the tree whose voicecraft_b200 package (and library) to measure,
for A/B runs against another build.

--ras: repetition-aware sampling off against windows of 10 and 32 tokens, on a window that never fires (threshold = the
window: a token would have to fill all of it, which top-k 40 over random weights does not do) and on one that fires at
every step after the first (the heads biased +30 towards audio token 5 in every codebook, threshold 1), one JSON line
per batch, model and setting.

usage: bench_sampler.py [--root DIR] [--batches 32,64] [--warmup 20] [--steps 200] [--ras]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--batches", default="32,64")
ap.add_argument("--warmup", type=int, default=20)
ap.add_argument("--steps", type=int, default=200)
ap.add_argument("--ras", action="store_true")
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import torch  # noqa: E402

import bench  # noqa: E402
from voicecraft_b200 import _lib  # noqa: E402
from voicecraft_b200.voicecraft import VoiceCraft  # noqa: E402

batches = [int(b) for b in args.batches.split(",")]
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()


class A:
    model, batch, codebooks, text_len, prompt = "830M", max(batches), 4, 80, 150


cfg, sd, utts = bench.make_model_inputs(A)
m = None
lib = _lib.load()


def sampler_us(B, **kw):
    """sampler_kernel microseconds per decode step of B utterances (profile class 4) and launches per step"""
    sess = m.open_tts_session([u[0].cuda() for u in utts[:B]], [u[2].cuda() for u in utts[:B]], top_k=40,
                              seeds=list(range(B)), **kw)
    try:
        sess.sample()
        for _ in range(args.warmup):
            sess.step()
        torch.cuda.synchronize()
        lib.vcb_set_option(sess.eng, b"profile", 1)
        for _ in range(args.steps):
            sess.step()
        torch.cuda.synchronize()
        ms, cnt = (C.c_double * 7)(), (C.c_int64 * 7)()
        _lib.check(lib.vcb_profile_read(sess.eng, ms, cnt, 7))
        lib.vcb_set_option(sess.eng, b"profile", 0)
    finally:
        sess.close()
    return 1e3 * ms[4] / args.steps, cnt[4] / args.steps


def load(state_dict):
    global m
    m = VoiceCraft(cfg)
    m.load_state_dict(state_dict)
    m = m.cuda().eval()
    m.configure_engine(max_slots=max(batches), max_seq_len=1024, max_new_tokens=args.warmup + args.steps + 8)


if not args.ras:
    load(sd)
    for B in batches:
        us, launches = sampler_us(B)
        print(json.dumps(dict(root=os.path.abspath(args.root), B=B, steps=args.steps, sampler_us_per_step=us,
                              sampler_launches_per_step=launches, card=card)), flush=True)
    sys.exit(0)

biased = {k: v.clone() if k.startswith("predict_layer.") else v for k, v in sd.items()}
for k in range(cfg.n_codebooks):
    biased[f"predict_layer.{k}.2.bias"][5] += 30.0
for model, state_dict, tau in (("random", sd, 1.0), ("biased", biased, None)):
    load(state_dict)
    for B in batches:
        for W in (0, 10, 32):
            kw = dict(ras_window=W, ras_tau=tau if tau is not None else 1.0 / W) if W else {}
            us, launches = sampler_us(B, **kw)
            print(json.dumps(dict(root=os.path.abspath(args.root), B=B, steps=args.steps, model=model, ras_window=W,
                                  ras_threshold=m._sampling(40, 1.0, 1.0, 3, [], **kw).ras_threshold,
                                  fires="never" if model == "random" else "every step", sampler_us_per_step=us,
                                  sampler_launches_per_step=launches, card=card)), flush=True)
