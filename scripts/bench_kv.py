"""bf16 against fp8 KV cache at bench.py's 830M TTS workload (text 80, 150-frame prompts: contexts 231 -> 881), the timed
window centred on the mean context as bench.py centres it.  For each batch size and policy, alternating the policies in
every round, one JSON line with
  step_ms, tokens_per_s      device time of --steps decode steps (events), codec tokens / s
  attn_ms_per_step           attention (profile class 1) per step, from a separate profile-mode pass after the window
  attn_bytes_per_step        K / V bytes the attention fetches per step at the profiled contexts (whole 64-token slabs,
                             fp8 scales included), computed from shapes
  attn_gbs                   attn_bytes_per_step / attn_ms_per_step
  kv_bytes_per_token         vcb_counter
  max_slots_in_budget        slots of this max_seq_len whose pools fit in --pool-gb (computed, not allocated)
and first a line with the card name, power limit and SM clocks.

  python scripts/bench_kv.py --batches 32 64 128 --rounds 2
Needs a GPU; no fall-back."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [s.strip() for s in out.stdout.splitlines()[0].split(",")])) if out.returncode == 0 else {}


def run(model, cfg, B, kv, args):
    import torch
    import bench
    from voicecraft_b200 import _lib
    lib = _lib.load()
    text_len, prompt = 80, 150
    cap = text_len * (cfg.encodec_sr // 5)
    S_total = cap - (prompt + 1) - 2
    start = max(args.warmup, (S_total - args.steps) // 2)
    max_seq_len = (text_len + cap + 64 + 255) // 256 * 256
    model.configure_engine(max_slots=B, max_seq_len=max_seq_len, kv_dtype=kv, max_new_tokens=cap + 64)
    a = argparse.Namespace(text_len=text_len, prompt=prompt)
    utts = bench.make_utterances(a, cfg, range(B))
    sess = model.open_tts_session([u[0].cuda() for u in utts], [u[2].cuda() for u in utts], seeds=[1 + i for i in range(B)],
                                  top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
    try:
        eng = sess.eng
        sess.sample()
        for _ in range(start):
            sess.step()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(args.steps):
            sess.step()
        ev1.record()
        torch.cuda.synchronize()
        ms = ev0.elapsed_time(ev1) / args.steps
        nprof = 8
        ctx = text_len + prompt + 1 + start + args.steps           # context of the first profiled step
        msb, cnt = bench.profile_pass(lib, eng, sess, nprof)
        per_tok = lib.vcb_counter(eng, b"kv_bytes_per_token")
        # what the TMA copies: every row fetches each page of its context (keys 0..pos) whole, K and V slab of every head in
        # every layer, scales included -- 64 * kv_bytes_per_token per page; pos = ctx + s at profiled step s
        attn_bytes = B * 64 * per_tok * sum((ctx + s) // 64 + 1 for s in range(nprof)) / nprof
        attn_ms = msb[1] / nprof
        return dict(kv=kv, B=B, steps=args.steps, ctx_window=[text_len + prompt + 1 + start, ctx], step_ms=ms,
                    tokens_per_s=B * cfg.n_codebooks / (ms * 1e-3), attn_ms_per_step=attn_ms,
                    attn_launches_per_step=cnt[1] / nprof, attn_bytes_per_step=attn_bytes,
                    attn_gbs=attn_bytes / (attn_ms * 1e-3) / 1e9, kv_bytes_per_token=per_tok,
                    max_slots_in_budget=int(args.pool_gb * 2 ** 30 // (max_seq_len * per_tok)), pool_gb=args.pool_gb,
                    max_seq_len=max_seq_len)
    finally:
        sess.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--pool-gb", type=float, default=40.0, help="KV pool budget of the max_slots_in_budget column")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_kv needs a GPU")
    import bench
    from voicecraft_b200.voicecraft import VoiceCraft
    print(json.dumps({"card": card()}), flush=True)
    cfg, sd = bench.make_model(argparse.Namespace(model="830M", codebooks=4))
    model = VoiceCraft(cfg)
    model.load_state_dict(sd)
    model = model.cuda().eval()
    for r in range(args.rounds):
        for B in args.batches:
            for kv in (("bf16", "fp8") if r % 2 == 0 else ("fp8", "bf16")):
                print(json.dumps(dict(run(model, cfg, B, kv, args), round=r)), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
