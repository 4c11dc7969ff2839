"""Best-of-N sessions at bench.py's 830M shapes (text 80, 150-frame prompts: 231 prompt positions, 3 full KV pages):
U utterances through open_tts_session(best_of=N), U*N <= 128 rows.  One JSON line per (U, N) with
  prefill_ms        device time of the session's prefill (events around session creation)
  step_ms           mean decode step over a window centred in the generation
  attn_ms_per_step  attention (profile class 1) per step, from a separate profile-mode pass
  kv_pages_free     free KV pages after the prefill (-1: the library has no such counter)
  tokens_sha        hash of every utterance's token rows over the timed window (equal across builds: same output)

  python scripts/bench_best_of.py                         this build
  python scripts/bench_best_of.py --ab PARENT_TREE --rounds 2  this build and the built checkout PARENT_TREE (its library
                                                                through VCB_LIB), alternating processes, then each tree's
                                                                bench.py --gpus 1 alternating the same way
Needs a GPU; no fall-back."""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SHAPES = [(8, 3), (8, 5), (16, 3), (16, 5), (32, 3)]           # (U, N), U * N <= 128


def run_arm(args):
    import torch
    from voicecraft_b200 import _lib, synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    if not torch.cuda.is_available():
        raise SystemExit("bench_best_of needs a GPU")
    if os.environ.get("VCB_LIB"):
        # another build (--ab) may predate debug hooks of this one: bind only the symbols it exports
        other = C.CDLL(_lib.LIB_PATH)
        for name in [n for n in _lib.PROTOTYPES if not hasattr(other, n)]:
            del _lib.PROTOTYPES[name]
    cfg = synthetic.make_config("830M")
    sd = synthetic.make_state_dict(cfg, seed=0)
    end = cfg.eos if cfg.eos > 0 else cfg.eog
    for k in range(cfg.n_codebooks):                       # only the length cap ends generation, as in bench.py
        sd[f"predict_layer.{k}.2.bias"][end] = -1e4
        sd[f"predict_layer.{k}.2.bias"][cfg.eog] = -1e4
    model = VoiceCraft(cfg)
    model.load_state_dict(sd)
    model = model.to("cuda").eval()
    text, prompt = 80, 150
    cap = text * (cfg.encodec_sr // 5)
    total_steps = cap - (prompt + 1) - 2
    model.configure_engine(max_slots=128, max_seq_len=(text + cap + 64 + 255) // 256 * 256, kv_dtype="bf16",
                           max_new_tokens=cap + 64)
    lib = _lib.load()
    kw = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
    for U, N in SHAPES:
        utts = [synthetic.synthetic_utterance(cfg, 100 + i, text, prompt) for i in range(U)]
        xs, ys = [u[0].cuda() for u in utts], [u[2].cuda() for u in utts]
        seeds = [1 + i for i in range(U)]
        start = (total_steps - args.steps) // 2
        out = {"U": U, "N": N, "rows": U * N}
        for rep in range(2):                                # rep 0 warms every shape up
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            torch.cuda.synchronize()
            ev[0].record()
            sess = model.open_tts_session(xs, ys, seeds=seeds, best_of=N, **kw)
            ev[1].record()
            try:
                out["kv_pages_free"] = int(lib.vcb_counter(sess.eng, b"kv_pages_free"))
                sess.sample()
                for _ in range(start):
                    sess.step()
                ev[2].record()
                for _ in range(args.steps):
                    sess.step()
                ev[3].record()
                torch.cuda.synchronize()
                h = hashlib.sha256()
                st = sess.poll()
                for i, s in enumerate(sess.slots):
                    h.update(model._read_rows(sess.eng, s, st[i].n_steps, sess.stream).tobytes())
                lib.vcb_set_option(sess.eng, b"profile", 1)
                msb, cnt = (C.c_double * 7)(), (C.c_int64 * 7)()
                lib.vcb_profile_read(sess.eng, msb, cnt, 7)
                for _ in range(args.prof_steps):
                    sess.step()
                lib.vcb_profile_read(sess.eng, msb, cnt, 7)
                lib.vcb_set_option(sess.eng, b"profile", 0)
            finally:
                sess.close()
        out.update(prefill_ms=round(ev[0].elapsed_time(ev[1]), 3), step_ms=round(ev[2].elapsed_time(ev[3]) / args.steps, 4),
                   attn_ms_per_step=round(msb[1] / args.prof_steps, 4), tokens_sha=h.hexdigest()[:16],
                   lib=os.environ.get("VCB_LIB", "this build"))
        print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--prof-steps", type=int, default=20)
    ap.add_argument("--ab", metavar="PARENT_TREE", default=None)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not args.ab:
        return run_arm(args)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_best_of needs a GPU")
    me = [sys.executable, os.path.abspath(__file__), "--steps", str(args.steps), "--prof-steps", str(args.prof_steps)]
    sha = {}                                                # (arm, U, N) -> token hashes of every round
    for r in range(args.rounds):
        for name, tree in (("new", ROOT), ("parent", os.path.abspath(args.ab))):
            env = dict(os.environ)
            env.pop("VCB_LIB", None)
            if tree != ROOT:
                env["VCB_LIB"] = os.path.join(tree, "voicecraft_b200", "libvcb200.so")
            bench = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--no-cpu"]
            for cmd, cwd in ((me, ROOT), (bench, tree)):
                p = subprocess.run(cmd, env=env if cwd == ROOT else {k: v for k, v in env.items() if k != "VCB_LIB"},
                                   cwd=cwd, capture_output=True, text=True)
                for line in p.stdout.splitlines():
                    if line.startswith("{"):
                        rec = json.loads(line)
                        if "tokens_sha" in rec:
                            sha.setdefault((name, rec["U"], rec["N"]), set()).add(rec["tokens_sha"])
                        print(json.dumps({"round": r, "arm": name, "cmd": os.path.basename(cmd[1]), **rec}), flush=True)
                if p.returncode:
                    sys.stderr.write(p.stderr[-3000:])
                    raise SystemExit(f"{name} {cmd[1]} failed with {p.returncode}")
    shapes = sorted({k[1:] for k in sha})
    same = {f"U{U}_N{N}": sha.get(("new", U, N)) == sha.get(("parent", U, N)) and len(sha.get(("new", U, N), ())) == 1
            for U, N in shapes}
    print(json.dumps({"equal_tokens": same, "all_equal": all(same.values())}), flush=True)


if __name__ == "__main__":
    main()
