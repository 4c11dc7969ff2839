"""KV pool budget at bench.py's 830M shapes.  One JSON line per measurement, card name and power limit in each.

  python scripts/bench_kv_pool.py --swap             vcb_swap_out / vcb_swap_in of one 1000-position utterance (text 80,
                                                     919-frame prompt), bf16 and fp8 KV: ms per call (host clock around
                                                     the blocking call) and GB/s of snapshot bytes; the KV bytes of the
                                                     first and last layer are checked equal after the round trips
  python scripts/bench_kv_pool.py --queue 64         ContinuousBatcher.stream() of 64 bench.py-shaped tickets (text 80,
                                                     150-frame prompt) at max_concurrency 32, alternating an unconstrained
                                                     pool and a --pool-pages budget that forces preemptions: seconds to
                                                     all audio, p50 / p90 time to first audio, cb.stats, equal tokens
  python scripts/bench_kv_pool.py --ab PARENT_TREE   each tree's `bench.py --gpus 1 --steps 100 --warmup 10 --no-cpu`,
                                                     alternating processes for --rounds rounds (the parent's own Python
                                                     binding: this build's declares symbols the parent library lacks)
Needs a GPU; no fall-back."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402


def card():
    from bench_stream import gpu_identity
    return gpu_identity(0)


def model_830m(kv, max_slots, max_seq_len, max_new_tokens, pool_gb=None, codec_safe=False):
    import bench
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg, sd = bench.make_model(argparse.Namespace(model="830M", codebooks=4))
    if codec_safe:                              # no frame may hold a token without a waveform
        for k in range(cfg.n_codebooks):
            for t in (cfg.empty_token, cfg.audio_pad_token):
                sd[f"predict_layer.{k}.2.bias"][t] = -1e4
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    m = m.to("cuda").eval()
    m.configure_engine(max_slots=max_slots, max_seq_len=max_seq_len, max_new_tokens=max_new_tokens, kv_dtype=kv,
                       kv_pool_gb=pool_gb)
    return cfg, m


def swap(args):
    import ctypes as C
    from voicecraft_b200 import _lib, synthetic
    from voicecraft_b200.voicecraft import _Prompt, _prefill
    lib = _lib.load()
    for kv in ("bf16", "fp8"):
        cfg, m = model_830m(kv, 2, 1024, 256)
        eng = m._engine()
        stream = torch.cuda.current_stream().cuda_stream
        x, _, y = synthetic.synthetic_utterance(cfg, 100, 80, 919)
        p = _Prompt(m, x.cuda(), y.cuda())
        assert p.total == 1000
        _prefill(eng, [(p, 0, 1, 1, 0)], stream)
        page = lib.vcb_counter(eng, b"kv_page_bytes")
        n_pages = (p.total + 63) // 64

        def pages(layer):
            kb, vb = (C.c_uint8 * (n_pages * page // (2 * cfg.num_decoder_layers)))(), \
                (C.c_uint8 * (n_pages * page // (2 * cfg.num_decoder_layers)))()
            _lib.check(lib.vcb_debug_kv_pages(eng, layer, 0, 0, n_pages, kb, vb))
            return bytes(kb) + bytes(vb)
        before = [pages(0), pages(cfg.num_decoder_layers - 1)]
        t_out, t_in = [], []
        for rep in range(args.reps + 1):                      # rep 0: warm-up (the engine's staging region)
            snap = C.c_void_p()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _lib.check(lib.vcb_swap_out(eng, 0, C.byref(snap), stream))
            t1 = time.perf_counter()
            _lib.check(lib.vcb_swap_in(eng, snap, 0, stream))
            t2 = time.perf_counter()
            lib.vcb_snapshot_free(snap)
            if rep:
                t_out.append(t1 - t0)
                t_in.append(t2 - t1)
        same = [pages(0), pages(cfg.num_decoder_layers - 1)] == before
        _lib.check(lib.vcb_release(eng, 0, 1))
        gb = n_pages * page / 1e9
        out_ms, in_ms = statistics.median(t_out) * 1e3, statistics.median(t_in) * 1e3
        print(json.dumps({"measure": "swap", "kv": kv, "positions": p.total, "pages": n_pages, "snapshot_gb": round(gb, 4),
                          "swap_out_ms": round(out_ms, 3), "swap_in_ms": round(in_ms, 3),
                          "swap_out_gb_s": round(gb / out_ms * 1e3, 2), "swap_in_gb_s": round(gb / in_ms * 1e3, 2),
                          "kv_bytes_equal_after_round_trips": same, "reps": args.reps, "gpu": card(),
                          "note": "median over reps; host clock around the blocking calls"}), flush=True)
        m._drop_engine()
        del m


def queue(args):
    from oracle import encodec_oracle as eo
    from voicecraft_b200 import _lib, synthetic
    from voicecraft_b200.tokenizer import AudioTokenizer
    from voicecraft_b200.voicecraft import ContinuousBatcher
    B, N, text, prompt = 32, args.queue, 80, 150
    cap = text * 10
    seq = (text + cap + 64 + 255) // 256 * 256
    cfg, m = model_830m("bf16", B, seq, cap + 64, codec_safe=True)
    page = _lib.load().vcb_counter(m._engine(), b"kv_page_bytes")
    ccfg = eo.default_config()
    tok = AudioTokenizer(device="cuda:0", config=ccfg, state_dict=eo.make_state_dict(ccfg, seed=0))
    utts = [synthetic.synthetic_utterance(cfg, 100 + i, text, prompt) for i in range(N)]
    xs, ys, seeds = [u[0].cuda() for u in utts], [u[2].cuda() for u in utts], [1 + i for i in range(N)]
    kw = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
    pools = {"unconstrained": None, "budget": (args.pool_pages + 0.5) * page / 1e9}

    def run(pool_gb):
        m.configure_engine(kv_pool_gb=pool_gb)
        m._engine()
        cb = ContinuousBatcher(m, max_concurrency=B, poll_every=8, **kw)
        for x, y, s in zip(xs, ys, seeds):
            cb.submit(x, y, seed=s)
        first = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for t, _, _ in cb.stream(tok, chunk_frames=25):
            first.setdefault(t, time.perf_counter() - t0)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        fa = sorted(first.values())
        return dict(seconds_to_all_audio=round(total, 3), first_audio_ms_p50=round(statistics.median(fa) * 1e3, 1),
                    first_audio_ms_p90=round(fa[int(0.9 * (len(fa) - 1))] * 1e3, 1), stats=dict(cb.stats)), \
            [r[1] for r in cb.results]
    for name, gb in pools.items():                           # warm-up of each pool
        run(gb)
    gens = {}
    for r in range(args.rounds):
        for name, gb in pools.items():
            rec, g = run(gb)
            gens.setdefault(name, g)
            print(json.dumps({"measure": "queue", "round": r, "pool": name, "pool_pages": args.pool_pages if gb else None,
                              "tickets": N, "max_concurrency": B, **rec, "gpu": card()}), flush=True)
    same = all(torch.equal(a, b) for a, b in zip(gens["unconstrained"], gens["budget"]))
    print(json.dumps({"measure": "queue", "equal_tokens": same}), flush=True)


def ab(args):
    runs = {}
    for r in range(args.rounds):
        for name, tree in (("new", ROOT), ("parent", os.path.abspath(args.ab))):
            env = {k: v for k, v in os.environ.items() if k != "VCB_LIB"}
            p = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", "100", "--warmup",
                                "10", "--no-cpu"], env=env, cwd=tree, capture_output=True, text=True)
            if p.returncode:
                sys.stderr.write(p.stderr[-3000:])
                raise SystemExit(f"{name} bench.py failed with {p.returncode}")
            rec = json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("{")][-1])
            runs.setdefault(name, []).append(rec["value"])
            print(json.dumps({"measure": "ab", "round": r, "arm": name, "value": rec["value"], "unit": rec.get("unit"),
                              "e2e": rec.get("e2e")}), flush=True)
    print(json.dumps({"measure": "ab", "values": runs, "gpu": card(),
                      "mean": {k: statistics.mean(v) for k, v in runs.items()}}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--swap", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--queue", type=int, default=0)
    ap.add_argument("--pool-pages", type=int, default=300, help="--queue: pages of the budget arm (32 slots peak at 448)")
    ap.add_argument("--ab", metavar="PARENT_TREE", default=None)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kv_pool.py needs a CUDA device")
    if args.swap:
        swap(args)
    if args.queue:
        queue(args)
    if args.ab:
        ab(args)


if __name__ == "__main__":
    main()
