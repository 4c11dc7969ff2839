"""Golden fixture of the int8 weight policy at the HEADLINE shape: make_golden_830m.py Part B (the bench checkpoint, the
same 32 utterances, 64 decode steps, CPU-generator noise 1 + i, the same trace points) decoded by the oracle under the bf16
KV policy (kv_round_bf16=True) on the dequantized checkpoint (tests/weight_int8_ref.py::dequantize_state_dict, DESIGN.md
section 2.2).  Stored: the sampled rows [32, 64, K], the sensitivity of every sample (make_golden_830m.py's rule) and the
logits at the traced (utterance, step) points.  Against lm_830m_b32.npz's bf16 policy on the checkpoint itself, this is
how far int8 weights move the oracle.  The oracle only: no reference import.

    python tests/golden/make_golden_830m_int8.py      # ~5 min on 8 cores
"""
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from make_golden_830m import KW, N_STEPS, PROMPTS, SILENCE, TEXT_LEN, TRACE_STEPS, TRACE_UTTS, bench_checkpoint, \
    cpu_noise, utterance  # noqa: E402
from make_golden_830m_fp8 import sensitivity_spy  # noqa: E402


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    from oracle import lm_oracle
    from weight_int8_ref import dequantize_state_dict
    t0 = time.time()
    cfg, sd = bench_checkpoint()
    oracle = lm_oracle.OracleLM(cfg, dequantize_state_dict(sd), kv_round_bf16=True)
    del sd
    orig = lm_oracle.sample_rows
    rows_all, marg_all, traces = [], [], {}
    try:
        for i in range(32):
            x, xl, y = utterance(cfg, i)
            margins = []
            lm_oracle.sample_rows = sensitivity_spy(lm_oracle, margins)
            rows = oracle.inference_tts(x, xl, y, silence_tokens=SILENCE, noise_fn=cpu_noise(1 + i), max_steps=N_STEPS,
                                        trace_logits=True, **KW)
            assert rows.shape == (N_STEPS, cfg.n_codebooks)
            rows_all.append(rows.numpy())
            marg_all.append(np.stack(margins))                     # [N, K]
            if i in TRACE_UTTS:
                traces[i] = np.stack([oracle.logit_trace[s].numpy() for s in TRACE_STEPS])
            print(f"int8 utt {i}: ctx {TEXT_LEN + PROMPTS[i % 8] + 1} ({time.time() - t0:.0f}s)", flush=True)
    finally:
        lm_oracle.sample_rows = orig
    np.savez_compressed(os.path.join(HERE, "lm_830m_b32_int8.npz"), rows_int8=np.stack(rows_all).astype(np.int16),
                        sens_int8=np.stack(marg_all).astype(np.float32),
                        logits_int8=np.stack([traces[i] for i in TRACE_UTTS]).astype(np.float32))
    print("written", time.time() - t0)


if __name__ == "__main__":
    main()
