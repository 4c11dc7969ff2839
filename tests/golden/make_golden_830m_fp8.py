"""Golden fixture of the fp8 KV policy at the HEADLINE shape: make_golden_830m.py Part B (the bench checkpoint, the same
32 utterances, 64 decode steps, CPU-generator noise 1 + i, the same trace points) decoded by the oracle with K / V stored
as e4m3 with a power-of-two scale per token and head (tests/kv_fp8_ref.py::OracleLMFp8, DESIGN.md section 2.2).
Stored: the sampled rows [32, 64, K], the sensitivity of every sample (the rule of make_golden_830m.py's module
docstring) and the logits at the traced (utterance, step) points.  The oracle only: no reference import.

    python tests/golden/make_golden_830m_fp8.py       # ~10 min on 8 cores
"""
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from make_golden_830m import KW, N_STEPS, PROMPTS, SILENCE, TEXT_LEN, TRACE_STEPS, TRACE_UTTS, bench_checkpoint, \
    cpu_noise, utterance  # noqa: E402


def sensitivity_spy(lm_oracle, margins):
    """lm_oracle.sample_rows plus, per row, the smallest per-logit move that could change the sampled token, appended to
    `margins` (the same rule as make_golden_830m.py's Part B, whose copy is local to that script)"""
    def spy(logits, top_k, top_p, temperature, noise_fn):
        assert top_p >= 1.0 and temperature == 1.0 and top_k > 0
        raw = logits.clone()
        lg = lm_oracle.filter_top_k_top_p(logits.clone(), top_k=top_k, top_p=top_p)
        p = F.softmax(lg, dim=-1)
        q = noise_fn(tuple(p.shape))
        win = torch.argmax(p / q, dim=-1)
        sens = []
        for row in range(raw.shape[0]):
            L = raw[row].double()
            s = L - torch.log(q[row].double())                    # log-domain score (the softmax normaliser cancels)
            k = min(top_k, L.numel())
            srt = torch.sort(L, descending=True)[0]
            kth, nxt = srt[k - 1], (srt[k] if k < L.numel() else torch.tensor(-1e30, dtype=torch.float64))
            kept = L >= kth
            w = int(win[row])
            others = s.clone()
            others[~kept] = -1e30
            others[w] = -1e30
            d1 = (s[w] - others.max()) / 2                         # another kept token overtakes the winner
            d2 = (L[w] - nxt) / 2                                  # the winner drops below the top-k threshold
            exc = ~kept
            d3 = torch.tensor(1e30, dtype=torch.float64)
            if exc.any():                                          # an excluded token enters the top-k and beats the winner
                d3 = torch.maximum((kth - L[exc]) / 2, (s[w] - s[exc]) / 2).min()
            sens.append(float(torch.minimum(torch.minimum(d1, d2), d3).clamp(min=0)))
        margins.append(np.array(sens))
        return win.unsqueeze(-1)
    return spy


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    from kv_fp8_ref import OracleLMFp8
    from oracle import lm_oracle
    t0 = time.time()
    cfg, sd = bench_checkpoint()
    oracle = OracleLMFp8(cfg, sd)
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
            print(f"fp8 utt {i}: ctx {TEXT_LEN + PROMPTS[i % 8] + 1} ({time.time() - t0:.0f}s)", flush=True)
    finally:
        lm_oracle.sample_rows = orig
    np.savez_compressed(os.path.join(HERE, "lm_830m_b32_fp8.npz"), rows_fp8=np.stack(rows_all).astype(np.int16),
                        sens_fp8=np.stack(marg_all).astype(np.float32),
                        logits_fp8=np.stack([traces[i] for i in TRACE_UTTS]).astype(np.float32))
    print("written", time.time() - t0)


if __name__ == "__main__":
    main()
