"""The CPU oracle against the fixtures the real reference produced (tests/golden/make_golden.py).
Token ids must be identical; traced logits within 2e-5 (they are bit-identical for the B=1 flows)."""
import numpy as np
import pytest
import torch

import golden_util as gu
from oracle import lm_oracle

CASES = gu.load_cases()


def _run_oracle(name, case, **okw):
    cfg, sd, x, x_lens, y, g = gu.build_case(name, case)
    oracle = lm_oracle.OracleLM(cfg, sd, **okw)
    kw = dict(case["kw"], silence_tokens=gu.SILENCE, kvcache=1, noise_fn=gu.cpu_noise_fn(case["seed"]))
    trace = []
    orig = lm_oracle.sample_rows

    def spy(logits, *a, **k):
        trace.append(logits.detach().clone())
        return orig(logits, *a, **k)
    lm_oracle.sample_rows = spy
    try:
        if case["kind"] == "tts":
            res, gen = oracle.inference_tts(x, x_lens, y, **kw)
        elif case["kind"] == "batch":
            res, gen = oracle.inference_tts_batch(x, x_lens, y, batch_size=case["batch_size"], **kw)
        else:
            res = oracle.inference(x, x_lens, y, torch.from_numpy(g["mask_interval"]), **kw)
    finally:
        lm_oracle.sample_rows = orig
    return res, trace, g


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_reference(name):
    torch.set_num_threads(min(8, torch.get_num_threads()))
    res, trace, g = _run_oracle(name, CASES[name])
    assert np.array_equal(res.numpy(), g["res"]), "oracle token ids differ from the reference fixture"
    assert len(trace) == int(g["n_steps"])
    for step, ref in zip(g["trace_steps"], g["trace_logits"]):
        got = trace[int(step)].reshape(-1, ref.shape[-1]).numpy()
        assert np.abs(got - ref).max() <= 2e-5


def test_invariants():
    """SURVEY.md section 4: steps = gen_len + K; first K-1 steps force empty on late codebooks; kvcache on/off."""
    name = "tts_topk40"
    case = CASES[name]
    cfg, sd, x, x_lens, y, g = gu.build_case(name, case)
    assert int(g["kvcache0_equal"]) == 1          # measured on the real reference when the fixture was made
    K = cfg.n_codebooks
    gen_len = g["res"].shape[2] - y.shape[1]
    assert int(g["n_steps"]) == gen_len + K
    # length cap: y_len > x_len * (encodec_sr // 5) ends generation (voicecraft.py:1042)
    assert g["res"].shape[2] == case["text_len"] * (cfg.encodec_sr // 5)
    oracle = lm_oracle.OracleLM(cfg, sd)
    kw = dict(case["kw"], silence_tokens=gu.SILENCE, noise_fn=gu.cpu_noise_fn(case["seed"]))
    res0, _ = oracle.inference_tts(x, x_lens, y, kvcache=0, **kw)
    assert np.array_equal(res0.numpy(), g["res"])


def test_topk1_is_argmax():
    case = CASES["tts_greedy"]
    cfg, sd, x, x_lens, y, g = gu.build_case("tts_greedy", case)
    a = lm_oracle.OracleLM(cfg, sd).inference_tts(x, x_lens, y, silence_tokens=gu.SILENCE,
                                                  noise_fn=gu.cpu_noise_fn(1), **case["kw"])[0]
    b = lm_oracle.OracleLM(cfg, sd).inference_tts(x, x_lens, y, silence_tokens=gu.SILENCE,
                                                  noise_fn=gu.cpu_noise_fn(2), **case["kw"])[0]
    assert torch.equal(a, b) and np.array_equal(a.numpy(), g["res"])


def test_kv_bf16_policy_is_close():
    """Rounding cached K/V to bf16 (the H100 default) moves logits by ~1e-3 at most on the tiny model."""
    name = "tts_topk40"
    res, trace, g = _run_oracle(name, CASES[name], kv_round_bf16=True)
    ref0 = g["trace_logits"][0]
    got0 = trace[0].reshape(-1, ref0.shape[-1]).numpy()
    live = ref0 > -9999
    assert np.abs(got0 - ref0)[live].max() < 5e-2


def test_oracle_reproduces_config1_prefix():
    """BASELINE.json configs[0] on the CPU oracle: the first sampled steps of the 323M / head_dim-64 utterance equal the
    unmodified reference's fixture (the full 254-step equality is asserted when the fixture is generated)."""
    import os
    import numpy as np
    import torch
    import golden_util as gu
    from oracle import lm_oracle
    from voicecraft_b200 import synthetic
    g = np.load(os.path.join(gu.GOLDEN, "lm_cfg1_330m.npz"))
    cfg = synthetic.make_config("330M")
    sd = gu.suppress_end_tokens(cfg, synthetic.make_state_dict(cfg, seed=0))
    x, xl, y = torch.from_numpy(g["x"]), torch.from_numpy(g["x_lens"]), torch.from_numpy(g["y"])
    n = 6
    rows = lm_oracle.OracleLM(cfg, sd).inference_tts(x, xl, y, silence_tokens=gu.SILENCE, noise_fn=gu.cpu_noise_fn(1),
                                                     max_steps=n, top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
    K, T = cfg.n_codebooks, y.shape[1]
    res = g["res"].astype(np.int64)[0]              # [K, T + G], un-delayed: frame t of codebook k was sampled at step t + k
    for k in range(K):
        assert np.array_equal(rows[k: n, k].numpy(), res[k, T: T + n - k]), k
