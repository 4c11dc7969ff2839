"""-m gpu: the CUDA path (through the C ABI) against the golden fixtures of the real reference and the CPU oracle.

Numerics policy under test: GEMM weights bf16 (the synthetic checkpoints are bf16-representable, so
the fp32 reference saw the same weights), activations split hi+lo bf16 (>= 16 mantissa bits), fp32 accumulation
and fp32 everywhere else.  With kv_dtype=fp32 the engine follows the unmodified reference; with the default
bf16 KV cache it follows the oracle's kv_round_bf16 policy.  Token ids must be IDENTICAL; raw logits agree to
1e-3 absolute (fp32 summation-order noise is ~1e-5).
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import golden_util as gu

pytestmark = pytest.mark.gpu
CASES = gu.load_cases()
LOGIT_TOL = 2e-3

def _case_params(names):
    return list(names)


def _model(cfg, sd, kv="fp32"):
    from voicecraft_b200.voicecraft import VoiceCraft
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    m = m.to("cuda").eval()
    m.configure_engine(kv_dtype=kv, max_slots=8, max_seq_len=512)
    return m


@pytest.mark.parametrize("simt", [1, 0])
@pytest.mark.parametrize("shape", [(256, 256, 4), (768, 256, 32), (2052, 1024, 32), (1024, 4096, 128), (6144, 2048, 7)])
def test_gemm_wgmma_vs_fp32(shape, simt):
    """Bring-up check of the wgmma/TMA GEMM (and its CUDA-core cross-check twin) against torch fp32: the engine's split
    count (0) and every split count the kernel accepts for the shape."""
    from voicecraft_b200 import _lib
    lib = _lib.load()
    N, K, B = shape
    g = torch.Generator(device="cpu").manual_seed(N + K + B)
    W = torch.randn(N, K, generator=g).to(torch.bfloat16).float().cuda()
    X = torch.randn(B, K, generator=g).cuda()
    ref = (X.double() @ W.double().t()).float()
    scale = ref.abs().max().item()
    bpad = 16 if B <= 16 else 32 if B <= 32 else 64 if B <= 64 else 128
    kb = K // 64
    legal = [s for s in (1, 2, 4, 8) if bpad % s == 0 and bpad // s >= 2 and (s - 1) * ((kb + s - 1) // s) < kb]
    for splits in [0] + ([] if simt else legal):
        out = torch.zeros(B, N, device="cuda")
        _lib.check(lib.vcb_debug_gemm(W.data_ptr(), X.data_ptr(), out.data_ptr(), N, K, B, splits, simt))
        err = (out - ref).abs().max().item()
        assert err <= 2e-4 * max(scale, 1.0), f"shape={shape} simt={simt} splits={splits} err={err} scale={scale}"


def _run_case(name, case, kv):
    cfg, sd, x, x_lens, y, g = gu.build_case(name, case)
    m = _model(cfg, sd, kv)
    m.noise_fn = gu.cpu_noise_fn(case["seed"])
    m.trace_logits = []
    kw = dict(case["kw"], silence_tokens=gu.SILENCE, kvcache=1)
    if case["kind"] == "tts":
        res, gen = m.inference_tts(x.cuda(), x_lens.cuda(), y.cuda(), **kw)
    elif case["kind"] == "batch":
        res, gen = m.inference_tts_batch(x.cuda(), x_lens.cuda(), y.cuda(), batch_size=case["batch_size"], **kw)
    else:
        res = m.inference(x.cuda(), x_lens.cuda(), y.cuda(), torch.from_numpy(g["mask_interval"]).cuda(), **kw)
    return res, m.trace_logits, g


@pytest.mark.parametrize("name", _case_params(sorted(CASES)))
def test_tokens_match_reference_fixture_kv_fp32(name):
    res, trace, g = _run_case(name, CASES[name], "fp32")
    # logits first: a numerical bug shows up here before it flips a token
    for step, ref in zip(g["trace_steps"], g["trace_logits"]):
        got = trace[int(step)].cpu().numpy()
        live = ref > -9999          # the fixture holds post-edit logits (-10000 writes), ours are pre-edit
        diff = np.abs(got - ref)[live]
        bad = int((diff > LOGIT_TOL).sum())
        assert bad <= 1, f"step {step}: {bad} logits off by > {LOGIT_TOL} (max {diff.max()})"   # <=1: silence penalty slot
    assert len(trace) == int(g["n_steps"])
    assert np.array_equal(res.cpu().numpy(), g["res"]), "token ids differ from the reference fixture"


@pytest.mark.parametrize("name", ["tts_topk40", "tts_topp", "edit2", "batch3"])
def test_tokens_match_oracle_kv_bf16(name):
    """Default engine policy (bf16 paged KV) against the oracle with the same rounding."""
    from oracle import lm_oracle
    case = CASES[name]
    cfg, sd, x, x_lens, y, g = gu.build_case(name, case)
    oracle = lm_oracle.OracleLM(cfg, sd, kv_round_bf16=True)
    kw = dict(case["kw"], silence_tokens=gu.SILENCE, kvcache=1, noise_fn=gu.cpu_noise_fn(case["seed"]))
    if case["kind"] == "tts":
        ores = oracle.inference_tts(x, x_lens, y, **kw)[0]
    elif case["kind"] == "batch":
        ores = oracle.inference_tts_batch(x, x_lens, y, batch_size=case["batch_size"], **kw)[0]
    else:
        ores = oracle.inference(x, x_lens, y, torch.from_numpy(g["mask_interval"]), **kw)
    res, _, _ = _run_case(name, case, "bf16")
    assert np.array_equal(res.cpu().numpy(), ores.numpy())


@pytest.mark.parametrize("numel,offset", [(4 * 2052, 0), (5 * 4 * 2052, 4), (32 * 4 * 2052, 40), (8 * 2051, 12), (1_500_000, 8), (7, 0)])
def test_device_exponential_is_bit_identical_to_torch(numel, offset):
    """The sampler's in-kernel Exp(1) generator (Philox4x32-10 + ATen's exponential transform) against
    torch.empty(numel, device='cuda').exponential_(1) at the same (seed, offset): bit-identical, and torch's generator
    advanced by exactly the offset the engine accounts per draw."""
    from voicecraft_b200 import _lib
    from voicecraft_b200.voicecraft import VoiceCraft
    lib = _lib.load()
    seed = 0x1234ABCD5678 + numel
    gen = torch.cuda.default_generators[0]
    torch.manual_seed(seed)
    gen.set_offset(offset)
    ref = torch.empty(numel, device="cuda").exponential_(1)
    advanced = gen.get_offset() - offset
    threads = VoiceCraft._rng_threads(torch.device("cuda", 0), numel)
    out = torch.zeros(numel, device="cuda")
    _lib.check(lib.vcb_debug_exponential(out.data_ptr(), numel, seed, offset, threads, None))
    torch.cuda.synchronize()
    assert torch.equal(out, ref), f"{int((out != ref).sum())} of {numel} values differ"
    assert advanced == ((numel - 1) // (4 * threads) + 1) * 4


def test_per_utterance_streams_batch_rows_equal_single_calls():
    """SURVEY.md section 7 'RNG parity': one generator per utterance.  Row i of a sampled (top-k 40) batch of 8 equals
    `torch.manual_seed(s_i); inference_tts(utterance i)` -- what the reference does per call
    (inference_tts_scale.py:128-135, voicecraft.py:85) -- and the default generator is left where the single call leaves it."""
    from voicecraft_b200 import synthetic
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=44)
    sd["predict_layer.0.2.bias"][cfg.eos] += 4.0
    m = _model(cfg, sd, "bf16")
    m.configure_engine(max_slots=8, max_seq_len=512, kv_dtype="bf16")
    utts = [synthetic.synthetic_utterance(cfg, 600 + i, text_len=4 + i % 3, prompt_frames=12 + 5 * i) for i in range(8)]
    seeds = [900 + 17 * i for i in range(8)]
    kw = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
    singles, offsets = [], []
    for (x, xl, y), sd_i in zip(utts, seeds):
        torch.manual_seed(sd_i)
        singles.append(m.inference_tts(x.cuda(), xl.cuda(), y.cuda(), **kw)[0])
        offsets.append(torch.cuda.default_generators[0].get_offset())
        assert offsets[-1] == 4 * m.last_stats["steps"]          # one [K,V] draw per sampling step, as the reference
    many = m.inference_tts_many([u[0] for u in utts], [u[2] for u in utts], seeds=seeds, poll_every=3, **kw)
    assert len({tuple(s.shape) for s in singles}) > 1, "utterances should end at different lengths"
    for i, (a, (b, _)) in enumerate(zip(singles, many)):
        assert torch.equal(a, b), f"utterance {i}: batched row differs from its single call"


def test_per_utterance_noise_batch_rows_equal_oracle():
    """Same statement against the CPU oracle: utterance i of a sampled batch, fed the CPU-generator noise of seed s_i,
    equals the oracle's (= the reference algorithm's) inference_tts of utterance i under that seed."""
    from oracle import lm_oracle
    from voicecraft_b200 import synthetic
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=45)
    sd["predict_layer.0.2.bias"][cfg.eos] += 4.0
    utts = [synthetic.synthetic_utterance(cfg, 700 + i, text_len=4 + i % 3, prompt_frames=10 + 4 * i) for i in range(8)]
    kw = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
    oracle = lm_oracle.OracleLM(cfg, sd)
    refs = [oracle.inference_tts(x, xl, y, silence_tokens=gu.SILENCE, noise_fn=gu.cpu_noise_fn(50 + i), **kw)[0]
            for i, (x, xl, y) in enumerate(utts)]
    m = _model(cfg, sd, "fp32")
    many = m.inference_tts_many([u[0] for u in utts], [u[2] for u in utts], poll_every=1,
                                noise_fns=[gu.cpu_noise_fn(50 + i) for i in range(8)], **kw)
    for i, (r, (b, _)) in enumerate(zip(refs, many)):
        assert np.array_equal(b.cpu().numpy(), r.numpy()), f"utterance {i}"


def test_generator_stream_matches_torch_multinomial_on_device():
    """Default noise path: the sampler consumes the CUDA generator's Philox stream exactly as torch.multinomial's
    exponential_ draw would.  Same seed twice -> same tokens; and the generator advanced by one draw per step."""
    name = "tts_topk40"
    case = CASES[name]
    cfg, sd, x, x_lens, y, g = gu.build_case(name, case)
    m = _model(cfg, sd, "bf16")
    kw = dict(case["kw"], silence_tokens=gu.SILENCE)
    torch.manual_seed(5)
    a = m.inference_tts(x.cuda(), x_lens.cuda(), y.cuda(), **kw)[0]
    after = torch.empty(4, device="cuda").exponential_(1)
    torch.manual_seed(5)
    b = m.inference_tts(x.cuda(), x_lens.cuda(), y.cuda(), **kw)[0]
    assert torch.equal(a, b)
    # replay the same number of draws by hand
    torch.manual_seed(5)
    K, V = cfg.n_codebooks, 2048 + cfg.n_special
    for _ in range(m.last_stats["steps"]):
        torch.empty(K, V, device="cuda").exponential_(1)
    assert torch.equal(after, torch.empty(4, device="cuda").exponential_(1))


def test_bpad32_best_of_20_matches_oracle():
    """Best-of-20 on the 512-d model: 20 rows -> Bpad 32 (UMMA N = 64; the fixtures only reach Bpad 16).  Oracle with the
    same rounding policy and the same noise."""
    from oracle import lm_oracle
    from voicecraft_b200 import synthetic
    cfg = synthetic.make_config("small")
    sd = synthetic.make_state_dict(cfg, seed=31)
    x, x_lens, y = synthetic.synthetic_utterance(cfg, 77, text_len=4, prompt_frames=10)
    kw = dict(top_k=30, top_p=0.9, temperature=1.0, stop_repetition=3, silence_tokens=gu.SILENCE, kvcache=1)
    ores = lm_oracle.OracleLM(cfg, sd, kv_round_bf16=True).inference_tts_batch(
        x, x_lens, y, batch_size=20, noise_fn=gu.cpu_noise_fn(3), **kw)[0]
    m = _model(cfg, sd, "bf16")
    m.configure_engine(max_slots=24, max_seq_len=512, kv_dtype="bf16")
    m.noise_fn = gu.cpu_noise_fn(3)
    res = m.inference_tts_batch(x.cuda(), x_lens.cuda(), y.cuda(), batch_size=20, **kw)[0]
    assert np.array_equal(res.cpu().numpy(), ores.numpy())


def test_batched_sessions_match_single_calls():
    """inference_tts_many / inference_many (independent utterances in one batch) return, row by row, what the reference-shaped
    single calls return when each row is fed the same noise rows."""
    from voicecraft_b200 import synthetic
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=41)
    sd["predict_layer.0.2.bias"][cfg.eog] += 3.0
    m = _model(cfg, sd, "bf16")
    K, V = cfg.n_codebooks, 2048 + cfg.n_special
    utts = [synthetic.synthetic_utterance(cfg, 500 + i, text_len=5 + i, prompt_frames=30 + 3 * i) for i in range(3)]
    spans = [torch.tensor([[[5, 9]]]), torch.tensor([[[4, 8], [15, 20]]]), torch.tensor([[[10, 12]]])]
    kw = dict(top_k=1, top_p=1.0, temperature=1.0)      # greedy: independent of how noise rows are batched
    singles_tts = [m.inference_tts(x.cuda(), xl.cuda(), y.cuda(), stop_repetition=3, **kw)[0] for x, xl, y in utts]
    many_tts = m.inference_tts_many([u[0] for u in utts], [u[2] for u in utts], poll_every=1, stop_repetition=3, **kw)
    for a, (b, _) in zip(singles_tts, many_tts):
        assert torch.equal(a, b)
    singles_ed = [m.inference(x.cuda(), xl.cuda(), y.cuda(), sp.cuda(), **kw) for (x, xl, y), sp in zip(utts, spans)]
    many_ed = m.inference_many([u[0] for u in utts], [u[2] for u in utts], spans, poll_every=1, **kw)
    for a, b in zip(singles_ed, many_ed):
        assert torch.equal(a, b)


def test_capacity_exhaustion_is_reported():
    from voicecraft_b200 import synthetic, _lib
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=42)
    end = cfg.eos
    sd["predict_layer.0.2.bias"][end] = -1e4
    m = _model(cfg, sd, "bf16")
    m.configure_engine(max_new_tokens=16, max_seq_len=512)
    x, xl, y = synthetic.synthetic_utterance(cfg, 9, text_len=8, prompt_frames=10)
    with pytest.raises(_lib.VcbError):
        m.inference_tts(x.cuda(), xl.cuda(), y.cuda(), top_k=10)


@pytest.mark.parametrize("wide", ["0", "1"])
def test_full_size_830M_first_steps_match_oracle(wide, monkeypatch):
    """BASELINE.json configs[1] at full size (giga830M: d=2048, 16 layers, 16 heads, K=4): prefill + the first sampling
    steps of one utterance, CUDA path (fp32 KV) vs the CPU oracle on the same synthetic checkpoint and the same Exp(1)
    noise.  Token ids identical, raw logits within LOGIT_TOL.  (Long generations at this size are covered by the
    size-independent checks: batched == single, generator stream, and scripts/parity_rate.py.)"""
    from oracle import lm_oracle
    from voicecraft_b200 import synthetic
    monkeypatch.setenv("VCB_PREFILL_WIDE", wide)       # prompt through the narrow (0) / rows-as-M (1) prefill GEMM
    n_steps = 24
    cfg = synthetic.make_config("830M")
    sd = synthetic.make_state_dict(cfg, seed=3)
    x, x_lens, y = synthetic.synthetic_utterance(cfg, 4242, 16, 24)
    kw = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3, silence_tokens=gu.SILENCE)
    torch.set_num_threads(max(1, min(16, torch.get_num_threads())))
    oracle = lm_oracle.OracleLM(cfg, sd)
    ref_rows = oracle.inference_tts(x, x_lens, y, noise_fn=gu.cpu_noise_fn(11), max_steps=n_steps, trace_logits=True, **kw)
    assert ref_rows.shape == (n_steps, cfg.n_codebooks), "the synthetic checkpoint must not end within the first steps"
    ref_trace = [t.numpy() for t in oracle.logit_trace]
    del oracle

    m = _model(cfg, sd, kv="fp32")
    m.noise_fn = gu.cpu_noise_fn(11)
    sess = m.open_tts_session([x.cuda()], [y.cuda()], **kw)
    try:
        sess.sample()
        t = torch.empty(cfg.n_codebooks, m.n_audio_tokens[0], device="cuda")
        lib = sess.lib
        traces = []
        def grab():
            from voicecraft_b200 import _lib
            _lib.check(lib.vcb_debug_logits(sess.eng, t.data_ptr(), cfg.n_codebooks))
            traces.append(t.cpu().numpy().copy())
        grab()
        for _ in range(n_steps - 1):
            sess.step()
            grab()
        rows = sess.raw_tokens(0)
    finally:
        sess.close()
    worst = 0.0
    for got, ref in zip(traces, ref_trace):
        live = ref > -9999
        worst = max(worst, float(np.abs(got - ref)[live].max()))
    assert worst <= LOGIT_TOL, f"max |logit - oracle| = {worst}"
    assert np.array_equal(rows[:n_steps], ref_rows.numpy()), "token ids differ from the oracle at full size"


@pytest.mark.parametrize("shape", [(256, 256, 40), (768, 256, 300), (1024, 4096, 1000), (6144, 2048, 513), (384, 512, 129)])
def test_gemm_rows_vs_fp32(shape):
    """Rows-as-M wgmma GEMM of the wide prefill path (csrc/gemm_rows.cu) against torch fp64: 256-wide tiles (even number
    of 128-feature blocks), 128-wide tiles (odd: 384), ragged last row tile."""
    from voicecraft_b200 import _lib
    lib = _lib.load()
    N, K, R = shape
    g = torch.Generator(device="cpu").manual_seed(N + K + R)
    W = torch.randn(N, K, generator=g).to(torch.bfloat16).float().cuda()
    X = torch.randn(R, K, generator=g).cuda()
    out = torch.zeros(R, N, device="cuda")
    _lib.check(lib.vcb_debug_gemm_rows(W.data_ptr(), X.data_ptr(), out.data_ptr(), N, K, R))
    ref = (X.double() @ W.double().t()).float()
    err = (out - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 2e-4 * max(scale, 1.0), f"shape={shape} err={err} scale={scale}"


@pytest.mark.parametrize("name", ["tts_topk40", "batch3", "edit2"])
def test_wide_prefill_matches_reference_fixture(name, monkeypatch):
    """VCB_PREFILL_WIDE=1: the whole prompt goes through the rows-as-M GEMM path; tokens must still equal the reference's."""
    monkeypatch.setenv("VCB_PREFILL_WIDE", "1")
    res, trace, g = _run_case(name, CASES[name], "fp32")
    for step, ref in zip(g["trace_steps"], g["trace_logits"]):
        got = trace[int(step)].cpu().numpy()
        live = ref > -9999
        diff = np.abs(got - ref)[live]
        assert int((diff > LOGIT_TOL).sum()) <= 1, f"step {step}: max {diff.max()}"
    assert np.array_equal(res.cpu().numpy(), g["res"]), "token ids differ from the reference fixture"


def test_wide_prefill_bf16_kv_matches_oracle(monkeypatch):
    """Default KV policy (bf16 pages) with the prompt going through the rows-as-M GEMM: its vectorised bf16 KV append must
    round exactly like the oracle's kv_round_bf16 policy."""
    from oracle import lm_oracle
    monkeypatch.setenv("VCB_PREFILL_WIDE", "1")
    name = "tts_topk40"
    case = CASES[name]
    cfg, sd, x, x_lens, y, g = gu.build_case(name, case)
    oracle = lm_oracle.OracleLM(cfg, sd, kv_round_bf16=True)
    kw = dict(case["kw"], silence_tokens=gu.SILENCE, kvcache=1, noise_fn=gu.cpu_noise_fn(case["seed"]))
    ores = oracle.inference_tts(x, x_lens, y, **kw)[0]
    res, _, _ = _run_case(name, case, "bf16")
    assert np.array_equal(res.cpu().numpy(), ores.numpy())



# ==========================================================================================================================
# Headline shape (BASELINE.json configs[1]): giga830M, B = 32 independent utterances, K = 4, top-k 40 sampling, one random
# stream per utterance.  Fixtures: tests/golden/lm_830m_b32.* (make_golden_830m.py: the oracle, pinned to the unmodified
# reference on two full-length 830M utterances).  64 decode steps; contexts 191..541 cross KV-page boundaries, 256 and 512.
# ==========================================================================================================================
SENS_TOL = {"fp32": 1e-4, "bf16": LOGIT_TOL}    # a token may differ only where a logit move of this size can change it


def _headline_run(kv):
    meta, g = gu.headline_fixture()
    cfg, sd = gu.headline_checkpoint(meta["ckpt_seed"])
    N = meta["n_steps"]
    m = _model(cfg, sd, kv)
    m.configure_engine(max_slots=32, max_seq_len=1024, kv_dtype=kv, max_new_tokens=128)
    utts = [gu.headline_utterance(cfg, meta, i) for i in range(32)]
    sess = m.open_tts_session([u[0] for u in utts], [u[2] for u in utts], noise_fns=[gu.cpu_noise_fn(1 + i) for i in range(32)],
                              silence_tokens=gu.SILENCE, **meta["kw"])
    K, V = cfg.n_codebooks, m.n_audio_tokens[0]
    t = torch.empty(32 * K, V, device="cuda")
    logits = {}
    try:
        from voicecraft_b200 import _lib
        for step in range(N):
            sess.sample() if step == 0 else sess.step()
            if step in meta["trace_steps"]:
                _lib.check(sess.lib.vcb_debug_logits(sess.eng, t.data_ptr(), 32 * K))
                logits[step] = t.cpu().numpy().reshape(32, K, V).copy()
        rows = np.stack([sess.raw_tokens(i)[:N] for i in range(32)])
    finally:
        sess.close()
    return meta, g, rows, logits


@pytest.mark.parametrize("kv", ["fp32", "bf16"])
def test_headline_830M_b32_matches_oracle(kv):
    """Token ids of all 32 utterances over 64 sampled steps against the oracle under the same KV policy.
    fp32 KV (the reference's arithmetic): identical, full stop.  bf16 KV pages (the benchmarked policy; oracle
    kv_round_bf16=True): every K/V element is rounded to bf16 from an fp32 value that differs from the CPU's in its last
    bits (a 2^-9 relative jump when the rounding goes the other way), so logits carry ~1e-3 of noise and a sample can
    legitimately change where that is enough to (i) swap the two best p/q scores, (ii) push the winner out of the top-k,
    or (iii) let an excluded token into the top-k that then wins.  The fixture stores, per sample, the smallest such logit
    move (`sens`, make_golden_830m.py).  Required: (a) raw logits within LOGIT_TOL of the oracle on the traced steps of
    still-identical utterances, (b) every utterance identical up to its first differing sample, and that sample's
    sensitivity below SENS_TOL, (c) at least 24 of 32 utterances identical throughout."""
    meta, g, rows, logits = _headline_run(kv)
    ref = g[f"rows_{kv}"].astype(np.int64)
    margin = g[f"sens_{kv}"]
    identical, first_div = 0, {}
    for i in range(32):
        neq = np.argwhere(rows[i] != ref[i])
        if len(neq) == 0:
            identical += 1
            continue
        s, k = (int(v) for v in neq[0])              # argwhere is row-major: first differing step, then codebook
        first_div[i] = (s, k, float(margin[i, s, k]))
    worst = 0.0
    for ui, u in enumerate(meta["trace_utts"]):
        for si, s in enumerate(meta["trace_steps"]):
            if u in first_div and first_div[u][0] < s:
                continue                              # inputs differ after a divergence: logits are no longer comparable
            refl = g[f"logits_{kv}"][ui, si]
            live = refl > -9999
            worst = max(worst, float(np.abs(logits[s][u] - refl)[live].max()))
    print(f"kv={kv}: {identical}/32 identical, divergences {first_div}, max |logit - oracle| {worst:.3g}")
    assert worst <= LOGIT_TOL, f"max |logit - oracle| = {worst}"
    for i, (s, k, mg) in first_div.items():
        assert mg < SENS_TOL[kv], f"utterance {i} differs at step {s} codebook {k} where the oracle's decision is robust to {mg:.3g}"
    # 109 of the 8192 bf16-policy samples sit within SENS_TOL of a flip; with ~1e-3 of logit noise a handful of them may go
    # the other way.  More than 8 divergent utterances would mean noise well above that.
    assert identical >= (32 if kv == "fp32" else 24), f"{identical}/32 utterances token-identical ({first_div})"


@pytest.mark.parametrize("j", [0, 1])
def test_headline_830M_reference_pinned_utterance(j):
    """The UNMODIFIED reference's inference_tts at full size (fixture pin{j}_res, generation ended by the reference's own
    length cap incl. the K-step end cascade) against the CUDA path with fp32 KV and the same CPU-generator noise."""
    meta, g = gu.headline_fixture()
    from voicecraft_b200 import synthetic
    cfg, sd = gu.headline_checkpoint(meta["pinned_ckpt_seed"])
    pc = meta["pinned"][j]
    x, xl, y = synthetic.synthetic_utterance(cfg, 7000 + j, pc["text_len"], pc["prompt"])
    m = _model(cfg, sd, "fp32")
    m.noise_fn = gu.cpu_noise_fn(pc["seed"])
    res = m.inference_tts(x.cuda(), xl.cuda(), y.cuda(), silence_tokens=gu.SILENCE, **meta["kw"])[0]
    assert np.array_equal(res.cpu().numpy(), g[f"pin{j}_res"].astype(np.int64)), "token ids differ from the reference at 830M"


def test_config1_330M_head_dim_64_matches_reference():
    """BASELINE.json configs[0] (SURVEY.md section 8d config 1): 323M stand-in, d=1024, 24 layers, 16 heads -> head_dim 64,
    one utterance, 3 s prompt -> 5 s generated (250 frames + the K-step end cascade), top-k 40, seed 1.  The fixture is
    the UNMODIFIED reference's output (tests/golden/make_golden_cfg1.py); fp32 KV, same CPU-generator noise.
    head_dim 64 takes the per-kernel decode path (attn_rows_kernel<*, 64>, d=1024 GEMM shapes)."""
    from voicecraft_b200 import synthetic
    g = np.load(os.path.join(gu.GOLDEN, "lm_cfg1_330m.npz"))
    cfg = synthetic.make_config("330M")
    sd = gu.suppress_end_tokens(cfg, synthetic.make_state_dict(cfg, seed=0))
    x, xl, y = torch.from_numpy(g["x"]), torch.from_numpy(g["x_lens"]), torch.from_numpy(g["y"])
    m = _model(cfg, sd, "fp32")
    m.noise_fn = gu.cpu_noise_fn(1)
    m.trace_logits = []
    res = m.inference_tts(x.cuda(), xl.cuda(), y.cuda(), silence_tokens=gu.SILENCE, top_k=40, top_p=1.0, temperature=1.0,
                          stop_repetition=3)[0]
    for step, ref in zip(g["trace_steps"], g["trace_logits"]):
        got = m.trace_logits[int(step)].cpu().numpy()
        live = ref > -9999
        assert float(np.abs(got - ref)[live].max()) <= LOGIT_TOL, f"step {step}"
    assert len(m.trace_logits) == int(g["n_steps"])
    assert np.array_equal(res.cpu().numpy(), g["res"].astype(np.int64)), "token ids differ from the reference on config 1"


def test_continuous_batching_equals_single_calls():
    """SURVEY.md section 8f row f2: 10 utterances of different lengths through 4 slots with refill-on-finish; every result
    equals `torch.manual_seed(seed_i); inference_tts(utterance i)`."""
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import ContinuousBatcher
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=46)
    sd["predict_layer.0.2.bias"][cfg.eos] += 4.5
    m = _model(cfg, sd, "bf16")
    utts = [synthetic.synthetic_utterance(cfg, 800 + i, text_len=3 + i % 4, prompt_frames=8 + 6 * (i % 5)) for i in range(10)]
    seeds = [300 + 7 * i for i in range(10)]
    kw = dict(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3)
    singles = []
    for (x, xl, y), s in zip(utts, seeds):
        torch.manual_seed(s)
        singles.append(m.inference_tts(x.cuda(), xl.cuda(), y.cuda(), **kw)[0])
    cb = ContinuousBatcher(m, max_concurrency=4, poll_every=3, **kw)
    for (x, xl, y), s in zip(utts, seeds):
        cb.submit(x, y, seed=s)
    out = cb.run()
    assert cb.stats["prefills"] >= 3 and cb.stats["max_active"] == 4
    for i, (a, (b, _)) in enumerate(zip(singles, out)):
        assert torch.equal(a, b), f"utterance {i}"


# ==========================================================================================================================
# The persistent decode-step kernel (csrc/mega_step.cu, opt-in: VCB_MEGA=1) against the same fixtures / oracle.
# ==========================================================================================================================
@pytest.mark.parametrize("name", ["tts_topk40", "tts_small", "batch3", "batch2_k8", "edit2", "edit3_noeos"])
def test_persistent_kernel_matches_reference_fixture(name, monkeypatch):
    monkeypatch.setenv("VCB_MEGA", "1")
    res, trace, g = _run_case(name, CASES[name], "fp32")
    for step, ref in zip(g["trace_steps"], g["trace_logits"]):
        got = trace[int(step)].cpu().numpy()
        live = ref > -9999
        diff = np.abs(got - ref)[live]
        assert int((diff > LOGIT_TOL).sum()) <= 1, f"step {step}: max {diff.max()}"
    assert np.array_equal(res.cpu().numpy(), g["res"]), "token ids differ from the reference fixture"


@pytest.mark.parametrize("kv", ["fp32", "bf16"])
def test_persistent_kernel_headline_830M_b32(kv, monkeypatch):
    """Same requirement as test_headline_830M_b32_matches_oracle, decode steps through the persistent kernel."""
    monkeypatch.setenv("VCB_MEGA", "1")
    test_headline_830M_b32_matches_oracle(kv)


def test_persistent_kernel_rows_do_not_depend_on_the_batch(monkeypatch):
    monkeypatch.setenv("VCB_MEGA", "1")
    test_per_utterance_streams_batch_rows_equal_single_calls()
