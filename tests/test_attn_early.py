"""Decode attention's early start and live-token copies (VCB_ATT_EARLY, DESIGN.md sections 4.1 and 7) against the issue
order and whole-page copies of VCB_ATT_EARLY=0, bit for bit: the logits of every step, every layer's K / V bytes and the
tokens.  The knob moves when and which bytes the attention producer copies, never the order of a sum.

  * bf16 / fp32 / fp8 KV at head dim 128 and 64; 1, 17 and 32 rows whose positions pass pos % 64 in {0, 1, 62, 63},
    and a row past 4096 tokens (split-context merge)
  * the attention ring filled with NaN before every launch (VCB_ATT_POISON): the unwritten tail of the last page is
    never read
  * after a swap-out / swap-in, and a best-of-N group (the grouped attention kernel)
"""
import numpy as np
import pytest
import torch

from test_decode_knobs import _build, _decode, _differences, _lib, gpu

# prompts of 60 .. 63 positions reach pos % 64 = 62, 63, 0, 1 within the steps; 4158 crosses 4159 -> 4160 (65 pages, five
# 16-page chunks)
ROWS = [(62,), (60, 61, 62, 63, 4158) + tuple(30 + 5 * i for i in range(12)), tuple(40 + 3 * i for i in range(31)) + (63,)]
STEPS = 4
_MODELS = {}


def _model(nhead):
    """tiny (d 256, 2 layers) with head dim 256 / nhead, kept for the module"""
    if nhead not in _MODELS:
        import golden_util as gu
        from voicecraft_b200 import synthetic
        from voicecraft_b200.voicecraft import VoiceCraft
        cfg = synthetic.make_config("tiny", nhead=nhead)
        sd = gu.suppress_end_tokens(cfg, synthetic.make_state_dict(cfg, seed=83))
        m = VoiceCraft(cfg)
        m.load_state_dict(sd)
        _MODELS[nhead] = m.to("cuda").eval()
    return _MODELS[nhead]


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    yield
    _MODELS.clear()


def _run(m, kv, env, rows=ROWS):
    eng = _build(m, env, kv=kv, max_slots=32, max_seq_len=4608)
    _, lib = _lib()
    want = int(env.get("VCB_ATT_EARLY", 1))
    assert lib.vcb_counter(eng, b"att_early") == want and lib.vcb_counter(eng, b"mega_grid") == 0
    return _decode(m, eng, kv, rows, STEPS)


CASES = [(kv, nh) for kv in ("bf16", "fp32", "fp8") for nh in (2, 4)]


@gpu
@pytest.mark.parametrize("kv,nhead", CASES, ids=[f"kv={k}-hd={256 // n}" for k, n in CASES])
def test_early_start_is_bit_identical(kv, nhead):
    m = _model(nhead)
    base = _run(m, kv, {"VCB_ATT_EARLY": 0})
    diff = _differences(base, _run(m, kv, {}))
    assert not diff, diff[:4]


@gpu
@pytest.mark.parametrize("kv", ["bf16", "fp8"])
def test_uncopied_tail_is_never_read(kv):
    """NaN in every ring byte the producer does not overwrite: a read of the last page's unwritten tail would put NaN into
    the scores or PV and so into the logits"""
    m = _model(2)
    base = _run(m, kv, {"VCB_ATT_EARLY": 0})
    poisoned = _run(m, kv, {"VCB_ATT_POISON": 1})
    diff = _differences(base, poisoned)
    assert not diff, diff[:4]
    assert all(torch.isfinite(t).all() for r in poisoned for t in r["logits"])


@gpu
def test_swap_in_then_early_start():
    """an utterance swapped out mid-page and into another slot, decoded with the early start, equals the uninterrupted
    run with VCB_ATT_EARLY=0"""
    import test_kv_pool as kp
    from voicecraft_b200.voicecraft import _Prompt
    out = []
    for env, swap in (({"VCB_ATT_EARLY": "0"}, False), ({}, True)):
        with pytest.MonkeyPatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            cfg, m = kp._lm("bf16", "bf16", 2, max_slots=4, max_seq_len=512)
            x, _, y = kp._utt(cfg, 12, 20, 100)
            if swap:
                filler = kp._utt(cfg, 13, 9, 150)
                out.append(kp._drive(m, cfg, x, y, None, swap_at=lambda i, st, seq: i == 40,
                                     filler=_Prompt(m, filler[0], filler[2])))
            else:
                out.append(kp._drive(m, cfg, x, y, None))
            assert _lib()[1].vcb_counter(m._engine(), b"att_early") == (1 if swap else 0)
    kp._same(out[1], out[0])


def _best_of(m, n, steps):
    """logits of every sampling step and the tokens of every copy of one best-of-n group"""
    import test_decode_knobs as dk
    from voicecraft_b200.voicecraft import DecodeSession
    _l, lib = _lib()
    x, y = dk._utts(m.args, (126,), 77)[0]          # one shared full page, the private one crosses 128
    sess = DecodeSession(m, [x], [y], m._sampling(**dk.SP), seeds=[5], best_of=n)
    rows_n = n * m.args.n_codebooks
    logits = []
    try:
        for s in range(steps + 1):
            sess.sample() if s == 0 else sess.step()
            t = torch.empty(rows_n, m.n_audio_tokens[0], device="cuda")
            _l.check(lib.vcb_debug_logits(sess.eng, t.data_ptr(), rows_n))
            logits.append(t)
        sess.poll()
        toks = [np.asarray(sess.raw_tokens(0))]
    finally:
        sess.close()
    return logits, toks


@gpu
def test_best_of_group_early_start():
    """a best-of-5 group (grouped attention: the shared prompt page read once, private pages per member) across the page
    boundary at 128"""
    m = _model(2)
    got = []
    for env in ({"VCB_ATT_EARLY": 0}, {}):
        eng = _build(m, env, kv="bf16", max_slots=8, max_seq_len=512)
        assert _lib()[1].vcb_counter(eng, b"att_early") == int(env.get("VCB_ATT_EARLY", 1))
        got.append(_best_of(m, 5, 6))
    (la, ta), (lb, tb) = got
    assert all(torch.equal(p, q) for p, q in zip(la, lb))
    assert all(np.array_equal(p, q) for p, q in zip(ta, tb))
