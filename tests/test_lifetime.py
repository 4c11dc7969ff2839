"""-m gpu: every device buffer, pinned buffer and event the library allocates belongs to the engine, stream or call that
made it, and is released by destroy (or by the call's return), including after a failed set-up.  Measured with the
process-wide counters vcb_counter(NULL, "live_bytes" / "live_handles"): each case must end exactly where it started."""
import ctypes as C
import gc

import pytest
import torch

from oracle import encodec_oracle as eo

pytestmark = pytest.mark.gpu


def _lib():
    from voicecraft_b200 import _lib
    return _lib, _lib.load()


def _live():
    gc.collect()
    torch.cuda.synchronize()
    _, lib = _lib()
    return lib.vcb_counter(None, b"live_bytes"), lib.vcb_counter(None, b"live_handles")


@pytest.fixture
def unchanged():
    """the live counts at the end of the test equal those at its start"""
    before = _live()
    yield before
    after = _live()
    assert after == before, f"live (bytes, handles): {before} before, {after} after"


def _tiny(seed=3):
    """tiny LM (head_dim 128) whose codebook 0 ends the utterance at once, so a call is a prefill plus the end cascade"""
    from voicecraft_b200 import synthetic
    from voicecraft_b200.voicecraft import VoiceCraft
    cfg = synthetic.make_config("tiny")
    sd = synthetic.make_state_dict(cfg, seed=seed)
    sd["predict_layer.0.2.bias"][cfg.eos] = 30.0
    m = VoiceCraft(cfg)
    m.load_state_dict(sd)
    return cfg, m.to("cuda:0").eval()


def _tts(m, cfg, batch_size=1):
    from voicecraft_b200 import synthetic
    x, xl, y = synthetic.synthetic_utterance(cfg, 21, text_len=12, prompt_frames=20)
    if batch_size == 1:
        return m.inference_tts(x.cuda(), xl, y.cuda(), top_k=40)
    return m.inference_tts_batch(x.cuda(), xl, y.cuda(), top_k=40, batch_size=batch_size)


def test_engine_create_finalize_destroy_three_times(unchanged):
    cfg, m = _tiny()
    for _ in range(3):
        m._engine()                      # vcb_create, vcb_load_weight of every tensor, vcb_load_pe, vcb_finalize_weights
        assert _live() != unchanged
        m._drop_engine()                 # vcb_destroy
        assert _live() == unchanged


@pytest.mark.parametrize("mode", ["mega_timeline", "profile"])
def test_voicecraft_rebuilds_and_drop_release_everything(mode, unchanged, monkeypatch):
    """inference_tts, a larger batch that grows the engine, configure_engine, another call -- then the model is dropped.
    mega_timeline: decode steps through the persistent kernel (VCB_MEGA=1) with its debug timeline recording; profile:
    the per-launch events of profile mode, read once."""
    _l, lib = _lib()
    if mode == "mega_timeline":
        monkeypatch.setenv("VCB_MEGA", "1")
    cfg, m = _tiny()

    def arm(eng):
        if mode == "mega_timeline":
            assert lib.vcb_counter(eng, b"mega_grid") > 0, "the persistent kernel is not set up"
            nph = C.c_int32()
            _l.check(lib.vcb_debug_mega_timeline(eng, None, 0, C.byref(nph)))
        else:
            _l.check(lib.vcb_set_option(eng, b"profile", 1))

    arm(m._engine())
    _tts(m, cfg)
    _tts(m, cfg, batch_size=9)           # more slots than the engine has: it is rebuilt larger
    arm(m._engine())
    _tts(m, cfg)
    m.configure_engine(max_seq_len=1024)
    eng = m._engine()
    arm(eng)
    _tts(m, cfg)
    if mode == "profile":
        ms, cnt = (C.c_double * 8)(), (C.c_int64 * 8)()
        _l.check(lib.vcb_profile_read(eng, ms, cnt, 8))
        assert sum(cnt) > 0
    del m, eng


def test_failed_finalize_then_destroy(unchanged):
    """a weight the finalize needs late (after the layers, the KV pools and the first heads) is missing"""
    from voicecraft_b200 import _lib as L
    cfg, m = _tiny()
    sd = {k: v for k, v in m.state_dict().items() if k != f"audio_embedding.{cfg.n_codebooks - 1}.word_embeddings.weight"}
    m.state_dict = lambda: sd
    with pytest.raises(L.VcbError, match="missing weight"):
        m._engine()                      # destroys the engine it failed to set up
    assert m._eng is None


def test_debug_hooks_release_their_buffers(unchanged):
    _l, lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(0)
    rnd = lambda *s: torch.randn(*s, generator=g).cuda()
    N = K = d = 256
    B = 4
    W, X, out = rnd(N, K), rnd(B, K), torch.empty(B, N, device="cuda")
    _l.check(lib.vcb_debug_gemm(W.data_ptr(), X.data_ptr(), out.data_ptr(), N, K, B, 0, 0))
    _l.check(lib.vcb_debug_gemm_rows(W.data_ptr(), X.data_ptr(), out.data_ptr(), N, K, B))
    # attention: 2 rows, 2 heads of 128, fp32 K / V pools [page][H][64][hd], pages listed per row
    H, hd = 2, 128
    q, Kp, Vp = rnd(2, H, hd), rnd(2, H, 64, hd), rnd(2, H, 64, hd)
    pages = torch.tensor([[0, 1], [1, 0]], dtype=torch.int32, device="cuda")
    pos = torch.tensor([10, 70], dtype=torch.int32, device="cuda")
    att = torch.empty(2, H * hd, device="cuda")
    _l.check(lib.vcb_debug_attention(q.data_ptr(), Kp.data_ptr(), Vp.data_ptr(), 1, pages.data_ptr(), None, None,
                                     pos.data_ptr(), 2, H, hd, 2, 1, 1, 1, att.data_ptr()))
    x, a, b1, gamma, beta, b2 = rnd(B, d), rnd(B, d), rnd(d), rnd(d), rnd(d), rnd(d)
    xn, y = torch.empty(B, d, device="cuda"), torch.empty(B, d, device="cuda")
    _l.check(lib.vcb_debug_fold_chain(x.data_ptr(), a.data_ptr(), W.data_ptr(), b1.data_ptr(), gamma.data_ptr(),
                                      beta.data_ptr(), W.data_ptr(), b2.data_ptr(), B, d, d, 0, 1, 0, 0, xn.data_ptr(),
                                      y.data_ptr()))
    # sampler: 2 rows of 3 codebooks over 2053 entries, top-k and top-p, noise drawn on the device
    V3 = 2053
    logits = rnd(2, 3, V3)
    sp = _l.vcb_sampling(top_k=40, top_p=0.8, temperature=1.0, stop_repetition=3, n_silence=0)
    state = (C.c_int32 * 14)(0, 0, 2, -1, 0, 1, 0, 1, 0, 2, -1, 0, 1, 0)
    tok, st_out = (C.c_int32 * 6)(), (C.c_int32 * 8)()
    _l.check(lib.vcb_debug_sampler(logits.data_ptr(), None, 5, 0, 256, C.byref(sp), 2, 3, V3, V3, V3 + 1, 0, 50, state, tok,
                                   st_out))
    assert all(0 <= t < V3 for t in tok)
    us = C.c_float()
    _l.check(lib.vcb_bench_gemm(N, K, B, 0, 0, 0, 3, 2, C.byref(us)))
    assert us.value > 0


def _tok(cfg, sd):
    from voicecraft_b200.tokenizer import AudioTokenizer
    return AudioTokenizer(device="cuda:0", config=cfg, state_dict=sd)


def _codes(cfg, B=2, T=40):
    return torch.randint(0, cfg.bins, (B, cfg.n_q, T), generator=torch.Generator().manual_seed(1)).cuda()


@pytest.mark.parametrize("tc", ["1", "0"])
def test_codec_decode_encode_and_drop(tc, unchanged, monkeypatch):
    """decode on the tensor-core decoder (or, VCB_CODEC_TC=0, the CUDA-core one, with its batch-chunk buffers) twice at
    a growing size, encode, then drop the tokenizer"""
    monkeypatch.setenv("VCB_CODEC_TC", tc)
    _, lib = _lib()
    cfg = eo.default_config()
    tok = _tok(cfg, eo.make_state_dict(cfg, seed=5, encoder=True))
    tok.decode_codes(_codes(cfg, 1, 20))
    wav = tok.decode_codes(_codes(cfg))
    assert lib.enc_counter(tok._engine(), b"tc_enabled") == int(tc)
    tok.encode_codes(wav[:, :, : 16 * tok.hop])
    del tok


def test_codec_refinalize_replaces_its_buffers(unchanged):
    _l, lib = _lib()
    cfg = eo.default_config()
    tok = _tok(cfg, eo.make_state_dict(cfg, seed=5, encoder=True))
    eng = tok._engine()                   # enc_create, enc_load_weight of every tensor, enc_finalize
    first = _live()
    _l.check(lib.enc_finalize(eng))
    assert _live() == first
    del tok, eng


def test_codec_stream_open_decode_reset_close(unchanged):
    cfg = eo.default_config()
    tok = _tok(cfg, eo.make_state_dict(cfg, seed=5))
    codes = _codes(cfg, 2, 12)
    with tok.open_stream(max_streams=3) as cs:
        cs.decode(codes)
        cs.reset([0])
        cs.decode(codes, ids=[0, 2])
    del tok
