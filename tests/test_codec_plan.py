"""The tensor-core EnCodec layer plans (-m gpu).  Decoder: launch counts of a decode and of a stream decode, the carried
state per stream, the frames a fresh stream needs, and the tensors enc_debug_tensor exposes, with their dims.  The values
were recorded on an H100 from the decoder as it was before its host side was driven by one plan; they pin the launches,
the stream-state layout and min_T of every configuration below.  Encoder: see test_encoder_plan_pinned."""
import ctypes as C
import json
import os

import pytest
import torch

from oracle import encodec_oracle as eo
from test_encode_numerics import ENC_CONFIGS, enc_tensors, min_accepted
from test_encode_numerics import hop as enc_hop

SMALL = dict(n_filters=8, dimension=32, bins=64)
B, T = 4, 100                 # one enc_decode
SB, ST = 3, 12                # one enc_stream_decode: the first push of SB fresh streams

# enc_debug_tensor name -> (C, halo + rows, halo) after a decode of B x T frames (dims[0] is the chunk's utterances)
DEFAULT_DBG = {
    "z": (128, 106, 6), "x0": (1024, 100, 0), "hs0": (1024, 101, 1), "hs1": (1024, 101, 1), "u0": (1024, 101, 1),
    "x1.elu": (512, 802, 2), "x1.raw": (512, 802, 2), "h1.0": (256, 802, 2), "o1.0": (512, 801, 1),
    "x2.elu": (256, 4002, 2), "x2.raw": (256, 4002, 2), "h2.0": (128, 4002, 2), "o2.0": (256, 4001, 1),
    "x3.elu": (128, 16002, 2), "x3.raw": (128, 16002, 2), "h3.0": (64, 16002, 2), "o3.0": (128, 16001, 1),
    "x4.elu": (64, 32002, 2), "x4.raw": (64, 32002, 2), "h4.0": (64, 32002, 2), "o4.0": (64, 32006, 6),
}
SMALL_STAGES = {
    "x1.elu": (64, 802, 2), "x1.raw": (64, 802, 2), "h1.0": (64, 802, 2), "o1.0": (64, 801, 1),
    "x2.elu": (64, 4002, 2), "x2.raw": (64, 4002, 2), "h2.0": (64, 4002, 2), "o2.0": (64, 4001, 1),
    "x3.elu": (64, 16002, 2), "x3.raw": (64, 16002, 2), "h3.0": (64, 16002, 2), "o3.0": (64, 16001, 1),
    "x4.elu": (64, 32002, 2), "x4.raw": (64, 32002, 2), "h4.0": (64, 32002, 2), "o4.0": (64, 32006, 6),
}
SMALL_LSTM2_DBG = dict(SMALL_STAGES, z=(64, 106, 6), x0=(128, 100, 0), hs0=(128, 101, 1), hs1=(128, 101, 1), u0=(128, 101, 1))
SMALL_LSTM1_DBG = dict(SMALL_STAGES, z=(64, 106, 6), x0=(128, 100, 0), hs0=(128, 101, 1), u0=(128, 101, 1))
TWO_RES_DBG = {
    "z": (64, 106, 6), "u0": (128, 101, 1),
    "x1.elu": (64, 802, 2), "x1.raw": (64, 802, 2), "h1.0": (64, 802, 2), "o1.0": (64, 804, 4), "h1.1": (64, 804, 4),
    "o1.1": (64, 801, 1),
    "x2.elu": (64, 4002, 2), "x2.raw": (64, 4002, 2), "h2.0": (64, 4002, 2), "o2.0": (64, 4004, 4), "h2.1": (64, 4004, 4),
    "o2.1": (64, 4001, 1),
    "x3.elu": (64, 16002, 2), "x3.raw": (64, 16002, 2), "h3.0": (64, 16002, 2), "o3.0": (64, 16004, 4),
    "h3.1": (64, 16004, 4), "o3.1": (64, 16001, 1),
    "x4.elu": (64, 32002, 2), "x4.raw": (64, 32002, 2), "h4.0": (64, 32002, 2), "o4.0": (64, 32004, 4),
    "h4.1": (64, 32004, 4), "o4.1": (64, 32006, 6),
}

# name: (config overrides, knobs, seed, decode launches, stream decode launches, stream_state_bytes, stream_min_frames,
#        utterances of the last chunk, debug tensors)
PLANS = {
    "default": ({}, {}, 5, 218, 60, 36352, 8, B, DEFAULT_DBG),
    "small_causal_reflect": (dict(SMALL, lstm=2), {}, 1, 218, 60, 8448, 8, B, SMALL_LSTM2_DBG),
    "small_constpad": (dict(SMALL, lstm=1, pad_mode="constant"), {}, 3, 117, 43, 7424, 8, B, SMALL_LSTM1_DBG),
    # two residual blocks per stage: min_T = (3 - 1) * 2 * 2 + 2 from the last block's dilation, not deepest halo + 2
    "two_res_no_lstm": (dict(SMALL, lstm=0, n_residual_layers=2), {}, 4, 24, 38, 10496, 10, B, TWO_RES_DBG),
    "convout_tc": ({}, {"VCB_CODEC_CONVOUT_TC": "1"}, 5, 217, 59, 36352, 8, B, DEFAULT_DBG),
    "lstm_wide": ({}, {"VCB_CODEC_LSTM_WIDE": "1"}, 5, 218, 60, 36352, 8, B, DEFAULT_DBG),
    # a 20 MB workspace: one utterance per chunk, so every launch of a decode repeats per utterance
    "ws_chunked": ({}, {"VCB_CODEC_WS_GB": "0.02"}, 6, 872, 180, 36352, 8, 1, DEFAULT_DBG),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PLANS))
def test_codec_plan_pinned(name, monkeypatch):
    from voicecraft_b200 import _lib
    from voicecraft_b200.tokenizer import AudioTokenizer
    over, knobs, seed, n_dec, n_stream, state_bytes, min_frames, chunk_b, dbg = PLANS[name]
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    cfg = eo.default_config(**over)
    tok = AudioTokenizer(device="cuda:0", config=cfg, state_dict=eo.make_state_dict(cfg, seed=seed))
    lib = _lib.load()
    eng = tok._engine()
    assert lib.enc_counter(eng, b"tc_enabled") == 1
    codes = torch.randint(0, cfg.bins, (B, cfg.n_q, T), generator=torch.Generator().manual_seed(seed)).cuda()

    n0 = lib.enc_counter(eng, b"launches")
    tok.decode_codes(codes)
    torch.cuda.synchronize()
    assert lib.enc_counter(eng, b"launches") - n0 == n_dec

    names = ["z", "u0", "x0", "hs0", "hs1"] + [f"x{i}.{f}" for i in range(1, 6) for f in ("elu", "raw")] + \
            [f"{p}{i}.{j}" for i in range(1, 6) for j in range(4) for p in ("h", "o")]
    got = {}
    for nm in names:
        d = (C.c_int32 * 4)()
        if lib.enc_debug_tensor(eng, nm.encode(), None, 0, d) == 0:
            assert d[0] == chunk_b, nm
            got[nm] = (d[1], d[2], d[3])
    assert got == dbg

    assert lib.enc_counter(eng, b"stream_state_bytes") == state_bytes
    assert lib.enc_counter(eng, b"stream_min_frames") == min_frames
    with tok.open_stream(max_streams=SB) as cs:
        n0 = lib.enc_counter(eng, b"launches")
        cs.decode(codes[:SB, :, :ST])
        torch.cuda.synchronize()
        assert lib.enc_counter(eng, b"launches") - n0 == n_stream


# ---- the tensor-core encoder: one seeded ragged encode_many batch per configuration of test_encode_numerics, per knob
ENC_KNOBS = {
    "plain": {},
    "lstm_wide": {"VCB_CODEC_LSTM_WIDE": "1"},
    "ws_small": {"VCB_CODEC_WS_GB": "0.01"},   # a 10.7 MB workspace limit: chunks of one to three rows
}
ENC_CASES = [(c, k) for c in ENC_CONFIGS for k in ENC_KNOBS]


def encoder_structure(name, knob, monkeypatch):
    """(launches, encode_rows, tc_encodes, workspace bytes) of the batch with VCB_CODEC_KEEP off, the workspace bytes being
    what the first encode of a fresh tokenizer adds to the process-wide live_bytes; then {enc.* name: (B, C, halo + rows,
    halo)} of the last chunk with VCB_CODEC_KEEP=1"""
    import gc

    from voicecraft_b200 import _lib
    from voicecraft_b200.tokenizer import AudioTokenizer
    lib = _lib.load()
    cfg = eo.default_config(**ENC_CONFIGS[name])
    sd = eo.make_state_dict(cfg, seed=11, encoder=True)
    g = torch.Generator().manual_seed(23)
    lens = [min_accepted(cfg)] + torch.randint(min_accepted(cfg), 25 * enc_hop(cfg) + 1, (4,), generator=g).tolist()
    wavs = [0.3 * torch.randn(1, n, generator=g) for n in lens]
    for k, v in ENC_KNOBS[knob].items():
        monkeypatch.setenv(k, v)
    out = {}
    for keep in ("0", "1"):
        monkeypatch.setenv("VCB_CODEC_KEEP", keep)
        gc.collect()
        tok = AudioTokenizer(device="cuda:0", config=cfg, state_dict=sd)
        eng = tok._engine()
        assert lib.enc_counter(eng, b"tc_encoder") == 1
        torch.cuda.synchronize()
        live0 = lib.enc_counter(None, b"live_bytes")
        counts0 = [lib.enc_counter(eng, c) for c in (b"launches", b"encode_rows", b"tc_encodes")]
        tok.encode_many(wavs)
        torch.cuda.synchronize()
        if keep == "0":
            out["launches"], out["encode_rows"], out["tc_encodes"] = \
                [lib.enc_counter(eng, c) - c0 for c, c0 in zip((b"launches", b"encode_rows", b"tc_encodes"), counts0)]
            out["ws_bytes"] = lib.enc_counter(None, b"live_bytes") - live0
        else:
            dims = {}
            for t in enc_tensors(cfg):
                for nm in (t["raw"], t["elu"]):
                    if nm is not None:
                        d = (C.c_int32 * 4)()
                        assert lib.enc_debug_tensor(eng, nm.encode(), None, 0, d) == 0, nm
                        dims[nm] = list(d)
            out["dbg"] = dims
        del tok, eng
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,knob", ENC_CASES)
def test_encoder_plan_pinned(name, knob, monkeypatch):
    """The encoder's launches, encode_rows (and so its chunking), tc_encodes, debug tensor dims and workspace bytes.  The
    values in golden/encoder_plan.json were recorded on an H100 from the encoder as it was when it had a plan, a workspace
    layout and an executor of its own, before it shared the decoder's; there the workspace bytes were checked to be
    exactly its workspace layout of the largest chunk, and nothing else."""
    with open(os.path.join(os.path.dirname(__file__), "golden", "encoder_plan.json")) as f:
        pinned = json.load(f)[f"{name}/{knob}"]
    assert encoder_structure(name, knob, monkeypatch) == pinned
