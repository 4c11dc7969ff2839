"""Stage-by-stage comparison of the tensor-core EnCodec decoder (csrc/codec_tc.cu) with the CPU oracle (GPU box, test infra).
usage: codec_tc_debug.py [n_filters] [B] [T] [lstm]     prints max |err| of every intermediate tensor and of the waveform."""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from oracle import encodec_oracle as eo
from voicecraft_b200 import _lib
from voicecraft_b200.tokenizer import AudioTokenizer

nf = int(sys.argv[1]) if len(sys.argv) > 1 else 16
B = int(sys.argv[2]) if len(sys.argv) > 2 else 3
T = int(sys.argv[3]) if len(sys.argv) > 3 else 37
nl = int(sys.argv[4]) if len(sys.argv) > 4 else 2
over = dict(n_filters=nf, lstm=nl)
if nf < 64:
    over.update(dimension=64, bins=256)
cfg = eo.default_config(**over)
sd = eo.make_state_dict(cfg, seed=3)
codes = torch.randint(0, cfg.bins, (B, cfg.n_q, T), generator=torch.Generator().manual_seed(1))

wav_ref, ref = eo.decode(cfg, sd, codes, return_intermediates=True)
del ref["wav"]

os.environ["VCB_CODEC_KEEP"] = "1"        # every stage tensor keeps rows of its own: what is printed is what the stage stored
tok = AudioTokenizer(device="cuda:0", config=cfg, state_dict=sd)
wav = tok.decode_codes(codes.cuda()).cpu()
lib = _lib.load()
eng = tok._engine()
print("tc_enabled", lib.enc_counter(eng, b"tc_enabled"), "tc_decodes", lib.enc_counter(eng, b"tc_decodes"))


def fetch(name):
    dims = (C.c_int32 * 4)()
    if lib.enc_debug_tensor(eng, name.encode(), None, 0, dims):
        return None, 0
    b, c, tp, halo = list(dims)
    out = np.empty((b, c, tp), dtype=np.float32)
    _lib.check(lib.enc_debug_tensor(eng, name.encode(), out.ctypes.data, out.size, dims))
    return out, halo


for name, r in ref.items():
    got, halo = fetch(name)
    if got is None:
        print(f"{name:10s} (not recorded)")
        continue
    r = r.numpy()
    if name[0] == "c" and name[1:].isdigit():
        r = r[:, :, -1:]                  # the decoder keeps the cell state after the last step only
    g = got[:, : r.shape[1], halo:]
    err = np.abs(g - r)
    pad = np.abs(got[:, r.shape[1]:, halo:]).max() if got.shape[1] > r.shape[1] else 0.0
    bad_t = np.unique(np.argwhere(err > 1e-3 * max(1.0, np.abs(r).max()))[:, 2])[:12] if err.size else []
    print(f"{name:10s} shape {tuple(r.shape)}  max|ref| {np.abs(r).max():9.4f}  max err {err.max():.3e}  pad-channels max {pad:.2e}  "
          f"halo {halo}  first bad t {list(bad_t)}")
err = (wav - wav_ref).abs()
print(f"waveform   max|ref| {wav_ref.abs().max():.4f}  max err {err.max():.3e}   SNR {10 * torch.log10((wav_ref ** 2).sum() / ((wav - wav_ref) ** 2).sum()).item():.1f} dB")
