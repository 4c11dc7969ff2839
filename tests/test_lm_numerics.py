"""The codec LM stage by stage against float64 (tests/lm_ref.py), as test_codec_numerics.py does for EnCodec.

A pass is run once per stage with vcb_set_option("stop_stage", s): the run stopped after stage s leaves that stage's output,
and the inputs it read are what the pass itself stored before it (read back with vcb_debug_stage_read, K / V with
vcb_debug_kv_pages, logits with vcb_debug_logits after an unstopped run).  Each bound therefore covers one stage's
arithmetic.  Stages are numbered as the persistent kernel's phases: 5 l + {0 QKV, 1 attention, 2 out-projection, 3 FFN1,
4 FFN2}, then 5 L (final LayerNorm + first head stage, GELU) and 5 L + 1 (second head stage, the logits).  The separate runs
are comparable because the engine is deterministic: test_stopped_runs_are_deterministic asserts it, and that an unset stop
changes nothing.

Bounds (|.| elementwise; A = sum |a||w| + |b| over the stage's GEMM, lm_ref.*_abs):
  * GEMM on a hi/lo operand (prefill, VCB_FOLD=0, out-projection, FFN2, second head stage): the operand read back is hi + lo
    exactly, the weights are bf16 values and every product is exact in fp32, so the error is the fp32 accumulation: at
    most one rounding of 2^-23 of a partial sum (<= A) per wgmma k16 step, per split-K / hi-lo / bias add, i.e.
    GEMM(K) = 2^-22 (K / 16 + 20) A.  A residual epilogue adds two fp32 roundings: 2^-23 |x_new|.
  * folded LayerNorm (QKV / FFN1 / first head stage of a decode step): y = rstd (W (gamma x) - mean W gamma) + b + W beta
    on the hi/lo operand gamma x (split error 2^-17 |gamma x|), with the statistics in fp32: (GEMM(K) + 2^-16) A_fold,
    A_fold = rstd |W gamma| (|x| + |mean|) + |W| |beta| + |b| (lm_ref.fold_abs).  This is the class-free form of
    test_kernel_numerics.FOLD_BOUND: the fold's error grows with |mean| because the mean is subtracted after the product.
  * two-pass LayerNorm rows (unfolded): fp32 arithmetic then the hi/lo split: 2^-17 |y| + 2^-20 (rstd (|x| + |mean|) |gamma|
    + |beta|).
  * an activation epilogue: ReLU is 1-Lipschitz, GELU 1.13-Lipschitz; then the hi/lo split, 2^-17 |out|.
  * attention over the pages the pass stored: 1e-5 max|V| (test_kernel_numerics) plus the hi/lo split of its output.
  * bf16 K / V: the GEMM bound plus half an ulp of the stored value.  fp8 K / V: the stored bytes dequantized with
    tests/kv_fp8_ref.py, within the GEMM bound plus the quantizer's error 2^-4 |v| + 2^-10 scale
    (test_kv_fp8.test_quantizer_relative_error_and_scale_rule).  Q is compared before storage on every engine.
  * the folded pass's operand gamma x (step_prep for layer 0, the residual epilogues after): the hi/lo split of the fp32
    product, 2^-17 (1 + 2^-7) |gamma x|.  The split's bound is 2^-17, not 2^-16: |x - hi| < 2^-8 2^e for x in [2^e, 2^(e+1)),
    so x - hi lies below 2^(e-8) and its own rounding is at most 2^(e-17).
  * embeddings (embed_rows_kernel, the sampler's next-input embedding, step_prep's copy of it): bit-exact against torch fp32
    in the kernels' order (lm_ref.prompt_rows / next_input).
Every check prints its worst error as a fraction of its bound.

The stages reach every layer of each case.  Cases: prefill through the decode GEMM in one chunk and in two (the second chunk
attends to K / V the first one wrote), through the rows-as-M GEMM (wide), text / audio boundaries, an edit prompt with mask
rows, prompts ending at positions 63 and 64; the first sampling step after a prefill (unfolded heads); decode steps folded
(bpad 16 / 32 / 64 / 128 through n = 1, 16, 17, 32, 33, 128), unfolded (VCB_FOLD=0) and through the persistent kernel
(VCB_MEGA=1), at positions 63, 64 and 1100 (the split-context merge); head dims 128 (tiny, 830M) and 64 (330M); fp32, bf16
and fp8 K / V; V = 2051 (no eos: a last logit tile with 3 valid columns); a residual offset of 20 (+20 on every
out-projection and FFN2 bias, and on the embeddings); a far offset (3000 on the embeddings, 2000 times the rows' spread)
where the layer-0 statistics of step_prep_kernel need their two passes: the fold's bound grows like mean / std, the error
of a one-pass variance E[x^2] - mean^2 like (mean / std)^2, and only past a mean / std of about 1000 does the second
outgrow the first at d = 256; and a quiet input (embeddings x 3e-3, variance near the LayerNorm epsilon) where a wrong
epsilon shows.
"""
import contextlib

import numpy as np
import pytest
import torch

import golden_util as gu
import lm_ref

# ==========================================================================================================================
# CPU: the stages chained reproduce the oracle
# ==========================================================================================================================


@pytest.mark.parametrize("name", ["tts_topk40", "tts_k8_noeos", "tts_small", "batch3"])
def test_stages_chained_reproduce_oracle(name):
    """lm_ref's stages chained over a fixture's prompt and its first sampled rows give OracleLM's logits at every traced
    step and its K / V cache, within fp32 noise (the oracle runs in fp32, the stages in fp64)."""
    from oracle import lm_oracle
    case = gu.load_cases()[name]
    cfg, sd, x, x_lens, y, _ = gu.build_case(name, case)
    oracle = lm_oracle.OracleLM(cfg, sd)
    kw = dict(case["kw"], silence_tokens=gu.SILENCE, noise_fn=gu.cpu_noise_fn(case["seed"]))
    rows = oracle.inference_tts(x, x_lens, y, max_steps=4, trace_logits=True, **kw)
    assert rows.shape[0] == 4
    K = cfg.n_codebooks
    # the oracle's own embedding rows: text, the delayed prompt, then the sampled rows but the last
    prompt = oracle._delay(y[0].transpose(1, 0))[:, : -(K - 1)]
    toks = torch.cat([prompt, rows[:-1].transpose(1, 0)], dim=1)
    emb = torch.cat([oracle.embed_text(x), oracle.pos_audio(oracle.embed_codes(toks.unsqueeze(-1)).transpose(1, 0))], 1)[0]
    sd64 = lm_ref.double(sd)
    logits, kv = lm_ref.forward(sd64, cfg, emb.double())
    xl, T = x.shape[1], emb.shape[0]
    for t, ref in enumerate(oracle.logit_trace):
        got = logits[T - len(oracle.logit_trace) + t].clone()
        if cfg.eos > 0:
            got[:, cfg.eog] = -10000.0
        err = float((got - ref.double()).abs().max())
        assert err <= 2e-4 * float(ref.abs().max()), f"step {t}: max |logit - oracle| {err:.3g}"
    # the oracle's K / V cache of the prompt (a first dec_forward with the cache on)
    cache = dict(kv=None, on=True)
    n_prompt = xl + prompt.shape[1]
    oracle.dec_forward(emb[None, :xl], emb[None, xl:n_prompt], cache)
    for l, (k, v) in enumerate(cache["kv"]):
        for what, a, b in (("K", k, kv[l][0]), ("V", v, kv[l][1])):
            a = a[0].transpose(0, 1).double()                 # [T, H, hd]
            err = float((a - b[:n_prompt]).abs().max())
            assert err <= 1e-5 * float(a.abs().max()), f"layer {l} {what}: max err {err:.3g}"


def test_fold_abs_bounds_the_folded_form():
    """lm_ref.fold_abs bounds |rstd (W (gamma x) - mean W gamma)| termwise: with every x replaced by |x| + |mean| and the
    weights by their magnitudes it can only grow, and it does at a large offset"""
    g = torch.Generator().manual_seed(0)
    W, gamma, beta, b = (torch.randn(*s, generator=g, dtype=torch.float64) for s in ((8, 16), (16,), (16,), (8,)))
    for off in (0.0, 20.0):
        x = torch.randn(3, 16, generator=g, dtype=torch.float64) + off
        mean, rstd = lm_ref.ln_parts(x)
        folded = rstd * ((x @ (W * gamma).t()) - mean * (W * gamma).sum(1)) + beta @ W.t() + b
        ref = lm_ref.layer_norm(x, gamma, beta) @ W.t() + b
        assert torch.allclose(folded, ref, atol=1e-9)
        assert torch.all(lm_ref.fold_abs(W, gamma, beta, b, x) >= folded.abs() - 1e-9)


# ==========================================================================================================================
# GPU
# ==========================================================================================================================
def _gemm_c(K):
    return 2.0 ** -22 * (K / 16 + 20)


SPLIT = 2.0 ** -17
GELU_LIP = 1.13


def _lib():
    from voicecraft_b200 import _lib
    return _lib, _lib.load()


def _half_ulp_bf16(v):
    """half an ulp of bf16 values v (0 for 0)"""
    _, e = torch.frexp(v)
    return torch.where(v == 0, torch.zeros_like(v), torch.ldexp(torch.ones_like(v), e - 9))


class Worst:
    """the worst |got - ref| / bound of each check, and the checks over their bound"""

    def __init__(self, label):
        self.label, self.worst, self.bad = label, {}, []

    def check(self, name, got, ref, bound):
        got, ref, bound = got.double(), ref.double(), bound.double()
        assert got.shape == ref.shape, f"{name}: shape {tuple(got.shape)} != {tuple(ref.shape)}"
        assert torch.isfinite(got).all(), f"{self.label} {name}: non-finite values"
        r = float(((got - ref).abs() / bound.clamp_min(1e-300)).max())
        self.worst[name] = max(self.worst.get(name, 0.0), r)
        if r > 1.0:
            self.bad.append(f"{name}: {r:.3g}")

    def exact(self, name, got, ref):
        n = int((got != ref).sum())
        self.worst[name] = max(self.worst.get(name, 0.0), float(n))
        if n:
            self.bad.append(f"{name}: {n} values differ")

    def done(self):
        summary = ", ".join(f"{k} {v:.3g}" for k, v in sorted(self.worst.items()))
        print(f"{self.label}: worst error / bound: {summary}")
        assert not self.bad, f"{self.label}: {len(self.bad)} over the bound (first: {self.bad[:8]})"


def _checkpoint(cfg_name, seed, regime="plain", **over):
    from voicecraft_b200 import synthetic
    cfg = synthetic.make_config(cfg_name, **over)
    sd = synthetic.make_state_dict(cfg, seed=seed)
    K, L = cfg.n_codebooks, cfg.num_decoder_layers
    if regime == "offset":
        for l in range(L):
            sd[f"decoder.layers.{l}.self_attn.out_proj.bias"] += 20.0
            sd[f"decoder.layers.{l}.linear2.bias"] += 20.0
        for k in range(K):
            sd[f"audio_embedding.{k}.word_embeddings.weight"] += 20.0 / K
        sd["text_embedding.word_embeddings.weight"] += 20.0
        sd["mask_embedding"] += 20.0
    elif regime == "far":
        for k in range(K):
            sd[f"audio_embedding.{k}.word_embeddings.weight"] += 3000.0 / K
        sd["text_embedding.word_embeddings.weight"] += 3000.0
        sd["mask_embedding"] += 3000.0
    elif regime == "quiet":
        for key in [f"audio_embedding.{k}.word_embeddings.weight" for k in range(K)] + [
                "text_embedding.word_embeddings.weight", "mask_embedding", "text_positional_embedding.alpha",
                "audio_positional_embedding.alpha"]:
            sd[key] *= 3e-3
    return cfg, sd


class Case:
    """one engine and a batch of prompts, run once per stage"""

    def __init__(self, cfg_name, kv="bf16", regime="plain", totals=(100,), mode="decode", edit=False, seed=5,
                 weight_dtype="bf16", max_seq_len=512, **over):
        from voicecraft_b200 import synthetic
        from voicecraft_b200.voicecraft import VoiceCraft
        self.cfg, sd = _checkpoint(cfg_name, seed, regime, **over)
        cfg = self.cfg
        self.mode, self.kv, self.edit = mode, kv, edit
        self.m = VoiceCraft(cfg)
        self.m.load_state_dict(sd)
        self.m = self.m.to("cuda").eval()
        self.m.configure_engine(kv_dtype=kv, max_slots=max(len(totals), 1), max_seq_len=max_seq_len,
                                weight_dtype=weight_dtype)
        self.eng = self.m._engine()
        if weight_dtype == "int8":
            from weight_int8_ref import dequantize_state_dict
            sd = dequantize_state_dict(sd)
        self.sd = {k: v.cuda() for k, v in lm_ref.double(sd).items()}
        self.sdf = {k: v.float() for k, v in sd.items() if "embedding" in k}   # the fp32 embedding tables, alphas
        self.L, self.K, self.H = cfg.num_decoder_layers, cfg.n_codebooks, cfg.nhead
        self.d = cfg.d_model
        self.hd = self.d // self.H
        self.utts, self.spans = [], []
        for i, total in enumerate(totals):
            text = 6 + i % 5
            x, xl, y = synthetic.synthetic_utterance(cfg, 700 + 31 * i + seed, text_len=text, prompt_frames=total - text - 1)
            self.utts.append((x, y))
            if edit:
                T = y.shape[1]
                self.spans.append(torch.tensor([[[T // 5, T // 5 + 4], [T // 2, T // 2 + 6]]]))
        self.seeds = [1000 + i for i in range(len(totals))]
        from voicecraft_b200.voicecraft import sine_pe
        self.pe = sine_pe(max(4000, max_seq_len), self.d)

    @contextlib.contextmanager
    def run(self, stop, pre_steps=0):
        """a session stopped after `stop` stages of its prefill (mode "prefill"), its first sampling step ("sample") or its
        decode step after pre_steps unstopped ones ("decode"); stop = 0 runs everything"""
        from voicecraft_b200.voicecraft import DecodeSession
        _l, lib = _lib()
        sp = self.m._sampling(top_k=40, top_p=1.0, temperature=1.0, stop_repetition=3, silence_tokens=gu.SILENCE)
        _l.check(lib.vcb_set_option(self.eng, b"stop_stage", stop if self.mode == "prefill" else 0))
        sess = None
        try:
            sess = DecodeSession(self.m, [u[0] for u in self.utts], [u[1] for u in self.utts], sp,
                                 mask_intervals=self.spans if self.edit else None, seeds=self.seeds)
            assert sess.eng == self.eng, "the engine was rebuilt: its options are gone"
            if self.mode == "sample":
                _l.check(lib.vcb_set_option(self.eng, b"stop_stage", stop))
            if self.mode != "prefill":
                sess.sample()
            if self.mode == "decode":
                for _ in range(pre_steps):
                    sess.step()
                _l.check(lib.vcb_set_option(self.eng, b"stop_stage", stop))
                sess.step()
            torch.cuda.synchronize()
            yield View(self, sess)
        finally:
            _l.check(lib.vcb_set_option(self.eng, b"stop_stage", 0))
            if sess is not None:
                sess.close()

    def prefill_rows(self, sess):
        """(utterance, position) of every prefill row, and the embedding rows lm_ref expects"""
        rows, emb = [], []
        for i, p in enumerate(sess.prompts):
            mask = None if p.mask_rows is None else p.mask_rows.cpu()
            emb.append(lm_ref.prompt_rows(self.sdf, self.pe, p.x_ids.cpu(), p.y_tok.cpu(), mask))
            rows += [(i, t) for t in range(p.total)]
        return rows, torch.cat(emb)


class View:
    """what a (stopped) run left: its rows, buffers, K / V pages and, unstopped, its logits"""

    def __init__(self, case, sess):
        self.c, self.sess = case, sess
        c = case
        n = len(sess.slots)
        if c.mode == "prefill":
            rows, self.emb_all = c.prefill_rows(sess)
            chunk = c.chunk
            first = (len(rows) - 1) // chunk * chunk            # the last chunk's rows
            self.rows, self.emb = rows[first:], self.emb_all[first:]
        else:
            st = sess.poll()
            self.rows = []
            for i in range(n):
                total = sess.prompts[i].total
                steps = st[i].n_steps
                self.rows.append((i, total + steps - (1 if c.mode == "decode" else 0)))
            if c.mode == "sample":
                self.rows = [(i, sess.prompts[i].total - 1) for i in range(n)]
        self.n = len(self.rows)
        self._kv = {}

    def read(self, name):
        _l, lib = _lib()
        c = self.c
        width = {"ffn": 4 * c.d, "heads": c.K * (int(c.cfg.audio_vocab_size) // 2)}.get(name, c.d)
        out = torch.empty(self.n, width, device="cuda")
        if lib.vcb_debug_stage_read(self.sess.eng, name.encode(), out.data_ptr(), self.n) != 0:
            return None
        return out.double()

    def kv(self, l, i):
        """layer l's K, V of utterance i over positions 0 .. its last row's, values as attention reads them [T, H, hd], and
        the fp8 scales [T, H] (None otherwise)"""
        if (l, i) in self._kv:
            return self._kv[l, i]
        _l, lib = _lib()
        c = self.c
        T = max(p for u, p in self.rows if u == i) + 1
        npg = (T + 63) // 64
        slab = {"fp32": 64 * c.hd * 4, "bf16": 64 * c.hd * 2, "fp8": 64 * (c.hd + 4)}[c.kv]
        kb = np.zeros(npg * c.H * slab, np.uint8)
        vb = np.zeros_like(kb)
        _l.check(lib.vcb_debug_kv_pages(self.sess.eng, l, self.sess.slots[i], 0, npg, kb.ctypes.data, vb.ctypes.data))
        out = []
        for raw in (kb, vb):
            t = torch.from_numpy(raw)
            if c.kv == "fp8":
                from kv_fp8_ref import split_slabs
                q, s = split_slabs(t, c.H, c.hd)
                vals = q.view(torch.float8_e4m3fn).float() * s[..., None]
                out.append((vals.transpose(1, 2).reshape(-1, c.H, c.hd)[:T].cuda().double(),
                            s.transpose(1, 2).reshape(-1, c.H)[:T].cuda().double()))
            else:
                dt = torch.float32 if c.kv == "fp32" else torch.bfloat16
                vals = t.view(dt).reshape(npg, c.H, 64, c.hd).transpose(1, 2).reshape(-1, c.H, c.hd)[:T]
                out.append((vals.float().cuda().double(), None))
        self._kv[l, i] = out
        return out

    def logits(self):
        _l, lib = _lib()
        c = self.c
        V = int(c.cfg.audio_vocab_size) + c.cfg.n_special
        out = torch.empty(self.n * c.K, V, device="cuda")
        _l.check(lib.vcb_debug_logits(self.sess.eng, out.data_ptr(), self.n * c.K))
        return out.double().reshape(self.n, c.K, V)


# ---- the checks of one stage -------------------------------------------------------------------------------------------
def _ln_check(w, name, got, x, g, b):
    ref = lm_ref.layer_norm(x, g, b)
    mean, rstd = lm_ref.ln_parts(x)
    bound = SPLIT * ref.abs() + 2.0 ** -20 * (rstd * (x.abs() + mean.abs()) * g.abs() + b.abs())
    w.check(name, got, ref, bound)
    return ref


def _operand_check(w, name, got, gamma, x):
    gx = gamma * x
    w.check(name, got, gx, SPLIT * (1 + 2.0 ** -7) * gx.abs() + 1e-300)


def _gemm_in(case, v, which, l, x, fold, w, tag):
    """the normalized operand of a QKV / FFN1 / head GEMM and its bound's A: folded, LN(x) from the pass's x in fp64;
    unfolded, the LayerNorm rows the pass stored (checked here)"""
    sd, K = case.sd, case.K
    W, g, b_, bias = lm_ref.heads_weights(sd, K) if which == "heads" else lm_ref.layer_weights(sd, l, which)
    if fold:
        h = lm_ref.layer_norm(x, g, b_)
        return h, (_gemm_c(x.shape[1]) + 2.0 ** -16) * lm_ref.fold_abs(W, g, b_, bias, x)
    h = v.read("opnd")
    _ln_check(w, f"{tag} LayerNorm", h, x, g, b_)
    return h, _gemm_c(x.shape[1]) * (h.abs() @ W.abs().t() + bias.abs())


def _check_stage(case, i, v, prev, w, fold):
    """stage i of a run stopped after it (v), with the previous run's x (prev)"""
    sd, L, d, H, hd, K = case.sd, case.L, case.d, case.H, case.hd, case.K
    l, t = divmod(i, 5)
    x = v.read("x")
    tag = f"L{l}" if l < L else "heads"
    if i == 0:
        if case.mode == "prefill":
            w.exact("embed_rows", x.float().cpu(), v.emb)
        else:
            st = v.sess.poll()
            for r, (u, pos) in enumerate(v.rows):
                if case.mode != "decode":
                    continue
                toks = torch.from_numpy(case.m._read_rows(v.sess.eng, v.sess.slots[u], st[u].n_steps, v.sess.stream)[-1])
                j = pos - v.sess.prompts[u].x_ids.shape[0]
                w.exact("next-input embedding", x[r].float().cpu(), lm_ref.next_input(case.sdf, case.pe, toks, j))
    if l < L and t == 0:
        if fold:
            _operand_check(w, f"{tag} gamma1 x", v.read("opnd"), sd[f"decoder.layers.{l}.norm1.weight"], x)
        h, A = _gemm_in(case, v, "qkv", l, x, fold, w, tag)
        ref = lm_ref.qkv(sd, l, h)
        bound = A
        w.check(f"{tag} Q", v.read("q"), ref[:, :d], bound[:, :d])
        for r, (u, pos) in enumerate(v.rows):
            kvs = v.kv(l, u)
            for part, (vals, scale) in enumerate(kvs):
                got = vals[pos].reshape(-1)
                rr = ref[r, (part + 1) * d:(part + 2) * d]
                bb = bound[r, (part + 1) * d:(part + 2) * d]
                if case.kv == "bf16":
                    bb = bb + _half_ulp_bf16(got)
                elif case.kv == "fp8":
                    bb = bb + 2.0 ** -4 * (rr.abs() + bb) + 2.0 ** -10 * scale[pos].repeat_interleave(hd)
                w.check(f"{tag} {'KV'[part]} ({case.kv})", got, rr, bb)
    elif l < L and t == 1:
        q = v.read("q").reshape(-1, H, hd)
        att = v.read("att")
        for r, (u, pos) in enumerate(v.rows):
            (Kv, _), (Vv, _) = v.kv(l, u)
            ref = lm_ref.attention(q[r], Kv[:pos + 1], Vv[:pos + 1])
            bound = 1e-5 * Vv[:pos + 1].abs().max() + SPLIT * ref.abs()
            w.check(f"{tag} attention", att[r], ref, bound)
    elif l < L and t == 2:
        att = v.read("att")
        ref = lm_ref.out_proj(sd, l, att, prev["x"])
        w.check(f"{tag} out-proj + residual", x, ref, _gemm_c(d) * lm_ref.out_proj_abs(sd, l, att) + 2.0 ** -23 * ref.abs())
        if fold:
            _operand_check(w, f"{tag} gamma2 x", v.read("opnd"), sd[f"decoder.layers.{l}.norm2.weight"], x)
    elif l < L and t == 3:
        h, A = _gemm_in(case, v, "ffn1", l, x, fold, w, tag)
        ref = lm_ref.ffn1(sd, l, h)
        w.check(f"{tag} FFN1 + ReLU", v.read("ffn"), ref, A + SPLIT * ref.abs())
    elif l < L and t == 4:
        f = v.read("ffn")
        ref = lm_ref.ffn2(sd, l, f, prev["x"])
        w.check(f"{tag} FFN2 + residual", x, ref, _gemm_c(4 * d) * lm_ref.ffn2_abs(sd, l, f) + 2.0 ** -23 * ref.abs())
        if fold:
            g = sd[f"decoder.layers.{l + 1}.norm1.weight"] if l + 1 < L else sd["decoder.norm.weight"]
            _operand_check(w, f"{tag} gamma_next x", v.read("opnd"), g, x)
    elif i == 5 * L:
        h, A = _gemm_in(case, v, "heads", None, x, fold, w, tag)
        ref = lm_ref.heads1(sd, K, h)
        w.check("heads stage 1 + GELU", v.read("heads"), ref, GELU_LIP * A + SPLIT * ref.abs())


def _check_logits(case, heads, v, w):
    """the second head stage: the logits of an unstopped run against the first stage's output of the stopped one"""
    Hh = heads.shape[1] // case.K
    ref = lm_ref.heads2(case.sd, case.K, heads)
    bound = _gemm_c(Hh) * lm_ref.heads2_abs(case.sd, case.K, heads)
    w.check("heads stage 2 (logits)", v.logits(), ref, bound)


def _run_case(case, label, pre_steps=0, fold=True, mega=False):
    """every stage of the case's pass, each against the run stopped one stage earlier"""
    _l, lib = _lib()
    w = Worst(label)
    L = case.L
    if mega:
        assert lib.vcb_counter(case.eng, b"mega_grid") > 0, "the persistent decode kernel is not available"
    stages = range(5 * L, 5 * L + 1) if case.mode == "sample" else range(5 * L + (0 if case.mode == "prefill" else 1))
    prev, heads = None, None
    for i in stages:
        with case.run(i + 1, pre_steps) as v:
            _check_stage(case, i, v, prev, w, fold)
            prev = {"x": v.read("x")}
            if i == 5 * L:
                heads = v.read("heads")
    if case.mode != "prefill":
        with case.run(0, pre_steps) as v:
            _check_logits(case, heads, v, w)
    w.done()


# ---- the cases ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kv", ["fp32", "bf16", "fp8"])
def test_prefill_narrow_two_chunks(kv, monkeypatch):
    """the decode GEMM's prefill, 164 rows in chunks of 128 and 36 (the second attends to K / V the first wrote): a prompt
    ending at position 63 and one across the text / audio boundary of the second chunk"""
    monkeypatch.setenv("VCB_PREFILL_WIDE", "0")
    case = Case("tiny", kv=kv, totals=(64, 100), mode="prefill")
    case.chunk = 128
    _run_case(case, f"narrow prefill 2 chunks kv={kv}", fold=False)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,regime,kv", [("tiny", "plain", "bf16"), ("tiny", "offset", "bf16"),
                                                ("tiny", "quiet", "fp32"), ("330M", "plain", "bf16")])
def test_prefill_narrow_one_chunk(cfg_name, regime, kv, monkeypatch):
    """one chunk of the decode GEMM's prefill: prompts ending at positions 63 and 64 (hd 64 at 330M)"""
    monkeypatch.setenv("VCB_PREFILL_WIDE", "0")
    case = Case(cfg_name, kv=kv, regime=regime, totals=(64, 65), mode="prefill")
    case.chunk = 128
    _run_case(case, f"narrow prefill {cfg_name} {regime} kv={kv}", fold=False)


@pytest.mark.gpu
def test_prefill_edit_prompt_mask_rows(monkeypatch):
    """an edit prompt of two spans: the mask-embedding rows of embed_rows_kernel"""
    monkeypatch.setenv("VCB_PREFILL_WIDE", "0")
    case = Case("tiny", totals=(90,), mode="prefill", edit=True)
    case.chunk = 128
    _run_case(case, "edit prompt prefill", fold=False)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,regime,kv,totals", [("tiny", "plain", "bf16", (1100,)), ("tiny", "offset", "fp8", (1100,)),
                                                       ("830M", "plain", "bf16", (1100,))])
def test_prefill_wide(cfg_name, regime, kv, totals):
    """the rows-as-M prefill (gemm_rows.cu) of about 1100 rows: attention contexts past 1024 (split-context merge)"""
    case = Case(cfg_name, kv=kv, regime=regime, totals=totals, mode="prefill", max_seq_len=2048)
    case.chunk = 1 << 30
    _run_case(case, f"wide prefill {cfg_name} {regime} kv={kv}", fold=False)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,n,over", [("tiny", 1, {}), ("tiny", 5, {"eos": -1}), ("tiny", 33, {}),
                                             ("830M", 5, {})])
def test_first_sample_heads(cfg_name, n, over):
    """vcb_sample after a prefill: explicit final LayerNorm rows, then both head stages (V = 2051 without eos)"""
    case = Case(cfg_name, totals=tuple(20 + 3 * i for i in range(n)), mode="sample", **over)
    _run_case(case, f"first sample {cfg_name} n={n} {over}", fold=False)


DECODE = [
    ("tiny", "bf16", "plain", (62,), {}),
    ("tiny", "bf16", "plain", tuple(40 + 2 * i for i in range(16)), {}),
    ("tiny", "fp32", "offset", tuple(60 + i for i in range(17)), {}),
    ("tiny", "fp8", "plain", tuple(30 + 3 * i for i in range(33)), {}),
    ("tiny", "bf16", "quiet", (62, 63, 1099), {}),
    ("tiny", "bf16", "far", tuple(40 + i for i in range(5)), {}),
    ("tiny", "bf16", "plain", tuple(20 + i for i in range(128)), {"eos": -1}),
    ("330M", "bf16", "plain", tuple(50 + i for i in range(17)), {}),
    ("830M", "bf16", "plain", tuple(60 + 7 * i for i in range(31)) + (1099,), {}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,kv,regime,totals,over", DECODE, ids=[f"{c}-{k}-{r}-n{len(t)}" for c, k, r, t, _ in DECODE])
def test_decode_chain_folded(cfg_name, kv, regime, totals, over):
    """a decode step on the per-kernel path with LayerNorm folded into the GEMM epilogues"""
    case = Case(cfg_name, kv=kv, regime=regime, totals=totals, mode="decode", max_seq_len=2048, **over)
    _run_case(case, f"decode folded {cfg_name} kv={kv} {regime} n={len(totals)} {over}", pre_steps=1)


@pytest.mark.gpu
def test_decode_chain_unfolded(monkeypatch):
    """VCB_FOLD=0: the decode step with explicit LayerNorm rows"""
    monkeypatch.setenv("VCB_FOLD", "0")
    case = Case("tiny", totals=(30, 40, 50, 63, 64), mode="decode")
    _run_case(case, "decode VCB_FOLD=0", pre_steps=1, fold=False)


MEGA = [
    ("tiny", "bf16", "plain", (62,), {}),
    ("tiny", "fp32", "plain", tuple(40 + 2 * i for i in range(16)), {}),
    ("tiny", "bf16", "offset", tuple(60 + i for i in range(17)), {}),
    ("tiny", "bf16", "far", (62, 63, 70), {}),
    ("tiny", "bf16", "plain", tuple(30 + i for i in range(31)) + (1099,), {"eos": -1}),
    ("830M", "bf16", "plain", tuple(60 + 7 * i for i in range(31)) + (1099,), {}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,kv,regime,totals,over", MEGA, ids=[f"{c}-{k}-{r}-n{len(t)}" for c, k, r, t, _ in MEGA])
def test_decode_persistent_kernel(cfg_name, kv, regime, totals, over, monkeypatch):
    """VCB_MEGA=1: every phase of the persistent step kernel (its epilogues, its attention, its heads)"""
    monkeypatch.setenv("VCB_MEGA", "1")
    case = Case(cfg_name, kv=kv, regime=regime, totals=totals, mode="decode", max_seq_len=2048, **over)
    _run_case(case, f"persistent kernel {cfg_name} kv={kv} {regime} n={len(totals)} {over}", pre_steps=1, mega=True)


@pytest.mark.gpu
def test_decode_chain_int8_weights():
    """int8 weights: the reference runs on W_deq"""
    case = Case("830M", totals=tuple(60 + 7 * i for i in range(32)), mode="decode", weight_dtype="int8")
    _run_case(case, "decode int8 830M n=32", pre_steps=1)


# ---- what the comparison relies on --------------------------------------------------------------------------------------
def _snapshot(case, v):
    out = {k: v.read(k) for k in ("x", "q", "opnd", "att", "ffn", "heads")}
    for l in range(case.L):
        for u in range(len(case.utts)):
            out[f"kv{l}.{u}"] = torch.cat([t[0] for t in v.kv(l, u)])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("mega", ["0", "1"])
def test_stopped_runs_are_deterministic(mega, monkeypatch):
    """two runs stopped at the same stage leave the same bits, and stop_stage = 0 leaves logits, K / V pages and tokens
    bit-identical to an engine that never set the option"""
    monkeypatch.setenv("VCB_MEGA", mega)
    _l, lib = _lib()
    case = Case("tiny", totals=(63, 64, 70), mode="decode")
    for stop in (3, 5 * case.L + 1):
        with case.run(stop, 1) as v:
            a = _snapshot(case, v)
        with case.run(stop, 1) as v:
            b = _snapshot(case, v)
        for k in a:
            assert (a[k] is None) == (b[k] is None)
            assert a[k] is None or torch.equal(a[k], b[k]), f"stop {stop}: {k} differs between two runs"
    outs = []
    for fresh in (True, False):
        c = Case("tiny", totals=(63, 64, 70), mode="decode") if fresh else case
        if not fresh:
            _l.check(lib.vcb_set_option(c.eng, b"stop_stage", 0))
        with c.run(0, 3) as v:
            toks = [c.m._read_rows(v.sess.eng, s, 4, v.sess.stream) for s in v.sess.slots]
            outs.append((v.logits(), _snapshot(c, v), toks))
    (la, sa, ta), (lb, sb, tb) = outs
    assert torch.equal(la, lb), "logits differ"
    for k in sa:
        if k.startswith("kv"):
            assert torch.equal(sa[k], sb[k]), f"{k} differs"
    assert all(np.array_equal(p, q) for p, q in zip(ta, tb)), "tokens differ"


@pytest.mark.gpu
def test_stop_stage_rejects_out_of_range():
    _l, lib = _lib()
    case = Case("tiny", totals=(40,), mode="decode")
    L = case.L
    for bad in (-1, 5 * L + 3):
        assert lib.vcb_set_option(case.eng, b"stop_stage", bad) != 0
        assert b"stop_stage" in lib.vcb_last_error()
    assert lib.vcb_set_option(case.eng, b"stop_stage", 5 * L + 2) == 0
    assert lib.vcb_set_option(case.eng, b"stop_stage", 0) == 0
    with case.run(2, 0) as v:
        out = torch.empty(v.n + 1, case.d, device="cuda")
        assert lib.vcb_debug_stage_read(case.eng, b"x", out.data_ptr(), v.n + 1) != 0
        assert lib.vcb_debug_stage_read(case.eng, b"nope", out.data_ptr(), 1) != 0
        assert b"unknown" in lib.vcb_last_error()
