"""TEST INFRASTRUCTURE ONLY -- torch-CPU fp32 restatement of the VoiceCraft codec-LM decode path.

This is the checker for the CUDA path; it is never shipped or timed as the product.
It restates, with plain torch CPU ops and no dependence on /root/reference:

  embeddings        models/modules/embedding.py:44-48 (TokenEmbedding), :67-97 (sinusoidal PE, alpha)
  transformer stack models/modules/transformer.py:321-329 (pre-LN layer), :386-388 (ReLU FFN),
                    :473-488 (KV path), models/modules/activation.py:536-638 (packed QKV, KV concat,
                    SDPA with additive mask, out_proj)
  dec_forward       models/voicecraft.py:406-470 (causal mask over [text;audio], last-1 / last-3 slicing)
  sampling          models/voicecraft.py:26-86 (top-k / top-p / temperature / multinomial)
  state machines    models/voicecraft.py:1018-1067 (tts), :718-787 (edit), :1269-1325 (batch)
  loops + un-delay  models/voicecraft.py:908-1153 (inference_tts), :561-906 (inference),
                    :1156-1439 (inference_tts_batch)

Pinning: the reference has no tests for this path.  This restatement is pinned against the
reference itself, imported and run by tests/golden/make_golden.py (same weights, same seed ->
identical token ids and logits); fixtures are committed under tests/golden/.

Numerics policy knob: ``kv_round_bf16`` rounds projected K/V to bf16 before use/caching (what the
H100 path's bf16 paged KV cache does).  With it off, and noise drawn from the global CPU generator,
this module is operation-for-operation the reference's fp32 path.

torch.multinomial(p, 1) is restated as argmax(p / q), q ~ Exp(1) drawn with
``torch.empty_like(p).exponential_(1)`` -- that is ATen's own n_sample==1 fast path
(aten/src/ATen/native/Distributions.cpp multinomial_out), verified token-for-token by make_golden.py.
"""
import math
from types import SimpleNamespace

import torch
import torch.nn.functional as F


def _cfg_get(cfg, name, default=None):
    if isinstance(cfg, dict):
        return cfg.get(name, default)
    return getattr(cfg, name, default)


def normalize_config(cfg):
    """Apply the defaults VoiceCraft.__init__ applies (voicecraft.py:117-130)."""
    c = SimpleNamespace()
    for name in ("n_codebooks", "d_model", "nhead", "num_decoder_layers", "empty_token", "eog",
                 "audio_pad_token", "text_vocab_size", "text_pad_token", "encodec_sr", "max_n_spans"):
        setattr(c, name, _cfg_get(cfg, name))
    avs = _cfg_get(cfg, "audio_vocab_size")
    c.audio_vocab_size = int(eval(avs)) if isinstance(avs, str) else int(avs)
    c.n_special = _cfg_get(cfg, "n_special", 3) or 3
    c.special_first = _cfg_get(cfg, "special_first", 0) or 0
    c.eos = _cfg_get(cfg, "eos", -1)
    if c.eos is None:
        c.eos = -1
    c.reduced_eog = _cfg_get(cfg, "reduced_eog", 0) or 0
    c.shuffle_mask_embedding = _cfg_get(cfg, "shuffle_mask_embedding", 0) or 0
    c.n_audio_tokens = c.audio_vocab_size + c.n_special
    return c


def sine_pe(length, dim):
    """Sinusoidal table, reference embedding.py:67-92."""
    pe = torch.zeros(length, dim)
    position = torch.arange(0, length, dtype=torch.float32).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * -(math.log(10000.0) / dim))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe.unsqueeze(0)


def default_noise(shape):
    """Exp(1) noise exactly as ATen's multinomial draws it (global CPU generator)."""
    return torch.empty(shape, dtype=torch.float32).exponential_(1)


# ----------------------------------------------------------------------------- sampling

def filter_top_k_top_p(logits, top_k=0, top_p=1.0):
    """In-place top-k then nucleus filter on [N,V].  reference voicecraft.py:26-68."""
    if top_k > 0:
        k = min(max(top_k, 1), logits.size(-1))
        kth = torch.topk(logits, k)[0][..., -1, None]
        logits[logits < kth] = -float("inf")          # strict '<': ties with the k-th value survive
    if top_p < 1.0:
        srt, idx = torch.sort(logits, descending=True)
        cum = torch.cumsum(F.softmax(srt, dim=-1), dim=-1)
        rm = cum > top_p
        rm[..., 1:] = rm[..., :-1].clone()             # shift right: first token above threshold kept
        rm[..., 0] = 0
        rm = rm.scatter(1, idx, rm)
        logits[rm] = -float("inf")
    return logits


def sample_rows(logits, top_k, top_p, temperature, noise_fn):
    """reference voicecraft.py:71-86 with multinomial restated as argmax(p/q)."""
    if temperature != 1.0:
        logits = logits / temperature                  # copy: caller's tensor keeps unfiltered values
    logits = filter_top_k_top_p(logits, top_k=top_k, top_p=top_p)
    p = F.softmax(logits, dim=-1)
    q = noise_fn(tuple(p.shape))
    return torch.argmax(p / q, dim=-1, keepdim=True)


# ----------------------------------------------------------------------------- model

class OracleLM:
    """Functional fp32 model over a reference-format ``state_dict``."""

    def __init__(self, cfg, state_dict, kv_round_bf16=False):
        self.c = normalize_config(cfg)
        self.sd = {k: v.detach().to(torch.float32) if v.is_floating_point() else v.detach()
                   for k, v in state_dict.items()}
        self.kv_round_bf16 = kv_round_bf16
        self.pe = sine_pe(4000, self.c.d_model)
        self.alpha_t = self.sd["text_positional_embedding.alpha"]
        self.alpha_a = self.sd["audio_positional_embedding.alpha"]
        self.last_logits = None     # debugging / parity hooks
        self.logit_trace = None

    # -- embeddings -----------------------------------------------------------------
    def _pe(self, T):
        if self.pe.size(1) < T:
            self.pe = sine_pe(T, self.c.d_model)
        return self.pe[:, :T]

    def pos_text(self, emb):       # embedding.py:94-97
        return emb * 1.0 + self.alpha_t * self._pe(emb.size(1))

    def pos_audio(self, emb):
        return emb * 1.0 + self.alpha_a * self._pe(emb.size(1))

    def embed_text(self, x):       # voicecraft.py:950-951
        return self.pos_text(F.embedding(x, self.sd["text_embedding.word_embeddings.weight"]))

    def embed_codes(self, tok):
        """tok [K, ...] int64 -> sum_k E_k[tok[k]]  (voicecraft.py:978-982, 1102-1103)."""
        K = self.c.n_codebooks
        e = torch.stack([F.embedding(tok[k], self.sd[f"audio_embedding.{k}.word_embeddings.weight"])
                         for k in range(K)], dim=0)
        return e.sum(dim=0)

    # -- transformer ----------------------------------------------------------------
    def _mha(self, l, h, mask4, past_kv):
        """activation.py:536-638.  h [B,T,D]; mask4 float [B,H,T,S]; past_kv (pk,pv) or None."""
        c = self.c
        D, H = c.d_model, c.nhead
        hd = D // H
        pre = f"decoder.layers.{l}.self_attn."
        q_in = h.transpose(1, 0)                                             # [T,B,D]
        T, B, _ = q_in.shape
        proj = F.linear(q_in, self.sd[pre + "in_proj_weight"], self.sd[pre + "in_proj_bias"])
        proj = proj.unflatten(-1, (3, D)).unsqueeze(0).transpose(0, -2).squeeze(-2).contiguous()
        q, k, v = proj[0], proj[1], proj[2]
        if self.kv_round_bf16:
            k = k.to(torch.bfloat16).to(torch.float32)
            v = v.to(torch.bfloat16).to(torch.float32)
        q = q.view(T, B * H, hd).transpose(0, 1).view(B, H, T, hd)
        k = k.view(T, B * H, hd).transpose(0, 1).view(B, H, T, hd)
        v = v.view(T, B * H, hd).transpose(0, 1).view(B, H, T, hd)
        present = torch.stack([k, v], dim=0)
        if past_kv is not None:
            k = torch.cat([past_kv[0], k], dim=-2)
            v = torch.cat([past_kv[1], v], dim=-2)
        o = F.scaled_dot_product_attention(q, k, v, mask4, 0.0, is_causal=False)
        o = o.permute(2, 0, 1, 3).contiguous().view(B * T, D)
        o = F.linear(o, self.sd[pre + "out_proj.weight"], self.sd[pre + "out_proj.bias"])
        return o.view(T, B, D).transpose(1, 0), present

    def _layer(self, l, x, mask4, past_kv):
        """transformer.py:321-329 (norm_first), :386-388."""
        pre = f"decoder.layers.{l}."
        D = self.c.d_model
        h = F.layer_norm(x, (D,), self.sd[pre + "norm1.weight"], self.sd[pre + "norm1.bias"], 1e-5)
        a, present = self._mha(l, h, mask4, past_kv)
        x = x + a
        h = F.layer_norm(x, (D,), self.sd[pre + "norm2.weight"], self.sd[pre + "norm2.bias"], 1e-5)
        f = F.linear(F.relu(F.linear(h, self.sd[pre + "linear1.weight"], self.sd[pre + "linear1.bias"])),
                     self.sd[pre + "linear2.weight"], self.sd[pre + "linear2.bias"])
        return x + f, present

    def decoder(self, xy, mask4, past):
        """transformer.py:473-488.  past: list per layer of (k,v) or None -> (out, list of present)."""
        out = xy
        presents = []
        for l in range(self.c.num_decoder_layers):
            out, pres = self._layer(l, out, mask4, None if past is None else past[l])
            presents.append(pres)
        D = self.c.d_model
        out = F.layer_norm(out, (D,), self.sd["decoder.norm.weight"], self.sd["decoder.norm.bias"], 1e-5)
        return out, presents

    def _mask(self, B, S, last_n):
        """Causal 0/-inf mask over the concatenation (voicecraft.py:419-447), rows = last ``last_n``."""
        H = self.c.nhead
        rm = torch.triu(torch.ones(S, S), diagonal=1).bool()
        m = torch.zeros(S, S, dtype=torch.float32).masked_fill_(rm, float("-inf"))
        m = m[-last_n:]
        return m.unsqueeze(0).unsqueeze(0).expand(B, H, last_n, S).contiguous()

    def dec_forward(self, x_in, y_in, cache, last_n=1):
        """voicecraft.py:406-470.  cache: dict(kv=list|None, on=bool).  Returns y-part output."""
        Lx = x_in.size(1)
        xy = torch.cat([x_in, y_in], dim=1)
        B, S, _ = xy.shape
        if not cache["on"]:
            out, _ = self.decoder(xy, self._mask(B, S, S), None)
            return out[:, Lx:]
        if cache["kv"] is None:                       # first pass fills the cache
            out, pres = self.decoder(xy, self._mask(B, S, S), None)
            cache["kv"] = [(p[0], p[1]) for p in pres]
            return out[:, Lx:]
        out, pres = self.decoder(xy[:, -last_n:], self._mask(B, S, last_n), cache["kv"])
        cache["kv"] = [(torch.cat([cache["kv"][l][0], pres[l][0]], dim=-2),
                        torch.cat([cache["kv"][l][1], pres[l][1]], dim=-2))
                       for l in range(len(pres))]
        return out

    def heads(self, y_last):
        """predict_layer stack (voicecraft.py:181-185,1085-1086).  y_last [B,1,D] -> [B,K,V]."""
        outs = []
        for k in range(self.c.n_codebooks):
            h = F.linear(y_last, self.sd[f"predict_layer.{k}.0.weight"], self.sd[f"predict_layer.{k}.0.bias"])
            h = F.gelu(h)
            outs.append(F.linear(h, self.sd[f"predict_layer.{k}.2.weight"], self.sd[f"predict_layer.{k}.2.bias"]))
        return torch.stack(outs, dim=1).squeeze(2)

    # -- per-step state machine -----------------------------------------------------
    def _span_step(self, st, logits, samp, y_cur_len, x_len, noise_fn):
        """One step of sample_helper for a single utterance.

        st: dict(eog=[bool]*K, cur=int, prev=None|int, consec=int, mode='tts'|'edit')
        logits [K,V] (edited in place, as in the reference).  voicecraft.py:1018-1067 / :718-787.
        """
        c = self.c
        K = c.n_codebooks
        tts = st["mode"] == "tts"
        E = (c.eos if c.eos > 0 else c.eog) if tts else c.eog
        n_eog = sum(st["eog"])
        if n_eog == 0:
            for k in range(1, K):
                logits[k][E] = -10000
                logits[k][c.empty_token] = -10000
            if tts and st["cur"] <= c.encodec_sr // 5:
                logits[0][E] = -10000
            self._silence_penalty(logits[0], st["prev"], st["consec"], samp)
            s = sample_rows(logits, samp["top_k"], samp["top_p"], samp["temperature"], noise_fn)
            if st["cur"] < K - 1:
                for jj in range(1, K - st["cur"]):
                    s[-jj, 0] = c.empty_token
            cap = x_len * (c.encodec_sr // 5) if tts else x_len * 10
            if int(s[0, 0]) == E or int(torch.argmax(logits[0], dim=-1)) == E or y_cur_len > cap:
                s[0, 0] = E
                st["eog"][0] = True
            tok0 = int(s[0, 0])
            if tok0 in samp["silence_tokens"] and tok0 == st["prev"]:
                st["consec"] += 1
            else:
                st["consec"] = 0
            st["prev"] = tok0
        else:
            for k in range(n_eog + 1, K):
                logits[k][E] = -10000
                logits[k][c.empty_token] = -10000
            s = sample_rows(logits, samp["top_k"], samp["top_p"], samp["temperature"], noise_fn)
            for k in range(n_eog):
                s[k, 0] = c.empty_token
            s[n_eog, 0] = E
            st["eog"][n_eog] = True
        return s

    @staticmethod
    def _silence_penalty(row0, prev, consec, samp):
        """voicecraft.py:1027-1031."""
        r = samp["stop_repetition"]
        if r > 0 and prev is not None and prev in samp["silence_tokens"] and consec > r:
            if row0[prev] < 0:
                row0[prev] = row0[prev] * (consec - (r - 1))
            else:
                row0[prev] = row0[prev] / (consec - (r - 1))

    def _undelay(self, rows):
        """rows: list of [K] tensors (one per step) -> [K, n-K].  voicecraft.py:1126-1137."""
        K = self.c.n_codebooks
        span = torch.stack(rows, dim=0).transpose(1, 0)
        return torch.stack([span[k][k: span.shape[1] - (K - k)] for k in range(K)], dim=0)

    def _delay(self, seg):
        """[K,T] -> delayed [K,T+K] with empty_token fill (voicecraft.py:254-262)."""
        K, T = seg.shape
        out = torch.full((K, T + K), self.c.empty_token, dtype=seg.dtype)
        for k in range(K):
            out[k, 1 + k: 1 + k + T] = seg[k]
        return out

    # -- inference_tts --------------------------------------------------------------
    @torch.no_grad()
    def inference_tts(self, x, x_lens, y, top_k=-100, top_p=1.0, temperature=1.0, stop_repetition=3,
                      kvcache=1, silence_tokens=(1388, 1898, 131), noise_fn=None, max_steps=None,
                      trace_logits=False):
        c = self.c
        K = c.n_codebooks
        noise_fn = noise_fn or default_noise
        samp = dict(top_k=top_k, top_p=top_p, temperature=temperature, stop_repetition=stop_repetition,
                    silence_tokens=list(silence_tokens))
        assert x.ndim == 2 and x_lens.ndim == 1 and y.ndim == 3
        if c.special_first:
            y = y + int(c.n_special)
        y = y.transpose(2, 1)
        assert y.shape[0] == 1 and y.shape[1] == K
        x_in = self.embed_text(x)
        prompt = self._delay(y[0])[:, : -(K - 1)] if K > 1 else self._delay(y[0])   # :961-967
        emb = self.embed_codes(prompt.unsqueeze(-1)).transpose(1, 0)                 # [1,S,D]
        y_in = self.pos_audio(emb)
        st = dict(eog=[False] * K, cur=0, prev=None, consec=0, mode="tts")
        cache = dict(kv=None, on=bool(kvcache))
        rows = []
        self.logit_trace = [] if trace_logits else None
        while True:
            out = self.dec_forward(x_in, y_in, cache)
            logits = self.heads(out[:, -1:]).squeeze(0)                              # [K,V]
            if c.eos > 0:
                logits[:, c.eog] = -10000.0
            if self.logit_trace is not None:
                self.logit_trace.append(logits.clone())
            s = self._span_step(st, logits, samp, y_in.shape[1], int(x_lens[0]), noise_fn)
            st["cur"] += 1
            rows.append(s.squeeze(-1))
            if sum(st["eog"]) == K or (max_steps is not None and len(rows) >= max_steps):
                break
            emb = torch.cat([emb, self.embed_codes(s).sum(dim=0, keepdim=True).view(1, 1, -1)], dim=1)
            y_in = self.pos_audio(emb)
        if sum(st["eog"]) != K:        # truncated run (max_steps): return raw delayed rows
            return torch.stack(rows, dim=0)
        gen = self._undelay(rows)
        res = torch.cat([y[0], gen], dim=1).unsqueeze(0)
        if c.special_first:
            res = res - int(c.n_special)
            gen = gen - int(c.n_special)
        return res, gen.unsqueeze(0)

    # -- inference_tts_batch (best-of-N, first EOG wins) --------------------------------
    @torch.no_grad()
    def inference_tts_batch(self, x, x_lens, y, top_k=-100, top_p=1.0, temperature=1.0, stop_repetition=3,
                            kvcache=1, batch_size=5, silence_tokens=(1388, 1898, 131), noise_fn=None,
                            max_steps=None, on_step=None):
        c = self.c
        K, Bn = c.n_codebooks, batch_size
        noise_fn = noise_fn or default_noise
        E = c.eos if c.eos > 0 else c.eog
        silence_tokens = list(silence_tokens)
        if c.special_first:
            y = y + int(c.n_special)
        y = y.transpose(2, 1)
        x_in = self.embed_text(x).repeat(Bn, 1, 1)
        prompt = self._delay(y[0])[:, : -(K - 1)] if K > 1 else self._delay(y[0])
        emb = self.embed_codes(prompt.unsqueeze(-1)).transpose(1, 0).repeat(Bn, 1, 1)
        y_in = self.pos_audio(emb)
        x_len = int(x_lens[0])
        eog = [False] * K
        cur = 0
        prev = [None] * Bn
        consec = [0] * Bn
        keep = None
        per_b = [[] for _ in range(Bn)]
        kept_rows = None
        cache = dict(kv=None, on=bool(kvcache))
        while True:
            out = self.dec_forward(x_in, y_in, cache)
            logits = self.heads(out[:, -1:])                                        # [B,K,V]
            n_eog = sum(eog)
            if c.eos > 0:
                logits[:, :, c.eog] = -10000.0
            if n_eog == 0:                                                           # :1270-1308
                logits[:, 1:, E] = -10000
                logits[:, 1:, c.empty_token] = -10000
                if cur <= c.encodec_sr // 5:
                    logits[:, :, E] = -10000
                for b in range(Bn):
                    self._silence_penalty(logits[b, 0], prev[b], consec[b],
                                          dict(stop_repetition=stop_repetition, silence_tokens=silence_tokens))
                s = sample_rows(logits.reshape(Bn * K, -1), top_k, top_p, temperature, noise_fn)
                s = s.reshape(Bn, K, 1)
                for b in range(Bn):
                    if cur < K - 1:
                        for jj in range(1, K - cur):
                            s[b, -jj, 0] = c.empty_token
                    if (int(s[b, 0, 0]) == E or int(torch.argmax(logits[b, 0], dim=-1)) == E
                            or y_in.shape[1] > x_len * (c.encodec_sr // 5)):
                        s[b, 0, 0] = E
                        eog[0] = True
                        keep = b                           # last b in the step wins (:1302)
                    t0 = int(s[b, 0, 0])
                    if t0 in silence_tokens and t0 == prev[b]:
                        consec[b] += 1
                    else:
                        consec[b] = 0
                    prev[b] = t0
            else:                                                                    # :1309-1325
                for k in range(n_eog + 1, K):
                    logits[:, k, E] = -10000
                    logits[:, k, c.empty_token] = -10000
                s = sample_rows(logits.reshape(Bn * K, -1), top_k, top_p, temperature, noise_fn)
                s = s.reshape(Bn, K, 1)
                for k in range(n_eog):
                    s[keep, k, 0] = c.empty_token
                s[keep, n_eog, 0] = E
                eog[n_eog] = True
            cur += 1
            if sum(eog) == 0:
                for b in range(Bn):
                    per_b[b].append(s[b].squeeze(-1))
            elif sum(eog) == 1:
                kept_rows = per_b[keep]
                kept_rows.append(s[keep].squeeze(-1))
            else:
                kept_rows.append(s[keep].squeeze(-1))
            if on_step is not None:
                on_step(cur)
            if sum(eog) == K:
                break
            if max_steps is not None and cur >= max_steps and sum(eog) == 0:
                return None, None            # bounded timing sample (bench.py cpu_baseline), no result assembled
            step_emb = torch.stack([F.embedding(s[:, k], self.sd[f"audio_embedding.{k}.word_embeddings.weight"])
                                    for k in range(K)], dim=1).sum(dim=1)            # [B,1,D]
            emb = torch.cat([emb, step_emb], dim=1)
            y_in = self.pos_audio(emb)
        gen = self._undelay(kept_rows)
        res = torch.cat([y[0], gen], dim=1).unsqueeze(0)
        if c.special_first:
            res = res - int(c.n_special)
            gen = gen - int(c.n_special)
        return res, gen.unsqueeze(0)

    # -- speech editing -------------------------------------------------------------
    def edit_prompt(self, y, spans):
        """Build the editing prompt (voicecraft.py:239-320, 615-683).

        y [K,T] int64; spans list of (start,end).  Returns (tokens [K,T'], mask_pos, mask_val, more_vals,
        non_mask_intervals).
        """
        c = self.c
        K, T = y.shape
        M = len(spans)
        starts = [s for s, _ in spans] + [T]
        ends = [0] + [e for _, e in spans]
        non_mask = list(zip(ends, starts))
        col = lambda tok: torch.full((K, 1), tok, dtype=y.dtype)
        segs = []
        for i, (a, b) in enumerate(non_mask):
            seg = y[:, a:b]
            last = i == len(non_mask) - 1
            if c.eos > 0:
                assert c.reduced_eog
                if last:
                    seg = torch.cat([seg, col(c.eos)], dim=-1)
            elif c.reduced_eog:
                if last:
                    seg = torch.cat([seg, col(c.eog)], dim=-1)
            else:
                seg = torch.cat([seg, col(c.eog)], dim=-1)
            segs.append(seg)
        for (a, b) in spans:
            segs.append(torch.cat([y[:, a:b], col(c.eog)], dim=-1))
        shifted = [self._delay(s) for s in segs]
        assert not c.shuffle_mask_embedding, "shuffle_mask_embedding is a training-time option"
        vals = list(range(c.max_n_spans))[:M]
        mask_val = vals + vals
        pieces, mask_pos, run = [], [], 0
        for j in range(len(shifted) - 1):
            pieces.append(shifted[j])
            run += shifted[j].shape[1]
            mask_pos.append(run)
            pieces.append(col(c.eog))                 # placeholder; embedding is overwritten (:311-320)
            run += 1
        pieces.append(shifted[-1])
        cated = torch.cat(pieces, dim=1)
        cut = mask_pos[M] + 2                         # :672-679
        return cated[:, :cut], mask_pos[: M + 1], mask_val[: M + 1], mask_val[M + 1:], non_mask

    @torch.no_grad()
    def inference(self, x, x_lens, y, mask_interval, top_k=-100, top_p=1.0, temperature=1.0,
                  stop_repetition=-1, kvcache=1, silence_tokens=(1388, 1898, 131), noise_fn=None):
        c = self.c
        K = c.n_codebooks
        noise_fn = noise_fn or default_noise
        samp = dict(top_k=top_k, top_p=top_p, temperature=temperature, stop_repetition=stop_repetition,
                    silence_tokens=list(silence_tokens))
        if c.special_first:
            y = y + int(c.n_special)
        y = y.transpose(2, 1)
        assert y.shape[0] == 1 and y.shape[1] == K
        assert mask_interval.shape == torch.Size((1, mask_interval.shape[1], 2))
        spans = [(int(a), int(b)) for a, b in mask_interval[0]]
        tokens, mask_pos, mask_val, more_vals, non_mask = self.edit_prompt(y[0], spans)
        more_vals = list(more_vals)
        x_in = self.embed_text(x)
        emb = self.embed_codes(tokens.unsqueeze(-1)).transpose(1, 0)                 # [1,T',D]
        emb[0, mask_pos] = self.sd["mask_embedding"][mask_val]
        y_in = self.pos_audio(emb)
        st = dict(eog=[False] * K, cur=0, prev=None, consec=0, mode="edit")
        cache = dict(kv=None, on=bool(kvcache))
        generated, rows = [], []
        last_n = 1
        while True:
            out = self.dec_forward(x_in, y_in, cache, last_n=last_n)
            last_n = 1
            logits = self.heads(out[:, -1:]).squeeze(0)
            if c.eos > 0:
                logits[:, c.eos] = -10000.0
            s = self._span_step(st, logits, samp, y_in.shape[1], int(x_lens[0]), noise_fn)
            st["cur"] += 1
            rows.append(s.squeeze(-1))
            step_emb = self.embed_codes(s).sum(dim=0, keepdim=True).view(1, 1, -1)
            if sum(st["eog"]) == K:
                generated.append(rows)
                rows = []
                st = dict(eog=[False] * K, cur=0, prev=st["prev"], consec=st["consec"], mode="edit")
                if len(more_vals) > 0:                                               # :838-858
                    nxt = more_vals.pop(0)
                    mask_emb = self.sd["mask_embedding"][nxt].view(1, 1, -1)
                    empty_emb = self.embed_codes(torch.full((K, 1), c.empty_token, dtype=torch.long)
                                                 ).sum(dim=0, keepdim=True).view(1, 1, -1)
                    step_emb = torch.cat([step_emb, mask_emb, empty_emb], dim=1)
                    st["consec"], st["prev"] = 0, None
                    last_n = 3
                else:
                    break
            emb = torch.cat([emb, step_emb], dim=1)
            y_in = self.pos_audio(emb)
        pieces = []
        for (a, b), rows_ in zip(non_mask, generated):
            pieces.append(y[0, :, a:b])
            pieces.append(self._undelay(rows_))
        pieces.append(y[0, :, non_mask[-1][0]: non_mask[-1][1]])
        res = torch.cat(pieces, dim=1).unsqueeze(0)
        if c.special_first:
            res = res - int(c.n_special)
        return res
