/* vcb200.h -- C ABI of libvcb200.so, the H100 (sm_90a) codec-LM decode + EnCodec decode engine.
 *
 * Drop-in boundary for the VoiceCraft hot path (SURVEY.md section 8b).  The reference has no FFI of its
 * own (it is pure PyTorch); each entry point below names the reference code it replaces.  Plain pointers
 * and sizes only -- no torch types.  All `dev` pointers are CUDA device pointers owned by the caller;
 * `stream` is a cudaStream_t passed as void* (0 = legacy default stream).  Every function returns 0 on
 * success and a negative value on error; vcb_last_error() then describes it.  Nothing throws across the ABI.
 *
 * Threading: one engine per device; calls on one engine must be serialised by the caller (the reference is
 * single-threaded Python, inference_tts_scale.py:42).  Synchronisation contract, per entry point:
 *   vcb_sample / vcb_decode_step   asynchronous on `stream` (one small pinned H2D copy when the slot list changes, and
 *                                  one when a slot's KV page list grows);
 *                                  the decode loop never blocks the host
 *   vcb_prefill                    once per utterance batch: waits for `stream`, uploads the slot / page / row tables and
 *                                  the groups' sampling parameters with blocking copies, then enqueues the prefill kernels
 *                                  asynchronously
 *   vcb_poll / vcb_read_tokens /   wait for `stream`, then copy state / tokens / log-probabilities to the host
 *   vcb_read_logprobs
 *   vcb_poll_frames(_ex)           enqueues the frame gather on `stream` (_ex: after one small pinned H2D copy of the
 *                                  sources), then waits for `stream` once; the codes stay on the device, the status and
 *                                  per-slot results arrive in one small copy.  _ex reads each edit source's y0 on `stream`
 *   vcb_release                    waits for the device (the slot's KV pages go back to the free list)
 *   vcb_swap_out                   waits for `stream`, copies the slot's state and KV pages to library-owned pinned memory
 *                                  (one gather kernel and one D2H copy on `stream`), waits for `stream` again, then
 *                                  releases the slot as vcb_release does
 *   vcb_swap_in                    waits for `stream`, restores a snapshot with blocking copies and one H2D copy plus one
 *                                  scatter kernel on `stream`, and waits for `stream` before it returns (the snapshot may
 *                                  be freed at once)
 *   vcb_snapshot_free              host only
 *   vcb_create / vcb_load_* / vcb_finalize_weights / vcb_destroy   blocking set-up calls
 * A call that fails leaves no slot, group or KV page held (vcb_prefill validates every prompt before it mutates state).
 *
 * KV pool (DESIGN.md section 3): vcb_config.kv_pool_bytes sizes the page pool; a one-copy prompt holds the pages its
 * positions use and vcb_decode_step grows it by VCB_KV_GROW_PAGES pages at a time.  When the pool cannot cover a step,
 * vcb_decode_step returns VCB_ERR_KV_FULL and changes nothing; the caller frees pages (vcb_release, vcb_swap_out) and
 * calls again.
 */
#ifndef VCB200_H_
#define VCB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vcb_engine vcb_engine;

enum { VCB_MODE_TTS = 0, VCB_MODE_EDIT = 1 };
/* KV cache policy (DESIGN.md sections 2.2, 3): bf16, fp32, or e4m3 with a power-of-two fp32 scale per token and head */
enum { VCB_KV_BF16 = 0, VCB_KV_FP32 = 1, VCB_KV_FP8 = 2 };
/* GEMM weight policy (DESIGN.md section 2.2): bf16, or int8 with a power-of-two fp32 scale per output feature */
enum { VCB_W_BF16 = 0, VCB_W_INT8 = 1 };
/* vcb_decode_step: the KV pool has too few free pages for the listed slots' next positions; nothing was enqueued or taken,
 * and vcb_counter(e, "kv_pages_needed") is how many pages the call lacked */
enum { VCB_ERR_KV_FULL = -3 };
/* pages a one-copy utterance's page list grows by (64 positions each) */
enum { VCB_KV_GROW_PAGES = 4 };
/* largest vcb_config.align_text_cap, and the largest X of vcb_align_monotonic */
enum { VCB_ALIGN_MAX_TEXT = 4096 };

typedef struct vcb_snapshot vcb_snapshot;

/* Model hyper-parameters: the argparse Namespace the reference model is built from
 * (reference config.py:50-84, models/voicecraft.py:106-195). */
typedef struct {
    int32_t d_model, nhead, num_layers, n_codebooks;
    int32_t audio_vocab_size, n_special, text_vocab_rows; /* text_vocab_size + 1 */
    int32_t empty_token, eog, audio_pad_token, eos;       /* eos <= 0: unused */
    int32_t encodec_sr, max_n_spans;
    int32_t max_slots;      /* concurrently open utterances */
    int32_t max_seq_len;    /* text + audio columns per utterance, upper bound: sizes the page tables and the prefill row
                             * tables; KV pages are taken as positions are written */
    int32_t max_new_tokens; /* token-log capacity per utterance */
    int32_t kv_dtype;       /* VCB_KV_BF16 (default), VCB_KV_FP32 or VCB_KV_FP8; vcb_create rejects any other value */
    int32_t device;         /* CUDA device ordinal */
    int32_t weight_dtype;   /* VCB_W_BF16 (default) or VCB_W_INT8 (d_model and audio_vocab_size / 2 multiples of 128);
                             * vcb_create rejects any other value */
    int32_t align_text_cap; /* alignment (DESIGN.md section 4.6): text tokens an alignment row holds, in [0, VCB_ALIGN_MAX_TEXT];
                             * 0 = alignment unavailable.  The alignment log [max_slots][max_seq_len][align_text_cap] fp32 is
                             * allocated by the first prefill that asks for alignment (vcb_counter "align_bytes").  It sits in
                             * what was the padding before kv_pool_bytes: the struct's size and kv_pool_bytes' offset are
                             * unchanged, and a zero-initialised config leaves alignment off.  A caller built against
                             * the older header that fills the struct field by field without zeroing it first must now
                             * set this field (0), or vcb_create may reject or misread the padding's old bytes */
    int64_t kv_pool_bytes;  /* KV page pool: 0 = max_slots * ceil(max_seq_len / 64) pages (every slot can reach max_seq_len);
                             * > 0: floor(kv_pool_bytes / page bytes) pages, a page being 64 positions of K and V in every
                             * layer (vcb_counter "kv_page_bytes"); vcb_create rejects a negative value or one below a page */
} vcb_config;

/* Sampling arguments of inference_tts / inference / inference_tts_batch (voicecraft.py:908-920), then two controls the
 * reference lacks, both off at 0 (DESIGN.md section 2.2):
 *   Repetition-aware sampling (VALL-E 2), ras_window = W in [1, 256], ras_threshold = c in [1, W]: per slot and codebook,
 *   the token t drawn as the reference draws it (masks, temperature, top-k, top-p, argmax(p / q1)) is redrawn as
 *   argmax(p_full / q2) when t occurs >= c times among the last min(W, steps of the current generation) tokens of that
 *   codebook in the slot's token log.  p_full is the softmax of the row after the reference's masks and temperature,
 *   before top-k / top-p.  Tokens the state machine forces afterwards overwrite as before, and the end-token triggers
 *   see the final token.  A group with ras_window > 0 consumes two draws of [n_copies*K, V] per step whether or not a
 *   redraw fires (q1 at the stream's offset, q2 at the next), so it needs the device generator (vcb_prompt.rng_threads)
 *   and caller noise is rejected for it.
 *   Length bounds in generated frames (codebook-0 sampling steps of the TTS output or of each edit span): min_frames > 0
 *   masks the end token on codebook 0 while fewer have been generated; max_frames > 0 forces it at max_frames, as the
 *   reference's length cap does (the cap still applies).  min_frames <= max_frames when both are set. */
typedef struct {
    int32_t top_k;
    float top_p;
    float temperature;
    int32_t stop_repetition;
    int32_t n_silence;
    int32_t silence_tokens[8];
    int32_t ras_window;
    int32_t ras_threshold;
    int32_t min_frames;
    int32_t max_frames;
} vcb_sampling;

/* One utterance (or one best-of-N group) to prefill.  `y_tokens` is the already arranged prompt:
 * the delayed pattern of voicecraft.py:961-972 (TTS) or the segment/placeholder layout of :615-683 (edit),
 * [y_len][n_codebooks] int64 on the device. */
typedef struct {
    int32_t slot;            /* first slot; a group occupies slot .. slot+n_copies-1 */
    int32_t n_copies;        /* 1, or batch_size of inference_tts_batch (voicecraft.py:1329-1343): a best-of-N group, prefilled
                              * once; its copies share the KV pages of the prompt's full pages [0, (x_len+y_len)/64) and
                              * each get a copy of the partial tail page and of the last hidden state */
    int32_t mode;            /* VCB_MODE_TTS / VCB_MODE_EDIT */
    int32_t x_len;
    const int64_t* text_ids_dev;    /* [x_len] */
    int32_t y_len;
    const int64_t* y_tokens_dev;    /* [y_len][K] */
    const int32_t* mask_rows_dev;   /* [y_len] or NULL: >= 0 -> column embedding = mask_embedding[row] (:311-320) */
    int32_t n_more_spans;           /* edit: masked spans after the first (voicecraft.py:681, 838-858) */
    int32_t more_mask_rows[8];      /* mask_embedding row of each further span (at most 7 further spans: 8 per utterance) */
    /* Sampling noise generated by the engine itself (vcb_sample / vcb_decode_step with exp_noise_dev == NULL): the
     * utterance (or best-of-N group) owns the Philox4x32-10 stream of a torch CUDA generator at (rng_seed, rng_offset)
     * and every sampling step consumes exactly what `torch.multinomial(softmax(logits[n_copies*K, V]), 1)` consumes
     * from it (voicecraft.py:85; ATen: empty_like(p).exponential_(1), distribution_nullary_kernel).
     * rng_threads = 256 * grid of that ATen launch = 256 * min(ceil(n_copies*K*V / 256), SMs * (maxThreadsPerSM / 256));
     * 0 = no device generator, the caller passes the noise. */
    uint64_t rng_seed, rng_offset;
    int32_t rng_threads, rng_reserved;
    /* The group's own sampling parameters, used by vcb_sample / vcb_decode_step called with sp == NULL; NULL: none (those
     * calls then reject the group's slots).  Rejected with the prompt: n_silence outside [0, 8], a temperature that is not
     * finite and > 0, a NaN top_p, sampling controls outside the ranges vcb_sampling states, ras_window > 0 with
     * rng_threads == 0. */
    const vcb_sampling* sampling;
    /* Alignment (DESIGN.md section 4.6): host array [num_layers] of head bitmasks, or NULL (off).  Each audio row of the
     * group's copies -- the prompt's in vcb_prefill, each step's in vcb_decode_step -- records at its position the mean over
     * the selected (layer, head) pairs of that head's attention weights on the x_len text keys (vcb_read_alignment).  The
     * probe only reads: tokens, log-probabilities, logits and KV bytes are those of a run without it.  Rejected with the
     * prompt: a bit >= nhead, no bit set, x_len > vcb_config.align_text_cap, VCB_MODE_EDIT. */
    const uint32_t* align_heads;
} vcb_prompt;

/* Source of an edit slot's output frames for vcb_poll_frames_ex: the original codes y0 [K][T] int64 on the device, as the
 * engine saw them (the codes the prompt was built from), and the masked spans [start, end) in ascending order.  A TTS slot
 * takes { NULL, 0, 0 }. */
typedef struct {
    const int64_t* orig_dev;
    int32_t T;
    int32_t n_spans;
    int32_t spans[8][2];
} vcb_edit_source;

/* Per-slot status returned by vcb_poll. */
typedef struct {
    int32_t done;      /* 1: generation finished (all codebooks ended, all spans); 2: stopped, token-log / KV capacity exhausted */
    int32_t forced;    /* >0: the next decode step feeds a forced embedding and consumes no noise */
    int32_t n_steps;   /* sampling steps recorded so far */
    int32_t keep;      /* best-of-N: member index whose tokens are the result (-1 while undecided) */
    int32_t n_spans_done;
    int32_t span_ends[8];
    int32_t reserved;
    uint64_t rng_offset; /* Philox offset of the group's generator after the steps recorded so far */
} vcb_status;

const char* vcb_last_error(void);
int vcb_version(void);

/* ---- life cycle: replaces VoiceCraft.__init__ / load_state_dict (voicecraft.py:106-195) ------------ */
int vcb_create(const vcb_config* cfg, vcb_engine** out);
int vcb_destroy(vcb_engine* e);
/* key = reference state_dict key (SURVEY.md section 8b), data = fp32 device or host pointer, row-major. */
int vcb_load_weight(vcb_engine* e, const char* key, const float* data, const int64_t* shape, int32_t ndim,
                    int32_t is_device_ptr);
/* sinusoidal table of SinePositionalEmbedding (embedding.py:67-92), fp32 [rows][d_model] */
int vcb_load_pe(vcb_engine* e, const float* data, int32_t rows, int32_t is_device_ptr);
int vcb_finalize_weights(vcb_engine* e);   /* packs the GEMM operands (bf16 or int8), builds TMA descriptors */

/* ---- decode: replaces dec_forward + the sampling loop (voicecraft.py:406-470, 1018-1120) ----------- */
/* validates every prompt first (a group needs max_pages + (n_copies-1) * (max_pages - full prompt pages) free KV pages),
 * then runs one prefill per prompt, whatever its n_copies */
int vcb_prefill(vcb_engine* e, const vcb_prompt* prompts, int32_t n, void* stream);
/* final LayerNorm + logit heads + fused sampler on the last hidden state of each listed slot.
 * exp_noise_dev: [n * K][V] fp32 Exp(1) noise, the draw torch.multinomial makes (voicecraft.py:85); NULL = every listed
 * slot draws from its own generator (vcb_prompt.rng_*), one stream per utterance / best-of-N group.
 * sp: the sampling parameters of every listed slot; NULL = each slot uses its group's (vcb_prompt.sampling), and a slot whose
 * group was prefilled without them is rejected before anything is enqueued.  Also rejected before anything is enqueued:
 * exp_noise_dev set while a listed slot samples with ras_window > 0, an sp whose controls vcb_prefill would reject. */
int vcb_sample(vcb_engine* e, const int32_t* slots, int32_t n, const float* exp_noise_dev,
               const vcb_sampling* sp, void* stream);
/* one transformer step on the embeddings produced by the previous sample, then vcb_sample.  Before it enqueues anything,
 * every listed one-copy slot gets a page for the position it writes (the host bounds it by the slot's prompt length plus the
 * steps issued since, without reading the device), VCB_KV_GROW_PAGES at a time up to ceil(max_seq_len / 64); the new page-table
 * entries go up in one small pinned H2D copy on `stream`.  Returns VCB_ERR_KV_FULL, having done nothing, when the free list
 * cannot cover that. */
int vcb_decode_step(vcb_engine* e, const int32_t* slots, int32_t n, const float* exp_noise_dev,
                    const vcb_sampling* sp, void* stream);
int vcb_poll(vcb_engine* e, const int32_t* slots, int32_t n, vcb_status* out_host, void* stream);
/* copies the raw (still delayed) sampled tokens [n_steps][K] int32 to host memory */
int vcb_read_tokens(vcb_engine* e, int32_t slot, int32_t* out_host, int32_t max_steps, void* stream);
/* copies the log-probabilities of those tokens [n_steps][K] fp32 to host memory, row for row and entry for entry as
 * vcb_read_tokens.  Entry [t][k] = log p_model(token | context) under the softmax of that step's raw logit row of
 * codebook k (the heads' output with bias, what vcb_debug_logits reports): taken before the end / empty masks, the
 * silence-repetition scaling, temperature, top-k and top-p, so it does not depend on the sampling parameters.  Forced
 * tokens (the first steps' empty tokens, the end-token cascade, a forced end token) get the log-probability of the token
 * written.  Edit hand-over steps write no row.  Computed by the sampler in fp32 (DESIGN.md section 2.2). */
int vcb_read_logprobs(vcb_engine* e, int32_t slot, float* out_host, int32_t max_steps, void* stream);
/* waits for `stream`, then copies the alignment rows of positions first_pos .. first_pos+n_pos-1 of a slot prefilled with
 * align_heads to host memory: out_host [n_pos][x_len] fp32, x_len the slot's.  Row p holds what the probe recorded for the
 * row at position p (its attention weights on the text keys, averaged over the selected heads); rows of positions the slot
 * has not written, and text positions (< x_len), are unspecified.  Rejected: a slot that is not open or has no alignment,
 * first_pos < 0, n_pos < 1, first_pos + n_pos > max_seq_len. */
int vcb_read_alignment(vcb_engine* e, int32_t slot, float* out_host, int32_t first_pos, int32_t n_pos, void* stream);
/* Monotonic alignment search (Glow-TTS) on the device, one CTA: logp_dev [T][X] fp32 -> durations_dev [X] int32 summing to T,
 * the path from (0, 0) to (T-1, X-1) that assigns each frame one token, never goes back, and gives every token a frame,
 * maximising the fp32 sum of logp along it (accumulated frame by frame).  Ties stay on the current token.  Asynchronous on
 * `stream` (a stream-ordered scratch of T * X bytes).  Rejected: T < X, X < 1, X > VCB_ALIGN_MAX_TEXT, null pointers. */
int vcb_align_monotonic(const float* logp_dev, int32_t T, int32_t X, int32_t* durations_dev, void* stream);
/* closes slots slot .. slot+n_copies-1 (slots that are not open are skipped); a KV page goes back to the free list when
 * the last slot holding it is released, and a group's id with its last slot, in any release order */
int vcb_release(vcb_engine* e, int32_t slot, int32_t n_copies);
/* Swap a one-copy utterance out to host memory and back, byte for byte (DESIGN.md section 3).  vcb_swap_out copies what the
 * slot's continuation depends on -- the K and V slabs of its written pages in every layer, its SlotState and GroupState
 * (Philox offset included), its sampling parameters, token-log and log-probability rows [0, n_steps), its next-input and last-hidden rows,
 * its alignment rows [0, seq_len) when it aligns, and the slot's host record -- into a snapshot, then releases the slot.  Rejected before anything changes: a slot that is not
 * open or belongs to a best-of-N group.
 * vcb_swap_in restores a snapshot of this engine into the free `slot` on newly taken pages and a free group id; rejected
 * before anything changes: a snapshot of another engine, a slot that is open, no free group, fewer free pages than
 * vcb_snapshot_pages.  The snapshot stays valid (and owned by the caller) either way.
 * Snapshots hold pinned host memory (counted in "live_bytes" / "live_handles") until vcb_snapshot_free.  The engine keeps
 * a device staging region as large as the largest utterance it swapped, at most ceil(max_seq_len / 64) pages ("swap_stage_bytes"), until
 * vcb_destroy. */
int vcb_swap_out(vcb_engine* e, int32_t slot, vcb_snapshot** out, void* stream);
int vcb_swap_in(vcb_engine* e, const vcb_snapshot* snap, int32_t slot, void* stream);
int32_t vcb_snapshot_pages(const vcb_snapshot* snap);     /* KV pages vcb_swap_in takes */
int vcb_snapshot_free(vcb_snapshot* snap);                /* NULL: nothing */
/* Streaming: vcb_poll, plus the newly final frames of the listed slots, un-delayed, as codec codes.
 * Waits for `stream` once.  For listed slot i: final_host[i] = frames of the slot that are final (frame t is final once the
 * token log holds rows up to t+K-1 and rows[t][0] is not the end token; for a finished generation n_steps-K).
 * codes_dev[i][k][t] = tok_log[slot][from_host[i]+t+k][k] - code_offset for t < min(final - from, max_frames), 0 after.
 * bad_host[3*i..] = (frame, codebook, token) of the first written code outside [0, bins) (lowest frame, then codebook),
 * or (-1, -1, -1); frame counts from the start of the generation, token is the token-log entry.
 * Rejected before anything is enqueued or written: n < 1, max_frames < 1, a slot that is not open, an edit slot, a slot of
 * a best-of-N group, from_host[i] < 0 or above the final frames this call last reported for the slot (0 after prefill). */
int vcb_poll_frames(vcb_engine* e, const int32_t* slots, int32_t n, const int32_t* from_host, int32_t max_frames,
                    int64_t code_offset, int64_t bins, int64_t* codes_dev /*[n][K][max_frames]*/,
                    vcb_status* status_host, int32_t* final_host, int32_t* bad_host, void* stream);
/* vcb_poll_frames that also streams edit slots, given one source per listed slot (src[i]).  An edit's output is
 *   res = y0[:, 0:s1] ++ G1 ++ y0[:, e1:s2] ++ ... ++ GM ++ y0[:, eM:T]
 * with Gj the un-delayed token-log rows [span_ends[j-1], span_ends[j]) (the end token in codebook 0 is eog).  With
 * d = n_spans_done, the final output frames are the original pieces 0..d, the generated spans before d and, within span d,
 * the frames final by the TTS rule applied to the rows since span_ends[d-1]; all of them once every span is done.
 * codes_dev[i][k][t] = output frame from_host[i]+t of codebook k - code_offset, from y0 or the token log; bad_host reports
 * the y0 or token-log entry.  Everything else is vcb_poll_frames'.  Rejected before anything is enqueued or written: what
 * vcb_poll_frames rejects except edit slots, src == NULL, an edit slot without a source (n_spans == 0 or orig_dev NULL),
 * n_spans different from the slot's prompt, spans not ascending / overlapping / outside [0, T], a TTS slot given a source. */
int vcb_poll_frames_ex(vcb_engine* e, const int32_t* slots, int32_t n, const vcb_edit_source* src, const int32_t* from_host,
                       int32_t max_frames, int64_t code_offset, int64_t bins, int64_t* codes_dev /*[n][K][max_frames]*/,
                       vcb_status* status_host, int32_t* final_host, int32_t* bad_host, void* stream);

/* debug / parity hooks */
int vcb_debug_logits(vcb_engine* e, float* out_dev, int32_t n_rows);   /* last sampled logits [n*K][V] (pre-edit) */
/* the Exp(1) values the sampler generates for a draw of `numel` elements at (seed, offset): must equal
 * torch.empty(numel, device="cuda").exponential_(1) under that generator state (tests/test_gpu_parity.py) */
int vcb_debug_exponential(float* out_dev, int64_t numel, uint64_t seed, uint64_t offset, int32_t threads, void* stream);
/* one sampling step of the fused sampler (sampler_kernel, launched through the engine's SamplerArgs) over n rows, each a
 * one-member group with codebooks 0..K-1.  logits_dev [n][K][V] fp32 is copied into the engine's padded layout (column
 * k*Vpad + v, pad columns set to about +3e29); noise_dev [n*K][V] Exp(1), or NULL: every row draws [K][V] from the Philox
 * stream at (seed, offset, rng_threads), as with vcb_prompt.rng_*.  The next-input embedding reads zero tables
 * [K][V+2][32], so empty_token and eog may lie in [0, V+2); eos <= 0 is unused, else in [1, V+2).
 * state_host [n][7] = {mode, n_eog, cur_num_gen, prev_token (-1: none), consec, x_len, y_len} before the step;
 * out: tokens_host [n][K] (the row written to the token log), state_out_host [n][4] = {prev_token, consec, n_eog, done}.
 * Rejected before anything is allocated or launched: n < 1, K outside [1, 8], V outside [1, 3072], a special id out of
 * range, mode not in {0, 1}, n_eog outside [0, K), x_len < 0, y_len outside [0, 65536).  Synchronous. */
int vcb_debug_sampler(const float* logits_dev, const float* noise_dev, uint64_t seed, uint64_t offset, int32_t rng_threads,
                      const vcb_sampling* sp, int32_t n, int32_t K, int32_t V, int32_t empty_token, int32_t eog, int32_t eos,
                      int32_t encodec_sr, const int32_t* state_host, int32_t* tokens_host, int32_t* state_out_host);
/* vcb_debug_sampler that also returns lp_host [n][K]: the log-probability the step stores with each written token (as
 * vcb_read_logprobs reports it).  Tokens and state are vcb_debug_sampler's bit for bit; a written token id >= V gets -inf.
 * Rejected as vcb_debug_sampler, and lp_host == NULL. */
int vcb_debug_sampler_lp(const float* logits_dev, const float* noise_dev, uint64_t seed, uint64_t offset,
                         int32_t rng_threads, const vcb_sampling* sp, int32_t n, int32_t K, int32_t V, int32_t empty_token,
                         int32_t eog, int32_t eos, int32_t encodec_sr, const int32_t* state_host, int32_t* tokens_host,
                         int32_t* state_out_host, float* lp_host);
/* vcb_debug_sampler_lp with repetition-aware sampling on (sp->ras_window = W >= 1): hist_host [n][K][W] is each row's
 * token history per codebook, oldest first, of which the last min(W, cur_num_gen) entries are the token-log rows ahead of
 * the step.  noise2_dev [n*K][V] is the second Exp(1) plane (q2), given exactly when noise_dev is; with both NULL the rows
 * draw q1 at (seed, offset) and q2 at the next offset of the stream, as the engine does.  redrew_host [n][K] out: 1 where
 * the redraw fired, else 0.  lp_host may be NULL.  Rejected as vcb_debug_sampler, and: ras_window < 1, sampling controls
 * the engine rejects, hist_host or redrew_host NULL, exactly one of noise_dev / noise2_dev NULL, cur_num_gen < 0. */
int vcb_debug_sampler_ras(const float* logits_dev, const float* noise_dev, const float* noise2_dev, uint64_t seed,
                          uint64_t offset, int32_t rng_threads, const vcb_sampling* sp, int32_t n, int32_t K, int32_t V,
                          int32_t empty_token, int32_t eog, int32_t eos, int32_t encodec_sr, const int32_t* state_host,
                          const int32_t* hist_host, int32_t* tokens_host, int32_t* state_out_host, float* lp_host,
                          int32_t* redrew_host);
int vcb_debug_gemm(const float* W_dev /*[N][K]*/, const float* X_dev /*[B][K]*/, float* out_dev /*[B][N]*/, int32_t N,
                   int32_t K, int32_t B, int32_t splits /*<=0: auto*/, int32_t simt);
/* the int8 weight rule of vcb_finalize_weights on fp32 W [N][K]: q_out [N][K] int8 and e_out [N] with W_deq = q * 2^e.
 * Synchronous. */
int vcb_debug_weight_quantize(const float* W_dev, int32_t N, int32_t K, int8_t* q_out, int32_t* e_out);
/* vcb_debug_gemm through the int8-weight decode GEMM: W quantized by that rule (out = X W_deq^T), K % 128 == 0 */
int vcb_debug_gemm_w8(const float* W_dev /*[N][K]*/, const float* X_dev /*[B][K]*/, float* out_dev /*[B][N]*/, int32_t N,
                      int32_t K, int32_t B, int32_t splits /*<=0: auto*/);
/* same check for the rows-as-M prefill GEMM (csrc/gemm_rows.cu): any number of rows, N % 128 == 0, K % 64 == 0 */
int vcb_debug_gemm_rows(const float* W_dev /*[N][K]*/, const float* X_dev /*[rows][K]*/, float* out_dev /*[rows][N]*/,
                        int32_t N, int32_t K, int32_t rows);
/* paged attention of the decode / prefill path (attn_rows_kernel) with the engine's launch decisions (chunk count, grid,
 * balance): out[r][h*hd + e] = hi + lo of softmax(q[r][h] . K^T / sqrt(hd)) V over keys 0..pos[r] of row r's pages.
 * kpool / vpool: [page][H] slabs of kv_dtype (VCB_KV_*): [64][hd] bf16 or fp32 elements, or [64][hd] e4m3 bytes followed by
 * [64] fp32 scales.  Pages of row r: row_pages[r][*] (decode) or, with
 * row_pages null, page_table[row_slot[r]][*] (prefill); both max_pages wide.  pos[r] = -1: inactive row, out[r] untouched.
 * chunk_pages <= 0: the engine default; the workspace is sized for max_pages as the engine sizes it for max_seq_len.
 * `repeats` launches run on the same workspace and arrival counters. */
int vcb_debug_attention(const float* q_dev /*[rows][H][hd]*/, const void* kpool_dev, const void* vpool_dev, int32_t kv_dtype,
                        const int32_t* row_pages_dev, const int32_t* page_table_dev, const int32_t* row_slot_dev,
                        const int32_t* pos_dev, int32_t rows, int32_t H, int32_t hd, int32_t max_pages, int32_t chunk_pages,
                        int32_t balance, int32_t repeats, float* out_dev /*[rows][H*hd]*/);
/* the same over row groups (attn_rows_kernel<.., GMAX>, the decode step's instantiation for best-of-N groups), row-pages form:
 * group g = rows group_first[g] .. group_first[g+1]-1 (host arrays, group_first[0] = 0, group_first[n_groups] = rows), whose
 * first group_shared[g] pages are one page list: loaded once per group, head and chunk; groups larger than the kernel's GMAX
 * are split.  Rejected on the host: groups that do not tile the rows, members whose first group_shared[g] page ids differ,
 * members whose positions are neither equal nor -1.  Every row's output equals vcb_debug_attention's bit for bit. */
int vcb_debug_attention_groups(const float* q_dev, const void* kpool_dev, const void* vpool_dev, int32_t kv_dtype,
                               const int32_t* row_pages_dev, const int32_t* pos_dev, int32_t rows, int32_t H, int32_t hd,
                               int32_t max_pages, int32_t chunk_pages, int32_t balance, int32_t repeats,
                               float* out_dev /*[rows][H*hd]*/, const int32_t* group_first, const int32_t* group_shared,
                               int32_t n_groups);
/* the attention phase of the persistent decode-step kernel (csrc/mega_step.cu, VCB_MEGA=1) alone, through its cooperative
 * launch: out[r][h*128 + e] = hi + lo of softmax over keys 0..pos[r]-1 of row r's pages (row_pages[r][*], max_pages wide)
 * and the current key knew[r][h] / value vnew[r][h] at position pos[r], scores q[r][h] . k / sqrt(128).  kv_dtype
 * VCB_KV_BF16 or VCB_KV_FP32 (the kernel has no fp8 path); hd = 128.  pos[r] = -1: inactive row, whose image is left as
 * filled (every bit set), so out[r] reads back NaN.  Rows 1..16 run the kernel's BPAD 16 instantiation, 17..32 BPAD 32.
 * Work items are chunks of 4 pages of one (row, head); CTA c of a grid of G takes the chunks that start in its share
 * [c*U/G, (c+1)*U/G) of the U (row, head, page) units.  An item of up to 16 chunks (pos < 4096) that one CTA owns folds
 * on chip; an item shared between CTAs, or of more chunks, folds its chunk states through a workspace.
 * Launch i runs on grids[i] CTAs (host array, `launches` entries), all on one workspace and one set of arrival counters;
 * the image is refilled before each launch, and after each launch every arrival counter must be back at 0 (else -1).
 * Rejected on the host before anything is allocated or launched: rows outside [1, 32], H < 1, max_pages < 1, a kv_dtype
 * other than bf16 / fp32, a grid outside [1, the kernel's co-resident CTAs], a position beyond max_pages pages and
 * H * rows * max_pages * (grid + 1) >= 2^31 (the kernel's work split is 32-bit).  Synchronous. */
int vcb_debug_mega_attention(const float* q_dev /*[rows][H][128]*/, const float* knew_dev /*[rows][H][128]*/,
                             const float* vnew_dev, const void* kpool_dev, const void* vpool_dev, int32_t kv_dtype,
                             const int32_t* row_pages_dev /*[rows][max_pages]*/, const int32_t* pos_dev, int32_t rows,
                             int32_t H, int32_t max_pages, const int32_t* grids, int32_t launches,
                             float* out_dev /*[rows][H*128]*/);
/* the alignment probe of vcb_prompt.align_heads alone, one layer: for each row r with pos[r] >= x_len, out[r][j] (j < x_len)
 * = mean over the heads h of head_mask of softmax_j(q[r][h] . k_j / sqrt(hd)) over the keys 0..pos[r] of row r's pages
 * (row_pages[r][*], max_pages wide; pools as vcb_debug_attention's).  Rows with pos[r] < x_len are left untouched.
 * Rejected: H outside [1, 32], hd not 64 / 128, an empty mask or one with a bit >= H, x_len outside [1, VCB_ALIGN_MAX_TEXT].
 * Synchronous. */
int vcb_debug_align_probe(const float* q_dev /*[rows][H][hd]*/, const void* kpool_dev, int32_t kv_dtype,
                          const int32_t* row_pages_dev, const int32_t* pos_dev, int32_t rows, int32_t H, int32_t hd,
                          int32_t max_pages, uint32_t head_mask, int32_t x_len, float* out_dev /*[rows][x_len]*/);
/* the fp8 KV quantizer of the QKV epilogues on `rows` rows of hd fp32 values (hd 64 or 128): out gets the e4m3 bytes
 * [rows][hd], then the fp32 scales [rows].  Synchronous. */
int vcb_debug_kv_quantize(const float* x_dev /*[rows][hd]*/, int32_t rows, int32_t hd, uint8_t* out_dev);
/* raw KV slabs of pages first_page .. first_page+n_pages-1 of a slot's page list in layer `layer`, any policy:
 * k_host / v_host [n_pages][H][slab bytes] (slab: [64][hd] elements, fp8 followed by [64] fp32 scales).  Waits for the
 * device. */
int vcb_debug_kv_pages(vcb_engine* e, int32_t layer, int32_t slot, int32_t first_page, int32_t n_pages, void* k_host,
                       void* v_host);
/* What the last vcb_prefill (its last chunk) / vcb_sample / vcb_decode_step left in one of its buffers, as fp32
 * out_dev [rows][width] with hi/lo planes summed (the persistent kernel's tiled images included), rows <= that pass's rows:
 *   "x"     the residual rows (vcb_sample: each listed slot's last prefill hidden state)       width d
 *   "q"     the attention queries of the last QKV stage (not vcb_sample)                        width d
 *   "opnd"  the operand of the next QKV or FFN1 GEMM: LN(x) unfolded, gamma * x folded         width d
 *   "att"   the attention output                                                               width d
 *   "ffn"   the FFN1 output after ReLU                                                         width 4 d
 *   "heads" the first logit-head stage after GELU, codebooks side by side                      width K * audio_vocab/2
 * With vcb_set_option(e, "stop_stage", s) the three calls run their first s stages only: stage 5 l + {0 QKV, 1 attention,
 * 2 out-projection, 3 FFN1, 4 FFN2} of layer l, then 5 L (final LayerNorm + first head stage) and 5 L + 1 (second head
 * stage), the persistent kernel's phases; an unfolded pass's LayerNorm belongs to the GEMM stage after it.  A stopped call
 * launches nothing after stage s (no sampler, no last-row gather, no best-of-N fork) and leaves its slots mid-step: release
 * them.  A prefill of several chunks runs all but its last chunk whole.  s = 0 (the default) runs everything, bit for bit
 * as without the option.  Unknown names and rows above the last pass's are rejected.  Waits for the device. */
int vcb_debug_stage_read(vcb_engine* e, const char* name, float* out_dev, int32_t rows);
/* the decode pair "out-projection -> LN2 -> FFN1" on the per-kernel GEMM path (B <= 128 rows, d % 128 == 0, d <= 4096):
 *   x_new = x + a W1^T + b1;  y = LN(x_new; gamma, beta, eps 1e-5) W2^T + b2, ReLU'd when relu != 0 (EPI_ACT, hi + lo)
 * fold = 1: the residual GEMM emits gamma * x_new and per-tile row statistics, the second GEMM folds the LayerNorm into its
 * epilogue (decode steps); fold = 0: ln_rows_kernel, then a plain GEMM (prefill).  splits* <= 0: the engine's choice. */
int vcb_debug_fold_chain(const float* x_dev /*[B][d]*/, const float* a_dev /*[B][d]*/, const float* W1_dev /*[d][d]*/,
                         const float* b1_dev, const float* gamma_dev, const float* beta_dev, const float* W2_dev /*[N2][d]*/,
                         const float* b2_dev, int32_t B, int32_t d, int32_t N2, int32_t relu, int32_t fold, int32_t splits1,
                         int32_t splits2, float* xnew_dev /*[B][d]*/, float* y_dev /*[B][N2]*/);
/* debug timeline: enable=1 starts recording (tag, globaltimer ns) pairs from CTA 0 of each kernel; enable=0 stops and
 * copies up to max_records pairs to out_host.  The marks are compiled in only by `make TIMELINE=1` (even disabled they cost
 * 2.7 % of a decode step); a default build returns an error for enable != 0. */
int vcb_timeline(int32_t enable, uint64_t* out_host, int32_t max_records, int32_t* n_out);
/* micro-benchmark of the GEMM kernel alone (HBM-resident weights): average microseconds per launch; splits <= 0: the
 * engine's choice, stages <= 0 or the kernel's own (see vcb_gemm_launch_shape) */
int vcb_bench_gemm(int32_t N, int32_t K, int32_t B, int32_t splits, int32_t stages, int32_t pdl, int32_t iters,
                   int32_t ncopies, float* us_out);
/* the launch shape the decode GEMM takes for N x K at B rows: out[0] = split count (= cluster size) after the fallback to
 * the largest cluster the device can place, out[1] = pipeline stages.  splits <= 0: the engine's choice; stages > 0 must
 * be the depth the kernel for B rows is built with (one per row padding); cluster_cap > 0: as if the device could place
 * no cluster larger than that.  Fails as the launch would (split count not a power of two <= 16, not leaving 2 rows per
 * CTA or a k-block per split). */
int vcb_gemm_launch_shape(int32_t N, int32_t K, int32_t B, int32_t splits, int32_t stages, int32_t cluster_cap,
                          int32_t* out /*[2]*/);
/* the persistent kernel's ring configuration for VCB_MEGA_NS / _NB / _FLIGHT = ns / nb / flight, as an engine built with
 * them runs it: out = {ns, nb, flight clamped to [1, ns]}.  Fails, as building the engine does, unless 2 <= ns <= 12,
 * 3 <= nb <= 8 and ns * 16 KB + nb * 8 KB <= 224 KB. */
int vcb_mega_ring_config(int32_t ns, int32_t nb, int32_t flight, int32_t* out /*[3]*/);
/* debug timeline of the persistent decode-step kernel (first call enables it): [2 CTAs][n_phases][8 events] globaltimer ns */
int vcb_debug_mega_timeline(vcb_engine* e, uint64_t* out_host, int32_t max_records, int32_t* n_phases);
/* "gemm_simt", "pdl", "profile", "stop_stage" (0 .. 5 L + 2, see vcb_debug_stage_read) */
int vcb_set_option(vcb_engine* e, const char* name, int32_t value);
/* profile mode: summed device ms and launch counts per kernel class since the last read
 * (0 gemm, 1 attention, 2 layernorm/reduce, 3 bias/act/qkv finish, 4 sampler, 5 misc) */
int vcb_profile_read(vcb_engine* e, double* ms_by_class, int64_t* count_by_class, int32_t n_classes);
/* "launches", "kv_bytes", "kv_pages_free", "kv_pages_total" (pool size), "kv_pages_needed" (pages the last refused
 * vcb_decode_step lacked), "kv_page_bytes" (one page: 64 positions of K and V in every layer), "align_bytes" (the alignment log and masks, 0 until a prefill asked for alignment), "swap_stage_bytes" (device
 * staging of the swap kernels), "prefill_rows" (rows through the prefill since create), "wide_rows" (rows per pass of
 * the rows-as-M prefill, fixed by its first use; 0 until a prefill took that path), "weight_bytes" (device
 * bytes of the packed GEMM operands with their int8 scales, and the int8 prefill scratch once a prefill allocated it),
 * "mega_grid" (the persistent kernel's grid, 0: not available), "mega_ns" / "mega_nb" / "mega_flight" / "mega_pf" (the ring
 * configuration it runs, 0 without it), ...; "live_bytes" / "live_handles" (any e, NULL included): device and pinned bytes, and allocations
 * plus events, the library holds now across every engine, codec engine and stream of the process */
int64_t vcb_counter(vcb_engine* e, const char* name);

/* ---- delayed codebook pattern on the device: Pattern.build_pattern_sequence
 *      (codebooks_patterns.py:151-176 with DelayedPatternProvider :336-352, delays = 0..K-1) -------- */
int vcb_delay_pattern(const int64_t* z_dev /*[B][K][T]*/, int64_t* out_dev /*[B][K][T+K]*/, int32_t B, int32_t K,
                      int32_t T, int64_t special_token, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VCB200_H_ */
