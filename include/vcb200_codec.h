/* vcb200_codec.h -- C ABI of the EnCodec decoder (token -> waveform) and encoder (waveform -> token) in libvcb200.so.
 *
 * Replaces AudioTokenizer.decode (reference data/tokenizer.py:131-133), i.e. audiocraft's
 * EncodecModel.decode = ResidualVectorQuantizer.decode + SEANetDecoder, with hand-written sm_90a kernels
 * (RVQ gather-sum, implicit-GEMM Conv1d / ConvTranspose1d with fused ELU / bias / residual, LSTM).
 * Same conventions as vcb200.h: plain pointers, 0 on success, vcb_last_error() for the message.
 */
#ifndef VCB200_CODEC_H_
#define VCB200_CODEC_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct enc_engine enc_engine;

/* SEANet / RVQ hyper-parameters (audiocraft config `seanet.*`, `rvq.*`; defaults of the 16 kHz / 50 Hz / 4x2048 codec) */
typedef struct {
    int32_t n_q, bins, dimension, n_filters;
    int32_t n_ratios, ratios[8];
    int32_t kernel_size, last_kernel_size, residual_kernel_size, dilation_base, n_residual_layers, compress;
    int32_t lstm;          /* LSTM layers (0 = none) */
    int32_t causal;        /* causal convolutions (left padding / right trim) */
    int32_t pad_reflect;   /* 1 = 'reflect' padding, 0 = zeros */
    int32_t true_skip;     /* 1 = identity skip in residual blocks, 0 = 1x1 conv shortcut */
    int32_t channels;
    float trim_right_ratio;
    int32_t device;
} enc_config;

int enc_create(const enc_config* cfg, enc_engine** out);
int enc_destroy(enc_engine* e);
/* name = "vq.{q}.embed", "dec.conv_in.weight", "dec.lstm.weight_ih_l0", "dec.up{i}.convtr.weight",
 * "dec.up{i}.res{j}.conv1.weight", ... (weight-norm already folded: w = g * v / ||v||), fp32 row-major. */
int enc_load_weight(enc_engine* e, const char* name, const float* data, const int64_t* shape, int32_t ndim,
                    int32_t is_device_ptr);
int enc_finalize(enc_engine* e);
/* codes [B][n_q][T] int64 (device) -> wav [B][channels][T * hop] fp32 (device) */
int enc_decode(enc_engine* e, const int64_t* codes_dev, float* wav_dev, int32_t B, int32_t T, void* stream);
/* wav [B][channels][N] fp32 (device) -> codes [B][n_q][T] int64 (device), T = N down-sampled by every ratio (rounded up).
 * Replaces AudioTokenizer.encode (reference data/tokenizer.py:127-129 -> audiocraft EncodecModel.encode = SEANetEncoder +
 * ResidualVectorQuantizer.encode).  Needs the "enc.*" weights: "enc.conv_in.weight", "enc.down{i}.res{j}.conv1.weight",
 * "enc.down{i}.conv.weight" (strided), "enc.lstm.*", "enc.conv_out.weight". */
int enc_encode(enc_engine* e, const float* wav_dev, int64_t* codes_dev, int32_t B, int32_t N, void* stream);
/* Ragged batch encode: wav [B][channels][N] fp32 (device), row b's first lens_host[b] samples -> codes [B][n_q][T_N] int64
 * (device), T_N = frames of N; row b's first frames_host[b] frames are the codes of its own lens_host[b] samples, 0 after.
 * Mono rows long enough for every reflect padding of the encoder run on the tensor-core encoder (codec_tc.cu): sorted by
 * length and cut into chunks under VCB_CODEC_WS_GB, each chunk's planes sized for its longest row, every layer causal, so a
 * row's codes are bit-identical whatever the batch, its order or the chunking.  Its latent follows the fp32 encoder within
 * the 3-pass bf16 products' error (DESIGN.md section 4.4); the RVQ search is the fp32 one of enc_encode, so the codes are
 * exactly the nearest codes of that latent.  Every other row (too short, a configuration the tensor-core encoder does not
 * cover, VCB_CODEC_TC=0) goes alone through the CUDA-core encoder: bit-identical to enc_encode of that row alone.
 * Rejected before anything is enqueued: B < 1, any lens outside [1, N], missing encoder weights.  Asynchronous on
 * `stream` (a larger workspace synchronises it first); it shares the engine's workspace with enc_decode and
 * enc_stream_decode, so calls on one engine must not overlap. */
int enc_encode_ragged(enc_engine* e, const float* wav_dev, const int32_t* lens_host, int32_t B, int32_t N, int64_t* codes_dev,
                      int32_t* frames_host, void* stream);
/* "launches", "hop", "flops_per_frame", "tc_enabled", "tc_decodes", "stream_decodes", "stream_min_frames" (frames a fresh
 * stream's first enc_stream_decode needs; -1 without the tensor-core decoder), "stream_state_bytes" (carried state per stream);
 * "tc_encoder" (the tensor-core encoder is built), "tc_encodes" (enc_encode_ragged calls that ran it), "encode_rows" (plane
 * rows of its first stage it ran: per chunk, rows x the chunk's longest row rounded up to the first stride);
 * "live_bytes" / "live_handles" as vcb_counter and "resample_launches" (kernels enc_resample / enc_resampler_push enqueued) are
 * process-wide, valid with a NULL engine */
int64_t enc_counter(enc_engine* e, const char* name);

/* Streaming decode: waveform chunk by chunk while the tokens are still being generated.  The decoder is causal, so a chunk
 * only needs the left context the previous chunk ended with: for every layer that reads earlier rows, the last rows of its
 * input (kept as the decoder keeps its activations), and the LSTM's (h, c).  With that state carried, the concatenated
 * chunks are bit-identical to one enc_decode of the whole sequence.
 *
 * Synchronisation: enc_stream_decode checks the codes on the device and waits for that check, and copies a small per-call
 * table to the device; the decode itself is asynchronous on `stream`.  One enc_stream is used from one CUDA stream, and the
 * calls of one enc_engine (enc_decode, enc_stream_decode) must not overlap: they share its workspace. */
typedef struct enc_stream enc_stream;
/* state for up to max_streams concurrent utterances; fails where the tensor-core decoder does not cover the codec
 * (non-causal codec, VCB_CODEC_TC=0, ...) */
int enc_stream_create(enc_engine* e, int32_t max_streams, enc_stream** out);
int enc_stream_destroy(enc_stream* s);
/* the listed streams start over at frame 0 on their next decode */
int enc_stream_reset(enc_stream* s, const int32_t* ids_host, int32_t n);
/* codes [B][n_q][T] int64 (device) -> wav [B][channels][T*hop] fp32 (device).  Row b continues stream ids_host[b]:
 * samples [0, lens_host[b]*hop) are the waveform of that stream's next lens_host[b] frames, bit-identical to the same
 * samples of enc_decode over the stream's whole code sequence; later samples are unspecified.
 * Rejected before any stream changes: an id outside [0, max_streams) or twice in the call, lens outside [1, T], a fresh
 * stream's first call with fewer than "stream_min_frames" frames, any code (padding included) outside [0, bins). */
int enc_stream_decode(enc_engine* e, enc_stream* s, const int32_t* ids_host, const int32_t* lens_host, int32_t B,
                      const int64_t* codes_dev, int32_t T, float* wav_dev, void* stream);
/* Debug / tests: an intermediate tensor of the last enc_decode on the tensor-core path ("z", "x0", "hs0", "u0", "x1.raw",
 * "x1.elu", "h1.0", "o1.0", with several residual blocks per stage also "o1.0.raw", ...), reassembled from its bf16 (hi, lo)
 * planes as fp32 [B][C][halo + T] on the host.  dims = {B, C, halo + T, halo}; host_out == NULL only queries dims.  "c0",
 * "c1", ... are the LSTM layers' fp32 cell states after the last step, dims {B, C, 1, 0}.  The up-sampling stages share two
 * workspace arenas, so after a full decode only the tensors of the last stage (and "z", "x0", "u0", "hs*", "c*") still hold
 * their values -- unless the engine was finalized under VCB_CODEC_KEEP=1, which gives every tensor rows of its own: same
 * kernels, launches and arithmetic, a larger workspace (tests/test_codec_numerics.py, scripts/codec_tc_debug.py).
 * "enc.latent": under VCB_CODEC_KEEP=1, the latent the last enc_encode or enc_encode_ragged quantised, fp32 dims
 * {B, dimension, T, 0} (ragged: row b's frames past frames_host[b] are 0); this name does not need the tensor-core decoder.
 * The tensor-core encoder's tensors of its last chunk (rows in the chunk's order: longest first): "enc.input" (the input
 * window planes), "enc.x0" / "enc.x0.elu" (enc.conv_in), per stage i and block j "enc.down{i}.res{j}.h" (ELU'd hidden),
 * "enc.down{i}.res{j}" / ".elu" (block output; the last block of a stage stores only ".elu", its right padding included),
 * "enc.down{i}.conv" / ".elu" (the strided conv; the last one is the LSTM input, time-major), "enc.hs{l}", "enc.lstm"
 * (ELU(LSTM + skip), enc.conv_out's input).  Any other name fails where the tensor-core decoder is not active. */
int enc_debug_tensor(enc_engine* e, const char* name, float* host_out, int64_t cap, int32_t* dims);

/* Resampling: torchaudio.transforms.Resample(orig_sr, new_sr) with its defaults (sinc_interp_hann, lowpass_filter_width 6,
 * rolloff 0.99), the conversion the reference's convert_audio applies to prompt audio (data/tokenizer.py:85-97), on the
 * device.  With g = gcd(orig_sr, new_sr), o = orig_sr / g, n = new_sr / g and w = ceil(6 o / (0.99 min(o, n))), output
 * sample b*n + p is sum_{i < 2w+o} table[p][i] * x[b*o + i - w] (x = 0 outside the row), summed in that order with fp32
 * FMA; a row of L samples gives ceil(n L / o).  The resampler is independent of any enc_engine.  Its calls enqueue work
 * on `stream` and never wait for the device; one resampler is used from one CUDA stream at a time. */
typedef struct enc_resampler enc_resampler;
/* table_host: fp32 [n][2w + o], the filter table torchaudio builds (voicecraft_b200.tokenizer.resample_table).  Rejected
 * before anything is allocated: a rate <= 0, a table over 16 MB, a down-sampling ratio whose one-output input window
 * does not fit in shared memory.  max_streams (>= 0) streams for enc_resampler_push. */
int enc_resampler_create(int32_t orig_sr, int32_t new_sr, const float* table_host, int32_t max_streams, int32_t device,
                         enc_resampler** out);
int enc_resampler_destroy(enc_resampler* r);
/* One-shot, over ragged rows: in [B][T] fp32 (device), row b's first lens_host[b] samples -> out [B][out_cap] (device),
 * row b's first out_lens_host[b] = ceil(n lens_host[b] / o) samples. */
int enc_resample(enc_resampler* r, const float* in_dev, const int32_t* lens_host, int32_t B, int32_t T, float* out_dev,
                 int32_t out_cap, int32_t* out_lens_host, void* stream);
/* Streaming: row b continues stream ids_host[b] with the first lens_host[b] (>= 0) samples of in [B][T] and emits every
 * output whose whole input window has arrived (block b once b*o + w + o <= samples so far); with final_host[b] set (null:
 * none) also the zero-padded tail up to ceil(n L / o), and the stream takes no more input until reset.  Row b's
 * out_lens_host[b] outputs go to out [B][out_cap]; the counts are written before anything is enqueued.  A stream's
 * outputs, concatenated, are bit-identical to enc_resample of its whole input.  Rejected before any stream changes: an id
 * outside [0, max_streams) or twice in the call, a length outside [0, T], a stream past its final push, a row whose
 * outputs exceed out_cap. */
int enc_resampler_push(enc_resampler* r, const int32_t* ids_host, const int32_t* lens_host, const int32_t* final_host,
                       int32_t B, const float* in_dev, int32_t T, float* out_dev, int32_t out_cap, int32_t* out_lens_host,
                       void* stream);
/* the listed streams start over with no input */
int enc_resampler_reset(enc_resampler* r, const int32_t* ids_host, int32_t n);

#ifdef __cplusplus
}
#endif
#endif /* VCB200_CODEC_H_ */
