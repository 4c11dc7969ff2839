// Interface between encodec.cu (C ABI, weight store, CUDA-core kernels) and codec_tc.cu (tensor-core decoder and encoder).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/vcb200_codec.h"
#include "vcb_internal.h"

namespace vcb {

struct TcCodec;
struct TcCodecDelete {                 // the owner synchronises first: nothing queued may still use the decoder's buffers
    void operator()(TcCodec* c) const;
};
using TcCodecPtr = std::unique_ptr<TcCodec, TcCodecDelete>;

// 0: built; 1: this configuration is outside what the tensor-core path covers (why -> *reason, static string); -1: error.
int tc_codec_build(const enc_config& cfg, const std::map<std::string, DevBuf<float>>& w_dev,
                   const std::map<std::string, std::vector<int64_t>>& shapes, TcCodecPtr* out, const char** reason);
// Stream decode (enc_stream_decode): utterance b of the call continues stream table[4b] with table[4b+1] valid frames;
// table[4b+2] = 1 if that stream has decoded frames before (its left context and LSTM state come from `state`), 0 if fresh.
struct TcStreamCtx {
    const int* table;                  // device [B][4]: id, valid frames, continuing, unused
    uint8_t* state;                    // device [max_streams][tc_stream_state_bytes]
};

// whether (B, T) can run here (T long enough for every reflect padding)
bool tc_codec_accepts(const TcCodec* c, int B, int T);
// sc == nullptr: a whole-utterance decode; otherwise every row b < lens continues its stream (rows past it are unspecified)
int tc_codec_decode(TcCodec* c, const int64_t* codes_dev, float* wav_dev, int B, int T, cudaStream_t st, int64_t* launches,
                    const TcStreamCtx* sc = nullptr);
size_t tc_stream_state_bytes(const TcCodec* c);
// frames a fresh stream's first decode needs (every reflect padding mirrors valid rows)
int tc_stream_min_frames(const TcCodec* c);
// *bad_host = whether any of the n codes lies outside [0, bins); waits for the stream
int tc_codes_check(const int64_t* codes_dev, long long n, int bins, int* bad_dev, int* bad_host, cudaStream_t st);
// per-layer device times of the last decode when VCB_CODEC_PROFILE=1 (name, ms), in launch order
const std::vector<std::pair<std::string, float>>& tc_codec_profile(const TcCodec* c);

// debug: tensor `name` of the last decoded chunk as fp32 [B][C][halo + T] (hi + lo); dims = {B, C, halo + T, halo}.  With
// VCB_CODEC_KEEP=1 at tc_codec_build no two tensors share rows, so every one of them holds what its layer stored.
int tc_codec_debug_tensor(TcCodec* c, const char* name, float* host_out, int64_t cap, int32_t* dims);

// ---- tensor-core encoder (built with the decoder when the enc.* weights are loaded and it is covered)
bool tc_encoder_active(const TcCodec* c);
// whether an utterance of len samples can run here (every stage longer than the padding it reflects)
bool tc_encoder_accepts(const TcCodec* c, int len);
// workspace of a chunk of B utterances of at most N samples; the VCB_CODEC_WS_GB limit the host chunks under
size_t tc_encoder_ws_bytes(const TcCodec* c, int B, int N);
size_t tc_ws_limit(const TcCodec* c);
// plane rows a chunk of B utterances of at most N samples runs through (its first stage)
int64_t tc_encoder_rows(const TcCodec* c, int B, int N);
// the chunk's fp32 latent [B][dimension][T] (the RVQ search consumes it as its residual), scores scratch [B][bins][T] and
// codes [B][n_q][T], all in the workspace; T = frames of the chunk's longest utterance
struct TcEncOut {
    float* latent;
    float* scores;
    int64_t* codes;
    int T;
};
// utterance b = wav row rows[b] (fp32 at wav + rows[b] * wav_ld) with lens[b] samples; asynchronous on st (the
// workspace may be reallocated first, after a stream synchronisation).  Debug names "enc.*" (tc_codec_debug_tensor).
int tc_encoder_encode(TcCodec* c, const float* wav, long long wav_ld, const int* rows, const int* lens, int B, cudaStream_t st,
                      int64_t* launches, TcEncOut* out);

}  // namespace vcb
