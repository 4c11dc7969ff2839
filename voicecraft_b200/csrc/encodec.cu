// EnCodec token -> waveform decode (include/vcb200_codec.h): RVQ gather-sum + SEANet decoder as explicit kernels.
//
// Replaces AudioTokenizer.decode (reference data/tokenizer.py:131-133 -> audiocraft EncodecModel.decode).
// Round-1 kernels are fp32 on CUDA cores (waveform parity to ~1e-5 against the oracle):
//   rvq_decode_kernel   sum_q codebook_q[code]  -> latent [B, D, T]              (integer gather + fp32 add, coalesced)
//   conv_gemm_kernel    Conv1d (stride 1, dilation, causal/reflect padding) and ConvTranspose1d (stride r, k = 2r: one
//                       2*Cin-deep GEMM per output phase) as an implicit GEMM, 64x64x16 smem tiles, 4x4 register tiles,
//                       ELU fused on the input gather, bias + residual fused in the epilogue
//   lstm_step_kernel    one time step of one LSTM layer: gates = pre[:, t] + W_hh h ; c, h update ; (+ skip)
// Since round 2 enc_decode runs the tensor-core decoder of codec_tc.cu whenever the configuration is one it covers (the
// default 16 kHz codec is); the kernels here remain the path for everything else and for enc_encode.  enc_encode_ragged
// runs the tensor-core encoder of codec_tc.cu on the rows it covers and these kernels, one row at a time, on the others;
// both end in the RVQ search here (rvq_encode).
#include "../../include/vcb200_codec.h"
#include "codec_tc.h"
#include "vcb_internal.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

namespace vcb {

__global__ void rvq_decode_kernel(const long long* __restrict__ codes, const float* const* __restrict__ embed,
                                  float* __restrict__ out, int K, int D, int T) {
    // block: 32 time steps x all D channels, transposed through smem so both sides are coalesced
    extern __shared__ float tile[];                     // [32][D+1]
    const int b = blockIdx.y, t0 = blockIdx.x * 32;
    for (int i = threadIdx.x; i < 32 * D; i += blockDim.x) {
        const int tt = i / D, c = i - tt * D;
        const int t = t0 + tt;
        float acc = 0.f;
        if (t < T)
            for (int q = 0; q < K; ++q)
                acc += embed[q][static_cast<size_t>(codes[(static_cast<size_t>(b) * K + q) * T + t]) * D + c];
        tile[tt * (D + 1) + c] = acc;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * D; i += blockDim.x) {
        const int c = i / 32, tt = i - c * 32;
        if (t0 + tt < T) out[(static_cast<size_t>(b) * D + c) * T + t0 + tt] = tile[tt * (D + 1) + c];
    }
}

struct ConvArgs {
    const float* A;        // conv: [Cout][Cin*ks] ; convT: [r phases][Cout][2*Cin]
    const float* bias;     // [Cout]
    const float* in;       // [B][Cin][Tin]
    float* out;            // [B][Cout][Tout]
    const float* residual; // [B][Cout][Tout] or null
    int Cin, Cout, Tin, Tout, ks, dil, padL, reflect, elu_in;
    int convT, r;          // transposed conv: stride r, kernel 2r, one GEMM per phase (blockIdx.z % r)
    int stride;            // forward conv stride (encoder down-sampling: stride r, kernel 2r); 1 in the decoder
    int Lp;                // reflect padding mirrors a signal of this length (= Tin, or max_pad + 1 zero-extended: audiocraft pad1d)
};

__device__ __forceinline__ float elu1(float x) { return x > 0.f ? x : expm1f(x); }

template <bool CONVT>
__global__ void __launch_bounds__(256) conv_gemm_kernel(const ConvArgs a) {
    __shared__ float As[16][68];
    __shared__ float Xs[16][68];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int phase = CONVT ? blockIdx.z % a.r : 0;
    const int b = CONVT ? blockIdx.z / a.r : blockIdx.z;
    const int co0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
    const int Ktot = CONVT ? 2 * a.Cin : a.Cin * a.ks;
    const float* A = a.A + (CONVT ? static_cast<size_t>(phase) * a.Cout * Ktot : 0);
    const float* in = a.in + static_cast<size_t>(b) * a.Cin * a.Tin;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < Ktot; k0 += 16) {
        // A tile: 64 rows x 16 k   (thread -> row tid/4, 4 consecutive k)
        {
            const int row = tid >> 2, kk = (tid & 3) * 4;
            const int co = co0 + row;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int k = k0 + kk + u;
                As[kk + u][row] = (co < a.Cout && k < Ktot) ? A[static_cast<size_t>(co) * Ktot + k] : 0.f;
            }
        }
        // X tile: 16 k x 64 columns, gathered from the input with padding / ELU   (thread -> k tid/16, 4 columns)
        {
            const int kk = tid >> 4, nn = (tid & 15) * 4;
            const int k = k0 + kk;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int n = n0 + nn + u;
                float v = 0.f;
                if (k < Ktot) {
                    int ci, src;
                    bool ok;
                    if (CONVT) {
                        const int tap = k / a.Cin;
                        ci = k - tap * a.Cin;
                        src = n - tap;
                        ok = src >= 0 && src < a.Tin;
                    } else {
                        ci = k / a.ks;
                        const int kx = k - ci * a.ks;
                        src = n * a.stride + kx * a.dil - a.padL;
                        ok = n < a.Tout;
                        if (ok && (src < 0 || src >= a.Tin)) {
                            if (a.reflect) {
                                // audiocraft pad1d: an input no longer than the padding is first zero-extended to Lp samples
                                if (src < 0) src = -src;
                                else if (src >= a.Lp) src = 2 * (a.Lp - 1) - src;
                                ok = src >= 0 && src < a.Tin;
                            } else {
                                ok = false;
                            }
                        }
                    }
                    if (ok) {
                        v = in[static_cast<size_t>(ci) * a.Tin + src];
                        if (a.elu_in) v = elu1(v);
                    }
                }
                Xs[kk][nn + u] = v;
            }
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < 16; ++kk) {
            const float4 av = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 xv = *reinterpret_cast<const float4*>(&Xs[kk][tx * 4]);
            const float ar[4] = {av.x, av.y, av.z, av.w};
            const float xr[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], xr[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int co = co0 + ty * 4 + i;
        if (co >= a.Cout) continue;
        const float bv = a.bias[co];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            const int t = CONVT ? phase + a.r * n - a.padL : n;
            if (t < 0 || t >= a.Tout) continue;
            const size_t o = (static_cast<size_t>(b) * a.Cout + co) * a.Tout + t;
            float v = acc[i][j] + bv;
            if (a.residual) v += a.residual[o];
            a.out[o] = v;
        }
    }
}

// One LSTM time step for one layer.  Warp = one hidden unit j, 4 batch rows; gate order i, f, g, o (torch.nn.LSTM).
// pre [B][4H][T] = W_ih x + (b_ih + b_hh) computed by conv_gemm_kernel (k = 1); h/c state [B][H].
__global__ void __launch_bounds__(256)
lstm_step_kernel(const float* __restrict__ pre, const float* __restrict__ Whh, const float* __restrict__ h_in,
                 float* __restrict__ h_out, float* __restrict__ c, float* __restrict__ seq_out,
                 const float* __restrict__ skip, int B, int H, int T, int t) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int j = blockIdx.x * 8 + warp;
    const int b0 = blockIdx.y * 4;
    if (j >= H) return;
    float acc[4][4];
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int bb = 0; bb < 4; ++bb) acc[g][bb] = 0.f;
    for (int k = lane * 4; k < H; k += 128) {
        float4 w[4], hv[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) w[g] = *reinterpret_cast<const float4*>(Whh + (static_cast<size_t>(g) * H + j) * H + k);
#pragma unroll
        for (int bb = 0; bb < 4; ++bb)
            hv[bb] = (b0 + bb < B) ? *reinterpret_cast<const float4*>(h_in + static_cast<size_t>(b0 + bb) * H + k)
                                   : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int g = 0; g < 4; ++g)
#pragma unroll
            for (int bb = 0; bb < 4; ++bb)
                acc[g][bb] += w[g].x * hv[bb].x + w[g].y * hv[bb].y + w[g].z * hv[bb].z + w[g].w * hv[bb].w;
    }
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int bb = 0; bb < 4; ++bb) acc[g][bb] = warp_sum(acc[g][bb]);
    if (lane < 4 && b0 + lane < B) {
        const int b = b0 + lane;
        float gt[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            float s = 0.f;
#pragma unroll
            for (int bb = 0; bb < 4; ++bb) s = (bb == lane) ? acc[g][bb] : s;
            gt[g] = s + pre[(static_cast<size_t>(b) * 4 * H + g * H + j) * T + t];
        }
        const float ig = 1.f / (1.f + expf(-gt[0])), fg = 1.f / (1.f + expf(-gt[1]));
        const float gg = tanhf(gt[2]), og = 1.f / (1.f + expf(-gt[3]));
        const size_t sidx = static_cast<size_t>(b) * H + j;
        const float cn = fg * c[sidx] + ig * gg;
        const float hn = og * tanhf(cn);
        c[sidx] = cn;
        h_out[sidx] = hn;
        const size_t o = (static_cast<size_t>(b) * H + j) * T + t;
        seq_out[o] = skip ? hn + skip[o] : hn;
    }
}

// RVQ encode, one quantizer stage (audiocraft ResidualVectorQuantizer.encode / core_vq.py EuclideanCodebook.quantize):
// scores[b][c][t] = e_c . x - |e_c|^2 / 2 come from conv_gemm_kernel (k = 1, bias = -|e|^2/2); the nearest code is their
// argmax (first index wins), then the residual loses that code's embedding.  One thread per (b, t), coalesced over t.
__global__ void rvq_pick_kernel(const float* __restrict__ scores, const float* __restrict__ embed, float* __restrict__ resid,
                                long long* __restrict__ codes, int bins, int D, int T, int n_q, int q) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (t >= T) return;
    const float* sc = scores + static_cast<size_t>(b) * bins * T + t;
    float best = -INFINITY;
    int bi = 0;
    for (int c = 0; c < bins; ++c) {
        const float v = sc[static_cast<size_t>(c) * T];
        if (v > best) {
            best = v;
            bi = c;
        }
    }
    codes[(static_cast<size_t>(b) * n_q + q) * T + t] = bi;
    float* r = resid + static_cast<size_t>(b) * D * T + t;
    const float* e = embed + static_cast<size_t>(bi) * D;
    for (int c = 0; c < D; ++c) r[static_cast<size_t>(c) * T] -= e[c];
}

__global__ void half_sqnorm_neg_kernel(const float* __restrict__ embed, float* __restrict__ out, int bins, int D) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= bins) return;
    float s = 0.f;
    for (int i = 0; i < D; ++i) s = fmaf(embed[static_cast<size_t>(c) * D + i], embed[static_cast<size_t>(c) * D + i], s);
    out[c] = -0.5f * s;
}

// ConvTranspose1d weight [Cin][Cout][2r] -> per-phase GEMM operand [r][Cout][2*Cin]  (k = tap*Cin + ci, tap in {0,1})
__global__ void pack_convtr_kernel(const float* __restrict__ w, float* __restrict__ out, int Cin, int Cout, int r) {
    const size_t total = static_cast<size_t>(r) * Cout * 2 * Cin;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int k = static_cast<int>(i % (2 * Cin));
        const int co = static_cast<int>((i / (2 * Cin)) % Cout);
        const int q = static_cast<int>(i / (static_cast<size_t>(2 * Cin) * Cout));
        const int tap = k / Cin, ci = k - tap * Cin;
        out[i] = w[(static_cast<size_t>(ci) * Cout + co) * (2 * r) + q + tap * r];
    }
}

__global__ void add_vec_kernel(const float* a, const float* b, float* o, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) o[i] = a[i] + b[i];
}

}  // namespace vcb

using namespace vcb;

struct enc_engine {
    enc_config cfg;
    std::map<std::string, DevBuf<float>> w;       // loaded weights and the ones enc_finalize derives (names with "__")
    std::map<std::string, std::vector<int64_t>> shapes;
    DevBuf<float*> d_embed;
    int hop = 1;
    bool finalized = false, has_encoder = false;
    // activation buffers for a batch chunk
    DevBuf<float> buf[4];
    size_t buf_floats = 0;
    DevBuf<float> h0, h1, cst;
    int cap_B = 0, cap_T = 0;
    int64_t launches = 0;
    double flops_per_frame = 0;
    TcCodecPtr tc;                      // tensor-core decoder (codec_tc.cu); null = configuration not covered
    const char* tc_reason = "";
    int64_t tc_decodes = 0;
    int64_t stream_decodes = 0;
    int64_t tc_encodes = 0;             // enc_encode_ragged calls that ran the tensor-core encoder
    int64_t encode_rows = 0;            // plane rows (first stage) through the tensor-core encoder
    DevBuf<float> row_wav;              // enc_encode_ragged, CUDA-core rows: one utterance's [channels][len] samples
    DevBuf<int64_t> row_codes;          // ... and its codes [n_q][T]
    bool keep = false;                  // VCB_CODEC_KEEP=1: enc_encode keeps the latent it quantises ("enc.latent")
    DevBuf<float> latent;               // [lat_B][dimension][lat_T]
    int lat_B = 0, lat_T = 0;
};

struct enc_stream {
    enc_engine* e = nullptr;
    int max_streams = 0;
    DevBuf<uint8_t> state;              // [max_streams][tc_stream_state_bytes]
    DevBuf<int> table;                  // [max_streams][4] per-call table (TcStreamCtx)
    DevBuf<int> bad;                    // codes check flag
    std::vector<int64_t> frames;        // frames decoded so far, per stream (0 = fresh)
};

namespace {

int enc_need(enc_engine* e, const std::string& name, float** out) {
    auto it = e->w.find(name);
    if (it == e->w.end()) {
        set_error("codec: missing weight %s", name.c_str());
        return -1;
    }
    *out = it->second;
    return 0;
}

int conv_launch(enc_engine* e, ConvArgs a, int B, cudaStream_t st) {
    if (a.convT) {
        const int ncols = (a.Tout + a.padL + a.r - 1) / a.r + 1;
        dim3 grid((ncols + 63) / 64, (a.Cout + 63) / 64, B * a.r);
        conv_gemm_kernel<true><<<grid, 256, 0, st>>>(a);
    } else {
        dim3 grid((a.Tout + 63) / 64, (a.Cout + 63) / 64, B);
        conv_gemm_kernel<false><<<grid, 256, 0, st>>>(a);
    }
    VCB_CUDA_OK(cudaGetLastError());
    e->launches++;
    return 0;
}

// Conv1d, stride 1: padding as audiocraft StreamableConv1d (causal: all left; else split, extra on the left)
ConvArgs conv_args(const enc_engine* e, const float* A, const float* bias, const float* in, float* out, int Cin, int Cout,
                   int T, int ks, int dil, int elu_in, const float* residual) {
    ConvArgs a;
    memset(&a, 0, sizeof(a));
    a.A = A; a.bias = bias; a.in = in; a.out = out; a.residual = residual;
    a.Cin = Cin; a.Cout = Cout; a.Tin = T; a.Tout = T; a.ks = ks; a.dil = dil;
    const int total = (ks - 1) * dil;
    a.padL = e->cfg.causal ? total : total - total / 2;
    a.reflect = e->cfg.pad_reflect;
    a.elu_in = elu_in;
    a.stride = 1;
    const int max_pad = std::max(a.padL, total - a.padL);
    a.Lp = (a.reflect && T <= max_pad) ? max_pad + 1 : T;
    return a;
}

// Strided Conv1d of the encoder (audiocraft StreamableConv1d with stride r, kernel 2r): pad (k - stride) in total -- causal:
// all on the left -- plus whatever the last window lacks on the right (get_extra_padding_for_conv1d); Tout = ceil(Tin / r).
ConvArgs conv_args_strided(const enc_engine* e, const float* A, const float* bias, const float* in, float* out, int Cin, int Cout,
                           int Tin, int ks, int stride, int elu_in) {
    ConvArgs a = conv_args(e, A, bias, in, out, Cin, Cout, Tin, ks, 1, elu_in, nullptr);
    const int total = ks - stride;
    a.padL = e->cfg.causal ? total : total - total / 2;
    a.stride = stride;
    a.Tout = (Tin + stride - 1) / stride;
    const int extra = (a.Tout - 1) * stride + ks - total - Tin;    // right padding that completes the last window
    const int max_pad = std::max(a.padL, total - a.padL + extra);
    a.Lp = (a.reflect && Tin <= max_pad) ? max_pad + 1 : Tin;
    return a;
}

int ensure_buffers(enc_engine* e, int B, int T) {
    if (B <= e->cap_B && T <= e->cap_T) return 0;
    for (auto& p : e->buf) p.reset();   // all released before the larger ones are allocated
    e->h0.reset();
    e->h1.reset();
    e->cst.reset();
    const enc_config& c = e->cfg;
    // widest activation: channels * time over the stack, plus the 4H x T LSTM pre-activations
    int ch = c.n_filters << c.n_ratios;
    size_t widest = static_cast<size_t>(std::max(c.dimension, (c.lstm ? 4 : 1) * ch)) * T;
    int t = T;
    for (int i = 0; i < c.n_ratios; ++i) {
        t *= c.ratios[i];
        ch /= 2;
        widest = std::max(widest, static_cast<size_t>(ch) * t);
    }
    e->buf_floats = widest * B;
    for (auto& p : e->buf)
        if (p.alloc(e->buf_floats)) return -1;
    const size_t hs = static_cast<size_t>(B) * (c.n_filters << c.n_ratios);
    if (e->h0.alloc(hs) || e->h1.alloc(hs) || e->cst.alloc(hs)) return -1;
    e->cap_B = B;
    e->cap_T = T;
    return 0;
}

// StreamableLSTM with skip over x [B, ch, T] -> y (z, pre: scratch).  side = "dec" / "enc".
int lstm_stack(enc_engine* e, const char* side, const float* x, float* y, float* z, float* pre, int B, int ch, int T,
               cudaStream_t st) {
    const enc_config& c = e->cfg;
    char nm[128];
    const float* layer_in = x;
    for (int l = 0; l < c.lstm; ++l) {
        float *wih, *whh, *bsum;
        snprintf(nm, sizeof(nm), "%s.lstm.weight_ih_l%d", side, l);
        if (enc_need(e, nm, &wih)) return -1;
        snprintf(nm, sizeof(nm), "%s.lstm.weight_hh_l%d", side, l);
        if (enc_need(e, nm, &whh)) return -1;
        snprintf(nm, sizeof(nm), "%s.lstm.__bias_sum_l%d", side, l);
        if (enc_need(e, nm, &bsum)) return -1;
        // pre[B, 4H, T] = W_ih * in + (b_ih + b_hh)   (a k=1 convolution, zero padding irrelevant)
        ConvArgs a = conv_args(e, wih, bsum, layer_in, pre, ch, 4 * ch, T, 1, 1, 0, nullptr);
        if (conv_launch(e, a, B, st)) return -1;
        VCB_CUDA_OK(cudaMemsetAsync(e->h0, 0, static_cast<size_t>(B) * ch * 4, st));
        VCB_CUDA_OK(cudaMemsetAsync(e->cst, 0, static_cast<size_t>(B) * ch * 4, st));
        float* seq_out = (l == c.lstm - 1) ? y : z;
        const float* skip = (l == c.lstm - 1) ? x : nullptr;      // y = LSTM(x) + x   (skip on the stack input)
        float *hin = e->h0, *hout = e->h1;
        for (int t = 0; t < T; ++t) {
            lstm_step_kernel<<<dim3((ch + 7) / 8, (B + 3) / 4), 256, 0, st>>>(pre, whh, hin, hout, e->cst, seq_out, skip, B, ch, T, t);
            std::swap(hin, hout);
        }
        VCB_CUDA_OK(cudaGetLastError());
        e->launches += T;
        layer_in = seq_out;
    }
    return 0;
}

// Residual block shared by encoder and decoder: x -> shortcut(x) + conv k1(ELU(conv k3 dil(ELU(x)))).  Result in `pre`.
int res_block(enc_engine* e, const char* prefix, const float* x, float* y, float* z, float* pre, int B, int ch, int T, int dil,
              cudaStream_t st) {
    const enc_config& c = e->cfg;
    char nm[160];
    const int hidden = ch / c.compress;
    float *w1, *b1, *w2, *b2;
    snprintf(nm, sizeof(nm), "%s.conv1.weight", prefix);
    if (enc_need(e, nm, &w1)) return -1;
    snprintf(nm, sizeof(nm), "%s.conv1.bias", prefix);
    if (enc_need(e, nm, &b1)) return -1;
    snprintf(nm, sizeof(nm), "%s.conv2.weight", prefix);
    if (enc_need(e, nm, &w2)) return -1;
    snprintf(nm, sizeof(nm), "%s.conv2.bias", prefix);
    if (enc_need(e, nm, &b2)) return -1;
    if (conv_launch(e, conv_args(e, w1, b1, x, y, ch, hidden, T, c.residual_kernel_size, dil, 1, nullptr), B, st)) return -1;
    const float* res = x;
    if (!c.true_skip) {
        float *ws, *bsc;
        snprintf(nm, sizeof(nm), "%s.shortcut.weight", prefix);
        if (enc_need(e, nm, &ws)) return -1;
        snprintf(nm, sizeof(nm), "%s.shortcut.bias", prefix);
        if (enc_need(e, nm, &bsc)) return -1;
        if (conv_launch(e, conv_args(e, ws, bsc, x, z, ch, ch, T, 1, 1, 0, nullptr), B, st)) return -1;
        res = z;
    }
    return conv_launch(e, conv_args(e, w2, b2, y, pre, hidden, ch, T, 1, 1, 1, res), B, st);
}

int rvq_encode(enc_engine* e, float* y, float* pre, int64_t* codes, int B, int T, cudaStream_t st);

// wav [B, channels, N] -> codes [B, n_q, T]: SEANetEncoder (conv k7 -> n x [ResBlock, ELU, strided conv] -> LSTM + skip -> ELU ->
// conv k7) and residual vector quantisation.  (reference data/tokenizer.py:127-129 -> audiocraft EncodecModel.encode)
int encode_chunk(enc_engine* e, const float* wav, int64_t* codes, float* latent, int B, int N, cudaStream_t st) {
    const enc_config& c = e->cfg;
    char nm[128];
    float *x = e->buf[0], *y = e->buf[1], *z = e->buf[2], *pre = e->buf[3];
    float *wt, *bs;
    int ch = c.n_filters, t_cur = N;
    if (enc_need(e, "enc.conv_in.weight", &wt) || enc_need(e, "enc.conv_in.bias", &bs)) return -1;
    if (conv_launch(e, conv_args(e, wt, bs, wav, x, c.channels, ch, t_cur, c.kernel_size, 1, 0, nullptr), B, st)) return -1;
    for (int i = 0; i < c.n_ratios; ++i) {
        const int r = c.ratios[c.n_ratios - 1 - i];           // the encoder walks the ratios in reverse
        for (int j = 0; j < c.n_residual_layers; ++j) {
            int dil = 1;
            for (int u = 0; u < j; ++u) dil *= c.dilation_base;
            snprintf(nm, sizeof(nm), "enc.down%d.res%d", i, j);
            if (res_block(e, nm, x, y, z, pre, B, ch, t_cur, dil, st)) return -1;
            std::swap(x, pre);
        }
        snprintf(nm, sizeof(nm), "enc.down%d.conv.weight", i);
        if (enc_need(e, nm, &wt)) return -1;
        snprintf(nm, sizeof(nm), "enc.down%d.conv.bias", i);
        if (enc_need(e, nm, &bs)) return -1;
        ConvArgs a = conv_args_strided(e, wt, bs, x, y, ch, 2 * ch, t_cur, 2 * r, r, 1);
        if (conv_launch(e, a, B, st)) return -1;
        std::swap(x, y);
        ch *= 2;
        t_cur = a.Tout;
    }
    if (c.lstm > 0) {
        if (lstm_stack(e, "enc", x, y, z, pre, B, ch, t_cur, st)) return -1;
        std::swap(x, y);
    }
    if (enc_need(e, "enc.conv_out.weight", &wt) || enc_need(e, "enc.conv_out.bias", &bs)) return -1;
    if (conv_launch(e, conv_args(e, wt, bs, x, y, ch, c.dimension, t_cur, c.last_kernel_size, 1, 1, nullptr), B, st)) return -1;
    const int T = t_cur;
    if (latent != nullptr)
        VCB_CUDA_OK(cudaMemcpyAsync(latent, y, static_cast<size_t>(B) * c.dimension * T * 4, cudaMemcpyDeviceToDevice, st));
    return rvq_encode(e, y, pre, codes, B, T, st);
}

// residual vector quantisation of y = latent [B, D, T], consumed as the running residual; pre: scores scratch [B][bins][T]
int rvq_encode(enc_engine* e, float* y, float* pre, int64_t* codes, int B, int T, cudaStream_t st) {
    const enc_config& c = e->cfg;
    char nm[128];
    for (int q = 0; q < c.n_q; ++q) {
        float *emb, *hsn;
        snprintf(nm, sizeof(nm), "vq.%d.embed", q);
        if (enc_need(e, nm, &emb)) return -1;
        snprintf(nm, sizeof(nm), "vq.%d.__neg_half_sqnorm", q);
        if (enc_need(e, nm, &hsn)) return -1;
        // scores[b][code][t] = e_code . resid[b][:, t] - |e_code|^2 / 2   (k = 1 "convolution" with the codebook as weights)
        if (conv_launch(e, conv_args(e, emb, hsn, y, pre, c.dimension, c.bins, T, 1, 1, 0, nullptr), B, st)) return -1;
        rvq_pick_kernel<<<dim3((T + 127) / 128, B), 128, 0, st>>>(pre, emb, y, reinterpret_cast<long long*>(codes), c.bins,
                                                                   c.dimension, T, c.n_q, q);
        VCB_CUDA_OK(cudaGetLastError());
        e->launches++;
    }
    return 0;
}

int decode_chunk(enc_engine* e, const int64_t* codes, float* wav, int B, int T, cudaStream_t st) {
    const enc_config& c = e->cfg;
    char nm[128];
    float *x = e->buf[0], *y = e->buf[1], *z = e->buf[2], *pre = e->buf[3];
    // RVQ decode -> x [B, D, T]
    rvq_decode_kernel<<<dim3((T + 31) / 32, B), 256, 32 * (c.dimension + 1) * sizeof(float), st>>>(
        reinterpret_cast<const long long*>(codes), e->d_embed, x, c.n_q, c.dimension, T);
    VCB_CUDA_OK(cudaGetLastError());
    e->launches++;
    int ch = c.n_filters << c.n_ratios;
    float *wt, *bs;
    if (enc_need(e, "dec.conv_in.weight", &wt) || enc_need(e, "dec.conv_in.bias", &bs)) return -1;
    if (conv_launch(e, conv_args(e, wt, bs, x, y, c.dimension, ch, T, c.kernel_size, 1, 0, nullptr), B, st)) return -1;
    std::swap(x, y);                                    // x = conv_in output [B, ch, T]
    if (c.lstm > 0) {
        if (lstm_stack(e, "dec", x, y, z, pre, B, ch, T, st)) return -1;
        std::swap(x, y);                                // x = LSTM output (+ skip)
    }
    int t_cur = T;
    for (int i = 0; i < c.n_ratios; ++i) {
        const int r = c.ratios[i];
        snprintf(nm, sizeof(nm), "dec.up%d.convtr.__packed", i);
        if (enc_need(e, nm, &wt)) return -1;
        snprintf(nm, sizeof(nm), "dec.up%d.convtr.bias", i);
        if (enc_need(e, nm, &bs)) return -1;
        ConvArgs a;
        memset(&a, 0, sizeof(a));
        a.A = wt; a.bias = bs; a.in = x; a.out = y;
        a.Cin = ch; a.Cout = ch / 2; a.Tin = t_cur; a.Tout = t_cur * r; a.convT = 1; a.r = r; a.elu_in = 1; a.stride = 1; a.Lp = t_cur;
        const int total = r;                            // kernel 2r - stride r
        const int right = c.causal ? static_cast<int>(ceilf(total * c.trim_right_ratio)) : total / 2;
        a.padL = total - right;                         // samples trimmed on the left
        if (conv_launch(e, a, B, st)) return -1;
        std::swap(x, y);
        ch /= 2;
        t_cur *= r;
        for (int j = 0; j < c.n_residual_layers; ++j) {
            int dil = 1;
            for (int u = 0; u < j; ++u) dil *= c.dilation_base;
            snprintf(nm, sizeof(nm), "dec.up%d.res%d", i, j);
            if (res_block(e, nm, x, y, z, pre, B, ch, t_cur, dil, st)) return -1;
            std::swap(x, pre);
        }
    }
    if (enc_need(e, "dec.conv_out.weight", &wt) || enc_need(e, "dec.conv_out.bias", &bs)) return -1;
    ConvArgs a = conv_args(e, wt, bs, x, wav, ch, c.channels, t_cur, c.last_kernel_size, 1, 1, nullptr);
    return conv_launch(e, a, B, st);
}

}  // namespace

extern "C" {

int enc_create(const enc_config* cfg, enc_engine** out) {
    if (!cfg || !out) {
        set_error("null argument");
        return -1;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        set_error("no CUDA device: libvcb200 has no CPU fallback");
        return -2;
    }
    if (cfg->n_ratios < 1 || cfg->n_ratios > 8 || cfg->n_q < 1 || cfg->dimension % 4 || cfg->n_filters % 4) {
        set_error("codec: unsupported configuration");
        return -1;
    }
    VCB_CUDA_OK(cudaSetDevice(cfg->device));
    enc_engine* e = new enc_engine();
    e->cfg = *cfg;
    e->hop = 1;
    for (int i = 0; i < cfg->n_ratios; ++i) e->hop *= cfg->ratios[i];
    *out = e;
    return 0;
}

int enc_destroy(enc_engine* e) {
    if (!e) return 0;
    cudaSetDevice(e->cfg.device);
    cudaDeviceSynchronize();
    delete e;
    return 0;
}

int enc_load_weight(enc_engine* e, const char* name, const float* data, const int64_t* shape, int32_t ndim,
                    int32_t is_device_ptr) {
    VCB_CUDA_OK(cudaSetDevice(e->cfg.device));
    size_t n = 1;
    std::vector<int64_t> sh(shape, shape + ndim);
    for (auto s : sh) n *= static_cast<size_t>(s);
    DevBuf<float> d;
    if (d.alloc(n)) return -1;
    VCB_CUDA_OK(cudaMemcpy(d, data, n * sizeof(float), is_device_ptr ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
    e->w[name] = std::move(d);         // a reloaded name releases its previous buffer
    e->shapes[name] = sh;
    e->finalized = false;
    return 0;
}

int enc_finalize(enc_engine* e) {
    VCB_CUDA_OK(cudaSetDevice(e->cfg.device));
    e->finalized = false;              // the derived buffers below are replaced: unusable until this call succeeds
    const enc_config& c = e->cfg;
    char nm[128];
    std::vector<float*> emb(c.n_q);
    for (int q = 0; q < c.n_q; ++q) {
        snprintf(nm, sizeof(nm), "vq.%d.embed", q);
        if (enc_need(e, nm, &emb[q])) return -1;
    }
    if (e->d_embed.ensure(c.n_q)) return -1;
    VCB_CUDA_OK(cudaMemcpy(e->d_embed, emb.data(), c.n_q * sizeof(float*), cudaMemcpyHostToDevice));
    int ch = c.n_filters << c.n_ratios;
    double flops = 2.0 * c.dimension * ch * c.kernel_size;                     // per frame
    for (int l = 0; l < c.lstm; ++l) {
        float *bi, *bh;
        snprintf(nm, sizeof(nm), "dec.lstm.bias_ih_l%d", l);
        if (enc_need(e, nm, &bi)) return -1;
        snprintf(nm, sizeof(nm), "dec.lstm.bias_hh_l%d", l);
        if (enc_need(e, nm, &bh)) return -1;
        snprintf(nm, sizeof(nm), "dec.lstm.__bias_sum_l%d", l);
        DevBuf<float>& sum = e->w[nm];
        if (sum.alloc(4 * ch)) return -1;
        add_vec_kernel<<<(4 * ch + 255) / 256, 256>>>(bi, bh, sum, 4 * ch);
        flops += 2.0 * 2 * 4 * ch * ch;
    }
    double t_mult = 1;
    for (int i = 0; i < c.n_ratios; ++i) {
        const int r = c.ratios[i];
        float* wsrc;
        snprintf(nm, sizeof(nm), "dec.up%d.convtr.weight", i);
        if (enc_need(e, nm, &wsrc)) return -1;
        snprintf(nm, sizeof(nm), "dec.up%d.convtr.__packed", i);
        DevBuf<float>& packed = e->w[nm];
        if (packed.alloc(static_cast<size_t>(r) * (ch / 2) * 2 * ch)) return -1;
        pack_convtr_kernel<<<512, 256>>>(wsrc, packed, ch, ch / 2, r);
        t_mult *= r;
        flops += t_mult * 2.0 * (2 * ch) * (ch / 2);
        ch /= 2;
        const int hidden = ch / c.compress;
        flops += c.n_residual_layers * t_mult * 2.0 * (ch * hidden * c.residual_kernel_size + hidden * ch + (c.true_skip ? 0 : ch * ch));
    }
    flops += t_mult * 2.0 * ch * c.channels * c.last_kernel_size;
    e->flops_per_frame = flops;
    // encoder side (optional: only when the enc.* weights were loaded)
    e->has_encoder = e->w.count("enc.conv_in.weight") > 0;
    if (e->has_encoder) {
        const int che = c.n_filters << c.n_ratios;
        for (int l = 0; l < c.lstm; ++l) {
            float *bi, *bh;
            snprintf(nm, sizeof(nm), "enc.lstm.bias_ih_l%d", l);
            if (enc_need(e, nm, &bi)) return -1;
            snprintf(nm, sizeof(nm), "enc.lstm.bias_hh_l%d", l);
            if (enc_need(e, nm, &bh)) return -1;
            snprintf(nm, sizeof(nm), "enc.lstm.__bias_sum_l%d", l);
            DevBuf<float>& sum = e->w[nm];
            if (sum.alloc(4 * che)) return -1;
            add_vec_kernel<<<(4 * che + 255) / 256, 256>>>(bi, bh, sum, 4 * che);
        }
        for (int q = 0; q < c.n_q; ++q) {
            snprintf(nm, sizeof(nm), "vq.%d.__neg_half_sqnorm", q);
            DevBuf<float>& hsn = e->w[nm];
            if (hsn.alloc(c.bins)) return -1;
            half_sqnorm_neg_kernel<<<(c.bins + 255) / 256, 256>>>(emb[q], hsn, c.bins, c.dimension);
        }
    }
    VCB_CUDA_OK(cudaDeviceSynchronize());
    e->tc.reset();
    e->keep = getenv("VCB_CODEC_KEEP") && atoi(getenv("VCB_CODEC_KEEP")) != 0;
    if (tc_codec_build(e->cfg, e->w, e->shapes, &e->tc, &e->tc_reason) < 0) return -1;
    e->finalized = true;
    return 0;
}

int enc_decode(enc_engine* e, const int64_t* codes_dev, float* wav_dev, int32_t B, int32_t T, void* stream) {
    if (!e || !e->finalized) {
        set_error("codec engine not finalized");
        return -1;
    }
    if (B < 1 || T < 1) {
        set_error("codec: empty input (B=%d, T=%d)", B, T);
        return -1;
    }
    VCB_CUDA_OK(cudaSetDevice(e->cfg.device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (tc_codec_accepts(e->tc.get(), B, T)) {
        if (tc_codec_decode(e->tc.get(), codes_dev, wav_dev, B, T, st, &e->launches)) return -1;
        e->tc_decodes++;
        if (getenv("VCB_CODEC_PROFILE"))
            for (auto& pr : tc_codec_profile(e->tc.get())) fprintf(stderr, "[codec_tc] %-12s %9.3f ms\n", pr.first.c_str(), pr.second);
        return 0;
    }
    const int chunk = std::min(B, 16);
    if (ensure_buffers(e, chunk, T)) return -1;
    for (int b0 = 0; b0 < B; b0 += chunk) {
        const int nb = std::min(chunk, B - b0);
        if (decode_chunk(e, codes_dev + static_cast<size_t>(b0) * e->cfg.n_q * T,
                         wav_dev + static_cast<size_t>(b0) * e->cfg.channels * T * e->hop, nb, T, st))
            return -1;
    }
    return 0;
}

int enc_encode(enc_engine* e, const float* wav_dev, int64_t* codes_dev, int32_t B, int32_t N, void* stream) {
    if (!e || !e->finalized) {
        set_error("codec engine not finalized");
        return -1;
    }
    if (!e->has_encoder) {
        set_error("codec: encoder weights (enc.*) were not loaded");
        return -1;
    }
    if (B < 1 || N < 1) {
        set_error("codec: empty input (B=%d, N=%d)", B, N);
        return -1;
    }
    VCB_CUDA_OK(cudaSetDevice(e->cfg.device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int T = N;                                           // frames: every strided conv rounds up
    for (int i = e->cfg.n_ratios - 1; i >= 0; --i) T = (T + e->cfg.ratios[i] - 1) / e->cfg.ratios[i];
    const int chunk = std::min(B, 16);
    if (ensure_buffers(e, chunk, (N + e->hop - 1) / e->hop + 1)) return -1;
    const size_t lat = static_cast<size_t>(e->cfg.dimension) * T;
    e->lat_B = 0;
    if (e->keep) {
        if (e->latent.size() < B * lat && e->latent.alloc(B * lat)) return -1;
        e->lat_B = B;
        e->lat_T = T;
    }
    for (int b0 = 0; b0 < B; b0 += chunk) {
        const int nb = std::min(chunk, B - b0);
        if (encode_chunk(e, wav_dev + static_cast<size_t>(b0) * e->cfg.channels * N,
                         codes_dev + static_cast<size_t>(b0) * e->cfg.n_q * T, e->keep ? e->latent + b0 * lat : nullptr, nb, N, st))
            return -1;
    }
    return 0;
}

int enc_encode_ragged(enc_engine* e, const float* wav_dev, const int32_t* lens_host, int32_t B, int32_t N, int64_t* codes_dev,
                      int32_t* frames_host, void* stream) {
    if (!e || !e->finalized) {
        set_error("codec engine not finalized");
        return -1;
    }
    if (!e->has_encoder) {
        set_error("codec: encoder weights (enc.*) were not loaded");
        return -1;
    }
    if (!wav_dev || !lens_host || !codes_dev || !frames_host) {
        set_error("codec: null argument");
        return -1;
    }
    if (B < 1 || N < 1) {
        set_error("codec: empty input (B=%d, N=%d)", B, N);
        return -1;
    }
    for (int b = 0; b < B; ++b)
        if (lens_host[b] < 1 || lens_host[b] > N) {
            set_error("codec: row %d has %d samples, outside [1, N = %d]", b, lens_host[b], N);
            return -1;
        }
    const enc_config& c = e->cfg;
    auto frames = [&](int n) {
        for (int i = c.n_ratios - 1; i >= 0; --i) n = (n + c.ratios[i] - 1) / c.ratios[i];
        return n;
    };
    const int TN = frames(N);
    for (int b = 0; b < B; ++b) frames_host[b] = frames(lens_host[b]);
    VCB_CUDA_OK(cudaSetDevice(c.device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t lat = static_cast<size_t>(c.dimension) * TN;
    e->lat_B = 0;
    if (e->keep) {
        if (e->latent.size() < B * lat && e->latent.alloc(B * lat)) return -1;
        VCB_CUDA_OK(cudaMemsetAsync(e->latent, 0, B * lat * 4, st));
        e->lat_B = B;
        e->lat_T = TN;
    }
    VCB_CUDA_OK(cudaMemsetAsync(codes_dev, 0, static_cast<size_t>(B) * c.n_q * TN * 8, st));
    // the codes (and under VCB_CODEC_KEEP the latent) of utterance b, [n_q][T] with T >= its frames, into its output row
    auto place = [&](int b, const int64_t* codes, const float* latent, int T) -> int {
        const int f = frames_host[b];
        VCB_CUDA_OK(cudaMemcpy2DAsync(codes_dev + static_cast<size_t>(b) * c.n_q * TN, TN * 8, codes, static_cast<size_t>(T) * 8,
                                      static_cast<size_t>(f) * 8, c.n_q, cudaMemcpyDeviceToDevice, st));
        if (e->keep && latent != nullptr)
            VCB_CUDA_OK(cudaMemcpy2DAsync(e->latent + b * lat, TN * 4, latent, static_cast<size_t>(T) * 4, static_cast<size_t>(f) * 4,
                                          c.dimension, cudaMemcpyDeviceToDevice, st));
        return 0;
    };
    TcCodec* tc = e->tc.get();
    std::vector<int> tc_rows, cc_rows;
    for (int b = 0; b < B; ++b) (c.channels == 1 && tc_encoder_accepts(tc, lens_host[b]) ? tc_rows : cc_rows).push_back(b);
    // tensor-core rows, longest first, in chunks under the workspace limit; a chunk is sized for its longest row
    std::stable_sort(tc_rows.begin(), tc_rows.end(), [&](int a, int b) { return lens_host[a] > lens_host[b]; });
    for (size_t i0 = 0; i0 < tc_rows.size();) {
        const int Nmax = lens_host[tc_rows[i0]];
        size_t i1 = i0 + 1;
        while (i1 < tc_rows.size() && tc_encoder_ws_bytes(tc, static_cast<int>(i1 - i0 + 1), Nmax) <= tc_ws_limit(tc)) ++i1;
        const int nb = static_cast<int>(i1 - i0);
        std::vector<int> rows(tc_rows.begin() + i0, tc_rows.begin() + i1), lens(nb);
        for (int j = 0; j < nb; ++j) lens[j] = lens_host[rows[j]];
        TcEncOut out;
        if (tc_encoder_encode(tc, wav_dev, N, rows.data(), lens.data(), nb, st, &e->launches, &out)) return -1;
        // (the latent is kept, in stream order, before the search consumes it as its residual)
        if (e->keep)
            for (int j = 0; j < nb; ++j)
                VCB_CUDA_OK(cudaMemcpy2DAsync(e->latent + rows[j] * lat, TN * 4, out.latent + static_cast<size_t>(j) * c.dimension * out.T,
                                              static_cast<size_t>(out.T) * 4, static_cast<size_t>(frames_host[rows[j]]) * 4, c.dimension,
                                              cudaMemcpyDeviceToDevice, st));
        if (rvq_encode(e, out.latent, out.scores, out.codes, nb, out.T, st)) return -1;
        for (int j = 0; j < nb; ++j)
            if (place(rows[j], out.codes + static_cast<size_t>(j) * c.n_q * out.T, nullptr, out.T)) return -1;
        e->encode_rows += tc_encoder_rows(tc, nb, Nmax);
        i0 = i1;
    }
    if (!tc_rows.empty()) e->tc_encodes++;
    // every other row alone on the CUDA-core encoder: what enc_encode of that row alone computes
    for (int b : cc_rows) {
        const int L = lens_host[b], T = frames_host[b];
        if (e->row_wav.size() < static_cast<size_t>(c.channels) * L && e->row_wav.alloc(static_cast<size_t>(c.channels) * L)) return -1;
        if (e->row_codes.size() < static_cast<size_t>(c.n_q) * T && e->row_codes.alloc(static_cast<size_t>(c.n_q) * T)) return -1;
        VCB_CUDA_OK(cudaMemcpy2DAsync(e->row_wav, static_cast<size_t>(L) * 4, wav_dev + static_cast<size_t>(b) * c.channels * N,
                                      static_cast<size_t>(N) * 4, static_cast<size_t>(L) * 4, c.channels, cudaMemcpyDeviceToDevice, st));
        if (ensure_buffers(e, 1, (L + e->hop - 1) / e->hop + 1)) return -1;
        // (its latent, under VCB_CODEC_KEEP, in buf[2]: scratch of the encoder layers that the RVQ search leaves alone)
        if (encode_chunk(e, e->row_wav, e->row_codes, e->keep ? e->buf[2].get() : nullptr, 1, L, st)) return -1;
        if (place(b, e->row_codes, e->buf[2], T)) return -1;
    }
    return 0;
}

int enc_debug_tensor(enc_engine* e, const char* name, float* host_out, int64_t cap, int32_t* dims) {
    if (e && name && !strcmp(name, "enc.latent")) {
        if (e->lat_B == 0) {
            set_error("codec: no enc.latent: it is kept by an enc_encode of an engine finalized under VCB_CODEC_KEEP=1");
            return -1;
        }
        const int64_t n = static_cast<int64_t>(e->lat_B) * e->cfg.dimension * e->lat_T;
        dims[0] = e->lat_B; dims[1] = e->cfg.dimension; dims[2] = e->lat_T; dims[3] = 0;
        if (host_out == nullptr) return 0;
        if (cap < n) {
            set_error("codec: debug buffer too small");
            return -1;
        }
        VCB_CUDA_OK(cudaSetDevice(e->cfg.device));
        VCB_CUDA_OK(cudaDeviceSynchronize());
        VCB_CUDA_OK(cudaMemcpy(host_out, e->latent, n * 4, cudaMemcpyDeviceToHost));
        return 0;
    }
    if (!e || !e->tc) {
        set_error("codec: the tensor-core decoder is not active (%s)", e ? e->tc_reason : "null engine");
        return -1;
    }
    return tc_codec_debug_tensor(e->tc.get(), name, host_out, cap, dims);
}

int64_t enc_counter(enc_engine* e, const char* name) {
    if (!strcmp(name, "live_bytes")) return LiveCount::bytes;          // process-wide, valid with a null engine
    if (!strcmp(name, "live_handles")) return LiveCount::handles;
    if (!strcmp(name, "resample_launches")) return resample_launches();
    if (!strcmp(name, "launches")) return e->launches;
    if (!strcmp(name, "hop")) return e->hop;
    if (!strcmp(name, "flops_per_frame")) return static_cast<int64_t>(e->flops_per_frame);
    if (!strcmp(name, "tc_enabled")) return e->tc != nullptr;
    if (!strcmp(name, "tc_decodes")) return e->tc_decodes;
    if (!strcmp(name, "stream_decodes")) return e->stream_decodes;
    if (!strcmp(name, "tc_encodes")) return e->tc_encodes;
    if (!strcmp(name, "encode_rows")) return e->encode_rows;
    if (!strcmp(name, "tc_encoder")) return tc_encoder_active(e->tc.get());
    if (!strcmp(name, "stream_min_frames")) return e->tc ? tc_stream_min_frames(e->tc.get()) : -1;
    if (!strcmp(name, "stream_state_bytes")) return e->tc ? static_cast<int64_t>(tc_stream_state_bytes(e->tc.get())) : -1;
    return -1;
}

int enc_stream_create(enc_engine* e, int32_t max_streams, enc_stream** out) {
    if (!e || !out || !e->finalized) {
        set_error("codec stream: engine not finalized");
        return -1;
    }
    *out = nullptr;
    if (!e->tc) {
        set_error("codec stream: streaming runs only on the tensor-core decoder, which does not cover this codec (%s)", e->tc_reason);
        return -1;
    }
    if (max_streams < 1) {
        set_error("codec stream: max_streams = %d", max_streams);
        return -1;
    }
    VCB_CUDA_OK(cudaSetDevice(e->cfg.device));
    std::unique_ptr<enc_stream> s(new enc_stream());
    s->e = e;
    s->max_streams = max_streams;
    s->frames.assign(max_streams, 0);
    const size_t bytes = static_cast<size_t>(max_streams) * tc_stream_state_bytes(e->tc.get());
    if (s->state.alloc(bytes) || s->table.alloc(static_cast<size_t>(max_streams) * 4) || s->bad.alloc(1)) {
        set_error("codec stream: cannot allocate the state of %d streams (%zu bytes)", max_streams, bytes);
        return -1;
    }
    *out = s.release();
    return 0;
}

int enc_stream_destroy(enc_stream* s) {
    if (!s) return 0;
    cudaSetDevice(s->e->cfg.device);
    cudaDeviceSynchronize();
    delete s;
    return 0;
}

int enc_stream_reset(enc_stream* s, const int32_t* ids_host, int32_t n) {
    if (!s || (n > 0 && !ids_host)) {
        set_error("codec stream: null argument");
        return -1;
    }
    for (int i = 0; i < n; ++i)
        if (ids_host[i] < 0 || ids_host[i] >= s->max_streams) {
            set_error("codec stream: id %d outside [0, %d)", ids_host[i], s->max_streams);
            return -1;
        }
    for (int i = 0; i < n; ++i) s->frames[ids_host[i]] = 0;
    return 0;
}

int enc_stream_decode(enc_engine* e, enc_stream* s, const int32_t* ids_host, const int32_t* lens_host, int32_t B,
                      const int64_t* codes_dev, int32_t T, float* wav_dev, void* stream) {
    if (!e || !s || s->e != e || !ids_host || !lens_host || !codes_dev || !wav_dev) {
        set_error("codec stream: null argument or a stream of another engine");
        return -1;
    }
    if (B < 1 || B > s->max_streams || T < 1) {
        set_error("codec stream: B = %d (max_streams %d), T = %d", B, s->max_streams, T);
        return -1;
    }
    // everything is validated before any stream changes
    const int min_frames = tc_stream_min_frames(e->tc.get());
    std::vector<char> seen(s->max_streams, 0);
    std::vector<int> table(static_cast<size_t>(B) * 4);
    for (int b = 0; b < B; ++b) {
        const int id = ids_host[b], len = lens_host[b];
        if (id < 0 || id >= s->max_streams) {
            set_error("codec stream: row %d: id %d outside [0, %d)", b, id, s->max_streams);
            return -1;
        }
        if (seen[id]) {
            set_error("codec stream: id %d appears twice in one call", id);
            return -1;
        }
        seen[id] = 1;
        if (len < 1 || len > T) {
            set_error("codec stream: row %d: %d frames outside [1, T = %d]", b, len, T);
            return -1;
        }
        if (s->frames[id] == 0 && len < min_frames) {
            set_error("codec stream: stream %d starts with %d frames; a fresh stream needs at least %d", id, len, min_frames);
            return -1;
        }
        table[4 * b] = id;
        table[4 * b + 1] = len;
        table[4 * b + 2] = s->frames[id] > 0;
        table[4 * b + 3] = 0;
    }
    VCB_CUDA_OK(cudaSetDevice(e->cfg.device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int bad = 0;
    if (tc_codes_check(codes_dev, static_cast<long long>(B) * e->cfg.n_q * T, e->cfg.bins, s->bad, &bad, st)) return -1;
    if (bad) {
        set_error("codec stream: a code lies outside [0, %d)", e->cfg.bins);
        return -1;
    }
    VCB_CUDA_OK(cudaMemcpyAsync(s->table, table.data(), table.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    const TcStreamCtx ctx{s->table, s->state};
    if (tc_codec_decode(e->tc.get(), codes_dev, wav_dev, B, T, st, &e->launches, &ctx)) return -1;
    for (int b = 0; b < B; ++b) s->frames[ids_host[b]] += lens_host[b];
    e->stream_decodes++;
    return 0;
}

}  // extern "C"
