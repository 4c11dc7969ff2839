// EnCodec SEANet decoder on the tensor cores (wgmma).
//
// Replaces, for the configurations it covers, the CUDA-core kernels of encodec.cu behind the same entry point
// (enc_decode <- AudioTokenizer.decode, reference data/tokenizer.py:131-133 -> audiocraft EncodecModel.decode).
//
// Every layer of the decoder is one launch of ONE kernel, an implicit GEMM with the time steps as the MMA M dimension:
//
//   activations  channels-last bf16 "planes": x ~= hi + lo (split_bf16), tensor [2 planes][rows][C], a row = one time step of
//                one utterance, every utterance preceded by `halo` rows that hold its left padding (reflect or zero), so a
//                causal convolution tap is the same 128-row TMA box shifted up by (k-1-j)*dilation rows -- no im2col, no
//                gather.  C is padded to a multiple of 64 (one 128-byte swizzle row) with zero channels.
//   weights      fp32 -> (hi, lo) bf16, pre-tiled [n-tile][k-block][hi|lo][BN][64]: one TMA box per k-block.
//   arithmetic   D += Ahi*Bhi + Alo*Bhi + Ahi*Blo in fp32 registers: the "3-pass" product, relative error ~2^-16 per term, i.e.
//                fp32-level parity with the CUDA-core path (tests/test_codec.py states the waveform tolerance).
//   ConvTranspose1d (stride r, kernel 2r, causal trim): y[t*r+p] = W[:,:,p] x[t] + W[:,:,p+r] x[t-1]: a 2-tap convolution
//                with N = r*Cout whose output row [r*Cout] IS r consecutive channels-last output rows.
//   residual block  conv k3 -> hidden; then conv k1 (hidden) and the 1x1 shortcut (block input) are ONE GEMM with
//                K = hidden + C (two A sources), bias = b2 + bs.
//   epilogue     accumulators staged in shared memory, read back one row per thread: + bias, optional ELU, split to planes (raw and/or ELU'd form, as the consumers need),
//                mirror rows 1..pad into the halo (reflect) or zero it; or fp32 rows (LSTM pre-activations, waveform).
//   LSTM         W_ih for all steps is one GEMM; each step is one launch of the same kernel over h_{t-1} planes with the
//                gates interleaved (n = 4*unit + gate) so the epilogue owns complete cells: c/h update, h_t planes for the
//                next step, and for the last layer ELU(h + skip) straight into the first ConvTranspose's input.
//                800 steps x 2 layers = 1 600 dependent launches for the WHOLE batch (was: per 16 utterances), W_hh (16.8 MB
//                as planes) stays in L2; chained with programmatic dependent launch, weights in flight before the wait.
//
// The encoder (enc_encode_ragged) runs on the same kernel from a plan of its own (EncPlan): input staging to 7-sample
// windows (enc.conv_in = one k-block), the residual blocks as above, each strided conv (k = 2r, stride r) as a 2-tap conv
// over the input read as folded rows [rows / r][r * C] with its per-utterance right padding written by tc_pad_rows_kernel,
// the LSTM above, enc.conv_out to fp32 rows; the RVQ search stays the fp32 one of encodec.cu.
#include "codec_tc.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "vcb_internal.h"

namespace vcb {

static constexpr int TC_BM = 128;
static constexpr int TC_BK = 64;
static constexpr int TC_EPI_WARPS = 16;
static constexpr int TC_THREADS = 128 + 32 * TC_EPI_WARPS;
static constexpr int TC_MAX_KB = 128;               // k-blocks per GEMM: the encoder's last strided conv has K = 2*8*512
enum { TC_MODE_CONV = 0, TC_MODE_LSTM = 1 };

struct TcTap {
    short src;     // which A tensor map (0 / 1)
    short shift;   // rows above the output row
    int coff;      // first channel of this k-block
};

struct TcCall {
    int total_kb, ntiles, mtiles, rows_total, row_base;
    int rcap[2];                       // rows per plane of A source 0 / 1 (lo plane = + rcap rows)
    int in_store_halo;                 // 1: halo rows (t >= -in_halo) are computed and stored too
    int in_div, in_tm, in_halo, T_in, B;   // A row -> (b, t): utterance-major (row / Tp, row % Tp - halo) or time-major
    int mode, up, Cout, Nstore;        // GEMM column n -> (phase p = n / Cout, channel n % Cout); columns >= Nstore are padding
    const float* bias;
    __nv_bfloat16* raw;                // optional output planes, raw / ELU'd form; row(b, t') = b*o_sb + t'*o_st + o_off
    __nv_bfloat16* elu;
    long long o_plane, o_sb, o_st, o_off;
    int o_ld, o_halo, o_halo_zero;     // halo rows t' = -1..-o_halo: mirror of rows 1..o_halo (reflect) or zeros
    float* f32;                        // optional fp32 rows
    long long f_sb, f_st, f_off;
    int f_ld, f_valid, f_scalar;
    // LSTM step
    const float* pre;                  // [T][Bcap][4H] gate pre-activations (interleaved), bias included
    float* cst;                        // [Bcap][H]
    const float* skip;                 // [T][Bcap][H] or null
    __nv_bfloat16* hseq;               // planes [T+1][Bcap][H]; slot t+1 = h_t
    long long h_plane;
    int t_step, Bcap, H;
    const int* stab;                   // stream decode: per utterance {id, valid frames, continuing, 0}; c frozen past its frames
    TcTap taps[TC_MAX_KB];
};

template <int BN, int STAGES>
struct TcSmem {
    static constexpr int A_BYTES = TC_BM * TC_BK * 2;
    static constexpr int B_BYTES = BN * TC_BK * 2;
    static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
    static constexpr int ACC_LD = BN + 4;                   // staged accumulators [128][ACC_LD] fp32, conflict-free rows
    static constexpr int ACC_OFFSET = STAGES * STAGE_BYTES;
    static constexpr int BAR_OFFSET = ACC_OFFSET + TC_BM * ACC_LD * 4;
    static constexpr int TOTAL = BAR_OFFSET + 2 * STAGES * 8;
};

// ELU for the planes the next layer reads: exp through ex2.approx (absolute error ~2e-7, far below the 2^-17 relative
// error of the hi/lo split it feeds)
__device__ __forceinline__ float tc_elu(float x) { return x > 0.f ? x : __expf(x) - 1.f; }
__device__ __forceinline__ float tc_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// two fp32 -> packed bf16x2 hi parts and bf16x2 lo parts (same roundings as split_bf16)
__device__ __forceinline__ void tc_split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    hi = *reinterpret_cast<uint32_t*>(&h);
    __nv_bfloat162 l = __floats2bfloat162_rn(a - __uint_as_float(hi << 16), b - __uint_as_float(hi & 0xffff0000u));
    lo = *reinterpret_cast<uint32_t*>(&l);
}
__device__ __forceinline__ void tc_split8(const float* v, uint4& hi, uint4& lo) {
    tc_split2(v[0], v[1], hi.x, lo.x);
    tc_split2(v[2], v[3], hi.y, lo.y);
    tc_split2(v[4], v[5], hi.z, lo.z);
    tc_split2(v[6], v[7], hi.w, lo.w);
}

// 32 bytes per lane (two 16-byte stores): every lane writes a whole 32-byte sector
__device__ __forceinline__ void tc_st256(void* p, const uint4& a, const uint4& b) {
    reinterpret_cast<uint4*>(p)[0] = a;
    reinterpret_cast<uint4*>(p)[1] = b;
}

// CW consecutive channels of one row -> both planes (and the mirrored halo row, if any).
template <int CW>
__device__ __forceinline__ void tc_store_planes(__nv_bfloat16* base, long long plane, int ld, long long row, long long mirror,
                                                int co0, const float (&v)[CW], bool elu, bool zero_mirror) {
    uint4 hi[CW / 8], lo[CW / 8];
#pragma unroll
    for (int j = 0; j < CW / 8; ++j) {
        float w[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) w[u] = elu ? tc_elu(v[8 * j + u]) : v[8 * j + u];
        tc_split8(w, hi[j], lo[j]);
    }
    __nv_bfloat16* ph = base + row * ld + co0;
    __nv_bfloat16* pl = ph + plane;
#pragma unroll
    for (int j = 0; j < CW / 16; ++j) {
        tc_st256(ph + 16 * j, hi[2 * j], hi[2 * j + 1]);
        tc_st256(pl + 16 * j, lo[2 * j], lo[2 * j + 1]);
    }
    if (mirror >= 0) {
        __nv_bfloat16* mh = base + mirror * ld + co0;
        __nv_bfloat16* ml = mh + plane;
        const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int j = 0; j < CW / 16; ++j) {
            tc_st256(mh + 16 * j, zero_mirror ? z : hi[2 * j], zero_mirror ? z : hi[2 * j + 1]);
            tc_st256(ml + 16 * j, zero_mirror ? z : lo[2 * j], zero_mirror ? z : lo[2 * j + 1]);
        }
    }
}

template <int CW>
__device__ __forceinline__ void tc_epilogue_conv(const TcCall& c, int b, int t, int n0, float (&v)[CW], const float4 (&bias)[CW / 4]) {
    const int p = n0 / c.Cout, co0 = n0 - p * c.Cout;
    const int t_out = t * c.up + p;
#pragma unroll
    for (int j = 0; j < CW / 4; ++j) {
        v[4 * j] += bias[j].x; v[4 * j + 1] += bias[j].y; v[4 * j + 2] += bias[j].z; v[4 * j + 3] += bias[j].w;
    }
    if (c.f32 != nullptr) {
        float* dst = c.f32 + (b * c.f_sb + t_out * c.f_st + c.f_off) * c.f_ld + co0;
        if (c.f_scalar) {
#pragma unroll
            for (int j = 0; j < CW; ++j)
                if (co0 + j < c.f_valid) dst[j] = v[j];
        } else if (co0 < c.f_valid) {
            float4* d4 = reinterpret_cast<float4*>(dst);
#pragma unroll
            for (int j = 0; j < CW / 4; ++j)
                if (co0 + 4 * j < c.f_valid) d4[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
        }
    }
    if (c.raw != nullptr || c.elu != nullptr) {
        const long long row = b * c.o_sb + t_out * c.o_st + c.o_off;
        const long long mirror = (t_out >= 1 && t_out <= c.o_halo) ? row - 2ll * t_out * c.o_st : -1ll;
        if (c.raw != nullptr) tc_store_planes<CW>(c.raw, c.o_plane, c.o_ld, row, mirror, co0, v, false, c.o_halo_zero != 0);
        if (c.elu != nullptr) tc_store_planes<CW>(c.elu, c.o_plane, c.o_ld, row, mirror, co0, v, true, c.o_halo_zero != 0);
    }
}

// columns [n0, n0+CW) = gates (i, f, g, o) of hidden units [n0/4, n0/4 + CW/4) of utterance b at step c.t_step
template <int CW>
__device__ __forceinline__ void tc_epilogue_lstm(const TcCall& c, int b, int n0, float (&v)[CW]) {
    constexpr int U = CW / 4;
    const int j0 = n0 >> 2;
    const size_t tb = static_cast<size_t>(c.t_step) * c.Bcap + b;
    const float4* pr = reinterpret_cast<const float4*>(c.pre + tb * (4 * static_cast<size_t>(c.H)) + n0);
    float* cp = c.cst + static_cast<size_t>(b) * c.H + j0;
    float cs[U], h[U];
#pragma unroll
    for (int u = 0; u < U; u += 4) {
        const float4 c4 = *reinterpret_cast<const float4*>(cp + u);
        cs[u] = c4.x; cs[u + 1] = c4.y; cs[u + 2] = c4.z; cs[u + 3] = c4.w;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
        const float4 g = pr[u];
        const float ig = tc_sigmoid(v[4 * u] + g.x), fg = tc_sigmoid(v[4 * u + 1] + g.y);
        const float gg = tanhf(v[4 * u + 2] + g.z), og = tc_sigmoid(v[4 * u + 3] + g.w);
        cs[u] = fg * cs[u] + ig * gg;
        h[u] = og * tanhf(cs[u]);
    }
    if (c.stab == nullptr || c.t_step < c.stab[4 * b + 1]) {    // a stream's c stays at its last valid step
#pragma unroll
        for (int u = 0; u < U; u += 4) *reinterpret_cast<float4*>(cp + u) = make_float4(cs[u], cs[u + 1], cs[u + 2], cs[u + 3]);
    }
    __nv_bfloat16* hp = c.hseq + (tb + c.Bcap) * c.H + j0;          // slot t+1
    const float* sk = c.elu != nullptr ? c.skip + tb * c.H + j0 : nullptr;
    __nv_bfloat16* op = c.elu != nullptr ? c.elu + (b * c.o_sb + c.t_step * c.o_st + c.o_off) * c.o_ld + j0 : nullptr;
#pragma unroll
    for (int u = 0; u < U; u += 4) {
        uint2 hi, lo;
        tc_split2(h[u], h[u + 1], hi.x, lo.x);
        tc_split2(h[u + 2], h[u + 3], hi.y, lo.y);
        *reinterpret_cast<uint2*>(hp + u) = hi;
        *reinterpret_cast<uint2*>(hp + c.h_plane + u) = lo;
        if (op != nullptr) {
            const float4 s4 = *reinterpret_cast<const float4*>(sk + u);
            tc_split2(tc_elu(h[u] + s4.x), tc_elu(h[u + 1] + s4.y), hi.x, lo.x);
            tc_split2(tc_elu(h[u + 2] + s4.z), tc_elu(h[u + 3] + s4.w), hi.y, lo.y);
            *reinterpret_cast<uint2*>(op + u) = hi;
            *reinterpret_cast<uint2*>(op + c.o_plane + u) = lo;
        }
    }
}

// Persistent: CTA i works on tiles i, i + grid, ... (tile = m-tile * ntiles + n-tile, n fastest so the CTAs that run
// together share their A rows in L2).  The TMA producer runs ahead across tile boundaries through the shared-memory ring.
// Four warpgroups each multiply a quarter of the tile (64 rows x BN/2 columns), stage it in shared memory and then run
// the epilogue one row per thread.
template <int BN, int STAGES, int CW>
__global__ void __launch_bounds__(TC_THREADS)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
               const __grid_constant__ CUtensorMap tmW, const __grid_constant__ TcCall c) {
    using L = TcSmem<BN, STAGES>;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
    uint64_t* empty_bar = full_bar + STAGES;
    float* sacc = reinterpret_cast<float*>(smem + L::ACC_OFFSET);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int total_kb = c.total_kb;
    const int total_tiles = c.mtiles * c.ntiles;
    const int pre = min(total_kb, STAGES);

    pdl_launch_dependents();
    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA0);
        tma_prefetch_desc(&tmA1);
        tma_prefetch_desc(&tmW);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], TC_EPI_WARPS);        // one arrival per MMA warp
        }
        mbar_fence_init();
        if (static_cast<int>(blockIdx.x) < total_tiles) {   // weights never depend on the previous kernel
            const int ntile = blockIdx.x % c.ntiles;
            for (int i = 0; i < pre; ++i) {
                mbar_arrive_expect_tx(&full_bar[i], L::STAGE_BYTES);
                tma_load_2d(smem + i * L::STAGE_BYTES + 2 * L::A_BYTES, &tmW, &full_bar[i], 0, (ntile * total_kb + i) * 2 * BN);
            }
        }
    }
    __syncthreads();

    if (warp == 0) {
        if (lane == 0) {
            pdl_wait();                                     // the activation planes come from the previous kernel
            int g = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int ntile = tile % c.ntiles, mtile = tile / c.ntiles;
                const int r0 = c.row_base + mtile * TC_BM;
                for (int i = 0; i < total_kb; ++i, ++g) {
                    const int stage = g % STAGES, use = g / STAGES;
                    uint8_t* a = smem + stage * L::STAGE_BYTES;
                    if (g >= pre) {                         // (the first `pre` k-blocks were armed above, with their weights)
                        if (use > 0) mbar_wait(&empty_bar[stage], (use - 1) & 1);
                        mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
                        tma_load_2d(a + 2 * L::A_BYTES, &tmW, &full_bar[stage], 0, (ntile * total_kb + i) * 2 * BN);
                    }
                    const TcTap tp = c.taps[i];
                    const CUtensorMap* m = tp.src ? &tmA1 : &tmA0;
                    const int row = r0 - tp.shift;
                    tma_load_2d(a, m, &full_bar[stage], tp.coff, row);
                    tma_load_2d(a + L::A_BYTES, m, &full_bar[stage], tp.coff, c.rcap[tp.src] + row);
                }
            }
        }
    } else if (warp >= 4) {
        const int q = warp & 3;                             // warp inside its warpgroup; epilogue: rows [32 q, 32 q + 32)
        const int grp = (warp - 4) >> 2;                    // warpgroup; epilogue: which column chunk
        const int mrow = (grp & 1) * 64, ncol = (grp >> 1) * (BN / 2);   // this warpgroup's quarter of the MMA tile
        pdl_wait();                                         // what the epilogue overwrites may still be read upstream
        int g = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int ntile = tile % c.ntiles, mtile = tile / c.ntiles;
            const int row = c.row_base + mtile * TC_BM + q * 32 + lane;
            int b, t;
            bool valid;
            if (c.mode == TC_MODE_LSTM) {
                b = row - c.row_base;
                t = c.t_step;
                valid = b < c.B;
            } else {
                const int qd = row / c.in_div, rm = row - qd * c.in_div;
                if (c.in_tm) { t = qd - c.in_halo; b = rm; }
                else { b = qd; t = rm - c.in_halo; }
                valid = row < c.rows_total && b < c.B && t >= (c.in_store_halo ? -c.in_halo : 0) && t < c.T_in;
            }
            // BN / CW <= 4 chunks and 4 warp groups: a warp owns at most one chunk of every tile.  Its bias is fetched while
            // the accumulator is still being produced.
            static_assert(BN / CW <= TC_EPI_WARPS / 4, "one column chunk per epilogue warp");
            const bool has_chunk = grp < BN / CW;
            const int n0 = ntile * BN + grp * CW;
            float4 bias[CW / 4];
            if (has_chunk) {
                const float4* b4 = reinterpret_cast<const float4*>(c.bias + n0);
#pragma unroll
                for (int j = 0; j < CW / 4; ++j) bias[j] = b4[j];
            }
            float acc[BN / 4];
#pragma unroll
            for (int j = 0; j < BN / 4; ++j) acc[j] = 0.f;
            int prev = -1;
            for (int i = 0; i < total_kb; ++i, ++g) {
                const int stage = g % STAGES;
                mbar_wait(&full_bar[stage], (g / STAGES) & 1);
                const uint32_t a_addr = smem_u32(smem + stage * L::STAGE_BYTES) + mrow * 128;
                const uint32_t b_addr = smem_u32(smem + stage * L::STAGE_BYTES + 2 * L::A_BYTES) + ncol * 128;
                wg_fence();
                wg_mma_kblock<BN / 2>(acc, a_addr, b_addr);                              // Ahi * Bhi
                wg_mma_kblock<BN / 2>(acc, a_addr + L::A_BYTES, b_addr);                 // Alo * Bhi
                wg_mma_kblock<BN / 2>(acc, a_addr, b_addr + L::B_BYTES);                 // Ahi * Blo
                wg_commit();
                wg_wait1();                                 // k-block i-1's MMAs are complete, i's may still run
                __syncwarp();
                if (lane == 0 && prev >= 0) mbar_arrive(&empty_bar[prev]);
                prev = stage;
            }
            wg_wait0();
            __syncwarp();
            if (lane == 0 && prev >= 0) mbar_arrive(&empty_bar[prev]);
            wg_acc_fence(acc);
            // the previous tile's read-out is complete before the staged accumulators are overwritten
            asm volatile("bar.sync 1, %0;" ::"n"(32 * TC_EPI_WARPS) : "memory");
            {
                const int r = mrow + q * 16 + (lane >> 2);
#pragma unroll
                for (int j = 0; j < BN / 16; ++j) {
                    const int cc = ncol + 8 * j + 2 * (lane & 3);
                    *reinterpret_cast<float2*>(sacc + r * L::ACC_LD + cc) = make_float2(acc[4 * j], acc[4 * j + 1]);
                    *reinterpret_cast<float2*>(sacc + (r + 8) * L::ACC_LD + cc) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
                }
            }
            asm volatile("bar.sync 1, %0;" ::"n"(32 * TC_EPI_WARPS) : "memory");
            if (has_chunk) {
                float v[CW];
                const float* src = sacc + (q * 32 + lane) * L::ACC_LD + grp * CW;
#pragma unroll
                for (int j = 0; j < CW; j += 4) {
                    const float4 t4 = *reinterpret_cast<const float4*>(src + j);
                    v[j] = t4.x; v[j + 1] = t4.y; v[j + 2] = t4.z; v[j + 3] = t4.w;
                }
                if (valid && n0 < c.Nstore) {
                    if (c.mode == TC_MODE_LSTM) tc_epilogue_lstm<CW>(c, b, n0, v);
                    else tc_epilogue_conv<CW>(c, b, t, n0, v, bias);
                }
            }
        }
    }
}

// codes [B][K][T] -> latent planes (row (b, t) = b*Tp + halo + t, D channels of ld), halo mirrored / zeroed
__global__ void __launch_bounds__(128)
tc_rvq_planes_kernel(const long long* __restrict__ codes, const float* const* __restrict__ embed, __nv_bfloat16* out,
                     long long plane, int K, int D, int ld, int T, int Tp, int halo, int halo_zero) {
    const int b = blockIdx.y, t0 = blockIdx.x * 16;
    for (int tt = 0; tt < 16; ++tt) {
        const int t = t0 + tt;
        if (t >= T) break;
        for (int ch = threadIdx.x; ch < ld; ch += blockDim.x) {
            float acc = 0.f;
            if (ch < D)
                for (int q = 0; q < K; ++q)
                    acc += embed[q][static_cast<size_t>(codes[(static_cast<size_t>(b) * K + q) * T + t]) * D + ch];
            __nv_bfloat16 hi, lo;
            split_bf16(acc, hi, lo);
            const long long row = static_cast<long long>(b) * Tp + halo + t;
            out[row * ld + ch] = hi;
            out[plane + row * ld + ch] = lo;
            if (t >= 1 && t <= halo) {
                const long long mr = row - 2ll * t;
                out[mr * ld + ch] = halo_zero ? __float2bfloat16_rn(0.f) : hi;
                out[plane + mr * ld + ch] = halo_zero ? __float2bfloat16_rn(0.f) : lo;
            }
        }
    }
}

// Final convolution (C channels -> 1 channel, k taps), split so that the activation planes are read ONCE:
//   P[row][j] = sum_c w[c][j] * x[row][c]          one k = 1 GEMM with N = k columns (conv_tc_kernel, fp32 rows of 8)
//   out[t]    = bias + sum_j P[t - (k-1-j)][j]     this kernel: k shifted diagonals, staged through shared memory
// (as a k-tap implicit GEMM it would pull k shifted copies of every 128-row tile through shared memory for one output column).
static constexpr int DS_ROWS = 256;
static constexpr int DS_LD = 8;                            // floats per P row (k <= 8)
__global__ void __launch_bounds__(DS_ROWS)
tc_diag_sum_kernel(const float* __restrict__ P, int k, float bias, float* __restrict__ out, int rows_total, int Tp, int halo,
                   int T, int B) {
    __shared__ float ps[(DS_ROWS + DS_LD) * (DS_LD + 1)];
    const long long r0 = static_cast<long long>(blockIdx.x) * DS_ROWS - (k - 1);
    pdl_wait();
    const int W = DS_ROWS + k - 1;
    for (int i = threadIdx.x; i < W * DS_LD; i += DS_ROWS) {  // contiguous floats of P: coalesced
        const long long row = r0 + i / DS_LD;
        ps[(i / DS_LD) * (DS_LD + 1) + (i % DS_LD)] = (row >= 0 && row < rows_total) ? P[row * DS_LD + (i % DS_LD)] : 0.f;
    }
    __syncthreads();
    const long long row = static_cast<long long>(blockIdx.x) * DS_ROWS + threadIdx.x;
    if (row >= rows_total) return;
    const int b = static_cast<int>(row / Tp), t = static_cast<int>(row - static_cast<long long>(b) * Tp) - halo;
    if (b >= B || t < 0 || t >= T) return;
    float acc = bias;
    for (int j = 0; j < k; ++j) acc += ps[(threadIdx.x + j) * (DS_LD + 1) + j];   // window row threadIdx.x + j = t - (k-1-j)
    out[static_cast<size_t>(b) * T + t] = acc;
}

// Stream decode: carry the left context of one plane across calls.  Block b = utterance b of the call, which continues
// stream table[4b] with table[4b+1] valid frames (table[4b+2] = 1: the stream has decoded frames before).  Launched after the
// plane's producer and before its consumer:
//   restore  a continuing stream's halo rows t = -halo..-1 <- its saved tail (they replace the reflect / zero padding);
//   save     the stream's saved tail <- rows [len*up - halo, len*up), which reach back into the restored halo when len*up < halo.
// The saved tail is stored exactly as the plane stores it (bf16 hi and lo planes, or fp32), [plane][halo rows][row_bytes].
// One block owns one stream (the ids of a call are distinct), and the block barrier orders reading the old tail before
// writing the new one.
struct CarryArgs {
    uint8_t* base;                     // plane storage; the second plane (lo) at + plane_bytes (0: a single plane)
    long long plane_bytes;
    long long sb, st, off;             // row(b, t) = b*sb + t*st + off
    int row_bytes;                     // multiple of 16
    int halo, up;                      // rows carried; plane rows per frame
    int restore, save;
    const int* table;
    uint8_t* state;
    long long state_stride, state_off; // stream id's tail at state + id*state_stride + state_off
};

__global__ void __launch_bounds__(256) tc_carry_kernel(const __grid_constant__ CarryArgs a) {
    pdl_launch_dependents();
    pdl_wait();                                                     // the producer has written the plane
    const int b = blockIdx.x;
    const int id = a.table[4 * b], len = a.table[4 * b + 1], cont = a.table[4 * b + 2];
    const int per_row = a.row_bytes / 16, per_plane = a.halo * per_row;
    const int n = (a.plane_bytes ? 2 : 1) * per_plane;
    uint4* s = reinterpret_cast<uint4*>(a.state + id * a.state_stride + a.state_off);
    auto at = [&](int i, int t) {
        const int p = i / per_plane, r = i - p * per_plane, col = r % per_row;
        return reinterpret_cast<uint4*>(a.base + p * a.plane_bytes + (b * a.sb + t * a.st + a.off) * a.row_bytes) + col;
    };
    if (a.restore && cont)
        for (int i = threadIdx.x; i < n; i += blockDim.x) *at(i, (i % per_plane) / per_row - a.halo) = s[i];
    __syncthreads();
    if (a.save)
        for (int i = threadIdx.x; i < n; i += blockDim.x) s[i] = *at(i, len * a.up - a.halo + (i % per_plane) / per_row);
}

// Encoder input: fp32 wav rows -> planes whose channel j (< k) at row t holds sample t - (k-1) + j of the utterance, so that
// enc.conv_in is one k-block: its causal left padding is folded in (reflect, x[-s] = x[s]; or zeros).  Channels >= k and
// rows at or past the utterance's lens[b] samples are zero.  Chunk row b is wav row rows[b]; plane row(b, t) = b*Tp + t.
__global__ void __launch_bounds__(256)
tc_enc_input_kernel(const float* __restrict__ wav, long long wav_ld, const int* __restrict__ rows, const int* __restrict__ lens,
                    __nv_bfloat16* out, long long plane, int ld, int Tp, int T, int k, int reflect, int B) {
    const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (i >= static_cast<long long>(B) * T) return;
    const int b = static_cast<int>(i / T), t = static_cast<int>(i - static_cast<long long>(b) * T), L = lens[b];
    const float* x = wav + rows[b] * wav_ld;
    __nv_bfloat16* o = out + (static_cast<long long>(b) * Tp + t) * ld;
    for (int c0 = 0; c0 < ld; c0 += 8) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            int s = t - (k - 1) + c0 + u;
            if (s < 0 && reflect) s = -s;
            v[u] = (c0 + u < k && t < L && s >= 0 && s < L) ? x[s] : 0.f;
        }
        uint4 hi, lo;
        tc_split8(v, hi, lo);
        *reinterpret_cast<uint4*>(o + c0) = hi;
        *reinterpret_cast<uint4*>(o + plane + c0) = lo;
    }
}

// Padding rows of one plane form, block b = utterance b:
//   lens == null   its left halo, rows -1..-n <- rows 1..n (reflect) -- for a plane whose producer writes no halo (LSTM)
//   lens != null   the right padding of a strided conv (stride r) over its lens[b] rows: rows L .. ceil(L/r)*r - 1 <- rows
//                  L-2, L-3, ... (reflect; audiocraft get_extra_padding_for_conv1d), which differs per utterance
// or zeros (zero != 0).  Rows are [2 planes][rows][ld] bf16, row(b, t) = b*sb + t*st + off.
__global__ void __launch_bounds__(256)
tc_pad_rows_kernel(__nv_bfloat16* base, long long plane, int ld, long long sb, long long st, long long off, const int* lens, int n,
                   int r, int zero) {
    const int b = blockIdx.x;
    int cnt = n, d0 = -1, dstep = -1, s0 = 1, sstep = 1;
    if (lens != nullptr) {
        const int L = lens[b];
        cnt = (L + r - 1) / r * r - L;
        d0 = L; dstep = 1; s0 = L - 2; sstep = -1;
    }
    const int per_row = ld / 8, per_plane = cnt * per_row;
    for (int i = threadIdx.x; i < 2 * per_plane; i += blockDim.x) {
        const int p = i / per_plane, rr = i - p * per_plane, j = rr / per_row, col = rr - j * per_row;
        const long long dst = b * sb + static_cast<long long>(d0 + dstep * j) * st + off;
        const long long src = b * sb + static_cast<long long>(s0 + sstep * j) * st + off;
        uint4* d = reinterpret_cast<uint4*>(base + p * plane + dst * ld) + col;
        *d = zero ? make_uint4(0u, 0u, 0u, 0u) : *(reinterpret_cast<const uint4*>(base + p * plane + src * ld) + col);
    }
}

// latent rows [B][T][ld] fp32 -> [B][D][T] (the layout of the RVQ search), 32 frames per block through shared memory
__global__ void __launch_bounds__(256)
tc_latent_cm_kernel(const float* __restrict__ in, float* __restrict__ out, int D, int ld, int T) {
    extern __shared__ float tile[];                                 // [32][D + 1]
    const int b = blockIdx.y, t0 = blockIdx.x * 32;
    for (int i = threadIdx.x; i < 32 * D; i += blockDim.x) {
        const int tt = i / D, c = i - tt * D;
        tile[tt * (D + 1) + c] = t0 + tt < T ? in[(static_cast<size_t>(b) * T + t0 + tt) * ld + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * D; i += blockDim.x) {
        const int c = i / 32, tt = i - c * 32;
        if (t0 + tt < T) out[(static_cast<size_t>(b) * D + c) * T + t0 + tt] = tile[tt * (D + 1) + c];
    }
}

// codes outside [0, bins) -> *bad = 1
__global__ void tc_codes_check_kernel(const long long* __restrict__ codes, long long n, int bins, int* bad) {
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x)
        if (codes[i] < 0 || codes[i] >= bins) *bad = 1;
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
namespace {

inline int cpad(int c) { return (c + 63) / 64 * 64; }
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

inline uint16_t f2bf(float f) {                                // round to nearest even, like __float2bfloat16_rn
    uint32_t u;
    memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x40);
    u += 0x7fffu + ((u >> 16) & 1u);
    return static_cast<uint16_t>(u >> 16);
}
inline float bf2f(uint16_t h) {
    uint32_t u = static_cast<uint32_t>(h) << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}

struct TcGemm {
    DevBuf<__nv_bfloat16> tiles;
    DevBuf<float> bias;
    int N = 0, BN = 0, ntiles = 0, total_kb = 0;
    int Cout = 0, up = 1;              // column n -> (n / Cout, n % Cout)
    CUtensorMap tmW;
    std::vector<TcTap> taps;
};

struct Plane {                         // an activation tensor in the workspace
    __nv_bfloat16* raw = nullptr;
    __nv_bfloat16* elu = nullptr;
    int C = 0;                         // padded channels (= ld)
    int rcap = 0;                      // rows per plane
    long long sb = 0, st = 1, off = 0; // row(b, t)
    int Tp = 0, halo = 0, halo_zero = 0, T = 0, tm = 0;
    long long plane() const { return static_cast<long long>(rcap) * C; }
};

// ---- the decoder plan: the layer sequence over a table of tensors, independent of (B, T).  The launches, the workspace,
// the stream-state layout and min_T are all derived from it.
enum { FORM_RAW = 1, FORM_ELU = 2 };
// HALO_UNWRITTEN: the rows exist (the tensor shares its block input's row geometry) but nothing stores or reads them
enum { HALO_REFLECT, HALO_ZERO, HALO_UNWRITTEN };
enum { HOME_ARENA0, HOME_ARENA1, HOME_HIDDEN, HOME_FIXED };   // ping-pong arenas of the stages, hidden arena, fixed region

struct PlanTensor {
    int C = 0, halo = 0, halo_kind = HALO_ZERO;
    int up = 1;                        // rows per frame: the product of the ratios so far
    bool tm = false;                   // time-major, row = (t + halo) * Bcap + b (LSTM planes); else utterance-major
    int forms = 0;                     // FORM_RAW | FORM_ELU stored
    int home = HOME_FIXED;
    bool carried = false;              // stream decode carries its halo rows (of the ELU'd form if stored, else raw) ...
    size_t state_off = 0;              // ... at this offset of a stream's state
    std::string dbg_raw, dbg_elu;      // enc_debug_tensor names of the two forms ("": not exposed)
};

enum { L_RVQ, L_CONV, L_LSTM_IH, L_LSTM_STEPS, L_CONV_OUT_SPLIT, L_CONV_OUT };
enum { F32_NONE, F32_X0, F32_PRE, F32_COPART, F32_WAV, F32_LAT };   // fp32 destination of a GEMM

struct PlanLayer {
    int kind = L_CONV;
    const char* label = "";            // VCB_CODEC_PROFILE
    const TcGemm* g = nullptr;
    int in = -1, in_form = FORM_RAW;   // A source 0
    int in2 = -1;                      // A source 1, raw form: the block input of a residual tail (shortcut)
    int out = -1, out_forms = 0;
    int f32 = F32_NONE;
    int nstore = 0;                    // GEMM columns stored
    int lstm = -1;                     // LSTM layer
    size_t h_off = 0, c_off = 0;       // LSTM steps: the layer's carried h and c in a stream's state
};

struct PlanStage { int up, C, Ch; };   // rows per frame, padded channels of the block tensors and of the hidden tensor

// ---- the encoder plan (SEANetEncoder, oracle/encodec_oracle.py::encoder_plan), over a table of tensors like the decoder's.
// A tensor belongs to a stage s (its rows are frames of stage s: the input's samples for s = 0, then one stage per strided
// conv) and holds, per utterance, `halo` rows of left padding and the stage's rows rounded up to the next strided conv's
// stride.  The input of a strided conv (stride r) has halo r and is read as folded rows [rows / r][r * C] (fold = r).
enum { E_INPUT, E_CONV, E_DOWN, E_RPAD, E_LSTM_IH, E_LSTM_STEPS, E_LPAD, E_CONV_OUT };

struct EncTensor {
    int C = 0, halo = 0, halo_kind = HALO_ZERO, stage = 0, fold = 1;
    bool tm = false;                   // time-major (LSTM planes)
    int forms = 0, home = HOME_FIXED;  // home: HOME_FIXED or the arena of its stage (HOME_ARENA0 + stage % 2)
    std::string dbg_raw, dbg_elu;
};

struct EncLayer {
    int kind = E_CONV;
    const char* label = "";
    const TcGemm* g = nullptr;
    int in = -1, in_form = FORM_RAW, in2 = -1, out = -1, out_forms = 0, f32 = F32_NONE, nstore = 0, lstm = -1;
    int stage = 0, r = 1;              // E_DOWN / E_RPAD: the stage and stride of the strided conv
};

struct EncPlan {
    std::vector<EncTensor> tensors;
    std::vector<EncLayer> layers;
    std::vector<int> ratios;           // stride of stage s's strided conv (the config's ratios reversed)
};

struct TcEncoder {
    TcGemm conv_in, conv_out;
    std::vector<TcGemm> down, pre, step;
    std::vector<std::vector<TcGemm>> res1, res2;
    EncPlan plan;
};

struct TcPlan {
    std::vector<PlanTensor> tensors;
    std::vector<PlanLayer> layers;
    std::vector<PlanStage> stages;
    int u0 = -1;                       // input of the first ConvTranspose (its zero halo is cleared before every chunk)
    int arena_halo = 1;                // halo rows every arena is sized for
    int min_T = 8;
    size_t stream_bytes = 0;           // carried state of one stream
};

}  // namespace

struct TcCodec {
    enc_config cfg;
    int hop = 1, D = 0, Dp = 0, ch0 = 0, num_sms = 132;
    DevBuf<const float*> d_embed;
    TcGemm conv_in, conv_out;
    TcGemm conv_out_p;                 // final conv as per-tap partial products (N = k), summed by tc_diag_sum_kernel
    bool co_split = false;
    float co_bias = 0.f;
    std::vector<TcGemm> pre, step, up; // step: 64-column tiles, or 128 with VCB_CODEC_LSTM_WIDE=1
    std::vector<std::vector<TcGemm>> res1, res2;
    TcPlan plan;
    DevBuf<uint8_t> ws;
    size_t ws_limit = 0;
    bool profile = false;
    bool keep = false;                 // VCB_CODEC_KEEP=1: every plan tensor has its own rows, so all survive a decode
    std::vector<std::pair<std::string, float>> prof;
    struct Dbg { Plane p; const __nv_bfloat16* ptr; int B; };
    std::map<std::string, Dbg> dbg;      // tensors of the last decoded chunk (debug read-back)
    std::map<std::string, Dbg> edbg;     // tensors of the last encoded chunk ("enc.*")
    std::unique_ptr<TcEncoder> enc;      // tensor-core encoder; null: no encoder weights or not covered (enc_reason)
    const char* enc_reason = "encoder weights (enc.*) not loaded";
    const float* dbg_cst = nullptr;      // its final LSTM cell states [layers][dbg_Bcap][ch0] ("c0", "c1", ...)
    int dbg_B = 0, dbg_Bcap = 0;
};

namespace {

inline int tc_num_sms(const TcCodec* tc) { return tc->num_sms; }

int upload_gemm(TcGemm& g, const std::vector<float>& W, const std::vector<float>& bias, int N, int Ktot, int bn_hint) {
    if (Ktot % TC_BK || Ktot / TC_BK > TC_MAX_KB) {
        set_error("codec_tc: K = %d outside the kernel's range", Ktot);
        return -1;
    }
    g.N = N;
    g.total_kb = Ktot / TC_BK;
    g.BN = bn_hint ? bn_hint : (N >= 128 ? 128 : (N >= 64 ? 64 : 32));
    g.ntiles = (N + g.BN - 1) / g.BN;
    const int Npad = g.ntiles * g.BN;
    std::vector<uint16_t> t(static_cast<size_t>(Npad) * Ktot * 2);
    size_t o = 0;
    for (int nt = 0; nt < g.ntiles; ++nt)
        for (int kb = 0; kb < g.total_kb; ++kb)
            for (int part = 0; part < 2; ++part)
                for (int r = 0; r < g.BN; ++r) {
                    const int n = nt * g.BN + r;
                    for (int kk = 0; kk < TC_BK; ++kk) {
                        const float w = n < N ? W[static_cast<size_t>(n) * Ktot + kb * TC_BK + kk] : 0.f;
                        const uint16_t hi = f2bf(w);
                        t[o++] = part == 0 ? hi : f2bf(w - bf2f(hi));
                    }
                }
    if (g.tiles.alloc(t.size())) return -1;
    VCB_CUDA_OK(cudaMemcpy(g.tiles, t.data(), t.size() * 2, cudaMemcpyHostToDevice));
    std::vector<float> bp(Npad, 0.f);
    for (int n = 0; n < N && n < static_cast<int>(bias.size()); ++n) bp[n] = bias[n];
    if (g.bias.alloc(bp.size())) return -1;
    VCB_CUDA_OK(cudaMemcpy(g.bias, bp.data(), bp.size() * 4, cudaMemcpyHostToDevice));
    return make_tmap_bf16_2d(&g.tmW, g.tiles, static_cast<uint64_t>(g.ntiles) * g.total_kb * 2 * g.BN, TC_BK, TC_BK, 2 * g.BN);
}

struct HostW {
    const std::map<std::string, DevBuf<float>>& dev;
    const std::map<std::string, std::vector<int64_t>>& shapes;
    int get(const std::string& name, std::vector<float>& out, std::vector<int64_t>* shape = nullptr) const {
        auto it = dev.find(name);
        auto is = shapes.find(name);
        if (it == dev.end() || is == shapes.end()) {
            set_error("codec: missing weight %s", name.c_str());
            return -1;
        }
        size_t n = 1;
        for (auto s : is->second) n *= static_cast<size_t>(s);
        out.resize(n);
        VCB_CUDA_OK(cudaMemcpy(out.data(), it->second, n * 4, cudaMemcpyDeviceToHost));
        if (shape) *shape = is->second;
        return 0;
    }
};

// Conv1d weight w[Cout][Cin][k] (stride 1, dilation dil, causal) -> GEMM [Cout_pad][k * Cin_pad], tap j reads row t - (k-1-j)*dil
int build_conv(TcGemm& g, const HostW& hw, const std::string& name, int Cin, int Cout, int k, int dil, int bn_hint = 0) {
    std::vector<float> w, b;
    if (hw.get(name + ".weight", w) || hw.get(name + ".bias", b)) return -1;
    const int Cip = cpad(Cin), Cop = Cout == 1 ? 1 : cpad(Cout);
    const int Ktot = k * Cip;
    std::vector<float> W(static_cast<size_t>(Cop) * Ktot, 0.f);
    for (int co = 0; co < Cout; ++co)
        for (int ci = 0; ci < Cin; ++ci)
            for (int j = 0; j < k; ++j) W[static_cast<size_t>(co) * Ktot + j * Cip + ci] = w[(static_cast<size_t>(co) * Cin + ci) * k + j];
    for (int j = 0; j < k; ++j)
        for (int cb = 0; cb < Cip / TC_BK; ++cb) g.taps.push_back(TcTap{0, static_cast<short>((k - 1 - j) * dil), cb * TC_BK});
    g.Cout = Cop == 1 ? 32 : Cop;
    g.up = 1;
    return upload_gemm(g, W, b, Cop, Ktot, bn_hint);
}

// ConvTranspose1d weight w[Cin][Cout][2r], stride r, causal trim of the last r samples -> GEMM [r * Cout_pad][2 * Cin_pad]
int build_convtr(TcGemm& g, const HostW& hw, const std::string& name, int Cin, int Cout, int r) {
    std::vector<float> w, b;
    if (hw.get(name + ".weight", w) || hw.get(name + ".bias", b)) return -1;
    const int Cip = cpad(Cin), Cop = cpad(Cout), Ktot = 2 * Cip, N = r * Cop;
    std::vector<float> W(static_cast<size_t>(N) * Ktot, 0.f), bias(N, 0.f);
    for (int p = 0; p < r; ++p)
        for (int co = 0; co < Cout; ++co) {
            const int n = p * Cop + co;
            bias[n] = b[co];
            for (int ci = 0; ci < Cin; ++ci) {
                const float* src = &w[(static_cast<size_t>(ci) * Cout + co) * 2 * r];
                W[static_cast<size_t>(n) * Ktot + ci] = src[p];               // x[t]
                W[static_cast<size_t>(n) * Ktot + Cip + ci] = src[p + r];     // x[t-1]
            }
        }
    for (int tap = 0; tap < 2; ++tap)
        for (int cb = 0; cb < Cip / TC_BK; ++cb) g.taps.push_back(TcTap{0, static_cast<short>(tap), cb * TC_BK});
    g.Cout = Cop;
    g.up = r;
    return upload_gemm(g, W, bias, N, Ktot, 0);
}

// residual block tail: conv2 (k = 1, on ELU(hidden)) + shortcut (k = 1, on the raw block input) as one GEMM
int build_res_tail(TcGemm& g, const HostW& hw, const std::string& prefix, int C, int hidden) {
    std::vector<float> w2, b2, ws, bs;
    if (hw.get(prefix + ".conv2.weight", w2) || hw.get(prefix + ".conv2.bias", b2) || hw.get(prefix + ".shortcut.weight", ws) ||
        hw.get(prefix + ".shortcut.bias", bs))
        return -1;
    const int Cp = cpad(C), Hp = cpad(hidden), Ktot = Hp + Cp;
    std::vector<float> W(static_cast<size_t>(Cp) * Ktot, 0.f), bias(Cp, 0.f);
    for (int co = 0; co < C; ++co) {
        bias[co] = b2[co] + bs[co];
        for (int ci = 0; ci < hidden; ++ci) W[static_cast<size_t>(co) * Ktot + ci] = w2[static_cast<size_t>(co) * hidden + ci];
        for (int ci = 0; ci < C; ++ci) W[static_cast<size_t>(co) * Ktot + Hp + ci] = ws[static_cast<size_t>(co) * C + ci];
    }
    for (int cb = 0; cb < Hp / TC_BK; ++cb) g.taps.push_back(TcTap{0, 0, cb * TC_BK});
    for (int cb = 0; cb < Cp / TC_BK; ++cb) g.taps.push_back(TcTap{1, 0, cb * TC_BK});
    g.Cout = Cp;
    g.up = 1;
    return upload_gemm(g, W, bias, Cp, Ktot, 0);
}

// LSTM matrix [4H][H] (gate-major rows i, f, g, o) -> gate-interleaved rows n = 4*unit + gate
int build_lstm(TcGemm& g, const HostW& hw, const std::string& wname, const std::string& b1, const std::string& b2,
               int H, int bn_hint) {
    std::vector<float> w, bi, bh;
    if (hw.get(wname, w)) return -1;
    std::vector<float> bias;
    if (!b1.empty()) {
        if (hw.get(b1, bi) || hw.get(b2, bh)) return -1;
        bias.assign(4 * H, 0.f);
    }
    std::vector<float> W(static_cast<size_t>(4) * H * H);
    for (int j = 0; j < H; ++j)
        for (int gt = 0; gt < 4; ++gt) {
            memcpy(&W[(static_cast<size_t>(4) * j + gt) * H], &w[(static_cast<size_t>(gt) * H + j) * H], static_cast<size_t>(H) * 4);
            if (!bias.empty()) bias[4 * j + gt] = bi[gt * H + j] + bh[gt * H + j];
        }
    for (int cb = 0; cb < H / TC_BK; ++cb) g.taps.push_back(TcTap{0, 0, cb * TC_BK});
    g.Cout = 4 * H;
    g.up = 1;
    return upload_gemm(g, W, bias, 4 * H, H, bn_hint);
}

template <int BN, int STAGES, int CW>
int tc_launch_t(const CUtensorMap& a0, const CUtensorMap& a1, const TcGemm& g, const TcCall& c, int num_sms, cudaStream_t st) {
    using L = TcSmem<BN, STAGES>;
    static bool attr_set = false;
    if (!attr_set) {
        VCB_CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<BN, STAGES, CW>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
        attr_set = true;
    }
    const long long tiles = static_cast<long long>(c.mtiles) * c.ntiles;
    VCB_CUDA_OK(launch_k_pdl(1, conv_tc_kernel<BN, STAGES, CW>, dim3(static_cast<unsigned>(std::min<long long>(tiles, num_sms))),
                             dim3(TC_THREADS), L::TOTAL, st, a0, a1, g.tmW, c));
    return 0;
}

int tc_launch(TcCodec* tc, const CUtensorMap& a0, const CUtensorMap& a1, const TcGemm& g, const TcCall& c, cudaStream_t st) {
    const int sms = tc_num_sms(tc);
    if (g.BN == 128) return tc_launch_t<128, 2, 32>(a0, a1, g, c, sms, st);
    if (g.BN == 64) return tc_launch_t<64, 4, 16>(a0, a1, g, c, sms, st);
    return tc_launch_t<32, 5, 16>(a0, a1, g, c, sms, st);
}

// A-side tensor map of an activation tensor form (raw / elu): [2 * rcap rows][C]
int plane_map(CUtensorMap* tm, const __nv_bfloat16* base, const Plane& p) {
    return make_tmap_bf16_2d(tm, base, 2ull * p.rcap, p.C, p.C, TC_BM);
}

inline int bcap(int B) { return (B + 127) / 128 * 128; }

// a plan tensor's rows for a chunk of B utterances of T frames: utterance-major, every utterance = halo rows + its rows; or
// time-major, row = (t + halo) * Bcap + b
Plane geometry(const PlanTensor& t, int B, int T) {
    Plane p;
    p.C = t.C;
    p.T = T * t.up;
    p.Tp = p.T + t.halo;
    p.halo = t.halo;
    p.halo_zero = t.halo_kind == HALO_ZERO;
    p.tm = t.tm;
    if (t.tm) {
        const int Bc = bcap(B);
        p.rcap = p.Tp * Bc;
        p.sb = 1;
        p.st = Bc;
        p.off = static_cast<long long>(t.halo) * Bc;
    } else {
        p.rcap = std::max(B * p.Tp, TC_BM);               // (a TMA box never taller than its tensor)
        p.sb = p.Tp;
        p.st = 1;
        p.off = t.halo;
    }
    return p;
}
size_t form_bytes(const Plane& p) { return static_cast<size_t>(p.rcap) * p.C * 2 * 2; }   // hi + lo planes of one form

struct Prof {
    TcCodec* tc;
    cudaStream_t st;
    struct Rec { std::string name; Event a, b; };
    std::vector<Rec> ev;
    void begin(const char* name) {
        if (!tc->profile) return;
        ev.push_back({name, Event(), Event()});
        ev.back().a.create();
        ev.back().b.create();
        cudaEventRecord(ev.back().a, st);
    }
    void end() {
        if (!tc->profile) return;
        cudaEventRecord(ev.back().b, st);
    }
    void finish() {
        if (!tc->profile) return;
        cudaStreamSynchronize(st);
        for (auto& e : ev) {
            float ms = 0.f;
            cudaEventElapsedTime(&ms, e.a, e.b);
            tc->prof.push_back({e.name, ms});
        }
    }
};

// The decoder's layers in launch order.  Every halo rule is here: a causal convolution reads (k-1)*dilation rows above its
// output row, so its input keeps that many halo rows, padded like the reference (reflect or zeros); a ConvTranspose reads
// x[t-1], so its input keeps one zero row.  A stream's state holds the carried tensors and the LSTM (h, c) per layer, in
// the order the carries run.
void build_plan(TcCodec* tc) {
    const enc_config& cf = tc->cfg;
    TcPlan& pl = tc->plan;
    const int H = tc->ch0, nl = cf.lstm, nres = cf.n_residual_layers;
    const int kres = cf.residual_kernel_size, kout = cf.last_kernel_size;
    const int pad = cf.pad_reflect ? HALO_REFLECT : HALO_ZERO;
    auto tensor = [&](int C, int halo, int kind, int up, bool tm, int forms, int home, bool carried, std::string dbg_raw,
                      std::string dbg_elu) {
        PlanTensor t;
        t.C = C; t.halo = halo; t.halo_kind = kind; t.up = up; t.tm = tm;
        t.forms = forms; t.home = tc->keep ? HOME_FIXED : home; t.carried = carried;
        t.dbg_raw = std::move(dbg_raw);
        t.dbg_elu = std::move(dbg_elu);
        pl.tensors.push_back(t);
        return static_cast<int>(pl.tensors.size()) - 1;
    };
    auto layer = [](int kind, const char* label, const TcGemm* g, int nstore, int in, int in_form, int out, int out_forms, int f32) {
        PlanLayer L;
        L.kind = kind; L.label = label; L.g = g; L.nstore = nstore;
        L.in = in; L.in_form = in_form; L.out = out; L.out_forms = out_forms; L.f32 = f32;
        return L;
    };
    auto add = [&](PlanLayer L) {
        if (L.kind == L_LSTM_STEPS) {
            L.h_off = pl.stream_bytes;
            L.c_off = pl.stream_bytes + static_cast<size_t>(H) * 4;
            pl.stream_bytes += static_cast<size_t>(H) * 8;
        }
        if (L.out >= 0) {
            PlanTensor& t = pl.tensors[L.out];
            if (t.carried && t.halo > 0) {
                t.state_off = pl.stream_bytes;
                pl.stream_bytes += static_cast<size_t>(t.halo) * t.C * 4;
            }
        }
        pl.layers.push_back(L);
    };
    // the input of a ConvTranspose, or of the final conv after the last stage
    auto feed = [&](bool last_stage, int& halo, int& kind) {
        halo = last_stage ? kout - 1 : 1;
        kind = last_stage ? pad : HALO_ZERO;
    };

    const int z = tensor(tc->Dp, cf.kernel_size - 1, pad, 1, false, FORM_RAW, HOME_FIXED, true, "z", "");
    pl.u0 = tensor(cpad(H), 1, HALO_ZERO, 1, false, FORM_ELU, HOME_FIXED, true, "", "u0");
    int x0 = -1, hs[2] = {-1, -1};
    if (nl > 0) {
        x0 = tensor(H, 0, HALO_ZERO, 1, true, FORM_RAW, HOME_FIXED, false, "x0", "");
        for (int l = 0; l < std::min(nl, 2); ++l)                 // h planes: slot t+1 = h_t, layers alternate
            hs[l] = tensor(H, 1, HALO_ZERO, 1, true, FORM_RAW, HOME_FIXED, false, "hs" + std::to_string(l), "");
    }
    add(layer(L_RVQ, "rvq", nullptr, 0, -1, 0, z, FORM_RAW, F32_NONE));
    if (nl > 0) add(layer(L_CONV, "conv_in", &tc->conv_in, cpad(H), z, FORM_RAW, x0, FORM_RAW, F32_X0));
    else add(layer(L_CONV, "conv_in", &tc->conv_in, cpad(H), z, FORM_RAW, pl.u0, FORM_ELU, F32_NONE));
    for (int l = 0; l < nl; ++l) {
        PlanLayer ih = layer(L_LSTM_IH, "lstm_ih", &tc->pre[l], 4 * H, l == 0 ? x0 : hs[(l - 1) & 1], FORM_RAW, -1, 0, F32_PRE);
        ih.lstm = l;
        add(ih);
        // the last layer's epilogue writes ELU(h + skip) straight into the first ConvTranspose's input
        const bool last = l == nl - 1;
        PlanLayer steps = layer(L_LSTM_STEPS, "lstm_steps", &tc->step[l], 4 * H, hs[l & 1], FORM_RAW, last ? pl.u0 : -1,
                                last ? FORM_ELU : 0, F32_NONE);
        steps.lstm = l;
        add(steps);
    }
    // up-sampling stages: ConvTranspose -> X; per residual block conv1 (on ELU(X)) -> hidden, then conv2 (on the hidden) +
    // shortcut (on raw X) -> O, the next block's X.  X and O alternate between the two arenas.
    int cur = pl.u0, ch = H, up = 1, side = HOME_ARENA0;
    for (int i = 0; i < cf.n_ratios; ++i) {
        const int r = cf.ratios[i], cout = ch / 2, hidden = cout / cf.compress;
        const bool last_stage = i == cf.n_ratios - 1;
        const std::string s = std::to_string(i + 1);
        ch = cout;
        up *= r;
        pl.stages.push_back(PlanStage{up, cpad(cout), cpad(hidden)});
        int halo = kres - 1, kind = pad;
        if (nres == 0) feed(last_stage, halo, kind);
        int x = tensor(cpad(cout), halo, kind, up, false, (nres > 0 ? FORM_RAW : 0) | FORM_ELU, side, true,
                       nres > 0 ? "x" + s + ".raw" : "", "x" + s + ".elu");
        add(layer(L_CONV, "convtr", &tc->up[i], r * cpad(cout), cur, FORM_ELU, x, pl.tensors[x].forms, F32_NONE));
        for (int j = 0, dil = 1; j < nres; ++j, dil *= cf.dilation_base) {
            const std::string sj = s + "." + std::to_string(j);
            const int hd = tensor(cpad(hidden), pl.tensors[x].halo, HALO_UNWRITTEN, up, false, FORM_ELU, HOME_HIDDEN, false, "",
                                  "h" + sj);
            add(layer(L_CONV, "res_conv1", &tc->res1[i][j], cpad(hidden), x, FORM_ELU, hd, FORM_ELU, F32_NONE));
            // the next block's conv1 reads (kres-1) * its dilation rows back.  min_T takes this term for the last block too.
            const int next = (kres - 1) * dil * cf.dilation_base;
            pl.min_T = std::max(pl.min_T, next + 2);
            halo = next;
            kind = pad;
            if (j == nres - 1) feed(last_stage, halo, kind);
            const int o = tensor(cpad(cout), halo, kind, up, false, (j < nres - 1 ? FORM_RAW : 0) | FORM_ELU, side ^ 1, true,
                                 j < nres - 1 ? "o" + sj + ".raw" : "", "o" + sj);
            PlanLayer tail = layer(L_CONV, "res_conv2", &tc->res2[i][j], cpad(cout), hd, FORM_ELU, o, pl.tensors[o].forms, F32_NONE);
            tail.in2 = x;
            add(tail);
            x = o;
            side ^= 1;
        }
        cur = x;
        side ^= 1;                                                 // the next ConvTranspose must not write over `cur`
    }
    // final conv: k <= DS_LD partial products (the first 16-column chunk), or one output column (f_valid = 1)
    if (tc->co_split) add(layer(L_CONV_OUT_SPLIT, "conv_out", &tc->conv_out_p, 16, cur, FORM_ELU, -1, 0, F32_COPART));
    else add(layer(L_CONV_OUT, "conv_out", &tc->conv_out, 32, cur, FORM_ELU, -1, 0, F32_WAV));
    pl.min_T = std::max(pl.min_T, std::max(cf.kernel_size, kout) + 1);
    for (const PlanTensor& t : pl.tensors)
        if (t.home != HOME_FIXED) pl.arena_halo = std::max(pl.arena_halo, t.halo);
}

// The workspace of a chunk: the fixed tensors, the fp32 buffers, the two stage arenas, the hidden arena, the final conv's
// partial products.  tensor[i] = offset of plan tensor i's first stored form (an ELU'd form follows a raw one).
struct WsLayout {
    std::vector<size_t> tensor;
    size_t x0f = 0, pre = 0, cst = 0, copart = 0, bytes = 0;
};

WsLayout ws_layout(const TcCodec* tc, int B, int T) {
    const TcPlan& pl = tc->plan;
    const int Bcap = bcap(B), H = tc->ch0, nl = tc->cfg.lstm;
    WsLayout w;
    w.tensor.resize(pl.tensors.size());
    size_t off = 0;
    auto take = [&](size_t bytes) {
        const size_t o = off;
        off += align_up(bytes, 1024);
        return o;
    };
    for (size_t i = 0; i < pl.tensors.size(); ++i) {
        const PlanTensor& t = pl.tensors[i];
        if (t.home != HOME_FIXED) continue;
        w.tensor[i] = off;
        for (int f : {FORM_RAW, FORM_ELU})
            if (t.forms & f) take(form_bytes(geometry(t, B, T)));
    }
    if (nl > 0) {
        w.x0f = take(static_cast<size_t>(T) * Bcap * H * 4);
        w.pre = take(static_cast<size_t>(T) * Bcap * 4 * H * 4);
        w.cst = take(static_cast<size_t>(nl) * Bcap * H * 4);
    }
    size_t ax = 0, ah = 0;
    for (const PlanStage& s : pl.stages) {
        const size_t rows = static_cast<size_t>(B) * (T * s.up + pl.arena_halo);
        ax = std::max(ax, align_up(rows * s.C * 4, 1024) * 2);
        ah = std::max(ah, align_up(rows * s.Ch * 4, 1024));
    }
    const size_t region[3] = {take(ax), take(ax), take(ah)};
    for (size_t i = 0; i < pl.tensors.size(); ++i)
        if (pl.tensors[i].home != HOME_FIXED) w.tensor[i] = region[pl.tensors[i].home];
    if (tc->co_split) {
        const PlanTensor& in = pl.tensors[pl.layers.back().in];
        w.copart = take((static_cast<size_t>(B) * (T * in.up + std::max(in.halo, 1)) + TC_BM) * DS_LD * 4);
    }
    w.bytes = off;
    return w;
}

// One chunk of B utterances.  sc = stream decode: every plane a layer reads as left context, and the LSTM state, continue
// the utterance's stream (tc_carry_kernel).
int decode_chunk_tc(TcCodec* tc, const int64_t* codes, float* wav, int B, int T, cudaStream_t st, int64_t* launches,
                    const TcStreamCtx* sc) {
    const TcPlan& pl = tc->plan;
    const enc_config& cf = tc->cfg;
    const int Bcap = bcap(B), H = tc->ch0, nl = cf.lstm;
    const WsLayout w = ws_layout(tc, B, T);
    std::vector<Plane> P(pl.tensors.size());
    tc->dbg.clear();
    for (size_t i = 0; i < P.size(); ++i) {
        const PlanTensor& t = pl.tensors[i];
        Plane& p = P[i];
        p = geometry(t, B, T);
        uint8_t* base = tc->ws + w.tensor[i];
        if (t.forms & FORM_RAW) {
            p.raw = reinterpret_cast<__nv_bfloat16*>(base);
            base += align_up(form_bytes(p), 1024);
        }
        if (t.forms & FORM_ELU) p.elu = reinterpret_cast<__nv_bfloat16*>(base);
        if (!t.dbg_raw.empty()) tc->dbg[t.dbg_raw] = TcCodec::Dbg{p, p.raw, B};
        if (!t.dbg_elu.empty()) tc->dbg[t.dbg_elu] = TcCodec::Dbg{p, p.elu, B};
    }
    float* x0f = reinterpret_cast<float*>(tc->ws + w.x0f);
    float* pre = reinterpret_cast<float*>(tc->ws + w.pre);
    float* cst = reinterpret_cast<float*>(tc->ws + w.cst);
    float* copart = reinterpret_cast<float*>(tc->ws + w.copart);
    tc->dbg_cst = nl > 0 ? cst : nullptr;
    tc->dbg_B = B;
    tc->dbg_Bcap = Bcap;

    // state that the kernels only ever read: U0's zero halo (the LSTM epilogue writes none), c_0 and h_{-1}
    const Plane& u0 = P[pl.u0];
    VCB_CUDA_OK(cudaMemset2DAsync(u0.elu, static_cast<size_t>(u0.Tp) * u0.C * 2, 0, static_cast<size_t>(u0.C) * 2, B, st));
    VCB_CUDA_OK(cudaMemset2DAsync(u0.elu + u0.plane(), static_cast<size_t>(u0.Tp) * u0.C * 2, 0, static_cast<size_t>(u0.C) * 2, B, st));
    auto clear_h0 = [&](const Plane& hs) -> int {
        VCB_CUDA_OK(cudaMemsetAsync(hs.raw, 0, static_cast<size_t>(Bcap) * H * 2, st));
        VCB_CUDA_OK(cudaMemsetAsync(hs.raw + hs.plane(), 0, static_cast<size_t>(Bcap) * H * 2, st));
        return 0;
    };
    if (nl > 0) {
        VCB_CUDA_OK(cudaMemsetAsync(cst, 0, static_cast<size_t>(nl) * Bcap * H * 4, st));
        for (const PlanLayer& L : pl.layers)
            if (L.kind == L_LSTM_STEPS && L.lstm < 2 && clear_h0(P[L.in])) return -1;
    }

    auto carry = [&](void* base, long long plane_bytes, long long sb, long long stt, long long off, int row_bytes, int halo, int up,
                     int restore, int save, size_t state_off) -> int {
        const CarryArgs a{static_cast<uint8_t*>(base), plane_bytes, sb, stt, off, row_bytes, halo, up, restore, save, sc->table,
                          sc->state, static_cast<long long>(pl.stream_bytes), static_cast<long long>(state_off)};
        VCB_CUDA_OK(launch_k_pdl(1, tc_carry_kernel, dim3(B), dim3(256), 0, st, a));
        ++*launches;
        return 0;
    };
    // a plane's halo: restore a continuing stream's tail over the padding the producer wrote, save the new tail
    auto carry_plane = [&](int i) -> int {
        const PlanTensor& t = pl.tensors[i];
        const Plane& p = P[i];
        if (sc == nullptr || !t.carried || p.halo == 0) return 0;
        return carry(p.elu ? p.elu : p.raw, p.plane() * 2, p.sb, p.st, p.off, p.C * 2, p.halo, t.up, 1, 1, t.state_off);
    };
    // stream decode: h_{-1} (slot 0) and c continue the stream; after the layer, h of the last valid step (slot frames) and
    // the frozen c are saved.  As a time-major plane with one halo row, row(b, t) = (t + 1) * Bcap + b.
    auto carry_lstm = [&](const PlanLayer& L, const Plane& hs, float* cl, int restore, int save) -> int {
        if (sc == nullptr) return 0;
        return carry(hs.raw, hs.plane() * 2, hs.sb, hs.st, hs.off, H * 2, 1, 1, restore, save, L.h_off) ||
               carry(cl, 0, 1, 0, 0, H * 4, 1, 1, restore, save, L.c_off);
    };
    // the call of a plan GEMM: its weights, its A rows, its epilogue (the LSTM steps then only move t_step and row_base)
    auto gemm_call = [&](const PlanLayer& L, TcCall& c) -> int {
        const TcGemm& g = *L.g;
        const Plane& in = P[L.in];
        c = TcCall{};
        c.mtiles = ((L.kind == L_LSTM_STEPS ? B : in.rcap) + TC_BM - 1) / TC_BM;
        if (static_cast<long long>(c.mtiles) * g.ntiles > 0x7fffffffll) {
            set_error("codec_tc: too many tiles");
            return -1;
        }
        c.total_kb = g.total_kb;
        c.ntiles = g.ntiles;
        c.bias = g.bias;
        c.up = g.up;
        c.Cout = g.Cout;
        std::copy(g.taps.begin(), g.taps.end(), c.taps);
        c.Nstore = L.nstore;
        c.rows_total = in.rcap;
        c.rcap[0] = in.rcap;
        c.B = B;
        if (L.kind != L_LSTM_STEPS) {
            c.in_tm = in.tm;
            c.in_div = in.tm ? static_cast<int>(in.st) : in.Tp;
            c.in_halo = in.halo;
            c.T_in = in.T;
        }
        if (L.in2 >= 0) c.rcap[1] = P[L.in2].rcap;
        if (L.out >= 0) {
            const Plane& o = P[L.out];
            c.raw = L.out_forms & FORM_RAW ? o.raw : nullptr;
            c.elu = L.out_forms & FORM_ELU ? o.elu : nullptr;
            c.o_plane = o.plane();
            c.o_ld = o.C;
            c.o_sb = o.sb;
            c.o_st = o.st;
            c.o_off = o.off;
            c.o_halo = pl.tensors[L.out].halo_kind == HALO_UNWRITTEN ? 0 : o.halo;
            c.o_halo_zero = o.halo_zero;
        }
        auto rows = [&](float* f, int ld, long long sb, long long stt, long long off) {
            c.f32 = f;
            c.f_ld = ld;
            c.f_valid = ld;
            c.f_sb = sb;
            c.f_st = stt;
            c.f_off = off;
        };
        if (L.f32 == F32_X0) rows(x0f, H, 1, Bcap, 0);                // time-major [T][Bcap][H]
        if (L.f32 == F32_PRE) rows(pre, 4 * H, 1, Bcap, 0);           // time-major [T][Bcap][4H]
        if (L.f32 == F32_COPART) {                                    // the input's rows, halo included
            rows(copart, DS_LD, in.sb, 1, in.off);
            c.in_store_halo = 1;
        }
        if (L.f32 == F32_WAV) {                                       // [B][T * hop]
            rows(wav, 1, in.T, 1, 0);
            c.f_scalar = 1;
        }
        if (L.kind == L_LSTM_STEPS) {
            c.mode = TC_MODE_LSTM;
            c.pre = pre;
            c.cst = cst + static_cast<size_t>(L.lstm) * Bcap * H;
            c.hseq = in.raw;
            c.h_plane = in.plane();
            c.Bcap = Bcap;
            c.H = H;
            if (L.out >= 0) c.skip = x0f;
            if (sc != nullptr) c.stab = sc->table;
        }
        return 0;
    };

    Prof pf{tc, st};
    CUtensorMap mA, mB;
    TcCall c;
    for (const PlanLayer& L : pl.layers) {
        pf.begin(L.label);
        if (L.kind == L_RVQ) {
            const Plane& z = P[L.out];
            tc_rvq_planes_kernel<<<dim3((T + 15) / 16, B), 128, 0, st>>>(reinterpret_cast<const long long*>(codes), tc->d_embed, z.raw,
                                                                         z.plane(), cf.n_q, tc->D, z.C, T, z.Tp, z.halo, z.halo_zero);
            VCB_CUDA_OK(cudaGetLastError());
            ++*launches;
        } else {
            const Plane& in = P[L.in];
            if (gemm_call(L, c) || plane_map(&mA, L.in_form == FORM_ELU ? in.elu : in.raw, in) ||
                (L.in2 >= 0 && plane_map(&mB, P[L.in2].raw, P[L.in2])))
                return -1;
            const CUtensorMap& a1 = L.in2 >= 0 ? mB : mA;
            if (L.kind == L_LSTM_STEPS) {
                if (L.lstm >= 2 && clear_h0(in)) return -1;
                if (carry_lstm(L, in, c.cst, 1, 0)) return -1;
                for (int t = 0; t < T; ++t) {
                    c.t_step = t;
                    c.row_base = t * Bcap;
                    if (tc_launch(tc, mA, a1, *L.g, c, st)) return -1;
                }
                *launches += T;
                if (carry_lstm(L, in, c.cst, 0, 1)) return -1;
            } else {
                if (tc_launch(tc, mA, a1, *L.g, c, st)) return -1;
                ++*launches;
            }
            if (L.kind == L_CONV_OUT_SPLIT) {
                VCB_CUDA_OK(launch_k_pdl(1, tc_diag_sum_kernel, dim3((in.rcap + DS_ROWS - 1) / DS_ROWS), dim3(DS_ROWS), 0, st,
                                         copart, cf.last_kernel_size, tc->co_bias, wav, in.rcap, in.Tp, in.halo, in.T, B));
                ++*launches;
            }
        }
        if (L.out >= 0 && carry_plane(L.out)) return -1;
        pf.end();
    }
    pf.finish();
    return 0;
}

// ---- encoder ---------------------------------------------------------------------------------------------------------

// enc.conv_in on the input planes: channel j of a row is tap j, so the whole k-tap conv is one k-block
int build_enc_conv_in(TcGemm& g, const HostW& hw, int k, int Cout) {
    std::vector<float> w, b;
    if (hw.get("enc.conv_in.weight", w) || hw.get("enc.conv_in.bias", b)) return -1;
    const int Cop = cpad(Cout);
    std::vector<float> W(static_cast<size_t>(Cop) * TC_BK, 0.f);
    for (int co = 0; co < Cout; ++co)
        for (int j = 0; j < k; ++j) W[static_cast<size_t>(co) * TC_BK + j] = w[static_cast<size_t>(co) * k + j];
    g.taps.push_back(TcTap{0, 0, 0});
    g.Cout = Cop;
    g.up = 1;
    return upload_gemm(g, W, b, Cop, TC_BK, 0);
}

// Strided Conv1d w[Cout][Cin][2r] (stride r, causal left pad r) over the folded input rows [rows / r][r * Cin_pad]: output
// frame t reads folded rows t-1 (taps 0..r-1) and t (taps r..2r-1), so K = 2 * r * Cin_pad with k = tap * Cin_pad + ci
int build_down(TcGemm& g, const HostW& hw, const std::string& name, int Cin, int Cout, int r) {
    std::vector<float> w, b;
    if (hw.get(name + ".weight", w) || hw.get(name + ".bias", b)) return -1;
    const int Cip = cpad(Cin), Cop = cpad(Cout), Ktot = 2 * r * Cip;
    std::vector<float> W(static_cast<size_t>(Cop) * Ktot, 0.f);
    for (int co = 0; co < Cout; ++co)
        for (int ci = 0; ci < Cin; ++ci)
            for (int j = 0; j < 2 * r; ++j) W[static_cast<size_t>(co) * Ktot + j * Cip + ci] = w[(static_cast<size_t>(co) * Cin + ci) * 2 * r + j];
    for (int half = 0; half < 2; ++half)
        for (int cb = 0; cb < r * Cip / TC_BK; ++cb) g.taps.push_back(TcTap{0, static_cast<short>(1 - half), cb * TC_BK});
    g.Cout = Cop;
    g.up = 1;
    return upload_gemm(g, W, b, Cop, Ktot, 0);
}

// the stage lengths of an utterance of N samples: L[0] = N, L[s+1] = ceil(L[s] / r_s)
std::vector<int> enc_chain(const EncPlan& pl, int N) {
    std::vector<int> L(1, N);
    for (int r : pl.ratios) L.push_back((L.back() + r - 1) / r);
    return L;
}

// plane rows per utterance of every stage: the stage length rounded up to its strided conv's stride
std::vector<int> enc_rows(const EncPlan& pl, const std::vector<int>& L) {
    std::vector<int> R(L);
    for (size_t s = 0; s < pl.ratios.size(); ++s) R[s] = (L[s] + pl.ratios[s] - 1) / pl.ratios[s] * pl.ratios[s];
    return R;
}

Plane enc_geometry(const EncTensor& t, int B, const std::vector<int>& R) {
    Plane p;
    p.C = t.C;
    p.T = R[t.stage];
    p.halo = t.halo;
    p.Tp = p.T + t.halo;
    p.halo_zero = t.halo_kind == HALO_ZERO;
    p.tm = t.tm;
    if (t.tm) {
        const int Bc = bcap(B);
        p.rcap = p.Tp * Bc;
        p.sb = 1;
        p.st = Bc;
        p.off = static_cast<long long>(t.halo) * Bc;
    } else {
        p.rcap = std::max(B * p.Tp, TC_BM * t.fold);     // (whole folded rows; a TMA box never taller than its tensor)
        p.sb = p.Tp;
        p.st = 1;
        p.off = t.halo;
    }
    return p;
}

// The encoder's layers in launch order.  Halo rule as in the decoder (a causal conv reads (k-1)*dilation rows above its output
// row); a strided conv's input keeps r rows (its causal left pad) plus the per-utterance right padding (E_RPAD).
void build_enc_plan(TcCodec* tc) {
    const enc_config& cf = tc->cfg;
    EncPlan& pl = tc->enc->plan;
    TcEncoder& E = *tc->enc;
    const int n = cf.n_ratios, nres = cf.n_residual_layers, nl = cf.lstm, H = tc->ch0;
    const int kres = cf.residual_kernel_size, kout = cf.last_kernel_size;
    const int pad = cf.pad_reflect ? HALO_REFLECT : HALO_ZERO;
    for (int s = 0; s < n; ++s) pl.ratios.push_back(cf.ratios[n - 1 - s]);
    auto tensor = [&](int C, int halo, int kind, int stage, int fold, bool tm, int forms, std::string dbg_raw, std::string dbg_elu) {
        EncTensor t;
        t.C = C; t.halo = halo; t.halo_kind = kind; t.stage = stage; t.fold = fold; t.tm = tm; t.forms = forms;
        t.home = (tc->keep || stage == n) ? HOME_FIXED : HOME_ARENA0 + (stage & 1);
        t.dbg_raw = std::move(dbg_raw);
        t.dbg_elu = std::move(dbg_elu);
        pl.tensors.push_back(t);
        return static_cast<int>(pl.tensors.size()) - 1;
    };
    auto layer = [&](int kind, const char* label, const TcGemm* g, int nstore, int in, int in_form, int out, int f32) {
        EncLayer L;
        L.kind = kind; L.label = label; L.g = g; L.nstore = nstore; L.in = in; L.in_form = in_form; L.out = out; L.f32 = f32;
        L.out_forms = out >= 0 ? pl.tensors[out].forms : 0;
        pl.layers.push_back(L);
        return &pl.layers.back();
    };
    // what stage s's first layer reads: its first residual block (conv1 reads kres-1 rows back), or its strided conv
    auto block_input = [&](int s, int C, const std::string& name) {
        if (nres > 0) return tensor(C, kres - 1, pad, s, 1, false, FORM_RAW | FORM_ELU, name, name + ".elu");
        return tensor(C, pl.ratios[s], pad, s, pl.ratios[s], false, FORM_ELU, "", name + ".elu");
    };
    int ch = cf.n_filters;
    const int in0 = tensor(TC_BK, 0, HALO_ZERO, 0, 1, false, FORM_RAW, "enc.input", "");
    layer(E_INPUT, "enc_input", nullptr, 0, -1, 0, in0, F32_NONE);
    int cur = block_input(0, cpad(ch), "enc.x0");
    layer(E_CONV, "enc_conv_in", &E.conv_in, cpad(ch), in0, FORM_RAW, cur, F32_NONE);
    int u = -1, x0 = -1;
    for (int s = 0; s < n; ++s) {
        const int r = pl.ratios[s], hidden = ch / cf.compress;
        const std::string si = "enc.down" + std::to_string(s);
        for (int j = 0, dil = 1; j < nres; ++j, dil *= cf.dilation_base) {
            const std::string sj = si + ".res" + std::to_string(j);
            const EncTensor& x = pl.tensors[cur];
            const int hd = tensor(cpad(hidden), x.halo, HALO_UNWRITTEN, s, x.fold, false, FORM_ELU, "", sj + ".h");
            layer(E_CONV, "enc_res_conv1", &E.res1[s][j], cpad(hidden), cur, FORM_ELU, hd, F32_NONE);
            const int o = j == nres - 1 ? tensor(cpad(ch), r, pad, s, r, false, FORM_ELU, "", sj + ".elu")
                                        : tensor(cpad(ch), (kres - 1) * dil * cf.dilation_base, pad, s, 1, false,
                                                 FORM_RAW | FORM_ELU, sj, sj + ".elu");
            layer(E_CONV, "enc_res_conv2", &E.res2[s][j], cpad(ch), hd, FORM_ELU, o, F32_NONE)->in2 = cur;
            cur = o;
        }
        EncLayer* rp = layer(E_RPAD, "enc_rpad", nullptr, 0, -1, 0, cur, F32_NONE);
        rp->stage = s;
        rp->r = r;
        ch *= 2;
        int next;
        if (s < n - 1) next = block_input(s + 1, cpad(ch), si + ".conv");
        else if (nl > 0) next = x0 = tensor(H, 0, HALO_ZERO, n, 1, true, FORM_RAW, si + ".conv", "");
        else next = u = tensor(cpad(ch), kout - 1, pad, n, 1, false, FORM_ELU, "", "enc.lstm");
        EncLayer* d = layer(E_DOWN, "enc_down", &E.down[s], cpad(ch), cur, FORM_ELU, next, next == x0 ? F32_X0 : F32_NONE);
        d->stage = s;
        d->r = r;
        cur = next;
    }
    if (nl > 0) {
        int hs[2] = {-1, -1};
        for (int l = 0; l < std::min(nl, 2); ++l)
            hs[l] = tensor(H, 1, HALO_ZERO, n, 1, true, FORM_RAW, "enc.hs" + std::to_string(l), "");
        u = tensor(cpad(H), kout - 1, pad, n, 1, false, FORM_ELU, "", "enc.lstm");
        for (int l = 0; l < nl; ++l) {
            layer(E_LSTM_IH, "enc_lstm_ih", &E.pre[l], 4 * H, l == 0 ? x0 : hs[(l - 1) & 1], FORM_RAW, -1, F32_PRE)->lstm = l;
            // the last layer's epilogue writes ELU(h + skip) into enc.conv_out's input, whose halo E_LPAD then fills
            layer(E_LSTM_STEPS, "enc_lstm_steps", &E.step[l], 4 * H, hs[l & 1], FORM_RAW, l == nl - 1 ? u : -1, F32_NONE)->lstm = l;
        }
        layer(E_LPAD, "enc_lpad", nullptr, 0, -1, 0, u, F32_NONE);
    }
    layer(E_CONV_OUT, "enc_conv_out", &E.conv_out, tc->Dp, u, FORM_ELU, -1, F32_LAT);
}

struct EncWs {
    std::vector<size_t> tensor;
    size_t x0f = 0, pre = 0, cst = 0, latf = 0, lat = 0, scores = 0, codes = 0, tab = 0, bytes = 0;
};

// The workspace of an encoder chunk of B utterances of at most N samples: fixed tensors (the LSTM stage's), two arenas that
// the stages alternate between (stage s's strided conv reads arena s % 2 and writes arena (s+1) % 2), the fp32 buffers,
// the RVQ scores and codes, the per-utterance table.
EncWs enc_ws_layout(const TcCodec* tc, int B, int N) {
    const EncPlan& pl = tc->enc->plan;
    const enc_config& cf = tc->cfg;
    const std::vector<int> R = enc_rows(pl, enc_chain(pl, N));
    const int n = static_cast<int>(pl.ratios.size()), Tn = R[n], Bcap = bcap(B), H = tc->ch0, nl = cf.lstm;
    EncWs w;
    w.tensor.resize(pl.tensors.size());
    size_t off = 0;
    auto take = [&](size_t bytes) {
        const size_t o = off;
        off += align_up(bytes, 1024);
        return o;
    };
    std::vector<size_t> stage_off(n + 1, 0);
    size_t arena[2] = {0, 0};
    for (size_t i = 0; i < pl.tensors.size(); ++i) {
        const EncTensor& t = pl.tensors[i];
        size_t bytes = 0;
        for (int f : {FORM_RAW, FORM_ELU})
            if (t.forms & f) bytes += align_up(form_bytes(enc_geometry(t, B, R)), 1024);
        if (t.home == HOME_FIXED) {
            w.tensor[i] = take(bytes);
        } else {
            w.tensor[i] = stage_off[t.stage];                  // offset inside its arena for now
            stage_off[t.stage] += bytes;
            arena[t.home - HOME_ARENA0] = std::max(arena[t.home - HOME_ARENA0], stage_off[t.stage]);
        }
    }
    const size_t a0 = take(arena[0]), a1 = take(arena[1]);
    for (size_t i = 0; i < pl.tensors.size(); ++i)
        if (pl.tensors[i].home != HOME_FIXED) w.tensor[i] += pl.tensors[i].home == HOME_ARENA0 ? a0 : a1;
    if (nl > 0) {
        w.x0f = take(static_cast<size_t>(Tn) * Bcap * H * 4);
        w.pre = take(static_cast<size_t>(Tn) * Bcap * 4 * H * 4);
        w.cst = take(static_cast<size_t>(nl) * Bcap * H * 4);
    }
    w.latf = take(static_cast<size_t>(B) * Tn * tc->Dp * 4);
    w.lat = take(static_cast<size_t>(B) * cf.dimension * Tn * 4);
    w.scores = take(static_cast<size_t>(B) * cf.bins * Tn * 4);
    w.codes = take(static_cast<size_t>(B) * cf.n_q * Tn * 8);
    w.tab = take(static_cast<size_t>(n + 2) * B * 4);
    w.bytes = off;
    return w;
}

// One chunk: utterance b = wav row rows[b] with lens[b] samples; the chunk's planes are sized for its longest utterance.
int encode_chunk_tc(TcCodec* tc, const float* wav, long long wav_ld, const int* rows, const int* lens, int B, cudaStream_t st,
                    int64_t* launches, TcEncOut* out) {
    const EncPlan& pl = tc->enc->plan;
    const enc_config& cf = tc->cfg;
    const int n = static_cast<int>(pl.ratios.size()), Bcap = bcap(B), H = tc->ch0, nl = cf.lstm;
    const int N = *std::max_element(lens, lens + B);
    const std::vector<int> R = enc_rows(pl, enc_chain(pl, N));
    const int Tn = R[n];
    const EncWs w = enc_ws_layout(tc, B, N);
    std::vector<Plane> P(pl.tensors.size());
    tc->edbg.clear();
    for (size_t i = 0; i < P.size(); ++i) {
        const EncTensor& t = pl.tensors[i];
        Plane& p = P[i];
        p = enc_geometry(t, B, R);
        uint8_t* base = tc->ws + w.tensor[i];
        if (t.forms & FORM_RAW) {
            p.raw = reinterpret_cast<__nv_bfloat16*>(base);
            base += align_up(form_bytes(p), 1024);
        }
        if (t.forms & FORM_ELU) p.elu = reinterpret_cast<__nv_bfloat16*>(base);
        if (!t.dbg_raw.empty()) tc->edbg[t.dbg_raw] = TcCodec::Dbg{p, p.raw, B};
        if (!t.dbg_elu.empty()) tc->edbg[t.dbg_elu] = TcCodec::Dbg{p, p.elu, B};
    }
    float* x0f = reinterpret_cast<float*>(tc->ws + w.x0f);
    float* pre = reinterpret_cast<float*>(tc->ws + w.pre);
    float* cst = reinterpret_cast<float*>(tc->ws + w.cst);
    float* latf = reinterpret_cast<float*>(tc->ws + w.latf);
    int* tab = reinterpret_cast<int*>(tc->ws + w.tab);         // [n+1][B] stage lengths, then [B] wav rows
    {
        std::vector<int> h(static_cast<size_t>(n + 2) * B);
        for (int b = 0; b < B; ++b) {
            const std::vector<int> L = enc_chain(pl, lens[b]);
            for (int s = 0; s <= n; ++s) h[static_cast<size_t>(s) * B + b] = L[s];
            h[static_cast<size_t>(n + 1) * B + b] = rows[b];
        }
        VCB_CUDA_OK(cudaMemcpyAsync(tab, h.data(), h.size() * 4, cudaMemcpyHostToDevice, st));   // pageable: staged at once
    }
    if (nl > 0) VCB_CUDA_OK(cudaMemsetAsync(cst, 0, static_cast<size_t>(nl) * Bcap * H * 4, st));
    auto clear_h0 = [&](const Plane& hs) -> int {
        VCB_CUDA_OK(cudaMemsetAsync(hs.raw, 0, static_cast<size_t>(Bcap) * H * 2, st));
        VCB_CUDA_OK(cudaMemsetAsync(hs.raw + hs.plane(), 0, static_cast<size_t>(Bcap) * H * 2, st));
        return 0;
    };
    for (const EncLayer& L : pl.layers)
        if (L.kind == E_LSTM_STEPS && L.lstm < 2 && clear_h0(P[L.in])) return -1;

    Prof pf{tc, st};
    CUtensorMap mA, mB;
    for (const EncLayer& L : pl.layers) {
        pf.begin(L.label);
        if (L.kind == E_INPUT) {
            const Plane& o = P[L.out];
            const long long items = static_cast<long long>(B) * o.T;
            tc_enc_input_kernel<<<static_cast<unsigned>((items + 255) / 256), 256, 0, st>>>(
                wav, wav_ld, tab + static_cast<size_t>(n + 1) * B, tab, o.raw, o.plane(), o.C, o.Tp, o.T, cf.kernel_size, cf.pad_reflect, B);
            VCB_CUDA_OK(cudaGetLastError());
            ++*launches;
        } else if (L.kind == E_RPAD || L.kind == E_LPAD) {
            const Plane& o = P[L.out];
            __nv_bfloat16* base = o.elu ? o.elu : o.raw;
            tc_pad_rows_kernel<<<B, 256, 0, st>>>(base, o.plane(), o.C, o.sb, o.st, o.off,
                                                  L.kind == E_RPAD ? tab + static_cast<size_t>(L.stage) * B : nullptr, o.halo, L.r,
                                                  o.halo_zero);
            VCB_CUDA_OK(cudaGetLastError());
            ++*launches;
        } else {
            const TcGemm& g = *L.g;
            Plane in = P[L.in];
            if (L.kind == E_DOWN) {                          // folded rows: r plane rows of C channels are one row of r*C
                const int r = L.r;
                in.C *= r; in.rcap /= r; in.Tp /= r; in.T /= r; in.halo = 1; in.sb = in.Tp; in.off = 1;
            }
            if (plane_map(&mA, L.in_form == FORM_ELU ? P[L.in].elu : P[L.in].raw, in) ||
                (L.in2 >= 0 && plane_map(&mB, P[L.in2].raw, P[L.in2])))
                return -1;
            TcCall c{};
            c.mtiles = ((L.kind == E_LSTM_STEPS ? B : in.rcap) + TC_BM - 1) / TC_BM;
            if (static_cast<long long>(c.mtiles) * g.ntiles > 0x7fffffffll) {
                set_error("codec_tc: too many tiles");
                return -1;
            }
            c.total_kb = g.total_kb;
            c.ntiles = g.ntiles;
            c.bias = g.bias;
            c.up = g.up;
            c.Cout = g.Cout;
            std::copy(g.taps.begin(), g.taps.end(), c.taps);
            c.Nstore = L.nstore;
            c.rows_total = in.rcap;
            c.rcap[0] = in.rcap;
            c.B = B;
            if (L.kind != E_LSTM_STEPS) {
                c.in_tm = in.tm;
                c.in_div = in.tm ? static_cast<int>(in.st) : in.Tp;
                c.in_halo = in.halo;
                c.T_in = in.T;
            }
            if (L.in2 >= 0) c.rcap[1] = P[L.in2].rcap;
            if (L.out >= 0) {
                const Plane& o = P[L.out];
                c.raw = L.out_forms & FORM_RAW ? o.raw : nullptr;
                c.elu = L.out_forms & FORM_ELU ? o.elu : nullptr;
                c.o_plane = o.plane();
                c.o_ld = o.C;
                c.o_sb = o.sb;
                c.o_st = o.st;
                c.o_off = o.off;
                c.o_halo = pl.tensors[L.out].halo_kind == HALO_UNWRITTEN ? 0 : o.halo;
                c.o_halo_zero = o.halo_zero;
            }
            auto rows_f32 = [&](float* f, int ld, int valid, long long sb, long long stt) {
                c.f32 = f; c.f_ld = ld; c.f_valid = valid; c.f_sb = sb; c.f_st = stt; c.f_off = 0;
            };
            if (L.f32 == F32_X0) rows_f32(x0f, H, H, 1, Bcap);                 // time-major [T][Bcap][H]
            if (L.f32 == F32_PRE) rows_f32(pre, 4 * H, 4 * H, 1, Bcap);        // time-major [T][Bcap][4H]
            if (L.f32 == F32_LAT) rows_f32(latf, tc->Dp, cf.dimension, Tn, 1); // [B][T][Dp]
            const CUtensorMap& a1 = L.in2 >= 0 ? mB : mA;
            if (L.kind == E_LSTM_STEPS) {
                c.mode = TC_MODE_LSTM;
                c.pre = pre;
                c.cst = cst + static_cast<size_t>(L.lstm) * Bcap * H;
                c.hseq = P[L.in].raw;
                c.h_plane = P[L.in].plane();
                c.Bcap = Bcap;
                c.H = H;
                if (L.out >= 0) c.skip = x0f;
                if (L.lstm >= 2 && clear_h0(P[L.in])) return -1;
                for (int t = 0; t < Tn; ++t) {
                    c.t_step = t;
                    c.row_base = t * Bcap;
                    if (tc_launch(tc, mA, a1, g, c, st)) return -1;
                }
                *launches += Tn;
            } else {
                if (tc_launch(tc, mA, a1, g, c, st)) return -1;
                ++*launches;
            }
            // The epilogue zeroes halo row -t from output row t, 1 <= t <= halo, and a GEMM writes in.T rows (a strided
            // conv ceil(L/r) of the chunk's longest utterance).  With constant padding an utterance may be shorter than a
            // halo (rows of any length are taken), and a chunk of only such utterances writes no row t for some halo
            // rows: they are cleared here, or they would keep whatever an earlier chunk left in the workspace.
            if (L.kind != E_LSTM_STEPS && L.out >= 0 && pl.tensors[L.out].halo_kind == HALO_ZERO && !P[L.out].tm &&
                in.T <= P[L.out].halo) {
                const Plane& o = P[L.out];
                for (__nv_bfloat16* base : {c.raw, c.elu}) {
                    if (base == nullptr) continue;
                    tc_pad_rows_kernel<<<B, 256, 0, st>>>(base, o.plane(), o.C, o.sb, o.st, o.off, nullptr, o.halo, 1, 1);
                    VCB_CUDA_OK(cudaGetLastError());
                    ++*launches;
                }
            }
        }
        pf.end();
    }
    float* lat = reinterpret_cast<float*>(tc->ws + w.lat);
    tc_latent_cm_kernel<<<dim3((Tn + 31) / 32, B), 256, 32 * (cf.dimension + 1) * 4, st>>>(latf, lat, cf.dimension, tc->Dp, Tn);
    VCB_CUDA_OK(cudaGetLastError());
    ++*launches;
    pf.finish();
    out->latent = lat;
    out->scores = reinterpret_cast<float*>(tc->ws + w.scores);
    out->codes = reinterpret_cast<int64_t*>(tc->ws + w.codes);
    out->T = Tn;
    return 0;
}

}  // namespace

int tc_codec_build(const enc_config& cfg, const std::map<std::string, DevBuf<float>>& w_dev,
                   const std::map<std::string, std::vector<int64_t>>& shapes, TcCodecPtr* out, const char** reason) {
    out->reset();
    const int ch0 = cfg.n_filters << cfg.n_ratios;
    auto no = [&](const char* why) {
        *reason = why;
        return 1;
    };
    if (!cfg.causal || cfg.trim_right_ratio != 1.0f) return no("non-causal / partial right trim");
    if (cfg.true_skip) return no("identity skip");
    if (cfg.channels != 1) return no("multi-channel output");
    if (cfg.lstm > 0 && ch0 % 64) return no("LSTM width not a multiple of 64");
    if (cfg.lstm == 0 && ch0 % 64) return no("first stage narrower than one k-block");
    if ((ch0 >> cfg.n_ratios) < 1 || cfg.compress < 1) return no("channel plan");
    if (2 * cpad(ch0) / TC_BK > TC_MAX_KB || cfg.kernel_size * cpad(cfg.dimension) / TC_BK > TC_MAX_KB ||
        cfg.residual_kernel_size * cpad(ch0 / 2) / TC_BK > TC_MAX_KB || cfg.last_kernel_size * cpad(cfg.n_filters) / TC_BK > TC_MAX_KB)
        return no("reduction deeper than the kernel's k-blocks");
    if (getenv("VCB_CODEC_TC") && atoi(getenv("VCB_CODEC_TC")) == 0) return no("disabled by VCB_CODEC_TC=0");
    TcCodecPtr tc(new TcCodec());
    tc->cfg = cfg;
    tc->D = cfg.dimension;
    tc->Dp = cpad(cfg.dimension);
    tc->ch0 = ch0;
    for (int i = 0; i < cfg.n_ratios; ++i) tc->hop *= cfg.ratios[i];
    {
        int dev = 0, sms = 0;
        if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && sms > 0)
            tc->num_sms = sms;
        if (getenv("VCB_CODEC_GRID")) tc->num_sms = std::max(1, atoi(getenv("VCB_CODEC_GRID")));
    }
    tc->profile = getenv("VCB_CODEC_PROFILE") && atoi(getenv("VCB_CODEC_PROFILE")) != 0;
    tc->keep = getenv("VCB_CODEC_KEEP") && atoi(getenv("VCB_CODEC_KEEP")) != 0;
    // LSTM step tiles: 128 columns move fewer bytes through L2 per step (VCB_CODEC_LSTM_WIDE=1); 64 keep more CTAs on the
    // 16-k-block pipeline of each step
    const int step_bn = getenv("VCB_CODEC_LSTM_WIDE") && atoi(getenv("VCB_CODEC_LSTM_WIDE")) > 0 ? 128 : 64;
    const char* lim = getenv("VCB_CODEC_WS_GB");
    tc->ws_limit = static_cast<size_t>((lim ? atof(lim) : 100.0) * (1ull << 30));
    HostW hw{w_dev, shapes};
    char nm[160];
    int rc = 0;
    {
        std::vector<const float*> emb(cfg.n_q);
        for (int q = 0; q < cfg.n_q && !rc; ++q) {
            snprintf(nm, sizeof(nm), "vq.%d.embed", q);
            auto it = w_dev.find(nm);
            if (it == w_dev.end()) {
                set_error("codec: missing weight %s", nm);
                rc = -1;
            } else {
                emb[q] = it->second;
            }
        }
        if (!rc && (tc->d_embed.alloc(cfg.n_q) ||
                    cudaMemcpy(tc->d_embed, emb.data(), cfg.n_q * sizeof(float*), cudaMemcpyHostToDevice) != cudaSuccess)) {
            set_error("codec_tc: codebook pointer table");
            rc = -1;
        }
    }
    if (!rc) rc = build_conv(tc->conv_in, hw, "dec.conv_in", cfg.dimension, ch0, cfg.kernel_size, 1);
    tc->pre.resize(cfg.lstm);
    tc->step.resize(cfg.lstm);
    for (int l = 0; l < cfg.lstm && !rc; ++l) {
        char a[96], b[96], c2[96];
        snprintf(a, sizeof(a), "dec.lstm.weight_ih_l%d", l);
        snprintf(b, sizeof(b), "dec.lstm.bias_ih_l%d", l);
        snprintf(c2, sizeof(c2), "dec.lstm.bias_hh_l%d", l);
        rc = build_lstm(tc->pre[l], hw, a, b, c2, ch0, 0);
        snprintf(a, sizeof(a), "dec.lstm.weight_hh_l%d", l);
        if (!rc) rc = build_lstm(tc->step[l], hw, a, "", "", ch0, step_bn);
    }
    tc->up.resize(cfg.n_ratios);
    tc->res1.resize(cfg.n_ratios);
    tc->res2.resize(cfg.n_ratios);
    int ch = ch0;
    for (int i = 0; i < cfg.n_ratios && !rc; ++i) {
        snprintf(nm, sizeof(nm), "dec.up%d.convtr", i);
        rc = build_convtr(tc->up[i], hw, nm, ch, ch / 2, cfg.ratios[i]);
        ch /= 2;
        tc->res1[i].resize(cfg.n_residual_layers);
        tc->res2[i].resize(cfg.n_residual_layers);
        for (int j = 0, dil = 1; j < cfg.n_residual_layers && !rc; ++j, dil *= cfg.dilation_base) {
            snprintf(nm, sizeof(nm), "dec.up%d.res%d.conv1", i, j);
            rc = build_conv(tc->res1[i][j], hw, nm, ch, ch / cfg.compress, cfg.residual_kernel_size, dil);
            snprintf(nm, sizeof(nm), "dec.up%d.res%d", i, j);
            if (!rc) rc = build_res_tail(tc->res2[i][j], hw, nm, ch, ch / cfg.compress);
        }
    }
    if (!rc) rc = build_conv(tc->conv_out, hw, "dec.conv_out", ch, 1, cfg.last_kernel_size, 1, 32);
    if (!rc && cfg.last_kernel_size <= DS_LD && !(getenv("VCB_CODEC_CONVOUT_TC") && atoi(getenv("VCB_CODEC_CONVOUT_TC")))) {
        std::vector<float> w, b;
        rc = hw.get("dec.conv_out.weight", w) || hw.get("dec.conv_out.bias", b) ? -1 : 0;
        if (!rc) {
            const int Cp = cpad(ch), k = cfg.last_kernel_size;
            std::vector<float> W(static_cast<size_t>(k) * Cp, 0.f);          // GEMM row j = tap j
            for (int ci = 0; ci < ch; ++ci)
                for (int j = 0; j < k; ++j) W[static_cast<size_t>(j) * Cp + ci] = w[static_cast<size_t>(ci) * k + j];
            TcGemm& g = tc->conv_out_p;
            for (int cb = 0; cb < Cp / TC_BK; ++cb) g.taps.push_back(TcTap{0, 0, cb * TC_BK});
            g.Cout = 32;
            g.up = 1;
            rc = upload_gemm(g, W, std::vector<float>(), k, Cp, 32);
            tc->co_bias = b[0];
            tc->co_split = rc == 0;
        }
    }
    if (rc) return -1;
    build_plan(tc.get());
    if (w_dev.count("enc.conv_in.weight")) {
        // the encoder: the decoder's coverage, plus an input window that fits one k-block and reductions within TC_MAX_KB
        const int n = cfg.n_ratios, kres = cfg.residual_kernel_size;
        bool deep = cfg.kernel_size > TC_BK || cfg.last_kernel_size * cpad(ch0) / TC_BK > TC_MAX_KB;
        for (int s = 0, c = cfg.n_filters; s < n; ++s, c *= 2)
            deep = deep || 2 * cfg.ratios[n - 1 - s] * cpad(c) / TC_BK > TC_MAX_KB || kres * cpad(c) / TC_BK > TC_MAX_KB;
        if (deep) {
            tc->enc_reason = "encoder reduction deeper than the kernel's k-blocks";
        } else {
            tc->enc.reset(new TcEncoder());
            TcEncoder& E = *tc->enc;
            rc = build_enc_conv_in(E.conv_in, hw, cfg.kernel_size, cfg.n_filters);
            E.down.resize(n);
            E.res1.resize(n);
            E.res2.resize(n);
            for (int s = 0, c = cfg.n_filters; s < n && !rc; ++s, c *= 2) {
                E.res1[s].resize(cfg.n_residual_layers);
                E.res2[s].resize(cfg.n_residual_layers);
                for (int j = 0, dil = 1; j < cfg.n_residual_layers && !rc; ++j, dil *= cfg.dilation_base) {
                    snprintf(nm, sizeof(nm), "enc.down%d.res%d.conv1", s, j);
                    rc = build_conv(E.res1[s][j], hw, nm, c, c / cfg.compress, kres, dil);
                    snprintf(nm, sizeof(nm), "enc.down%d.res%d", s, j);
                    if (!rc) rc = build_res_tail(E.res2[s][j], hw, nm, c, c / cfg.compress);
                }
                snprintf(nm, sizeof(nm), "enc.down%d.conv", s);
                if (!rc) rc = build_down(E.down[s], hw, nm, c, 2 * c, cfg.ratios[n - 1 - s]);
            }
            E.pre.resize(cfg.lstm);
            E.step.resize(cfg.lstm);
            for (int l = 0; l < cfg.lstm && !rc; ++l) {
                char a[96], b[96], c2[96];
                snprintf(a, sizeof(a), "enc.lstm.weight_ih_l%d", l);
                snprintf(b, sizeof(b), "enc.lstm.bias_ih_l%d", l);
                snprintf(c2, sizeof(c2), "enc.lstm.bias_hh_l%d", l);
                rc = build_lstm(E.pre[l], hw, a, b, c2, ch0, 0);
                snprintf(a, sizeof(a), "enc.lstm.weight_hh_l%d", l);
                if (!rc) rc = build_lstm(E.step[l], hw, a, "", "", ch0, step_bn);
            }
            if (!rc) rc = build_conv(E.conv_out, hw, "enc.conv_out", ch0, cfg.dimension, cfg.last_kernel_size, 1);
            if (rc) return -1;
            build_enc_plan(tc.get());
            tc->enc_reason = "";
        }
    }
    *out = std::move(tc);
    return 0;
}

bool tc_encoder_active(const TcCodec* c) { return c != nullptr && c->enc != nullptr; }

const char* tc_encoder_reason(const TcCodec* c) { return c ? c->enc_reason : "the tensor-core codec is not active"; }

// every stage longer than the padding its convolutions reflect (audiocraft pad1d zero-extends a shorter input instead)
bool tc_encoder_accepts(const TcCodec* c, int len) {
    if (!tc_encoder_active(c) || len < 1) return false;
    const enc_config& cf = c->cfg;
    if (!cf.pad_reflect) return true;
    const std::vector<int> L = enc_chain(c->enc->plan, len);
    int dmax = 1;
    for (int j = 1; j < cf.n_residual_layers; ++j) dmax *= cf.dilation_base;
    const int res_pad = cf.n_residual_layers > 0 ? (cf.residual_kernel_size - 1) * dmax : 0;
    if (L[0] <= cf.kernel_size - 1) return false;
    for (size_t s = 0; s < c->enc->plan.ratios.size(); ++s)
        if (L[s] <= res_pad || L[s] <= c->enc->plan.ratios[s]) return false;
    return L.back() > cf.last_kernel_size - 1;
}

size_t tc_encoder_ws_bytes(const TcCodec* c, int B, int N) { return enc_ws_layout(c, B, N).bytes; }

size_t tc_ws_limit(const TcCodec* c) { return c->ws_limit; }

int64_t tc_encoder_rows(const TcCodec* c, int B, int N) {
    return static_cast<int64_t>(B) * enc_rows(c->enc->plan, enc_chain(c->enc->plan, N))[0];
}

int tc_encoder_encode(TcCodec* tc, const float* wav, long long wav_ld, const int* rows, const int* lens, int B, cudaStream_t st,
                      int64_t* launches, TcEncOut* out) {
    tc->prof.clear();
    const size_t need = enc_ws_layout(tc, B, *std::max_element(lens, lens + B)).bytes;
    if (need > tc->ws.size()) {
        if (tc->ws) VCB_CUDA_OK(cudaStreamSynchronize(st));      // alloc releases the previous workspace first
        if (tc->ws.alloc(need)) {
            const std::string why = get_error();
            set_error("codec_tc: cannot allocate a %.2f GB encoder workspace for %d utterances (%s)", need / 1073741824.0, B,
                      why.c_str());
            return -1;
        }
    }
    return encode_chunk_tc(tc, wav, wav_ld, rows, lens, B, st, launches, out);
}

bool tc_codec_accepts(const TcCodec* c, int B, int T) { return c != nullptr && B >= 1 && T >= c->plan.min_T; }

int tc_codec_decode(TcCodec* tc, const int64_t* codes, float* wav, int B, int T, cudaStream_t st, int64_t* launches,
                    const TcStreamCtx* sc) {
    tc->prof.clear();
    // chunk the batch so the workspace stays under the limit -- and halve the chunk again if the device cannot give that much
    int chunk = B;
    for (;;) {
        const size_t need = ws_layout(tc, chunk, T).bytes;
        if (need > tc->ws_limit && chunk > 1) {
            chunk = (chunk + 1) / 2;
            continue;
        }
        if (need <= tc->ws.size()) break;
        if (tc->ws) VCB_CUDA_OK(cudaStreamSynchronize(st));   // alloc releases the previous workspace first
        if (tc->ws.alloc(need) == 0) break;
        if (chunk == 1) {
            const std::string why = get_error();
            set_error("codec_tc: cannot allocate a %.2f GB workspace for one utterance of %d frames (%s)", need / 1073741824.0, T,
                      why.c_str());
            return -1;
        }
        chunk = (chunk + 1) / 2;
    }
    for (int b0 = 0; b0 < B; b0 += chunk) {
        const int nb = std::min(chunk, B - b0);
        TcStreamCtx part;
        if (sc != nullptr) part = TcStreamCtx{sc->table + 4 * b0, sc->state};
        if (decode_chunk_tc(tc, codes + static_cast<size_t>(b0) * tc->cfg.n_q * T, wav + static_cast<size_t>(b0) * T * tc->hop, nb, T, st,
                            launches, sc != nullptr ? &part : nullptr))
            return -1;
    }
    return 0;
}

size_t tc_stream_state_bytes(const TcCodec* c) { return c->plan.stream_bytes; }

int tc_stream_min_frames(const TcCodec* c) { return c->plan.min_T; }

int tc_codes_check(const int64_t* codes, long long n, int bins, int* bad_dev, int* bad_host, cudaStream_t st) {
    VCB_CUDA_OK(cudaMemsetAsync(bad_dev, 0, sizeof(int), st));
    const long long blocks = std::min<long long>((n + 255) / 256, 1024);
    tc_codes_check_kernel<<<static_cast<unsigned>(std::max<long long>(blocks, 1)), 256, 0, st>>>(reinterpret_cast<const long long*>(codes),
                                                                                              n, bins, bad_dev);
    VCB_CUDA_OK(cudaGetLastError());
    VCB_CUDA_OK(cudaMemcpyAsync(bad_host, bad_dev, sizeof(int), cudaMemcpyDeviceToHost, st));
    VCB_CUDA_OK(cudaStreamSynchronize(st));
    return 0;
}

void TcCodecDelete::operator()(TcCodec* tc) const { delete tc; }

const std::vector<std::pair<std::string, float>>& tc_codec_profile(const TcCodec* c) { return c->prof; }

int tc_codec_debug_tensor(TcCodec* tc, const char* name, float* host_out, int64_t cap, int32_t* dims) {
    if (name[0] == 'c' && name[1] >= '0' && name[1] < '0' + tc->cfg.lstm && name[2] == 0 && tc->dbg_cst != nullptr) {
        const int B = tc->dbg_B, H = tc->ch0;                        // fp32 [B][H], the state after the last step
        dims[0] = B; dims[1] = H; dims[2] = 1; dims[3] = 0;
        if (host_out == nullptr) return 0;
        if (cap < static_cast<int64_t>(B) * H) {
            set_error("codec_tc: debug buffer too small");
            return -1;
        }
        VCB_CUDA_OK(cudaDeviceSynchronize());
        VCB_CUDA_OK(cudaMemcpy(host_out, tc->dbg_cst + static_cast<size_t>(name[1] - '0') * tc->dbg_Bcap * H,
                               static_cast<size_t>(B) * H * 4, cudaMemcpyDeviceToHost));
        return 0;
    }
    auto& m = strncmp(name, "enc.", 4) ? tc->dbg : tc->edbg;
    auto it = m.find(name);
    if (it == m.end()) {
        set_error("codec_tc: no tensor '%s' in the last decode or tensor-core encode", name);
        return -1;
    }
    const Plane& p = it->second.p;
    const int B = it->second.B;
    dims[0] = B; dims[1] = p.C; dims[2] = p.Tp; dims[3] = p.halo;
    const int64_t n = static_cast<int64_t>(B) * p.C * p.Tp;
    if (host_out == nullptr) return 0;
    if (cap < n) {
        set_error("codec_tc: debug buffer too small");
        return -1;
    }
    VCB_CUDA_OK(cudaDeviceSynchronize());
    std::vector<uint16_t> h(static_cast<size_t>(p.rcap) * p.C * 2);
    VCB_CUDA_OK(cudaMemcpy(h.data(), it->second.ptr, h.size() * 2, cudaMemcpyDeviceToHost));
    const size_t pl = static_cast<size_t>(p.plane());
    for (int b = 0; b < B; ++b)
        for (int t = -p.halo; t < p.T; ++t) {
            const long long row = b * p.sb + t * p.st + p.off;
            for (int ch = 0; ch < p.C; ++ch)
                host_out[(static_cast<size_t>(b) * p.C + ch) * p.Tp + (t + p.halo)] = bf2f(h[row * p.C + ch]) + bf2f(h[pl + row * p.C + ch]);
        }
    return 0;
}

}  // namespace vcb
