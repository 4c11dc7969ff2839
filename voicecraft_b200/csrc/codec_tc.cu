// EnCodec SEANet decoder and encoder on the tensor cores (wgmma).
//
// Replaces, for the configurations it covers, the CUDA-core kernels of encodec.cu behind the same entry points
// (enc_decode <- AudioTokenizer.decode, reference data/tokenizer.py:131-133 -> audiocraft EncodecModel.decode;
// enc_encode_ragged <- AudioTokenizer.encode_many).
//
// Every GEMM layer is one launch of ONE kernel, an implicit GEMM with the time steps as the MMA M dimension:
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
// The encoder: input staging to 7-sample windows (enc.conv_in = one k-block), the residual blocks as above, each strided
// conv (k = 2r, stride r) as a 2-tap conv over the input read as folded rows [rows / r][r * C] with its per-utterance right
// padding written by tc_pad_rows_kernel, the LSTM above, enc.conv_out to fp32 rows; the RVQ search stays the fp32 one of
// encodec.cu.
//
// Host side: each direction is one Plan (tensors, layers with their GEMMs, fp32 buffers) built by walking the model once
// (build_dec / build_enc); ws_layout derives a chunk's workspace from it and run_chunk every launch.  A GEMM whose K does not
// fit the kernel's k-blocks makes the configuration not covered.
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
struct Dbg { Plane p; const __nv_bfloat16* ptr; int B; };   // a tensor of the last chunk (debug read-back)

// ---- the layer plan of one direction: the layer sequence over a table of tensors, independent of the chunk.  The GEMMs,
// the launches and the workspace are derived from it, and for the decoder the stream-state layout and min_T.
//
// A tensor belongs to a stage: the chunk's plane rows per utterance of every stage are one vector (decoder: T * the product
// of the ratios so far; encoder: each stage's length, rounded up to its strided conv's stride, from the samples to the
// frames).  Utterance-major, every utterance holds `halo` rows of left padding and then its rows; the input of an encoder
// strided conv (stride r) is read as folded rows [rows / r][r * C] (fold = r) and gets its right padding from L_RPAD.
enum { FORM_RAW = 1, FORM_ELU = 2 };
// HALO_UNWRITTEN: the rows exist (the tensor shares its block input's row geometry) but nothing stores or reads them
enum { HALO_REFLECT, HALO_ZERO, HALO_UNWRITTEN };

struct Tensor {
    int C = 0, halo = 0, halo_kind = HALO_ZERO;
    int stage = 0, fold = 1;
    bool tm = false;                   // time-major, row = (t + halo) * Bcap + b (LSTM planes); else utterance-major
    int forms = 0;                     // FORM_RAW | FORM_ELU stored
    int arena = -1, group = 0;         // -1: own rows; else an arena, where the tensors of one group stack (see ws_layout)
    bool carried = false;              // decoder stream: its halo rows (of the ELU'd form if stored, else raw) are carried ...
    size_t state_off = 0;              // ... at this offset of a stream's state
    std::string dbg_raw, dbg_elu;      // enc_debug_tensor names of the two forms ("": not exposed)
};

// L_RPAD: the right padding of a strided conv's input over the stage's length table; L_LPAD: a left halo no producer writes
enum { L_RVQ, L_INPUT, L_RPAD, L_LPAD, L_CONV, L_LSTM_IH, L_LSTM_STEPS, L_CONV_OUT_SPLIT, L_CONV_OUT };
enum { F32_NONE, F32_X0, F32_PRE, F32_COPART, F32_WAV, F32_LAT };   // fp32 destination of a GEMM
// the workspace's fp32 buffers: LSTM input, pre-activations and cells; the decoder's final-conv partial products; the
// encoder's latent rows, latent [B][D][T], RVQ scores and codes, per-utterance table
enum { BUF_X0, BUF_PRE, BUF_CST, BUF_COPART, BUF_LATF, BUF_LAT, BUF_SCORES, BUF_CODES, BUF_TAB, NBUF };

struct Layer {
    int kind = L_CONV;
    std::string label;                 // VCB_CODEC_PROFILE
    const TcGemm* g = nullptr;
    int in = -1, in_form = FORM_RAW;   // A source 0
    int in2 = -1;                      // A source 1, raw form: the block input of a residual tail (shortcut)
    int out = -1;                      // stores every form the tensor has
    int f32 = F32_NONE;
    int nstore = 0;                    // GEMM columns stored
    int lstm = -1;                     // LSTM layer
    size_t h_off = 0, c_off = 0;       // decoder stream: the layer's carried h and c in a stream's state
};

struct Plan {
    std::vector<Tensor> tensors;
    std::vector<Layer> layers;
    std::vector<std::unique_ptr<TcGemm>> gemms;   // the layers' weights (a layer's pointer stays valid as more are added)
    std::vector<int> bufs;             // the fp32 buffers the layers use, in workspace order
    int top = 0;                       // the stage of the LSTM and the latent frames
    std::vector<int> up;               // decoder: plane rows per frame of every stage
    std::vector<int> ratios;           // encoder: stride of stage s's strided conv (the config's ratios reversed)
    int u0 = -1;                       // decoder: input of the first ConvTranspose (its zero halo is cleared before every chunk)
    int min_T = 8;
    size_t stream_bytes = 0;           // decoder: carried state of one stream
    std::map<std::string, Dbg> dbg;    // the tensors of the last chunk by debug name

    TcGemm& gemm() { return *gemms.emplace_back(std::make_unique<TcGemm>()); }
    Layer& layer(int kind, std::string label, const TcGemm* g, int nstore, int in, int in_form, int out, int f32) {
        Layer& L = layers.emplace_back();
        L.kind = kind; L.label = std::move(label); L.g = g; L.nstore = nstore;
        L.in = in; L.in_form = in_form; L.out = out; L.f32 = f32;
        return L;
    }
};

}  // namespace

struct TcCodec {
    enc_config cfg;
    int hop = 1, D = 0, Dp = 0, ch0 = 0, num_sms = 132;
    DevBuf<const float*> d_embed;
    float co_bias = 0.f;               // bias of the split final conv, added by tc_diag_sum_kernel
    Plan dec;
    std::unique_ptr<Plan> enc;         // tensor-core encoder; null: no encoder weights, or not covered
    DevBuf<uint8_t> ws;
    size_t ws_limit = 0;
    bool profile = false;
    bool keep = false;                 // VCB_CODEC_KEEP=1: every plan tensor has its own rows, so all survive a chunk
    std::vector<std::pair<std::string, float>> prof;
    const float* dbg_cst = nullptr;    // the last decoded chunk's final LSTM cell states [layers][dbg_Bcap][ch0] ("c0", ...)
    int dbg_B = 0, dbg_Bcap = 0;
};

namespace {

inline int tc_num_sms(const TcCodec* tc) { return tc->num_sms; }

// 0: uploaded; 1: K is outside the kernel's k-blocks (the configuration is not covered); -1: error
int upload_gemm(TcGemm& g, const std::vector<float>& W, const std::vector<float>& bias, int N, int Ktot, int bn_hint) {
    if (Ktot < TC_BK || Ktot > TC_MAX_KB * TC_BK) return 1;
    if (Ktot % TC_BK) {
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

// a plan tensor's rows for a chunk of B utterances with plane rows R per stage: utterance-major, every utterance = halo rows +
// its rows; or time-major, row = (t + halo) * Bcap + b
Plane geometry(const Tensor& t, int B, const std::vector<int>& R) {
    Plane p;
    p.C = t.C;
    p.T = R[t.stage];
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
        p.rcap = std::max(B * p.Tp, TC_BM * t.fold);     // (whole folded rows; a TMA box never taller than its tensor)
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

// enc.conv_in on the input planes: channel j of a row is tap j, so the whole k-tap conv is one k-block
int build_enc_conv_in(TcGemm& g, const HostW& hw, int k, int Cout) {
    if (k > TC_BK) return 1;                                       // the input window does not fit one k-block
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

// the decoder's final conv (k <= DS_LD) as per-tap partial products: GEMM row j = tap j, summed by tc_diag_sum_kernel
int build_conv_out_split(TcGemm& g, const HostW& hw, int C, int k, float* bias) {
    std::vector<float> w, b;
    if (hw.get("dec.conv_out.weight", w) || hw.get("dec.conv_out.bias", b)) return -1;
    const int Cp = cpad(C);
    std::vector<float> W(static_cast<size_t>(k) * Cp, 0.f);
    for (int ci = 0; ci < C; ++ci)
        for (int j = 0; j < k; ++j) W[static_cast<size_t>(j) * Cp + ci] = w[static_cast<size_t>(ci) * k + j];
    for (int cb = 0; cb < Cp / TC_BK; ++cb) g.taps.push_back(TcTap{0, 0, cb * TC_BK});
    g.Cout = 32;
    g.up = 1;
    *bias = b[0];
    return upload_gemm(g, W, std::vector<float>(), k, Cp, 32);
}

// One residual block (weights `name`, profile labels prefixed by `lp`): conv1 (kres taps, dilation dil) on ELU(x) -> the
// hidden tensor hd, then conv2 on hd and the 1x1 shortcut on raw x as one GEMM -> o.  C and hidden are real channels.
int res_block(Plan& pl, const HostW& hw, const std::string& name, const std::string& lp, int x, int hd, int o, int C,
              int hidden, int kres, int dil) {
    TcGemm& g1 = pl.gemm();
    if (int rc = build_conv(g1, hw, name + ".conv1", C, hidden, kres, dil)) return rc;
    pl.layer(L_CONV, lp + "res_conv1", &g1, cpad(hidden), x, FORM_ELU, hd, F32_NONE);
    TcGemm& g2 = pl.gemm();
    if (int rc = build_res_tail(g2, hw, name, C, hidden)) return rc;
    pl.layer(L_CONV, lp + "res_conv2", &g2, cpad(C), hd, FORM_ELU, o, F32_NONE).in2 = x;
    return 0;
}

// The LSTM stack (weights `dir`.lstm.*): per layer, W_ih for all steps as one GEMM into the fp32 pre-activations (layer 0
// reads x0, layer l the h planes of layer l-1), then the steps over the layer's h planes hs[l % 2].  The last layer's
// epilogue writes ELU(h + skip) straight into `out`.
int lstm_stack(Plan& pl, const HostW& hw, const std::string& dir, const std::string& lp, int H, int x0, const int* hs, int out,
               int step_bn, int nl) {
    for (int l = 0; l < nl; ++l) {
        const std::string w = dir + ".lstm.weight_", b = dir + ".lstm.bias_", sl = "_l" + std::to_string(l);
        TcGemm& ih = pl.gemm();
        if (int rc = build_lstm(ih, hw, w + "ih" + sl, b + "ih" + sl, b + "hh" + sl, H, 0)) return rc;
        pl.layer(L_LSTM_IH, lp + "lstm_ih", &ih, 4 * H, l == 0 ? x0 : hs[(l - 1) & 1], FORM_RAW, -1, F32_PRE).lstm = l;
        TcGemm& step = pl.gemm();
        if (int rc = build_lstm(step, hw, w + "hh" + sl, "", "", H, step_bn)) return rc;
        pl.layer(L_LSTM_STEPS, lp + "lstm_steps", &step, 4 * H, hs[l & 1], FORM_RAW, l == nl - 1 ? out : -1, F32_NONE).lstm = l;
    }
    return 0;
}

// The decoder's layers in launch order, each with its GEMM.  Every halo rule is here: a causal convolution reads
// (k-1)*dilation rows above its output row, so its input keeps that many halo rows, padded like the reference (reflect or
// zeros); a ConvTranspose reads x[t-1], so its input keeps one zero row.  A stream's state holds the carried tensors and
// the LSTM (h, c) per layer, in the order the carries run.  0: built; 1: not covered; -1: error.
int build_dec(TcCodec* tc, const HostW& hw, int step_bn) {
    const enc_config& cf = tc->cfg;
    Plan& pl = tc->dec;
    const int H = tc->ch0, nl = cf.lstm, nres = cf.n_residual_layers;
    const int kres = cf.residual_kernel_size, kout = cf.last_kernel_size;
    const int pad = cf.pad_reflect ? HALO_REFLECT : HALO_ZERO;
    enum { ARENA_X0, ARENA_X1, ARENA_HIDDEN };   // the stages' ping-pong arenas, and the hidden tensors'
    // arena tensors are each a group of their own: they all start at their arena's first byte
    auto tensor = [&](int C, int halo, int kind, int stage, bool tm, int forms, int arena, bool carried, std::string dbg_raw,
                      std::string dbg_elu) {
        Tensor t;
        t.C = C; t.halo = halo; t.halo_kind = kind; t.stage = stage; t.tm = tm;
        t.forms = forms; t.arena = tc->keep ? -1 : arena; t.group = static_cast<int>(pl.tensors.size()); t.carried = carried;
        t.dbg_raw = std::move(dbg_raw);
        t.dbg_elu = std::move(dbg_elu);
        pl.tensors.push_back(t);
        return static_cast<int>(pl.tensors.size()) - 1;
    };
    // the input of a ConvTranspose, or of the final conv after the last stage
    auto feed = [&](bool last_stage, int& halo, int& kind) {
        halo = last_stage ? kout - 1 : 1;
        kind = last_stage ? pad : HALO_ZERO;
    };
    char nm[96];

    pl.up.push_back(1);
    const int z = tensor(tc->Dp, cf.kernel_size - 1, pad, 0, false, FORM_RAW, -1, true, "z", "");
    pl.u0 = tensor(cpad(H), 1, HALO_ZERO, 0, false, FORM_ELU, -1, true, "", "u0");
    int x0 = -1, hs[2] = {-1, -1};
    if (nl > 0) {
        x0 = tensor(H, 0, HALO_ZERO, 0, true, FORM_RAW, -1, false, "x0", "");
        for (int l = 0; l < std::min(nl, 2); ++l)                 // h planes: slot t+1 = h_t, layers alternate
            hs[l] = tensor(H, 1, HALO_ZERO, 0, true, FORM_RAW, -1, false, "hs" + std::to_string(l), "");
        pl.bufs = {BUF_X0, BUF_PRE, BUF_CST};
    }
    pl.layer(L_RVQ, "rvq", nullptr, 0, -1, 0, z, F32_NONE);
    TcGemm& ci = pl.gemm();
    if (int rc = build_conv(ci, hw, "dec.conv_in", cf.dimension, H, cf.kernel_size, 1)) return rc;
    pl.layer(L_CONV, "conv_in", &ci, cpad(H), z, FORM_RAW, nl > 0 ? x0 : pl.u0, nl > 0 ? F32_X0 : F32_NONE);
    if (int rc = lstm_stack(pl, hw, "dec", "", H, x0, hs, pl.u0, step_bn, nl)) return rc;
    // up-sampling stages: ConvTranspose -> X; per residual block conv1 (on ELU(X)) -> hidden, then conv2 (on the hidden) +
    // shortcut (on raw X) -> O, the next block's X.  X and O alternate between the two arenas.
    int cur = pl.u0, ch = H, side = ARENA_X0;
    for (int i = 0; i < cf.n_ratios; ++i) {
        const int r = cf.ratios[i], cout = ch / 2, hidden = cout / cf.compress, stage = i + 1;
        const bool last_stage = i == cf.n_ratios - 1;
        const std::string s = std::to_string(i + 1);
        pl.up.push_back(pl.up.back() * r);
        int halo = kres - 1, kind = pad;
        if (nres == 0) feed(last_stage, halo, kind);
        int x = tensor(cpad(cout), halo, kind, stage, false, (nres > 0 ? FORM_RAW : 0) | FORM_ELU, side, true,
                       nres > 0 ? "x" + s + ".raw" : "", "x" + s + ".elu");
        TcGemm& up = pl.gemm();
        snprintf(nm, sizeof(nm), "dec.up%d.convtr", i);
        if (int rc = build_convtr(up, hw, nm, ch, cout, r)) return rc;
        pl.layer(L_CONV, "convtr", &up, r * cpad(cout), cur, FORM_ELU, x, F32_NONE);
        ch = cout;
        for (int j = 0, dil = 1; j < nres; ++j, dil *= cf.dilation_base) {
            const std::string sj = s + "." + std::to_string(j);
            const int hd = tensor(cpad(hidden), pl.tensors[x].halo, HALO_UNWRITTEN, stage, false, FORM_ELU, ARENA_HIDDEN, false,
                                  "", "h" + sj);
            // the next block's conv1 reads (kres-1) * its dilation rows back.  min_T takes this term for the last block too.
            const int next = (kres - 1) * dil * cf.dilation_base;
            pl.min_T = std::max(pl.min_T, next + 2);
            halo = next;
            kind = pad;
            if (j == nres - 1) feed(last_stage, halo, kind);
            const int o = tensor(cpad(cout), halo, kind, stage, false, (j < nres - 1 ? FORM_RAW : 0) | FORM_ELU, side ^ 1, true,
                                 j < nres - 1 ? "o" + sj + ".raw" : "", "o" + sj);
            snprintf(nm, sizeof(nm), "dec.up%d.res%d", i, j);
            if (int rc = res_block(pl, hw, nm, "", x, hd, o, cout, hidden, kres, dil)) return rc;
            x = o;
            side ^= 1;
        }
        cur = x;
        side ^= 1;                                                 // the next ConvTranspose must not write over `cur`
    }
    // final conv: k <= DS_LD partial products (the first 16-column chunk), or one output column (f_valid = 1)
    TcGemm& co = pl.gemm();
    if (int rc = build_conv(co, hw, "dec.conv_out", ch, 1, kout, 1, 32)) return rc;
    if (kout <= DS_LD && !(getenv("VCB_CODEC_CONVOUT_TC") && atoi(getenv("VCB_CODEC_CONVOUT_TC")))) {
        TcGemm& cop = pl.gemm();
        if (int rc = build_conv_out_split(cop, hw, ch, kout, &tc->co_bias)) return rc;
        pl.layer(L_CONV_OUT_SPLIT, "conv_out", &cop, 16, cur, FORM_ELU, -1, F32_COPART);
        pl.bufs.push_back(BUF_COPART);
    } else {
        pl.layer(L_CONV_OUT, "conv_out", &co, 32, cur, FORM_ELU, -1, F32_WAV);
    }
    pl.min_T = std::max(pl.min_T, std::max(cf.kernel_size, kout) + 1);
    for (Layer& L : pl.layers) {                                   // the stream state, in the order the carries run
        if (L.kind == L_LSTM_STEPS) {
            L.h_off = pl.stream_bytes;
            L.c_off = pl.stream_bytes + static_cast<size_t>(H) * 4;
            pl.stream_bytes += static_cast<size_t>(H) * 8;
        }
        Tensor* t = L.out >= 0 ? &pl.tensors[L.out] : nullptr;
        if (t && t->carried && t->halo > 0) {
            t->state_off = pl.stream_bytes;
            pl.stream_bytes += static_cast<size_t>(t->halo) * t->C * 4;
        }
    }
    return 0;
}

// The encoder's layers in launch order (SEANetEncoder, oracle/encodec_oracle.py::encoder_plan), each with its GEMM.  Stage
// s holds the rows of the s-th strided conv's input (stage 0: the samples; stage n: the frames).  Halo rule as in the
// decoder; a strided conv's input keeps r rows (its causal left pad) plus the per-utterance right padding (L_RPAD).
// 0: built; 1: not covered; -1: error.
int build_enc(TcCodec* tc, const HostW& hw, int step_bn) {
    const enc_config& cf = tc->cfg;
    Plan& pl = *tc->enc;
    const int n = cf.n_ratios, nres = cf.n_residual_layers, nl = cf.lstm, H = tc->ch0;
    const int kres = cf.residual_kernel_size, kout = cf.last_kernel_size;
    const int pad = cf.pad_reflect ? HALO_REFLECT : HALO_ZERO;
    for (int s = 0; s < n; ++s) pl.ratios.push_back(cf.ratios[n - 1 - s]);
    pl.top = n;
    // the stages alternate between two arenas (stage s's strided conv reads arena s % 2 and writes arena (s+1) % 2), where
    // the tensors of a stage stack; the LSTM stage's tensors have their own rows
    auto tensor = [&](int C, int halo, int kind, int stage, int fold, bool tm, int forms, std::string dbg_raw, std::string dbg_elu) {
        Tensor t;
        t.C = C; t.halo = halo; t.halo_kind = kind; t.stage = stage; t.fold = fold; t.tm = tm; t.forms = forms;
        t.arena = (tc->keep || stage == n) ? -1 : stage & 1;
        t.group = stage;
        t.dbg_raw = std::move(dbg_raw);
        t.dbg_elu = std::move(dbg_elu);
        pl.tensors.push_back(t);
        return static_cast<int>(pl.tensors.size()) - 1;
    };
    // what stage s's first layer reads: its first residual block (conv1 reads kres-1 rows back), or its strided conv
    auto block_input = [&](int s, int C, const std::string& name) {
        if (nres > 0) return tensor(C, kres - 1, pad, s, 1, false, FORM_RAW | FORM_ELU, name, name + ".elu");
        return tensor(C, pl.ratios[s], pad, s, pl.ratios[s], false, FORM_ELU, "", name + ".elu");
    };
    char nm[96];
    int ch = cf.n_filters;
    const int in0 = tensor(TC_BK, 0, HALO_ZERO, 0, 1, false, FORM_RAW, "enc.input", "");
    pl.layer(L_INPUT, "enc_input", nullptr, 0, -1, 0, in0, F32_NONE);
    int cur = block_input(0, cpad(ch), "enc.x0");
    TcGemm& ci = pl.gemm();
    if (int rc = build_enc_conv_in(ci, hw, cf.kernel_size, cf.n_filters)) return rc;
    pl.layer(L_CONV, "enc_conv_in", &ci, cpad(ch), in0, FORM_RAW, cur, F32_NONE);
    int u = -1, x0 = -1;
    for (int s = 0; s < n; ++s) {
        const int r = pl.ratios[s], hidden = ch / cf.compress;
        const std::string si = "enc.down" + std::to_string(s);
        for (int j = 0, dil = 1; j < nres; ++j, dil *= cf.dilation_base) {
            const std::string sj = si + ".res" + std::to_string(j);
            const Tensor x = pl.tensors[cur];
            const int hd = tensor(cpad(hidden), x.halo, HALO_UNWRITTEN, s, x.fold, false, FORM_ELU, "", sj + ".h");
            const int o = j == nres - 1 ? tensor(cpad(ch), r, pad, s, r, false, FORM_ELU, "", sj + ".elu")
                                        : tensor(cpad(ch), (kres - 1) * dil * cf.dilation_base, pad, s, 1, false,
                                                 FORM_RAW | FORM_ELU, sj, sj + ".elu");
            if (int rc = res_block(pl, hw, sj, "enc_", cur, hd, o, ch, hidden, kres, dil)) return rc;
            cur = o;
        }
        pl.layer(L_RPAD, "enc_rpad", nullptr, 0, -1, 0, cur, F32_NONE);
        int next;
        if (s < n - 1) next = block_input(s + 1, cpad(2 * ch), si + ".conv");
        else if (nl > 0) next = x0 = tensor(H, 0, HALO_ZERO, n, 1, true, FORM_RAW, si + ".conv", "");
        else next = u = tensor(cpad(2 * ch), kout - 1, pad, n, 1, false, FORM_ELU, "", "enc.lstm");
        TcGemm& d = pl.gemm();
        snprintf(nm, sizeof(nm), "enc.down%d.conv", s);
        if (int rc = build_down(d, hw, nm, ch, 2 * ch, r)) return rc;
        pl.layer(L_CONV, "enc_down", &d, cpad(2 * ch), cur, FORM_ELU, next, next == x0 ? F32_X0 : F32_NONE);
        cur = next;
        ch *= 2;
    }
    if (nl > 0) {
        int hs[2] = {-1, -1};
        for (int l = 0; l < std::min(nl, 2); ++l)
            hs[l] = tensor(H, 1, HALO_ZERO, n, 1, true, FORM_RAW, "enc.hs" + std::to_string(l), "");
        u = tensor(cpad(H), kout - 1, pad, n, 1, false, FORM_ELU, "", "enc.lstm");
        // the last layer's epilogue writes ELU(h + skip) into enc.conv_out's input, whose halo L_LPAD then fills
        if (int rc = lstm_stack(pl, hw, "enc", "enc_", H, x0, hs, u, step_bn, nl)) return rc;
        pl.layer(L_LPAD, "enc_lpad", nullptr, 0, -1, 0, u, F32_NONE);
        pl.bufs = {BUF_X0, BUF_PRE, BUF_CST};
    }
    TcGemm& co = pl.gemm();
    if (int rc = build_conv(co, hw, "enc.conv_out", H, cf.dimension, kout, 1)) return rc;
    pl.layer(L_CONV_OUT, "enc_conv_out", &co, tc->Dp, u, FORM_ELU, -1, F32_LAT);
    pl.bufs.insert(pl.bufs.end(), {BUF_LATF, BUF_LAT, BUF_SCORES, BUF_CODES, BUF_TAB});
    return 0;
}

// the stage lengths of an utterance of N samples: L[0] = N, L[s+1] = ceil(L[s] / r_s)
std::vector<int> enc_chain(const Plan& pl, int N) {
    std::vector<int> L(1, N);
    for (int r : pl.ratios) L.push_back((L.back() + r - 1) / r);
    return L;
}

// plane rows per utterance of every stage: the stage length rounded up to its strided conv's stride
std::vector<int> enc_rows(const Plan& pl, const std::vector<int>& L) {
    std::vector<int> R(L);
    for (size_t s = 0; s < pl.ratios.size(); ++s) R[s] = (L[s] + pl.ratios[s] - 1) / pl.ratios[s] * pl.ratios[s];
    return R;
}

// the decoder's plane rows per utterance of every stage for T frames
std::vector<int> dec_rows(const Plan& pl, int T) {
    std::vector<int> R;
    for (int u : pl.up) R.push_back(T * u);
    return R;
}

// The workspace of a chunk of B utterances with plane rows R per stage: the tensors with rows of their own, the arenas, the
// fp32 buffers.  In an arena, the tensors of a group stack, and every group starts at the arena's first byte: the arena is
// as large as its largest group.  tensor[i] = offset of plan tensor i's first stored form (an ELU'd form follows a raw one).
struct WsLayout {
    std::vector<size_t> tensor;
    size_t buf[NBUF] = {};
    size_t bytes = 0;
};

WsLayout ws_layout(const TcCodec* tc, const Plan& pl, int B, const std::vector<int>& R) {
    const enc_config& cf = tc->cfg;
    const size_t Bn = B, Bc = bcap(B), H = tc->ch0, Tn = R[pl.top];
    WsLayout w;
    w.tensor.resize(pl.tensors.size());
    size_t off = 0;
    auto take = [&](size_t bytes) {
        const size_t o = off;
        off += align_up(bytes, 1024);
        return o;
    };
    std::map<int, size_t> group_end;
    size_t arena[3] = {0, 0, 0};
    for (size_t i = 0; i < pl.tensors.size(); ++i) {
        const Tensor& t = pl.tensors[i];
        size_t bytes = 0;
        for (int f : {FORM_RAW, FORM_ELU})
            if (t.forms & f) bytes += align_up(form_bytes(geometry(t, B, R)), 1024);
        if (t.arena < 0) {
            w.tensor[i] = take(bytes);
        } else {
            w.tensor[i] = group_end[t.group];                     // offset inside its arena for now
            group_end[t.group] += bytes;
            arena[t.arena] = std::max(arena[t.arena], group_end[t.group]);
        }
    }
    const size_t a[3] = {take(arena[0]), take(arena[1]), take(arena[2])};
    for (size_t i = 0; i < pl.tensors.size(); ++i)
        if (pl.tensors[i].arena >= 0) w.tensor[i] += a[pl.tensors[i].arena];
    for (int b : pl.bufs) {
        size_t bytes = 0;
        switch (b) {
            case BUF_X0: bytes = Tn * Bc * H * 4; break;           // time-major [T][Bcap][H]
            case BUF_PRE: bytes = Tn * Bc * 4 * H * 4; break;      // time-major [T][Bcap][4H]
            case BUF_CST: bytes = cf.lstm * Bc * H * 4; break;     // [layers][Bcap][H]
            case BUF_COPART: {                                     // the final conv's input rows, halo included, + a tile
                const Tensor& in = pl.tensors[pl.layers.back().in];
                bytes = (Bn * (R[in.stage] + std::max(in.halo, 1)) + TC_BM) * DS_LD * 4;
                break;
            }
            case BUF_LATF: bytes = Bn * Tn * tc->Dp * 4; break;    // [B][T][Dp]
            case BUF_LAT: bytes = Bn * cf.dimension * Tn * 4; break;
            case BUF_SCORES: bytes = Bn * cf.bins * Tn * 4; break;
            case BUF_CODES: bytes = Bn * cf.n_q * Tn * 8; break;
            case BUF_TAB: bytes = (R.size() + 1) * Bn * 4; break;  // [stages][B] lengths, then [B] wav rows
        }
        w.buf[b] = take(bytes);
    }
    w.bytes = off;
    return w;
}

// grows the workspace to at least `need` bytes (alloc releases the previous one first, so the stream is drained before)
int grow_ws(TcCodec* tc, size_t need, cudaStream_t st, const std::string& what) {
    if (need <= tc->ws.size()) return 0;
    if (tc->ws) VCB_CUDA_OK(cudaStreamSynchronize(st));
    if (tc->ws.alloc(need) == 0) return 0;
    const std::string why = get_error();
    set_error("codec_tc: cannot allocate a %.2f GB %s (%s)", need / 1073741824.0, what.c_str(), why.c_str());
    return -1;
}

// what a chunk reads and writes outside the workspace
struct ChunkIO {
    const int64_t* codes = nullptr;    // decoder: codes [B][n_q][T]
    float* wav = nullptr;              // decoder: waveform [B][T * hop]
    const float* wav_in = nullptr;     // encoder: fp32 wav rows (the table's rows) of wav_ld samples
    long long wav_ld = 0;
    const TcStreamCtx* sc = nullptr;   // decoder stream: every plane a layer reads as left context, and the LSTM state,
                                       // continue the utterance's stream (tc_carry_kernel)
};

// One chunk of B utterances through plan pl, with plane rows R per stage, in the workspace laid out as w.
int run_chunk(TcCodec* tc, Plan& pl, const WsLayout& w, int B, const std::vector<int>& R, cudaStream_t st, int64_t* launches,
              const ChunkIO& io) {
    const enc_config& cf = tc->cfg;
    const int Bcap = bcap(B), H = tc->ch0, nl = cf.lstm;
    const TcStreamCtx* sc = io.sc;
    auto buf = [&](int b) { return reinterpret_cast<float*>(tc->ws + w.buf[b]); };
    int* tab = reinterpret_cast<int*>(buf(BUF_TAB));                // encoder: [stages][B] lengths, then [B] wav rows
    std::vector<Plane> P(pl.tensors.size());
    pl.dbg.clear();
    for (size_t i = 0; i < P.size(); ++i) {
        const Tensor& t = pl.tensors[i];
        Plane& p = P[i];
        p = geometry(t, B, R);
        uint8_t* base = tc->ws + w.tensor[i];
        if (t.forms & FORM_RAW) {
            p.raw = reinterpret_cast<__nv_bfloat16*>(base);
            base += align_up(form_bytes(p), 1024);
        }
        if (t.forms & FORM_ELU) p.elu = reinterpret_cast<__nv_bfloat16*>(base);
        if (!t.dbg_raw.empty()) pl.dbg[t.dbg_raw] = Dbg{p, p.raw, B};
        if (!t.dbg_elu.empty()) pl.dbg[t.dbg_elu] = Dbg{p, p.elu, B};
    }

    // state that the kernels only ever read: U0's zero halo (the LSTM epilogue writes none), c_0 and h_{-1}
    if (pl.u0 >= 0) {
        const Plane& u0 = P[pl.u0];
        VCB_CUDA_OK(cudaMemset2DAsync(u0.elu, static_cast<size_t>(u0.Tp) * u0.C * 2, 0, static_cast<size_t>(u0.C) * 2, B, st));
        VCB_CUDA_OK(cudaMemset2DAsync(u0.elu + u0.plane(), static_cast<size_t>(u0.Tp) * u0.C * 2, 0, static_cast<size_t>(u0.C) * 2, B, st));
    }
    auto clear_h0 = [&](const Plane& hs) -> int {
        VCB_CUDA_OK(cudaMemsetAsync(hs.raw, 0, static_cast<size_t>(Bcap) * H * 2, st));
        VCB_CUDA_OK(cudaMemsetAsync(hs.raw + hs.plane(), 0, static_cast<size_t>(Bcap) * H * 2, st));
        return 0;
    };
    if (nl > 0) {
        VCB_CUDA_OK(cudaMemsetAsync(buf(BUF_CST), 0, static_cast<size_t>(nl) * Bcap * H * 4, st));
        for (const Layer& L : pl.layers)
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
        const Tensor& t = pl.tensors[i];
        const Plane& p = P[i];
        if (sc == nullptr || !t.carried || p.halo == 0) return 0;
        return carry(p.elu ? p.elu : p.raw, p.plane() * 2, p.sb, p.st, p.off, p.C * 2, p.halo, pl.up[t.stage], 1, 1, t.state_off);
    };
    // stream decode: h_{-1} (slot 0) and c continue the stream; after the layer, h of the last valid step (slot frames) and
    // the frozen c are saved.  As a time-major plane with one halo row, row(b, t) = (t + 1) * Bcap + b.
    auto carry_lstm = [&](const Layer& L, const Plane& hs, float* cl, int restore, int save) -> int {
        if (sc == nullptr) return 0;
        return carry(hs.raw, hs.plane() * 2, hs.sb, hs.st, hs.off, H * 2, 1, 1, restore, save, L.h_off) ||
               carry(cl, 0, 1, 0, 0, H * 4, 1, 1, restore, save, L.c_off);
    };
    auto pad_rows = [&](__nv_bfloat16* base, const Plane& o, const int* lens, int r, int zero) -> int {
        tc_pad_rows_kernel<<<B, 256, 0, st>>>(base, o.plane(), o.C, o.sb, o.st, o.off, lens, o.halo, r, zero);
        VCB_CUDA_OK(cudaGetLastError());
        ++*launches;
        return 0;
    };

    Prof pf{tc, st};
    CUtensorMap mA, mB;
    for (const Layer& L : pl.layers) {
        pf.begin(L.label.c_str());
        if (L.kind == L_RVQ) {
            const Plane& z = P[L.out];
            tc_rvq_planes_kernel<<<dim3((z.T + 15) / 16, B), 128, 0, st>>>(reinterpret_cast<const long long*>(io.codes), tc->d_embed,
                                                                           z.raw, z.plane(), cf.n_q, tc->D, z.C, z.T, z.Tp, z.halo,
                                                                           z.halo_zero);
            VCB_CUDA_OK(cudaGetLastError());
            ++*launches;
        } else if (L.kind == L_INPUT) {
            const Plane& o = P[L.out];
            const long long items = static_cast<long long>(B) * o.T;
            tc_enc_input_kernel<<<static_cast<unsigned>((items + 255) / 256), 256, 0, st>>>(
                io.wav_in, io.wav_ld, tab + R.size() * B, tab, o.raw, o.plane(), o.C, o.Tp, o.T, cf.kernel_size, cf.pad_reflect, B);
            VCB_CUDA_OK(cudaGetLastError());
            ++*launches;
        } else if (L.kind == L_RPAD || L.kind == L_LPAD) {
            const Tensor& t = pl.tensors[L.out];
            const Plane& o = P[L.out];
            const bool right = L.kind == L_RPAD;
            if (pad_rows(o.elu ? o.elu : o.raw, o, right ? tab + static_cast<size_t>(t.stage) * B : nullptr, right ? t.fold : 1,
                         o.halo_zero))
                return -1;
        } else {
            const TcGemm& g = *L.g;
            Plane in = P[L.in];
            const int r = pl.tensors[L.in].fold;
            if (r > 1) {                                     // folded rows: r plane rows of C channels are one row of r*C
                in.C *= r; in.rcap /= r; in.Tp /= r; in.T /= r; in.halo = 1; in.sb = in.Tp; in.off = 1;
            }
            if (plane_map(&mA, L.in_form == FORM_ELU ? P[L.in].elu : P[L.in].raw, in) ||
                (L.in2 >= 0 && plane_map(&mB, P[L.in2].raw, P[L.in2])))
                return -1;
            const CUtensorMap& a1 = L.in2 >= 0 ? mB : mA;
            // the call of a plan GEMM: its weights, its A rows, its epilogue (the LSTM steps then only move t_step and row_base)
            TcCall c{};
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
                c.raw = o.raw;
                c.elu = o.elu;
                c.o_plane = o.plane();
                c.o_ld = o.C;
                c.o_sb = o.sb;
                c.o_st = o.st;
                c.o_off = o.off;
                c.o_halo = pl.tensors[L.out].halo_kind == HALO_UNWRITTEN ? 0 : o.halo;
                c.o_halo_zero = o.halo_zero;
            }
            auto rows = [&](float* f, int ld, int valid, long long sb, long long stt, long long off) {
                c.f32 = f; c.f_ld = ld; c.f_valid = valid; c.f_sb = sb; c.f_st = stt; c.f_off = off;
            };
            if (L.f32 == F32_X0) rows(buf(BUF_X0), H, H, 1, Bcap, 0);                  // time-major [T][Bcap][H]
            if (L.f32 == F32_PRE) rows(buf(BUF_PRE), 4 * H, 4 * H, 1, Bcap, 0);         // time-major [T][Bcap][4H]
            if (L.f32 == F32_COPART) {                                                // the input's rows, halo included
                rows(buf(BUF_COPART), DS_LD, DS_LD, in.sb, 1, in.off);
                c.in_store_halo = 1;
            }
            if (L.f32 == F32_WAV) {                                                   // [B][T * hop]
                rows(io.wav, 1, 1, in.T, 1, 0);
                c.f_scalar = 1;
            }
            if (L.f32 == F32_LAT) rows(buf(BUF_LATF), tc->Dp, cf.dimension, in.T, 1, 0);  // [B][T][Dp]
            if (L.kind == L_LSTM_STEPS) {
                c.mode = TC_MODE_LSTM;
                c.pre = buf(BUF_PRE);
                c.cst = buf(BUF_CST) + static_cast<size_t>(L.lstm) * Bcap * H;
                c.hseq = in.raw;
                c.h_plane = in.plane();
                c.Bcap = Bcap;
                c.H = H;
                if (L.out >= 0) c.skip = buf(BUF_X0);
                if (sc != nullptr) c.stab = sc->table;
                if (L.lstm >= 2 && clear_h0(in)) return -1;
                if (carry_lstm(L, in, c.cst, 1, 0)) return -1;
                for (int t = 0; t < in.T; ++t) {                                      // one step per row of its stage
                    c.t_step = t;
                    c.row_base = t * Bcap;
                    if (tc_launch(tc, mA, a1, g, c, st)) return -1;
                }
                *launches += in.T;
                if (carry_lstm(L, in, c.cst, 0, 1)) return -1;
            } else {
                if (tc_launch(tc, mA, a1, g, c, st)) return -1;
                ++*launches;
                // The epilogue zeroes halo row -t from output row t, 1 <= t <= halo, and a GEMM writes in.T rows (an
                // encoder strided conv ceil(L/r) of the chunk's longest utterance).  With constant padding an utterance
                // may be shorter than a halo (the encoder takes rows of any length), and a chunk of only such utterances
                // writes no row t for some halo rows: they are cleared here, or they would keep whatever an earlier chunk
                // left in the workspace.  The decoder's tensors are carried: its T >= min_T exceeds every halo, or (a stream
                // decode of continuing streams only) each halo is the stream's saved tail.
                const Tensor* t = L.out >= 0 ? &pl.tensors[L.out] : nullptr;
                if (t && t->halo_kind == HALO_ZERO && !t->tm && !t->carried && in.T <= t->halo)
                    for (__nv_bfloat16* base : {c.raw, c.elu})
                        if (base != nullptr && pad_rows(base, P[L.out], nullptr, 1, 1)) return -1;
            }
            if (L.kind == L_CONV_OUT_SPLIT) {
                VCB_CUDA_OK(launch_k_pdl(1, tc_diag_sum_kernel, dim3((in.rcap + DS_ROWS - 1) / DS_ROWS), dim3(DS_ROWS), 0, st,
                                         buf(BUF_COPART), cf.last_kernel_size, tc->co_bias, io.wav, in.rcap, in.Tp, in.halo, in.T, B));
                ++*launches;
            }
        }
        if (L.out >= 0 && carry_plane(L.out)) return -1;
        pf.end();
    }
    pf.finish();
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
    {
        std::vector<const float*> emb(cfg.n_q);
        for (int q = 0; q < cfg.n_q; ++q) {
            char nm[32];
            snprintf(nm, sizeof(nm), "vq.%d.embed", q);
            auto it = w_dev.find(nm);
            if (it == w_dev.end()) {
                set_error("codec: missing weight %s", nm);
                return -1;
            }
            emb[q] = it->second;
        }
        if (tc->d_embed.alloc(cfg.n_q) || cudaMemcpy(tc->d_embed, emb.data(), cfg.n_q * sizeof(float*), cudaMemcpyHostToDevice) != cudaSuccess) {
            set_error("codec_tc: codebook pointer table");
            return -1;
        }
    }
    const int rc = build_dec(tc.get(), hw, step_bn);
    if (rc > 0) return no("reduction deeper than the kernel's k-blocks");
    if (rc < 0) return -1;
    if (w_dev.count("enc.conv_in.weight")) {
        // the encoder where the decoder is covered, its input window fits one k-block and every reduction fits the kernel;
        // otherwise enc_encode_ragged encodes every row on the CUDA cores
        tc->enc.reset(new Plan());
        const int erc = build_enc(tc.get(), hw, step_bn);
        if (erc < 0) return -1;
        if (erc > 0) tc->enc.reset();
    }
    *out = std::move(tc);
    return 0;
}

bool tc_encoder_active(const TcCodec* c) { return c != nullptr && c->enc != nullptr; }

// every stage longer than the padding its convolutions reflect (audiocraft pad1d zero-extends a shorter input instead)
bool tc_encoder_accepts(const TcCodec* c, int len) {
    if (!tc_encoder_active(c) || len < 1) return false;
    const enc_config& cf = c->cfg;
    if (!cf.pad_reflect) return true;
    const std::vector<int> L = enc_chain(*c->enc, len);
    int dmax = 1;
    for (int j = 1; j < cf.n_residual_layers; ++j) dmax *= cf.dilation_base;
    const int res_pad = cf.n_residual_layers > 0 ? (cf.residual_kernel_size - 1) * dmax : 0;
    if (L[0] <= cf.kernel_size - 1) return false;
    for (size_t s = 0; s < c->enc->ratios.size(); ++s)
        if (L[s] <= res_pad || L[s] <= c->enc->ratios[s]) return false;
    return L.back() > cf.last_kernel_size - 1;
}

size_t tc_encoder_ws_bytes(const TcCodec* c, int B, int N) {
    return ws_layout(c, *c->enc, B, enc_rows(*c->enc, enc_chain(*c->enc, N))).bytes;
}

size_t tc_ws_limit(const TcCodec* c) { return c->ws_limit; }

int64_t tc_encoder_rows(const TcCodec* c, int B, int N) {
    return static_cast<int64_t>(B) * enc_rows(*c->enc, enc_chain(*c->enc, N))[0];
}

// One chunk: utterance b = wav row rows[b] with lens[b] samples; the chunk's planes are sized for its longest utterance.
int tc_encoder_encode(TcCodec* tc, const float* wav, long long wav_ld, const int* rows, const int* lens, int B, cudaStream_t st,
                      int64_t* launches, TcEncOut* out) {
    tc->prof.clear();
    const Plan& pl = *tc->enc;
    const int n = static_cast<int>(pl.ratios.size());
    const std::vector<int> R = enc_rows(pl, enc_chain(pl, *std::max_element(lens, lens + B)));
    const WsLayout w = ws_layout(tc, pl, B, R);
    if (grow_ws(tc, w.bytes, st, "encoder workspace for " + std::to_string(B) + " utterances")) return -1;
    {
        std::vector<int> h(static_cast<size_t>(n + 2) * B);
        for (int b = 0; b < B; ++b) {
            const std::vector<int> L = enc_chain(pl, lens[b]);
            for (int s = 0; s <= n; ++s) h[static_cast<size_t>(s) * B + b] = L[s];
            h[static_cast<size_t>(n + 1) * B + b] = rows[b];
        }
        VCB_CUDA_OK(cudaMemcpyAsync(tc->ws + w.buf[BUF_TAB], h.data(), h.size() * 4, cudaMemcpyHostToDevice, st));   // pageable: staged at once
    }
    ChunkIO io;
    io.wav_in = wav;
    io.wav_ld = wav_ld;
    if (run_chunk(tc, *tc->enc, w, B, R, st, launches, io)) return -1;
    const int Tn = R[n];
    const float* latf = reinterpret_cast<const float*>(tc->ws + w.buf[BUF_LATF]);
    float* lat = reinterpret_cast<float*>(tc->ws + w.buf[BUF_LAT]);
    tc_latent_cm_kernel<<<dim3((Tn + 31) / 32, B), 256, 32 * (tc->D + 1) * 4, st>>>(latf, lat, tc->D, tc->Dp, Tn);
    VCB_CUDA_OK(cudaGetLastError());
    ++*launches;
    out->latent = lat;
    out->scores = reinterpret_cast<float*>(tc->ws + w.buf[BUF_SCORES]);
    out->codes = reinterpret_cast<int64_t*>(tc->ws + w.buf[BUF_CODES]);
    out->T = Tn;
    return 0;
}

bool tc_codec_accepts(const TcCodec* c, int B, int T) { return c != nullptr && B >= 1 && T >= c->dec.min_T; }

int tc_codec_decode(TcCodec* tc, const int64_t* codes, float* wav, int B, int T, cudaStream_t st, int64_t* launches,
                    const TcStreamCtx* sc) {
    tc->prof.clear();
    const std::vector<int> R = dec_rows(tc->dec, T);
    // chunk the batch so the workspace stays under the limit -- and halve the chunk again if the device cannot give that much
    int chunk = B;
    for (;;) {
        const size_t need = ws_layout(tc, tc->dec, chunk, R).bytes;
        if (need > tc->ws_limit && chunk > 1) {
            chunk = (chunk + 1) / 2;
            continue;
        }
        if (grow_ws(tc, need, st, "workspace for one utterance of " + std::to_string(T) + " frames") == 0) break;
        if (chunk == 1) return -1;
        chunk = (chunk + 1) / 2;
    }
    for (int b0 = 0; b0 < B; b0 += chunk) {
        const int nb = std::min(chunk, B - b0);
        const WsLayout w = ws_layout(tc, tc->dec, nb, R);
        TcStreamCtx part;
        ChunkIO io;
        io.codes = codes + static_cast<size_t>(b0) * tc->cfg.n_q * T;
        io.wav = wav + static_cast<size_t>(b0) * T * tc->hop;
        if (sc != nullptr) {
            part = TcStreamCtx{sc->table + 4 * b0, sc->state};
            io.sc = &part;
        }
        tc->dbg_cst = tc->cfg.lstm > 0 ? reinterpret_cast<const float*>(tc->ws + w.buf[BUF_CST]) : nullptr;
        tc->dbg_B = nb;
        tc->dbg_Bcap = bcap(nb);
        if (run_chunk(tc, tc->dec, w, nb, R, st, launches, io)) return -1;
    }
    return 0;
}

size_t tc_stream_state_bytes(const TcCodec* c) { return c->dec.stream_bytes; }

int tc_stream_min_frames(const TcCodec* c) { return c->dec.min_T; }

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
    const Plan* plan = strncmp(name, "enc.", 4) ? &tc->dec : tc->enc.get();
    const auto it = plan ? plan->dbg.find(name) : std::map<std::string, Dbg>::const_iterator();
    if (plan == nullptr || it == plan->dbg.end()) {
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
