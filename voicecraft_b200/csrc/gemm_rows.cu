// Row-major ("rows as M") GEMM of the codec-LM for many token rows at once: prompt prefill.
//
//   out[r][n] = epilogue( sum_k (Xhi[r,k] + Xlo[r,k]) * W[n,k] + bias[n] )        r = token row, n = output feature
//
// gemm_wgmma.cu keeps the WEIGHTS as the 128-row operand and at most 128 token rows as the MMA N dimension: right
// for decode (every weight byte is used once per step), wrong for a prompt of thousands of rows, where it streams the
// whole matrix once per 128 rows and spends most of each launch in the per-row epilogue.  Here a CTA owns a
// [128 rows] x [BN features] output tile:
//   A operand = activations, bf16 [2][rcap][K]: plane 0 = hi parts, plane 1 = lo parts (x ~= hi + lo, split_bf16);
//               both 128 x 64 tiles of a k-block are multiplied with the SAME weight tile into the SAME accumulator
//               (D += Ahi.B^T ; D += Alo.B^T), so the second pass costs no extra weight traffic.
//   B operand = the pre-tiled weights of gemm_wgmma.cu, unchanged: BN/128 consecutive 16 KB blocks of one k-block,
//               stacked in shared memory, are exactly a K-major SWIZZLE_128B operand of BN rows.
//   D         = fp32 in registers (wgmma): each of two warpgroups multiplies 64 token rows x BN features, then stages
//               its accumulators in the (by then idle) pipeline shared memory, row = token, column = feature.
// No split-K, no cluster: with >= 512 rows there are enough tiles (e.g. QKV at d = 2048: 24 x rows/128 CTAs), and the
// weights (<= 34 MB per matrix) stay L2-resident across the row tiles.
// Warp roles as in gemm_wgmma.cu: w0 TMA producer, w1..w3 idle, w4..w11 MMA + epilogue (two warpgroups; in the
// epilogue each covers all 128 rows and takes half of the columns).
// Epilogues: EPI_QKV (q -> fp32 rows, k/v -> paged KV cache), EPI_RESID (x += y + b), EPI_ACT (ReLU/GELU -> hi/lo
// planes), EPI_LOGITS (plain fp32 rows; bring-up tests).  A thread owns one token row and 32 consecutive features
// per step, so every access is a run of 16-byte vectors.
#include "vcb_internal.h"

#include <algorithm>
#include <cstdio>

namespace vcb {

static constexpr int RG_BM = 128;     // token rows per CTA (2 x wgmma M)
static constexpr int RG_BK = 64;      // K elements per stage (one 128-byte swizzle row of bf16)
static constexpr int RG_EPI_WARPS = 8;
static constexpr int RG_THREADS = 128 + 32 * RG_EPI_WARPS;

template <int BN, int STAGES>
struct RowsSmem {
    static constexpr int A_BYTES = RG_BM * RG_BK * 2;               // one of the hi / lo tiles
    static constexpr int B_BYTES = BN * RG_BK * 2;
    static constexpr int STAGE_BYTES = 2 * A_BYTES + B_BYTES;
    static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
    static constexpr int TOTAL = BAR_OFFSET + 2 * STAGES * 8;
    static constexpr int ACC_LD = BN + 4;                           // staged accumulators [128][ACC_LD] fp32, conflict-free rows
    static_assert(RG_BM * ACC_LD * 4 <= BAR_OFFSET, "staged accumulators alias the pipeline stages");
};

__device__ __forceinline__ float act_fn(float v, int kind) {
    if (kind == 1) return fmaxf(v, 0.f);
    if (kind == 2) return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
    return v;
}

// 32 consecutive features [f0, f0+32) of token row `row`, accumulator values in v[]; `acc` points at the staged accumulator
// of feature f0 in the row, which holds every feature of f0's head (the fp8 KV scale is taken over the whole head).
// kv_amax / kv_head: the fp8 amax of the head whose first feature is kv_head, kept across the calls of one row, so each
// (row, head) amax is computed once
__device__ __forceinline__ void rows_epilogue32(const GemmEpilogue& ep, int row, int f0, float (&v)[32], const float* acc,
                                                float& kv_amax, int& kv_head) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] += ep.bias[f0 + j];         // same address in every lane: broadcast
    switch (ep.mode) {
        case EPI_QKV: {
            const int part = f0 / ep.d, cc = f0 - part * ep.d;
            if (part == 0) {
                float4* dst = reinterpret_cast<float4*>(ep.qbuf + static_cast<size_t>(row) * ep.d + cc);
#pragma unroll
                for (int j = 0; j < 8; ++j) dst[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                return;
            }
            const int pos = ep.row_pos[row];
            if (pos < 0) return;
            const int page = ep.row_page ? ep.row_page[row] : ep.page_table[ep.row_slot[row] * ep.max_pages + pos / ep.page_size];
            const int h = cc / ep.hd, e0 = cc - h * ep.hd;          // hd % 32 == 0: the 32 features share a head
            const size_t off = ((static_cast<size_t>(page) * ep.H + h) * ep.page_size + pos % ep.page_size) * ep.hd + e0;
            void* pool = (part == 1) ? ep.kpool : ep.vpool;
            if (ep.kv_fp8) {
                // the head's values are its staged accumulators plus bias, the same fp32 sums as v[]
                if (kv_head != f0 - e0) {
                    kv_head = f0 - e0;
                    kv_amax = 0.f;
                    for (int j = 0; j < ep.hd; ++j) kv_amax = fmaxf(kv_amax, fabsf(acc[j - e0] + ep.bias[kv_head + j]));
                }
                float inv;
                const float scale = kv_fp8_scale(kv_amax, inv);
                const int t = pos % ep.page_size;
                uint8_t* s = static_cast<uint8_t*>(pool) + (static_cast<size_t>(page) * ep.H + h) * kv_slab_bytes(KV_FP8, ep.hd);
                uint4* dst = reinterpret_cast<uint4*>(s + t * ep.hd + e0);
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    uint32_t w[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        w[i] = kv_fp8_pack2(v[16 * j + 4 * i], v[16 * j + 4 * i + 1], inv) |
                               (static_cast<uint32_t>(kv_fp8_pack2(v[16 * j + 4 * i + 2], v[16 * j + 4 * i + 3], inv)) << 16);
                    dst[j] = make_uint4(w[0], w[1], w[2], w[3]);
                }
                if (e0 == 0) reinterpret_cast<float*>(s + ep.page_size * ep.hd)[t] = scale;
            } else if (ep.kv_fp32) {
                float4* dst = reinterpret_cast<float4*>(static_cast<float*>(pool) + off);
#pragma unroll
                for (int j = 0; j < 8; ++j) dst[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
            } else {
                uint4* dst = reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(pool) + off);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    __nv_bfloat162 p0 = __floats2bfloat162_rn(v[8 * j], v[8 * j + 1]);
                    __nv_bfloat162 p1 = __floats2bfloat162_rn(v[8 * j + 2], v[8 * j + 3]);
                    __nv_bfloat162 p2 = __floats2bfloat162_rn(v[8 * j + 4], v[8 * j + 5]);
                    __nv_bfloat162 p3 = __floats2bfloat162_rn(v[8 * j + 6], v[8 * j + 7]);
                    dst[j] = make_uint4(*reinterpret_cast<uint32_t*>(&p0), *reinterpret_cast<uint32_t*>(&p1),
                                        *reinterpret_cast<uint32_t*>(&p2), *reinterpret_cast<uint32_t*>(&p3));
                }
            }
            break;
        }
        case EPI_RESID: {
            float4* px = reinterpret_cast<float4*>(ep.x + static_cast<size_t>(row) * ep.ld_out + f0);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float4 t = px[j];
                t.x += v[4 * j];
                t.y += v[4 * j + 1];
                t.z += v[4 * j + 2];
                t.w += v[4 * j + 3];
                px[j] = t;
            }
            break;
        }
        case EPI_ACT: {
            uint4* ph = reinterpret_cast<uint4*>(ep.act + static_cast<size_t>(row) * ep.ld_out + f0);
            uint4* pl = reinterpret_cast<uint4*>(ep.act + static_cast<size_t>(row + ep.bpad_out) * ep.ld_out + f0);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                uint32_t hw[4], lw[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    __nv_bfloat16 h0, l0, h1, l1;
                    split_bf16(act_fn(v[8 * j + 2 * u], ep.act_kind), h0, l0);
                    split_bf16(act_fn(v[8 * j + 2 * u + 1], ep.act_kind), h1, l1);
                    __nv_bfloat162 hh = __halves2bfloat162(h0, h1), ll = __halves2bfloat162(l0, l1);
                    hw[u] = *reinterpret_cast<uint32_t*>(&hh);
                    lw[u] = *reinterpret_cast<uint32_t*>(&ll);
                }
                ph[j] = make_uint4(hw[0], hw[1], hw[2], hw[3]);
                pl[j] = make_uint4(lw[0], lw[1], lw[2], lw[3]);
            }
            break;
        }
        default: {
            float4* dst = reinterpret_cast<float4*>(ep.out + static_cast<size_t>(row) * ep.ld_out + ep.col_off + f0);
#pragma unroll
            for (int j = 0; j < 8; ++j) dst[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
        }
    }
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(RG_THREADS)
gemm_rows_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const GemmEpilogue ep,
                 int rows, int rcap, int Nout, int total_kb) {
    using L = RowsSmem<BN, STAGES>;
    extern __shared__ __align__(1024) uint8_t smem[];       // SWIZZLE_128B tiles need 1024-byte alignment
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n0 = blockIdx.x * BN;                         // first output feature of this tile
    const int r0 = blockIdx.y * RG_BM;                      // first token row
    const int mt0 = n0 / 128;                               // first 128-feature weight block
    const int pre = min(total_kb, STAGES);

    pdl_launch_dependents();
    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmX);
        tma_prefetch_desc(&tmW);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], RG_EPI_WARPS);        // one arrival per MMA warp
        }
        mbar_fence_init();
        // weights never depend on the previous kernel: the first stages' weight tiles go in flight before the wait
        for (int i = 0; i < pre; ++i) {
            mbar_arrive_expect_tx(&full_bar[i], L::STAGE_BYTES);
            uint8_t* b = smem + i * L::STAGE_BYTES + 2 * L::A_BYTES;
#pragma unroll
            for (int j = 0; j < BN / 128; ++j)
                tma_load_2d(b + j * (128 * RG_BK * 2), &tmW, &full_bar[i], 0, ((mt0 + j) * total_kb + i) * 128);
        }
    }
    __syncthreads();

    if (warp == 0) {
        // ===== TMA producer ==========================================================================
        if (lane == 0) {
            pdl_wait();                                     // the activation planes come from the previous kernel
            for (int i = 0; i < pre; ++i) {
                uint8_t* a = smem + i * L::STAGE_BYTES;
                tma_load_2d(a, &tmX, &full_bar[i], i * RG_BK, r0);
                tma_load_2d(a + L::A_BYTES, &tmX, &full_bar[i], i * RG_BK, rcap + r0);
            }
            int stage = 0, phase = 0;
            for (int i = pre; i < total_kb; ++i) {
                mbar_wait(&empty_bar[stage], phase);        // the MMAs released this slot
                mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
                uint8_t* a = smem + stage * L::STAGE_BYTES;
                tma_load_2d(a, &tmX, &full_bar[stage], i * RG_BK, r0);
                tma_load_2d(a + L::A_BYTES, &tmX, &full_bar[stage], i * RG_BK, rcap + r0);
#pragma unroll
                for (int j = 0; j < BN / 128; ++j)
                    tma_load_2d(a + 2 * L::A_BYTES + j * (128 * RG_BK * 2), &tmW, &full_bar[stage], 0,
                                ((mt0 + j) * total_kb + i) * 128);
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        }
    } else if (warp >= 4) {
        // ===== MMA: warpgroup `half` multiplies token rows [64 half, 64 half + 64) x all BN features =====================
        const int q = warp & 3;
        const int half = (warp - 4) >> 2;
        float acc[BN / 2];
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
        int stage = 0, phase = 0, prev = -1;
        for (int i = 0; i < total_kb; ++i) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t a_addr = smem_u32(smem + stage * L::STAGE_BYTES) + half * 64 * 128;
            const uint32_t b_addr = smem_u32(smem + stage * L::STAGE_BYTES + 2 * L::A_BYTES);
            wg_fence();
            wg_mma_kblock<BN>(acc, a_addr, b_addr);
            wg_mma_kblock<BN>(acc, a_addr + L::A_BYTES, b_addr);
            wg_commit();
            wg_wait1();                                     // k-block i-1's MMAs are complete, i's may still run
            __syncwarp();
            if (lane == 0 && prev >= 0) mbar_arrive(&empty_bar[prev]);   // this warp's MMAs have read that slot
            prev = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        wg_wait0();
        wg_acc_fence(acc);
        // stage the accumulators in shared memory once BOTH warpgroups are done reading the pipeline slots
        float* sacc = reinterpret_cast<float*>(smem);
        asm volatile("bar.sync 1, %0;" ::"n"(32 * RG_EPI_WARPS) : "memory");
        {
            const int r = half * 64 + q * 16 + (lane >> 2);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int c = 8 * j + 2 * (lane & 3);
                *reinterpret_cast<float2*>(sacc + r * L::ACC_LD + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
                *reinterpret_cast<float2*>(sacc + (r + 8) * L::ACC_LD + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
            }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(32 * RG_EPI_WARPS) : "memory");
        // ===== epilogue: one token row per thread, 32 consecutive features per step =====================================
        const int row = r0 + q * 32 + lane;
        pdl_wait();                                         // residual rows / KV positions come from earlier kernels
        const float* arow = sacc + (q * 32 + lane) * L::ACC_LD;
        float kv_amax = 0.f;
        int kv_head = -1;
#pragma unroll 1
        for (int c = half * (BN / 2); c < (half + 1) * (BN / 2); c += 32) {
            float v[32];
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
                const float4 t = *reinterpret_cast<const float4*>(arow + c + j);
                v[j] = t.x; v[j + 1] = t.y; v[j + 2] = t.z; v[j + 3] = t.w;
            }
            if (row < rows && n0 + c < Nout) rows_epilogue32(ep, row, n0 + c, v, arow + c, kv_amax, kv_head);
        }
    }
}

template <int BN, int STAGES>
static int launch_rows(const RowsGemmCall& g, cudaStream_t st) {
    using L = RowsSmem<BN, STAGES>;
    static bool attr_set = false;
    if (!attr_set) {
        VCB_CUDA_OK(cudaFuncSetAttribute(gemm_rows_kernel<BN, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
        attr_set = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((g.Nout + BN - 1) / BN, (g.rows + RG_BM - 1) / RG_BM, 1);
    cfg.blockDim = dim3(RG_THREADS);
    cfg.dynamicSmemBytes = L::TOTAL;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = g.pdl ? 1 : 0;
    VCB_CUDA_OK(cudaLaunchKernelEx(&cfg, gemm_rows_kernel<BN, STAGES>, *g.tmX, *g.tmW, g.ep, g.rows, g.rcap, g.Nout,
                                   g.Kdim / RG_BK));
    return 0;
}

// Shapes this kernel takes: K a multiple of 64, Nout a multiple of 128 (whole weight blocks), hd a multiple of 32 for
// the QKV epilogue, rcap (rows per plane) a multiple of 128.
bool gemm_rows_supported(int Nout, int Kdim, int hd) {
    return Kdim % RG_BK == 0 && Nout % 128 == 0 && (hd == 0 || hd % 32 == 0);
}

int gemm_rows_launch(const RowsGemmCall& g, cudaStream_t st) {
    if (!gemm_rows_supported(g.Nout, g.Kdim, g.ep.mode == EPI_QKV ? g.ep.hd : 0) || g.rcap % RG_BM || g.rows < 1 ||
        g.rows > g.rcap) {
        set_error("gemm_rows: unsupported shape N=%d K=%d rows=%d rcap=%d", g.Nout, g.Kdim, g.rows, g.rcap);
        return -1;
    }
    // 256-feature tiles halve the activation re-reads; an odd number of 128-feature blocks runs 128-wide tiles
    if ((g.Nout / 128) % 2 == 0) return launch_rows<256, 3>(g, st);
    return launch_rows<128, 4>(g, st);
}

}  // namespace vcb
