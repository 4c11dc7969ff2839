// Weight-streaming GEMM of the codec-LM with cluster split-K and fused epilogues.
//
//   out[j][m] = epilogue( sum_k W[m,k] * (Xhi[j,k] + Xlo[j,k]) + bias[m] )        j = token row, m = output feature
//
//   A operand = weight matrix W [Nout, Kdim] bf16, PRE-TILED in HBM: tile (mt, kb) = W[mt*128.., kb*64..] is one
//               contiguous 16 KB block [128 rows][64 cols] at block index mt*KB + kb (pack_weight_tiles), so every
//               TMA box is a single sequential DRAM burst (a row-major matrix would scatter a box over 128 DRAM
//               pages).  TMA SWIZZLE_128B into smem.
//   B operand = activations  X [2*Bpad, Kdim] bf16: rows [0,Bpad) = hi parts, rows [Bpad,2*Bpad) = lo parts
//               (x ~= hi + lo, see split_bf16): one MMA of N = 2*Bpad columns covers both; this regime is HBM-bound,
//               so the tensor cores have the room, and the second half buys ~16 mantissa bits.
//   D         = fp32 accumulators in registers (wgmma): 128 output features x 2*Bpad columns per CTA, 64 features per
//               warpgroup issue (one warpgroup covers both 64-feature halves when Bpad <= 32)
//
// Split-K without a workspace: the S CTAs of a thread-block cluster each stream one K slice of the same 128-feature
// weight tile (so >=128 CTAs pull HBM even for a 2048 x 2048 matrix), then reduce-scatter their accumulators
// through distributed shared memory: CTA z owns token rows [z*R, (z+1)*R), every CTA writes its partial of those
// rows into the owner's smem with asynchronous stores that count their bytes on the owner's mbarrier (st.async ...
// mbarrier::complete_tx): the owner waits on its own barrier -- no cluster barrier after the start-up one -- then sums
// the S partials in fixed order (deterministic) and applies the fused epilogue:
//     EPI_QKV    q -> fp32 buffer, k/v -> appended to the paged KV cache    (activation.py:86-88, 626-631)
//     EPI_RESID  x += y + bias                                            (transformer.py:321-329)
//     EPI_ACT    ReLU / exact GELU -> bf16 hi/lo rows of the next GEMM      (transformer.py:387, voicecraft.py:183)
//     EPI_LOGITS fp32 logits                                              (voicecraft.py:1085)
// Warp roles: w0 TMA producer, w1..w3 idle (the MMA warpgroups must start on a warpgroup boundary), w4..w7 MMA +
// epilogue (plus w8..w11 for tiles with >= 64 token rows).  Prompt batches use the rows-as-M kernel in gemm_rows.cu instead.
#include "vcb_internal.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>

namespace vcb {

static constexpr int GEMM_BM = 128;   // output features per CTA (2 x wgmma M)
static constexpr int GEMM_BK = 64;    // K elements per pipeline stage (= 128 B of bf16 = one swizzle row)
static constexpr int GEMM_MAX_SPLITS = 16;   // cluster size = K splits
// threads per CTA: warpgroup 0 (w0 TMA), then one MMA + epilogue warpgroup; tiles with >= 64 token rows get a second one:
// each then multiplies 64 of the 128 features (accumulators: Bpad registers per thread) and takes half of the rows in
// the epilogue (the epilogue, not the weight stream, dominates those launches)
constexpr int gemm_epi_warps(int bn) { return bn >= 128 ? 8 : 4; }
constexpr int gemm_threads(int bn) { return 128 + 32 * gemm_epi_warps(bn); }

// W8: the stage holds one 128-k int8 weight tile (the same 16 KB) and the two 64-k activation boxes it multiplies
template <int BN, int STAGES, bool W8 = false>
struct GemmSmem {
    static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;
    static constexpr int B_BYTES = BN * GEMM_BK * 2 * (W8 ? 2 : 1);
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int RED_OFFSET = STAGES * STAGE_BYTES;
    static constexpr int RED_BYTES = (BN / 2) * GEMM_BM * 4;          // [S][R][128] fp32 with S*R = Bpad
    static constexpr int BAR_OFFSET = RED_OFFSET + RED_BYTES;
    static constexpr int TOTAL = BAR_OFFSET + (2 * STAGES + 1) * 8;           // full[S] empty[S] red_full
};

// Pipeline stages for `bpad` token rows: 4 (64 KB of weight tiles in flight per CTA), fewer only where 4 do not fit into
// the 227 KB of shared memory a block may opt in to on sm_90 (bpad 128: 3).  Measured on the H100 (DESIGN.md section
// 4.1): at bpad 32 deeper pipelines (6, 8) allow one CTA per SM instead of two and gain nothing once the split count
// follows that; at bpad 64, 4 stages beat 3 on every decode shape.
constexpr int gemm_stages(int bpad) {
    int s = 4;
    while (s > 2 && s * (GEMM_BM + 2 * bpad) * GEMM_BK * 2 + bpad * GEMM_BM * 4 + (2 * s + 1) * 8 > 227 * 1024) --s;
    return s;
}
static_assert(GemmSmem<64, gemm_stages(32)>::TOTAL <= 227 * 1024 && GemmSmem<256, gemm_stages(128)>::TOTAL <= 227 * 1024,
              "gemm_stages and GemmSmem disagree on the shared memory footprint");
// Int8 weights (W8): a stage carries twice the activation bytes.  The most stages (<= 4) that still fit and keep as many
// CTAs per SM as the bf16 kernel for `bpad`, whose occupancy chose the split count: bpad 16: 4, 32: 3, 64: 4, 128: 2.
constexpr int gemm_smem_bytes(int bpad, int s, bool w8) {
    return s * (GEMM_BM * GEMM_BK * 2 + (w8 ? 2 : 1) * 2 * bpad * GEMM_BK * 2) + bpad * GEMM_BM * 4 + (2 * s + 1) * 8;
}
constexpr int gemm_ctas_per_sm(int bytes) { return (228 * 1024) / (bytes + 1024); }
constexpr int gemm_stages_w8(int bpad) {
    int s = 4;
    while (s > 2 && (gemm_smem_bytes(bpad, s, true) > 227 * 1024 ||
                     gemm_ctas_per_sm(gemm_smem_bytes(bpad, s, true)) < gemm_ctas_per_sm(gemm_smem_bytes(bpad, gemm_stages(bpad), false))))
        --s;
    return s;
}
static_assert(GemmSmem<256, gemm_stages_w8(128), true>::TOTAL == gemm_smem_bytes(128, gemm_stages_w8(128), true) &&
              GemmSmem<256, gemm_stages_w8(128), true>::TOTAL <= 227 * 1024,
              "gemm_stages_w8 and GemmSmem disagree on the shared memory footprint");

// Int8 weight tiles (W8).  Tile (mt, cb) = rows mt*128.., k cb*128.. is one contiguous 16 KB block [128 rows][128 bytes] at
// block index mt*(K/128) + cb, one TMA box with SWIZZLE_128B.  Inside a row the k order is permuted so that thread t of a
// quad finds every A fragment value it needs for the tile's eight k16 steps in the 32 bytes [32t, 32t+32): byte 32t + 4s + j
// holds k = 16s + 2t + (j & 1) + 8 (j >> 1) -- the wgmma register fragment of A (rows g, g+8; k 2t, 2t+1, 2t+8, 2t+9) -- so
// each row costs a thread two 16-byte shared loads per tile, and the swizzle keeps a quarter warp's loads on distinct banks.
__host__ __device__ inline size_t w8_index(int m, int k, int Kdim) {
    const int kc = k % 128, s = kc / 16, w = kc % 16;
    const int pos = 32 * ((w & 7) >> 1) + 4 * s + (w & 1) + 2 * (w >> 3);
    return ((static_cast<size_t>(m / GEMM_BM) * (Kdim / 128) + k / 128) * GEMM_BM + (m % GEMM_BM)) * 128 + pos;
}

// 4 int8 (k 2t, 2t+1, 2t+8, 2t+9) -> two bf16x2 A-fragment registers, exactly: byte u = q + 128 becomes the fp32 2^23 + u,
// minus 2^23 + 128 gives q, whose upper 16 bits are q as a bf16 (|q| <= 128 has at most 8 significant bits)
__device__ __forceinline__ void w8_to_bf16x2(uint32_t w, uint32_t& lo, uint32_t& hi) {
    const uint32_t u = w ^ 0x80808080u;
    float f[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) f[j] = __uint_as_float(__byte_perm(u, 0x4B000000u, 0x7540 + j)) - 8388736.f;
    lo = __byte_perm(__float_as_uint(f[0]), __float_as_uint(f[1]), 0x7632);
    hi = __byte_perm(__float_as_uint(f[2]), __float_as_uint(f[3]), 0x7632);
}

// A fragments of the eight k16 steps of one 64-row block of an int8 tile in shared memory (SWIZZLE_128B: 16-byte chunk c of
// row r sits at chunk c ^ (r & 7)), for the thread at rows r, r + 8 and quad position t
__device__ __forceinline__ void w8_frags(const uint8_t* tile, int r, int t, uint32_t (&f)[8][4]) {
#pragma unroll
    for (int p = 0; p < 2; ++p) {
        const int row = r + 8 * p;
        const uint8_t* base = tile + row * 128;
        const uint4 a = *reinterpret_cast<const uint4*>(base + (((2 * t) ^ (row & 7)) << 4));
        const uint4 b = *reinterpret_cast<const uint4*>(base + (((2 * t + 1) ^ (row & 7)) << 4));
        const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
        for (int s = 0; s < 8; ++s) w8_to_bf16x2(w[s], f[s][p], f[s][2 + p]);
    }
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t cluster_nctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_smem_addr, uint32_t cta) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local_smem_addr), "r"(cta));
    return remote;
}
// Asynchronous store into a peer CTA's shared memory that counts its bytes on the peer's mbarrier: the owner of the
// rows learns that every partial has landed from its own barrier -- no cluster-wide barrier (and no GPU-scope
// membar, which is what barrier.cluster.arrive.release costs) between the accumulators and the epilogue.
__device__ __forceinline__ void st_async_f32x2(uint32_t remote_addr, uint32_t remote_bar, float a, float b) {
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];" ::"r"(remote_addr),
                 "f"(a), "f"(b), "r"(remote_bar)
                 : "memory");
}
// bounded wait: a byte-count mismatch would otherwise hang the GPU; ~1 s of polling, then trap (surfaces as a CUDA error)
__device__ __forceinline__ void mbar_wait_bounded(uint64_t* bar, uint32_t parity) {
    for (unsigned int spins = 0; !mbar_try_wait(bar, parity); ++spins)
        if (spins > (1u << 26)) __trap();
}

// Fused epilogue for up to 4 token rows of one output feature m.  All loads of the group are issued before the first
// dependent use (the per-row chains position -> page -> address would otherwise serialise on L2 latency).
__device__ __forceinline__ void apply_epilogue4(const GemmEpilogue& ep, int row0, int nrows, int m, const float (&sum)[4],
                                                float bias, float (&xnew)[4], int colx = 0, const float* xpre = nullptr) {
    switch (ep.mode) {
        case EPI_QKV: {
            int pos[4], slot[4], page[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                pos[u] = (u < nrows) ? ep.row_pos[row0 + u] : -1;
                slot[u] = (u < nrows && !ep.row_page) ? ep.row_slot[row0 + u] : 0;
                page[u] = (u < nrows && ep.row_page) ? ep.row_page[row0 + u] : 0;      // same batch of loads as pos
            }
            const int part = m / ep.d, cc = m - part * ep.d;
            if (part == 0) {
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (pos[u] >= 0) ep.qbuf[static_cast<size_t>(row0 + u) * ep.d + cc] = sum[u] + bias;
                return;
            }
            if (!ep.row_page) {         // (precomputed by step_prep / prefill otherwise: one L2 round trip instead of two)
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    page[u] = (pos[u] >= 0) ? ep.page_table[slot[u] * ep.max_pages + pos[u] / ep.page_size] : 0;
            }
            const int h = cc / ep.hd, e = cc - h * ep.hd;
            void* pool = (part == 1) ? ep.kpool : ep.vpool;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (pos[u] < 0) continue;
                const size_t off = ((static_cast<size_t>(page[u]) * ep.H + h) * ep.page_size + pos[u] % ep.page_size) * ep.hd + e;
                const float val = sum[u] + bias;
                if (ep.kv_fp32) static_cast<float*>(pool)[off] = val;
                else static_cast<__nv_bfloat16*>(pool)[off] = __float2bfloat16_rn(val);
            }
            break;
        }
        case EPI_RESID: {
            float xv[4];
#pragma unroll
            for (int u = 0; u < 4; ++u)
                xv[u] = xpre ? xpre[u] : ((u < nrows) ? ep.x[static_cast<size_t>(row0 + u) * ep.ld_out + m] : 0.f);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                xnew[u] = xv[u] + (sum[u] + bias);
                if (u < nrows) ep.x[static_cast<size_t>(row0 + u) * ep.ld_out + m] = xnew[u];
            }
            break;
        }
        case EPI_ACT: {
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (u >= nrows) continue;
                float v = sum[u] + bias;
                if (ep.act_kind == 1) v = fmaxf(v, 0.f);
                else if (ep.act_kind == 2) v = 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
                __nv_bfloat16 hi, lo;
                split_bf16(v, hi, lo);
                ep.act[static_cast<size_t>(row0 + u) * ep.ld_out + m] = hi;
                ep.act[static_cast<size_t>(row0 + u + ep.bpad_out) * ep.ld_out + m] = lo;
            }
            break;
        }
        default:
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (u < nrows) ep.out[static_cast<size_t>(row0 + u) * ep.ld_out + ep.col_off + colx + m] = sum[u] + bias;
    }
}

// KV8: the QKV launch of an fp8-KV engine (its own instantiation, so the other epilogues keep their register budget)
// W8: int8 weight tiles (w8_index) with a power-of-two scale per feature (wscale, or grp.wscale per group).  The K slices are
// the bf16 kernel's (total_kb / kb_per_split count 64-k blocks); a stage holds a 128-k tile, and a slice that begins or ends
// halfway through one skips that half's k16 steps.  The MMA warps convert each tile to bf16 A fragments in registers and issue
// the bf16 kernel's wgmmas in its k16 order; the fixed-order sum of the partials is multiplied by 2^e before the epilogue.
template <int BN, int STAGES, bool KV8 = false, bool W8 = false>
__global__ void __launch_bounds__(gemm_threads(BN))
gemm_w_xT_cluster(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const GemmEpilogue ep, int Nout, int total_kb, int kb_per_split, int b_col_off, int nvalid,
                  const void* pf_ptr, unsigned long long pf_bytes, const GemmGroup grp, const float* wscale) {
    using L = GemmSmem<BN, STAGES, W8>;
    constexpr int BPAD = BN / 2;
    constexpr int HALVES = gemm_epi_warps(BN) / 4;          // MMA + epilogue warpgroups
    constexpr int MH = 2 / HALVES;                          // 64-feature halves multiplied by each warpgroup
    constexpr int EPI_THREADS = 32 * gemm_epi_warps(BN);
    extern __shared__ __align__(1024) uint8_t smem[];       // SWIZZLE_128B tiles need 1024-byte alignment
    float* red = reinterpret_cast<float*>(smem + L::RED_OFFSET);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* red_full = empty_bar + STAGES;                // all S partials of my R rows have landed in `red`

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int S = static_cast<int>(cluster_nctarank());      // K splits = cluster size
    const int z = static_cast<int>(cluster_ctarank());
    const int mt = blockIdx.x / S;                          // 128-feature tile
    const int m0 = mt * GEMM_BM;
    // grouped launch (blockIdx.y = group): same shapes, per-group weight map / bias / column offsets (the K logit heads)
    const int grp_i = blockIdx.y;
    const CUtensorMap* pA = grp.tmA ? grp.tmA + grp_i : &tmA;
    b_col_off += grp_i * grp.b_stride;
    const int colx = grp_i * grp.col_stride;
    const int kb0 = z * kb_per_split;
    const int nkb = max(0, min(kb_per_split, total_kb - kb0));
    // pipeline items: 64-k blocks, or (W8) the 128-k tiles t0 .. t0 + nst - 1 that hold 64-k blocks kb0 .. kb0 + nkb - 1
    const int t0 = W8 ? kb0 / 2 : kb0;
    const int nst = W8 ? (nkb > 0 ? (kb0 + nkb - 1) / 2 - t0 + 1 : 0) : nkb;
    const int a_blocks = W8 ? total_kb / 2 : total_kb;      // weight tiles per 128-feature row of tiles
    const int pre = min(nst, STAGES);

    pdl_launch_dependents();        // dependents may be scheduled now; their griddepcontrol.wait still orders the data
    if (threadIdx.x == 0) { tl_mark(0x100 + ep.mode); tl_mark_all(0x100 + ep.mode); }
    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(pA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], gemm_epi_warps(BN));  // one arrival per MMA warp
        }
        mbar_init(red_full, 1);
        mbar_fence_init();
        // every CTA of the cluster sends all of my R rows x 128 features (fp32), armed before anyone can send
        mbar_arrive_expect_tx(red_full, static_cast<uint32_t>(BPAD) * GEMM_BM * 4);
        // Weights never depend on the previous kernel: their first STAGES tiles go in flight right away
        // (under PDL: while the producer grid is still draining); activations wait for griddepcontrol.wait.
        const uint64_t pol = l2_policy_evict_first();      // weight tiles are read once per step
        for (int i = 0; i < pre; ++i) {
            mbar_arrive_expect_tx(&full_bar[i], L::STAGE_BYTES);
            tma_load_2d_hint(smem + i * L::STAGE_BYTES, pA, &full_bar[i], 0, (mt * a_blocks + t0 + i) * GEMM_BM, pol);
        }
        // keep HBM busy across the kernel boundary: pull the NEXT GEMM's weights into L2 while this one runs
        // (bit 63 of pf_bytes: issue it after this CTA's last weight load instead -- HBM idles during the epilogue)
        if (!(pf_bytes >> 63)) prefetch_l2_slice(pf_ptr, pf_bytes, blockIdx.x, gridDim.x);
    }
    cluster_sync_all();             // CTA-wide sync + "every CTA of the cluster has started and armed its barrier"
    // per-feature epilogue constants (bias / LN-fold vector / next gamma) are model weights, never written by a kernel:
    // the epilogue warps fetch them while the mainloop runs, off the critical tail
    float w_bias = 0.f, w_cv = 0.f, w_gnext = 0.f;
    float e_mean = 0.f, e_rstd = 0.f;                       // LayerNorm statistics of row z*R + lane (BPAD <= 32, see below)
    float e_x[4] = {0.f, 0.f, 0.f, 0.f};                    // residual rows fetched early (R == 4)
    bool e_x_valid = false;
    if (warp >= 4) {
        const int m = m0 + (warp & 3) * 32 + lane;
        if (m < Nout) {
            const float* bias_ptr = grp.bias ? grp.bias[grp_i] : ep.bias;
            w_bias = bias_ptr[m];
            if (ep.ln_fold) w_cv = ep.cvec[m];
            if (ep.emit) w_gnext = ep.next_gamma[m];
        }
    }
    float w_scale = 1.f;                                    // W8: 2^e of the feature
    if constexpr (W8) {
        const int m = m0 + (warp & 3) * 32 + lane;
        if (warp >= 4 && m < Nout) w_scale = (grp.wscale ? grp.wscale[grp_i] : wscale)[m];
    }

    if (warp == 0) {
        // ===== TMA producer ==========================================================================
        if (lane == 0) {
            pdl_wait();
            tl_mark(0x110 + ep.mode);
            tl_mark_all(0x110 + ep.mode);
            for (int i = 0; i < pre; ++i) {
                if constexpr (W8) {
                    uint8_t* b = smem + i * L::STAGE_BYTES + L::A_BYTES;
                    tma_load_2d(b, &tmB, &full_bar[i], b_col_off + (t0 + i) * 2 * GEMM_BK, 0);
                    tma_load_2d(b + L::B_BYTES / 2, &tmB, &full_bar[i], b_col_off + ((t0 + i) * 2 + 1) * GEMM_BK, 0);
                } else {
                    tma_load_2d(smem + i * L::STAGE_BYTES + L::A_BYTES, &tmB, &full_bar[i],
                                b_col_off + (kb0 + i) * GEMM_BK, 0);
                }
            }
            int stage = 0, phase = 0;                       // state after the first `pre` fills
            const uint64_t pol = l2_policy_evict_first();
            for (int i = pre; i < nst; ++i) {
                mbar_wait(&empty_bar[stage], phase);        // the MMA released this slot
                mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
                uint8_t* a = smem + stage * L::STAGE_BYTES;
                tma_load_2d_hint(a, pA, &full_bar[stage], 0, (mt * a_blocks + t0 + i) * GEMM_BM, pol);
                if constexpr (W8) {
                    tma_load_2d(a + L::A_BYTES, &tmB, &full_bar[stage], b_col_off + (t0 + i) * 2 * GEMM_BK, 0);
                    tma_load_2d(a + L::A_BYTES + L::B_BYTES / 2, &tmB, &full_bar[stage],
                                b_col_off + ((t0 + i) * 2 + 1) * GEMM_BK, 0);
                } else {
                    tma_load_2d(a + L::A_BYTES, &tmB, &full_bar[stage], b_col_off + (kb0 + i) * GEMM_BK, 0);
                }
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            if (pf_bytes >> 63) prefetch_l2_slice(pf_ptr, pf_bytes & ~(1ull << 63), blockIdx.x, gridDim.x);
        }
    } else if (warp >= 4) {
        // ===== MMA mainloop, then reduce-scatter of the accumulators over the cluster (DSMEM) ==========
        const int q = warp & 3;                             // warp inside its warpgroup
        const int half = (warp - 4) >> 2;                   // which warpgroup (0 unless HALVES == 2)
        const int ml = q * 32 + lane;                       // feature inside the tile (epilogue part 2 layout)
        const int R = BPAD / S;                             // token rows owned by each CTA (power of two)
        const int shR = 31 - __clz(R);
        // While the mainloop runs: everything the epilogue needs from EARLIER kernels.  With a folded LayerNorm that is the
        // mean / rstd of my R rows, from the per-tile partial sums the producer kernel left (fixed tile order): lane r of every
        // warp computes row r (R <= 32 here) and the row groups below fetch it with a shuffle -- no shared memory (the scratch
        // area aliases a pipeline stage that is still in use now), no barrier, and the L2 round trip is off the critical tail.
        if constexpr (BPAD <= 32) {
            pdl_wait();
            if (ep.ln_fold && lane < R) {
                const int row = z * R + lane;
                if (row < nvalid) ln_row_stats(ep.stats, ep.stats_tiles, ep.ln_d, row, ep.inv_d, ep.ln_eps, e_mean, e_rstd);
            }
            // ... and, when this CTA owns a single group of 4 rows (the out-projection and FFN2 at B = 32: R = 4), the
            // residual rows it is going to update
            if (ep.mode == EPI_RESID && R == 4 && m0 + ml < Nout) {
                const int row0 = z * 4;
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    e_x[u] = (row0 + u < nvalid) ? ep.x[static_cast<size_t>(row0 + u) * ep.ld_out + m0 + ml] : 0.f;
                e_x_valid = true;
            }
        }
        // mainloop: this warpgroup's MH x 64 features x BN columns, every k-block of my K slice
        float acc[MH][BN / 2];
#pragma unroll
        for (int h = 0; h < MH; ++h)
#pragma unroll
            for (int j = 0; j < BN / 2; ++j) acc[h][j] = 0.f;
        if constexpr (W8) {
            // per tile: every thread converts its A fragments, the warpgroup issues the tile's k16 steps that lie in the slice,
            // and waits for them (the fragment registers are rewritten for the next tile) before releasing the slot
            int stage = 0, phase = 0;
            for (int i = 0; i < nst; ++i) {
                mbar_wait(&full_bar[stage], phase);
                const uint8_t* tile = smem + stage * L::STAGE_BYTES;
                const uint32_t b_addr = smem_u32(tile + L::A_BYTES);
                const int c0 = (t0 + i) * 8;                // first k16 step of the tile
                const int klo = max(kb0 * 4 - c0, 0), khi = min((kb0 + nkb) * 4 - c0, 8);
                uint32_t fa[MH][8][4];
#pragma unroll
                for (int h = 0; h < MH; ++h) w8_frags(tile, (half * MH + h) * 64 + q * 16 + (lane >> 2), lane & 3, fa[h]);
                wg_fence();
#pragma unroll
                for (int s = 0; s < 8; ++s) {
                    if (s < klo || s >= khi) continue;      // (uniform over the warpgroup)
#pragma unroll
                    for (int h = 0; h < MH; ++h) wg_mma_k16_ra<BN>(acc[h], fa[h][s], b_addr + (s >> 2) * (L::B_BYTES / 2), s & 3);
                }
                wg_commit();
                wg_wait0();
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[stage]);
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        } else {
            int stage = 0, phase = 0, prev = -1;
            for (int i = 0; i < nkb; ++i) {
                mbar_wait(&full_bar[stage], phase);
                const uint32_t a_addr = smem_u32(smem + stage * L::STAGE_BYTES);
                wg_fence();
#pragma unroll
                for (int h = 0; h < MH; ++h)
                    wg_mma_kblock<BN>(acc[h], a_addr + (half * MH + h) * 64 * 128, a_addr + L::A_BYTES);
                wg_commit();
                wg_wait1();                                 // k-block i-1's MMAs are complete, i's may still run
                __syncwarp();
                if (lane == 0 && prev >= 0) mbar_arrive(&empty_bar[prev]);   // this warp's MMAs have read that slot
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            wg_wait0();
            __syncwarp();
            if (lane == 0 && prev >= 0) mbar_arrive(&empty_bar[prev]);
        }
#pragma unroll
        for (int h = 0; h < MH; ++h) wg_acc_fence(acc[h]);
        if (threadIdx.x == 128) tl_mark(0x120 + ep.mode);
        const uint32_t red_addr = smem_u32(red);
        const uint32_t bar_addr = smem_u32(red_full);
        // red layout in the owner: [writer z][feature][R rows].  A thread holds two features (f, f + 8) x pairs of adjacent
        // token rows (8-byte stores; R >= 2 keeps a pair inside one owner).  All Bpad rows are sent, valid or not: the byte
        // count is a constant.
#pragma unroll
        for (int h = 0; h < MH; ++h) {
#pragma unroll
            for (int jb = 0; jb < BPAD / 8; ++jb) {
                const int row = 8 * jb + 2 * (lane & 3);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int f = (half * MH + h) * 64 + q * 16 + (lane >> 2) + 8 * e;
                    const float s0 = acc[h][4 * jb + 2 * e] + acc[h][4 * (jb + BPAD / 8) + 2 * e];
                    const float s1 = acc[h][4 * jb + 2 * e + 1] + acc[h][4 * (jb + BPAD / 8) + 2 * e + 1];
                    if (S == 1) {
                        // no split: the partials stay in this CTA -- plain shared stores, handed over by a named barrier
                        // (a 1-CTA cluster has no peer to st.async to)
                        *reinterpret_cast<float2*>(red + (static_cast<size_t>(f) << shR) + row) = make_float2(s0, s1);
                    } else {
                        const int owner = row >> shR, rr = row & (R - 1);
                        const uint32_t off = static_cast<uint32_t>((((z << 7) + f) << shR) + rr) << 2;
                        st_async_f32x2(mapa_u32(red_addr + off, owner), mapa_u32(bar_addr, owner), s0, s1);
                    }
                }
            }
        }
        if (threadIdx.x == 128) tl_mark(0x140 + ep.mode);
    }
    if (warp >= 4) {
        if (S == 1) asm volatile("bar.sync 4, %0;" ::"n"(EPI_THREADS) : "memory");   // every epilogue thread stored its partials
        else mbar_wait_bounded(red_full, 0);                // all S partials of my rows have landed (async stores counted)
        if (threadIdx.x == 128) tl_mark(0x150 + ep.mode);
        // ===== epilogue part 2: fixed-order sum of the S partials of my R rows + fused epilogue =======
        // scratch aliases pipeline stage 0: every TMA write / MMA read of this CTA's stages has retired (both warpgroups
        // sent their partials after their last wgmma completed), and peers only ever write into `red`.  (Static __shared__ here would cost the second resident CTA per SM.)
        float* s_mean = reinterpret_cast<float*>(smem);
        float* s_rstd = s_mean + GEMM_BM;
        float (*s_part_all)[4][4][2] = reinterpret_cast<float (*)[4][4][2]>(s_rstd + GEMM_BM);
        const int q = warp & 3;
        const int half = (warp - 4) >> 2;
        float (*s_part)[4][2] = s_part_all[half];
        const int ml = q * 32 + lane;
        const int et = static_cast<int>(threadIdx.x) - 128; // index among the epilogue threads
        const int m = m0 + ml;
        const int R = BPAD / S;
        const bool valid_m = m < Nout;
        pdl_wait();                                         // x / stats of earlier kernels are read below
        if (BPAD > 32 && ep.ln_fold) {
            // mean / rstd of my rows from the per-tile partial sums the producer kernel left (fixed tile order)
            for (int rr = et; rr < R; rr += EPI_THREADS) {
                const int row = z * R + rr;
                float mean = 0.f, rstd = 0.f;
                if (row < nvalid) {
                    // 16 tiles = one batch of independent 8-byte loads (a single L2 round trip), summed in tile order
                    ln_row_stats(ep.stats, ep.stats_tiles, ep.ln_d, row, ep.inv_d, ep.ln_eps, mean, rstd);
                }
                s_mean[rr] = mean;
                s_rstd[rr] = rstd;
            }
            asm volatile("bar.sync 4, %0;" ::"n"(EPI_THREADS) : "memory");
        }
        const float bias = w_bias, cv = w_cv, gnext = w_gnext;
        // the two warp sets (if any) alternate over the groups of 4 rows; each has its own named barrier (2 + half),
        // so they may run a different number of groups
        for (int rr0 = 4 * half; rr0 < R; rr0 += 4 * HALVES) {
            const int row0 = z * R + rr0;
            const int nrows = min(min(4, R - rr0), nvalid - row0);
            if (nrows <= 0) break;
            float sum[4], xnew[4] = {0.f, 0.f, 0.f, 0.f};
            // the S partials of rows rr0 .. rr0 + 3, summed in writer order.  With R >= 4 the four rows are one 16-byte
            // word per writer (R and rr0 are multiples of 4): one conflict-free vector load instead of four loads at a
            // stride of R words, which conflict 4- to 16-way.  Rows past nrows were sent too; they stay 0 as before.
            float part[4] = {0.f, 0.f, 0.f, 0.f};
            if (R >= 4) {
                for (int zz = 0; zz < S; ++zz) {
                    const float4 v = *reinterpret_cast<const float4*>(red + (zz * GEMM_BM + ml) * R + rr0);
                    part[0] += v.x;
                    part[1] += v.y;
                    part[2] += v.z;
                    part[3] += v.w;
                }
            } else {
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (u < nrows)
                        for (int zz = 0; zz < S; ++zz) part[u] += red[(zz * GEMM_BM + ml) * R + rr0 + u];
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                float a = u < nrows ? part[u] : 0.f;
                if constexpr (W8) a *= w_scale;             // exact: a power of two
                if (ep.ln_fold) {
                    float mean, rstd;
                    if constexpr (BPAD <= 32) {             // (uniform: every lane of the warp takes part in the shuffle)
                        mean = __shfl_sync(0xffffffffu, e_mean, (rr0 + u) & 31);
                        rstd = __shfl_sync(0xffffffffu, e_rstd, (rr0 + u) & 31);
                    } else {
                        mean = s_mean[(rr0 + u) & (R - 1)];
                        rstd = s_rstd[(rr0 + u) & (R - 1)];
                    }
                    if (u < nrows) a = rstd * (a - mean * cv);
                }
                sum[u] = a;
            }
            if (KV8 && m0 + GEMM_BM > ep.d) {
                // fp8 K / V (a tile of K or V features, or one that straddles Q|K): each row's amax over a head is a warp
                // max combined through shared memory behind the half's barrier, over the hd / 32 warps of the head
                // (heads are 64-aligned, so a head never crosses a warp pair); s_part is free, QKV tiles do not emit
                float val[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    val[u] = sum[u] + bias;
                    const float am = warp_max(u < nrows ? fabsf(val[u]) : 0.f);
                    if (lane == 0) s_part[q][u][0] = am;
                }
                if (half == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
                else asm volatile("bar.sync 3, 128;" ::: "memory");
                const int wph = ep.hd / 32, w0 = q & ~(wph - 1);
                float amax[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    amax[u] = s_part[w0][u][0];
                    for (int w = 1; w < wph; ++w) amax[u] = fmaxf(amax[u], s_part[w0 + w][u][0]);
                }
                if (half == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
                else asm volatile("bar.sync 3, 128;" ::: "memory");
                if (valid_m && m < ep.d) {
                    apply_epilogue4(ep, row0, nrows, m, sum, bias, xnew);
                } else if (valid_m) {
                    const int part = m / ep.d, cc = m - part * ep.d, h = cc / ep.hd, e = cc - h * ep.hd;
                    uint8_t* pool = static_cast<uint8_t*>(part == 1 ? ep.kpool : ep.vpool);
                    const int slab = kv_slab_bytes(KV_FP8, ep.hd);
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int pos = u < nrows ? ep.row_pos[row0 + u] : -1;
                        if (pos < 0) continue;
                        const int page = ep.row_page ? ep.row_page[row0 + u]
                                                     : ep.page_table[ep.row_slot[row0 + u] * ep.max_pages + pos / ep.page_size];
                        const int t = pos % ep.page_size;
                        uint8_t* s = pool + (static_cast<size_t>(page) * ep.H + h) * slab;
                        float inv;
                        const float scale = kv_fp8_scale(amax[u], inv);
                        s[t * ep.hd + e] = static_cast<uint8_t>(kv_fp8_pack2(val[u], 0.f, inv) & 0xff);
                        if (e == 0) reinterpret_cast<float*>(s + ep.page_size * ep.hd)[t] = scale;
                    }
                }
            } else if (valid_m) apply_epilogue4(ep, row0, nrows, m, sum, bias, xnew, colx, e_x_valid ? e_x : nullptr);
            if (ep.emit) {
                // next GEMM's operand gamma_next * x_new (hi/lo) and this tile's (sum x, M2 about the tile mean) per row:
                // each warp sums its 32 features, and their powers shifted by one of them (lane 0's, within the row's
                // spread of the others), which gives the warp's M2 without cancellation; the 4 warps combine below
                const int nw = min(32, max(0, Nout - (m0 + q * 32)));      // valid features of this warp
                float p1[4], p2[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const bool ok = valid_m && u < nrows;
                    if (ok) {
                        __nv_bfloat16 hi, lo;
                        split_bf16(gnext * xnew[u], hi, lo);
                        ep.next_act[static_cast<size_t>(row0 + u) * ep.next_ld + m] = hi;
                        ep.next_act[static_cast<size_t>(row0 + u + ep.next_bpad) * ep.next_ld + m] = lo;
                    }
                    const float dv = ok ? xnew[u] - __shfl_sync(0xffffffffu, xnew[u], 0) : 0.f;
                    p1[u] = warp_sum(ok ? xnew[u] : 0.f);
                    const float q1 = warp_sum(dv), q2 = warp_sum(dv * dv);
                    p2[u] = nw > 0 ? fmaxf(q2 - q1 * q1 / static_cast<float>(nw), 0.f) : 0.f;
                }
                if (lane == 0) {
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        s_part[q][u][0] = p1[u];
                        s_part[q][u][1] = p2[u];
                    }
                }
                if (half == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
                else asm volatile("bar.sync 3, 128;" ::: "memory");
                if (ml < 4 && ml < nrows) {
                    const int u = ml;
                    const float sum = s_part[0][u][0] + s_part[1][u][0] + s_part[2][u][0] + s_part[3][u][0];
                    const float tmean = sum / static_cast<float>(min(GEMM_BM, Nout - m0));
                    float m2 = 0.f;
#pragma unroll
                    for (int w = 0; w < 4; ++w) {
                        const int nw = min(32, Nout - (m0 + w * 32));
                        if (nw > 0) m2 += ln_tile_m2(static_cast<float>(nw), s_part[w][u][0], s_part[w][u][1], tmean);
                    }
                    *reinterpret_cast<float2*>(ep.stats_out + (static_cast<size_t>(mt) * STATS_ROWS + row0 + u) * 2) =
                        make_float2(sum, m2);
                }
                if (half == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
                else asm volatile("bar.sync 3, 128;" ::: "memory");
            }
        }
        if (threadIdx.x == 128) tl_mark(0x160 + ep.mode);
    }
    __syncthreads();
    if (threadIdx.x == 0) { tl_mark(0x130 + ep.mode); tl_mark_all(0x130 + ep.mode); }
}

void gemm_timeline_set(unsigned long long* buf, unsigned int* cnt) {
    cudaMemcpyToSymbol(g_tl_buf, &buf, sizeof(buf));
    cudaMemcpyToSymbol(g_tl_cnt, &cnt, sizeof(cnt));
}

// ---------------------------------------------------------------------------------------------------
// Bring-up / cross-check kernel: same contract on CUDA cores (one warp per output feature, no split).
// Selected with VCB_GEMM_IMPL=simt; never the default.  It exists so a wgmma descriptor bug can be told
// apart from a bug anywhere else in the step.
// ---------------------------------------------------------------------------------------------------
// element (m, k) of the pre-tiled weight layout
__host__ __device__ inline size_t packed_index(int m, int k, int Kdim) {
    const int KB = Kdim / GEMM_BK;
    return ((static_cast<size_t>(m / GEMM_BM) * KB + k / GEMM_BK) * GEMM_BM + (m % GEMM_BM)) * GEMM_BK + (k % GEMM_BK);
}

__global__ void gemm_w_xT_simt(const __nv_bfloat16* __restrict__ W, const __nv_bfloat16* __restrict__ X,
                               const GemmEpilogue ep, int Nout, int Kdim, int ldx, int bpad, int b_col_off, int nvalid) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= Nout) return;
    for (int j = 0; j < nvalid; ++j) {
        float acc = 0.f;
        for (int k = lane; k < Kdim; k += 32) {
            const float w = __bfloat162float(W[packed_index(warp, k, Kdim)]);
            const float xh = __bfloat162float(X[static_cast<size_t>(j) * ldx + b_col_off + k]);
            const float xl = __bfloat162float(X[static_cast<size_t>(j + bpad) * ldx + b_col_off + k]);
            acc = fmaf(w, xh, acc);
            acc = fmaf(w, xl, acc);
        }
        acc = warp_sum(acc);
        if (lane == 0) {
            if (ep.ln_fold) {
                float mean, rstd;
                ln_row_stats(ep.stats, ep.stats_tiles, ep.ln_d, j, ep.inv_d, ep.ln_eps, mean, rstd);
                acc = rstd * (acc - mean * ep.cvec[warp]);
            }
            const float sum[4] = {acc, 0.f, 0.f, 0.f};
            float xnew[4];
            apply_epilogue4(ep, j, 1, warp, sum, ep.bias[warp], xnew);
            if (ep.emit) {       // the row statistics of x_new follow in tile_stats_kernel, once every feature is written
                __nv_bfloat16 hi, lo;
                split_bf16(ep.next_gamma[warp] * xnew[0], hi, lo);
                ep.next_act[static_cast<size_t>(j) * ep.next_ld + warp] = hi;
                ep.next_act[static_cast<size_t>(j + ep.next_bpad) * ep.next_ld + warp] = lo;
            }
        }
    }
}

// Row statistics of the cross-check path's x_new (EPI_RESID + emit): per 128-feature tile and row, (sum x, M2 about the
// tile mean) -- what the tensor-core epilogue leaves.  One 128-thread CTA per (tile, row).
__global__ void __launch_bounds__(128) tile_stats_kernel(const float* __restrict__ x, int ld, int Nout, float* __restrict__ stats) {
    __shared__ float red[4];
    const int t = blockIdx.x, r = blockIdx.y, m = t * GEMM_BM + threadIdx.x;
    const int n = min(GEMM_BM, Nout - t * GEMM_BM);
    const float v = m < Nout ? x[static_cast<size_t>(r) * ld + m] : 0.f;
    auto block_sum = [&](float s) {
        s = warp_sum(s);
        __syncthreads();
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
        __syncthreads();
        return red[0] + red[1] + red[2] + red[3];
    };
    const float s1 = block_sum(v);
    const float dv = m < Nout ? v - s1 / static_cast<float>(n) : 0.f;
    const float m2 = block_sum(dv * dv);
    if (threadIdx.x == 0) *reinterpret_cast<float2*>(stats + (static_cast<size_t>(t) * STATS_ROWS + r) * 2) = make_float2(s1, m2);
}

// ---------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------
// fp32 row-major [N, K] -> bf16 tiles [ceil(N/128)][K/64][128][64], rows beyond N zero-filled
__global__ void pack_weight_tiles_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, int N, int Kdim) {
    const size_t total = static_cast<size_t>((N + GEMM_BM - 1) / GEMM_BM) * GEMM_BM * Kdim;
    const int KB = Kdim / GEMM_BK;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int c = static_cast<int>(i % GEMM_BK);
        const int r = static_cast<int>((i / GEMM_BK) % GEMM_BM);
        const size_t blk = i / (GEMM_BK * GEMM_BM);
        const int kb = static_cast<int>(blk % KB);
        const int mt = static_cast<int>(blk / KB);
        const int m = mt * GEMM_BM + r, k = kb * GEMM_BK + c;
        out[i] = (m < N) ? __float2bfloat16_rn(in[static_cast<size_t>(m) * Kdim + k]) : __float2bfloat16_rn(0.f);
    }
}

// element (m, k) of a packed weight as fp32: bf16 tiles, or int8 tiles times the row's 2^e (exactly W_deq)
struct PackedBf16 {
    const __nv_bfloat16* w;
    __device__ float operator()(int m, int k, int Kdim) const { return __bfloat162float(w[packed_index(m, k, Kdim)]); }
};
struct PackedW8 {
    const uint8_t* w;
    const float* scale;
    __device__ float operator()(int m, int k, int Kdim) const {
        return static_cast<float>(static_cast<int8_t>(w[w8_index(m, k, Kdim)])) * scale[m];
    }
};

// LayerNorm folding vectors from the pre-tiled weight: cvec[m] = sum_k gamma[k] W[m,k],
// bprime[m] = bias[m] + sum_k beta[k] W[m,k]; one warp per output feature, fp32.
template <typename WAt>
__global__ void ln_fold_vectors_kernel(const WAt Wp, const float* __restrict__ gamma,
                                       const float* __restrict__ beta, const float* __restrict__ bias,
                                       float* __restrict__ cvec, float* __restrict__ bprime, int N, int Kdim) {
    const int m = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (m >= N) return;
    float c = 0.f, b = 0.f;
    for (int k = lane; k < Kdim; k += 32) {
        const float w = Wp(m, k, Kdim);
        c = fmaf(gamma[k], w, c);
        b = fmaf(beta[k], w, b);
    }
    c = warp_sum(c);
    b = warp_sum(b);
    if (lane == 0) {
        cvec[m] = c;
        bprime[m] = bias[m] + b;
    }
}

int ln_fold_vectors(const __nv_bfloat16* Wp, const float* gamma, const float* beta, const float* bias, float* cvec,
                    float* bprime, int N, int Kdim) {
    ln_fold_vectors_kernel<<<(N * 32 + 255) / 256, 256>>>(PackedBf16{Wp}, gamma, beta, bias, cvec, bprime, N, Kdim);
    VCB_CUDA_OK(cudaGetLastError());
    return 0;
}

int ln_fold_vectors_w8(const uint8_t* W8, const float* scale, const float* gamma, const float* beta, const float* bias,
                       float* cvec, float* bprime, int N, int Kdim) {
    ln_fold_vectors_kernel<<<(N * 32 + 255) / 256, 256>>>(PackedW8{W8, scale}, gamma, beta, bias, cvec, bprime, N, Kdim);
    VCB_CUDA_OK(cudaGetLastError());
    return 0;
}

// The int8 rule (DESIGN.md section 2.2), one warp per row m of fp32 W [N, K]: e = the smallest integer >= -126 with
// max|W[m,:]| <= 127 * 2^e, q = round-half-even(W / 2^e) in [-127, 127].  With amax = f * 2^p, f in [1, 2): e = p - 6 when
// f <= 127/64 = 1.984375 (mantissa field <= 0x7e0000), else p - 5; zero or subnormal amax: -126.  Scaling by 2^-e
// (a normal fp32 for every such e) is exact where W / 2^e is, and rounds as the division does where it is not.
__global__ void weight_quantize_kernel(const float* __restrict__ W, int N, int Kdim, int8_t* __restrict__ q,
                                       int32_t* __restrict__ e_out, float* __restrict__ scale) {
    const int m = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (m >= N) return;
    const float* row = W + static_cast<size_t>(m) * Kdim;
    float amax = 0.f;
    for (int k = lane; k < Kdim; k += 32) amax = fmaxf(amax, fabsf(row[k]));
    amax = warp_max(amax);
    const uint32_t b = __float_as_uint(amax);
    const int e = (b >> 23) == 0 ? -126 : max(static_cast<int>(b >> 23) - 127 - 6 + ((b & 0x7fffffu) > 0x7e0000u), -126);
    const float inv = __uint_as_float(static_cast<uint32_t>(127 - e) << 23);
    int8_t* qrow = q + static_cast<size_t>(m) * Kdim;
    for (int k = lane; k < Kdim; k += 32) qrow[k] = static_cast<int8_t>(__float2int_rn(row[k] * inv));
    if (lane == 0) {
        if (e_out) e_out[m] = e;
        if (scale) scale[m] = __uint_as_float(static_cast<uint32_t>(127 + e) << 23);
    }
}

// int8 row-major [N, K] -> int8 tiles (w8_index), rows beyond N zero-filled
__global__ void pack_w8_tiles_kernel(const int8_t* __restrict__ q, uint8_t* __restrict__ out, int N, int Kdim) {
    const size_t total = static_cast<size_t>((N + GEMM_BM - 1) / GEMM_BM) * GEMM_BM * Kdim;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int m = static_cast<int>(i / Kdim), k = static_cast<int>(i % Kdim);
        out[w8_index(m, k, Kdim)] = m < N ? static_cast<uint8_t>(q[i]) : 0;
    }
}

// int8 tiles -> the bf16 tiles of pack_weight holding W_deq = q * 2^e (exact), for the rows-as-M prefill GEMM
__global__ void expand_w8_tiles_kernel(const uint8_t* __restrict__ in, const float* __restrict__ scale,
                                       __nv_bfloat16* __restrict__ out, int N, int Kdim) {
    const size_t total = static_cast<size_t>((N + GEMM_BM - 1) / GEMM_BM) * GEMM_BM * Kdim;
    const int KB = Kdim / GEMM_BK;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int c = static_cast<int>(i % GEMM_BK);
        const int r = static_cast<int>((i / GEMM_BK) % GEMM_BM);
        const size_t blk = i / (GEMM_BK * GEMM_BM);
        const int m = static_cast<int>(blk / KB) * GEMM_BM + r, k = static_cast<int>(blk % KB) * GEMM_BK + c;
        out[i] = __float2bfloat16_rn(m < N ? static_cast<float>(static_cast<int8_t>(in[w8_index(m, k, Kdim)])) * scale[m] : 0.f);
    }
}

static int make_tmap_w8(CUtensorMap* out, const void* base, uint64_t rows);

int weight_quantize(const float* W, int N, int Kdim, int8_t* q, int32_t* e, float* scale) {
    weight_quantize_kernel<<<(N * 32 + 255) / 256, 256>>>(W, N, Kdim, q, e, scale);
    VCB_CUDA_OK(cudaGetLastError());
    return 0;
}

int pack_weight_w8(const int8_t* q, uint8_t* out, int N, int Kdim, CUtensorMap* tm) {
    if (Kdim % 128) {
        set_error("int8 weights: K=%d not a multiple of 128", Kdim);
        return -1;
    }
    pack_w8_tiles_kernel<<<1024, 256>>>(q, out, N, Kdim);
    VCB_CUDA_OK(cudaGetLastError());
    return make_tmap_w8(tm, out, packed_weight_elems(N, Kdim) / 128);
}

int expand_weight_w8(const uint8_t* W8, const float* scale, __nv_bfloat16* out, int N, int Kdim, cudaStream_t st) {
    expand_w8_tiles_kernel<<<1024, 256, 0, st>>>(W8, scale, out, N, Kdim);
    VCB_CUDA_OK(cudaGetLastError());
    return 0;
}

size_t packed_weight_elems(int N, int Kdim) { return static_cast<size_t>((N + GEMM_BM - 1) / GEMM_BM) * GEMM_BM * Kdim; }

int pack_weight(const float* w_f32_dev, __nv_bfloat16* out, int N, int Kdim, CUtensorMap* tm) {
    if (Kdim % GEMM_BK) {
        set_error("pack_weight: K=%d not a multiple of %d", Kdim, GEMM_BK);
        return -1;
    }
    pack_weight_tiles_kernel<<<1024, 256>>>(w_f32_dev, out, N, Kdim);
    VCB_CUDA_OK(cudaGetLastError());
    const uint64_t rows = packed_weight_elems(N, Kdim) / GEMM_BK;       // 128-byte rows, 128 per tile
    return make_tmap_bf16_2d(tm, out, rows, GEMM_BK, GEMM_BK, GEMM_BM);
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess)
            return nullptr;
        fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
    return fn;
}

// 2D bf16 row-major [rows, cols] tensor, box = [box_rows, 64 cols], 128B swizzle, OOB -> 0
int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                      uint32_t box_rows) {
    PFN_encodeTiled fn = get_encode_fn();
    if (!fn) {
        set_error("cuTensorMapEncodeTiled entry point unavailable");
        return -1;
    }
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {ld_elems * 2};
    cuuint32_t box[2] = {GEMM_BK, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed: %d (rows=%llu cols=%llu ld=%llu box_rows=%u)", (int)r,
                  (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld_elems, box_rows);
        return -1;
    }
    return 0;
}

// int8 weight tiles as `rows` rows of 128 bytes, box = one 16 KB tile, 128B swizzle
static int make_tmap_w8(CUtensorMap* out, const void* base, uint64_t rows) {
    PFN_encodeTiled fn = get_encode_fn();
    if (!fn) {
        set_error("cuTensorMapEncodeTiled entry point unavailable");
        return -1;
    }
    cuuint64_t gdim[2] = {128, rows};
    cuuint64_t gstride[1] = {128};
    cuuint32_t box[2] = {128, GEMM_BM};
    cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled (int8 weights) failed: %d (rows=%llu)", (int)r, (unsigned long long)rows);
        return -1;
    }
    return 0;
}

// Co-residency of one instantiation, from the occupancy API: clusters[i] = clusters of 2^i CTAs the device can hold at
// once, 0 where it cannot place one (a cluster of 16 is non-portable: all of its CTAs must fit into one GPC at once).
struct GemmOccupancy {
    int clusters[5] = {};       // cluster sizes 1, 2, 4, 8, 16
    int max_cluster = 0;        // largest size it can place; 0: the queries failed (error set)
};

// Queried once per instantiation, after opting in to its shared memory and to non-portable cluster sizes.
template <int BN, int STAGES, bool W8 = false>
static const GemmOccupancy& occupancy() {
    static GemmOccupancy occ;
    if (occ.max_cluster) return occ;
    using L = GemmSmem<BN, STAGES, W8>;
    const auto kern = gemm_w_xT_cluster<BN, STAGES, false, W8>;
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL);
    if (err == cudaSuccess) err = cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (err != cudaSuccess) {
        set_error("gemm<%d,%d>: cudaFuncSetAttribute: %s", BN, STAGES, cudaGetErrorString(err));
        return occ;
    }
    GemmOccupancy q;
    for (int i = 0; i < 5; ++i) {
        cudaLaunchAttribute at;
        at.id = cudaLaunchAttributeClusterDimension;
        at.val.clusterDim.x = 1 << i;
        at.val.clusterDim.y = 1;
        at.val.clusterDim.z = 1;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(1 << i);
        cfg.blockDim = dim3(gemm_threads(BN));
        cfg.dynamicSmemBytes = L::TOTAL;
        cfg.attrs = &at;
        cfg.numAttrs = 1;
        int n = 0;
        if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) {
            (void)cudaGetLastError();       // a size the device rejects outright counts as "cannot be placed"
            n = 0;
        }
        if (n < 1) break;
        q.clusters[i] = n;
        q.max_cluster = 1 << i;
    }
    if (!q.max_cluster) {
        set_error("gemm<%d,%d>: the occupancy API places no CTA of %d B shared memory", BN, STAGES, L::TOTAL);
        return occ;
    }
    if (getenv("VCB_DEBUG_OCC"))
        fprintf(stderr, "[vcb] gemm<%d,%d>: %d B smem, resident clusters of 1/2/4/8/16: %d %d %d %d %d (occupancy API)\n",
                BN, STAGES, L::TOTAL, q.clusters[0], q.clusters[1], q.clusters[2], q.clusters[3], q.clusters[4]);
    return occ = q;
}

template <int BN, int STAGES, bool W8 = false>
static int launch_one(const GemmCall& g, int splits, cudaStream_t st) {
    using L = GemmSmem<BN, STAGES, W8>;
    const int tiles = (g.Nout + GEMM_BM - 1) / GEMM_BM;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(tiles * splits, g.grp.tmA ? g.groups : 1, 1);
    cfg.blockDim = dim3(gemm_threads(BN));
    cfg.dynamicSmemBytes = L::TOTAL;
    cfg.stream = st;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = splits;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = g.pdl ? 2 : 1;
    const int total_kb = g.Kdim / GEMM_BK;
    const int kbps = (total_kb + splits - 1) / splits;
    auto kern = gemm_w_xT_cluster<BN, STAGES, false, W8>;
    if (g.ep.mode == EPI_QKV && g.ep.kv_fp8) {
        // same shared memory and cluster shapes as the plain instantiation, whose occupancy chose the split count
        kern = gemm_w_xT_cluster<BN, STAGES, true, W8>;
        static bool attr_set = false;
        if (!attr_set) {
            VCB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
            VCB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
            attr_set = true;
        }
    }
    VCB_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, *g.tmA, *g.tmB, g.ep, g.Nout, total_kb, kbps, g.b_col_off, g.nvalid, g.pf_ptr,
                                   static_cast<unsigned long long>(g.pf_bytes), g.grp, g.wscale));
    return 0;
}

struct GemmVariant {
    const GemmOccupancy& (*occupancy)() = nullptr;
    int (*launch)(const GemmCall&, int, cudaStream_t) = nullptr;
};
template <int BN, int STAGES, bool W8 = false>
static GemmVariant variant() {
    return {occupancy<BN, STAGES, W8>, launch_one<BN, STAGES, W8>};
}

// The kernel for `bpad` token rows (2 * bpad hi/lo activation rows per tile); empty for any other padding.
static GemmVariant find_variant(int bpad) {
    switch (bpad) {
        case 16: return variant<32, gemm_stages(16)>();
        case 32: return variant<64, gemm_stages(32)>();
        case 64: return variant<128, gemm_stages(64)>();
        case 128: return variant<256, gemm_stages(128)>();
        default: return {};
    }
}
// ... and with int8 weights
static GemmVariant find_variant_w8(int bpad) {
    switch (bpad) {
        case 16: return variant<32, gemm_stages_w8(16), true>();
        case 32: return variant<64, gemm_stages_w8(32), true>();
        case 64: return variant<128, gemm_stages_w8(64), true>();
        case 128: return variant<256, gemm_stages_w8(128), true>();
        default: return {};
    }
}

// A split count the kernel can run: a power of two <= 16 that leaves each CTA of the cluster two or more token rows (the
// reduce-scatter sends pairs of adjacent rows to one owner) and at least one k-block.
static bool splits_legal(int s, int bpad, int total_kb) {
    return s >= 1 && s <= GEMM_MAX_SPLITS && !(s & (s - 1)) && bpad % s == 0 && bpad / s >= 2 &&
           (s - 1) * ((total_kb + s - 1) / s) < total_kb;
}

int gemm_launch_shape(const GemmCall& g, int cluster_cap, int& splits, int& stages) {
    if (g.Kdim % GEMM_BK != 0 || g.Kdim <= 0) {
        set_error("gemm: K=%d not a positive multiple of %d", g.Kdim, GEMM_BK);
        return -1;
    }
    const GemmVariant v = find_variant(g.bpad);
    if (!v.launch) {
        set_error("gemm: unsupported bpad %d", g.bpad);
        return -1;
    }
    const int total_kb = g.Kdim / GEMM_BK;
    if (!splits_legal(g.splits, g.bpad, total_kb)) {
        set_error("gemm: bad split count %d for %d k-blocks, bpad %d", g.splits, total_kb, g.bpad);
        return -1;
    }
    int placeable = v.occupancy().max_cluster;
    if (!placeable) return -1;
    if (cluster_cap > 0) placeable = std::min(placeable, cluster_cap);
    // a cluster the device cannot place falls back to the largest that it can: halving keeps the split count legal
    splits = g.splits;
    while (splits > placeable) splits /= 2;
    stages = gemm_stages(g.bpad);
    return 0;
}

int gemm_launch(const GemmCall& g, cudaStream_t st) {
    if (g.Kdim % GEMM_BK != 0) {
        set_error("gemm: K=%d not a multiple of %d", g.Kdim, GEMM_BK);
        return -1;
    }
    if (g.simt) {
        if (g.w8) {
            set_error("gemm: the CUDA-core cross-check GEMM has no int8-weight path");
            return -1;
        }
        dim3 grid((g.Nout * 32 + 255) / 256, 1, 1);
        gemm_w_xT_simt<<<grid, 256, 0, st>>>(g.W, g.X, g.ep, g.Nout, g.Kdim, g.ldx, g.bpad, g.b_col_off, g.nvalid);
        VCB_CUDA_OK(cudaGetLastError());
        if (g.ep.emit && g.nvalid > 0) {
            tile_stats_kernel<<<dim3((g.Nout + GEMM_BM - 1) / GEMM_BM, g.nvalid), GEMM_BM, 0, st>>>(g.ep.x, g.ep.ld_out, g.Nout,
                                                                                                  g.ep.stats_out);
            VCB_CUDA_OK(cudaGetLastError());
        }
        return 0;
    }
    int splits = 0;
    if (gemm_tc_splits(g, splits)) return -1;
    return (g.w8 ? find_variant_w8(g.bpad) : find_variant(g.bpad)).launch(g, splits, st);
}

// The split count the tensor-core launch of g runs, or -1 with the reason where gemm_launch would refuse it.
int gemm_tc_splits(const GemmCall& g, int& splits) {
    int stages = 0;
    if (gemm_launch_shape(g, 0, splits, stages)) return -1;
    if (!g.w8) return 0;
    // int8 weights: the bf16 kernel's launch shape (split count and K slices), on 128-k tiles
    if (g.Kdim % 128) {
        set_error("gemm: int8 weights need K %% 128 == 0 (K=%d)", g.Kdim);
        return -1;
    }
    const int placeable = find_variant_w8(g.bpad).occupancy().max_cluster;
    if (placeable < splits) {
        if (placeable) set_error("gemm: the int8-weight kernel for bpad %d places clusters of at most %d, not %d", g.bpad, placeable, splits);
        return -1;
    }
    return 0;
}

// Cluster size (= K splits) of a launch of `groups` x ceil(Nout / 128) tiles.  `room` = CTAs of this kernel the device
// holds at once (occupancy API).  Measured on the H100 (DESIGN.md section 4.1, scripts/bench_gemm.py), a launch is fastest
// with about half of `room` in its grid: the weight stream then has enough CTAs pulling HBM, and the next launch in the
// chain finds room for its CTAs, whose weight loads PDL starts under this launch's tail.  More splits than that cost more
// in the reduce-scatter and in the successor's start than the shorter K slice gains.  So: the most splits whose grid fits
// in room / 2; then one doubling more if that grid fills less than 3/4 of room / 2 (or the split is 1, which streams the
// whole K per CTA), as long as the doubled grid still runs as one wave of co-resident clusters.
int gemm_pick_splits(int Nout, int Kdim, int bpad, int groups) {
    const GemmVariant v = find_variant(bpad);
    if (!v.launch) return 1;                                        // (gemm_launch reports the padding)
    const GemmOccupancy& occ = v.occupancy();
    if (!occ.max_cluster) return 1;
    const int clusters = (Nout + GEMM_BM - 1) / GEMM_BM * std::max(1, groups);
    const int total_kb = Kdim / GEMM_BK, half = occ.clusters[0] / 2;
    auto fits = [&](int s) {                // legal, placeable, and one wave
        const int i = 31 - __builtin_clz(s);
        return s <= occ.max_cluster && splits_legal(s, bpad, total_kb) && occ.clusters[i] >= clusters;
    };
    int s = 1;
    while (fits(2 * s) && clusters * 2 * s <= half) s *= 2;
    if ((s == 1 || 4 * clusters * s < 3 * half) && fits(2 * s)) s *= 2;
    return s;
}

}  // namespace vcb
