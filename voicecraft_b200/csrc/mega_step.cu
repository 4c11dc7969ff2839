// Persistent decode-step kernel: every transformer layer of one decode step (QKV -> attention -> out-proj -> FFN1 -> FFN2,
// x L, then the logit heads) in ONE launch on a grid of one CTA per SM.  (transformer.py:321-329, 473-488; activation.py:536-638;
// voicecraft.py:181-185, 1085-1087.)
//
// Why: as 84 separate kernels the step is a latency chain -- every GEMM stops the HBM stream for a launch boundary, a
// pipeline ramp and an epilogue tail.  Neither the weights nor the cached K/V pages depend on the activations of the step, so here ONE producer
// thread per SM streams them, in schedule order, through a single ring of 16 KB shared-memory slots and never waits for
// anything but a free slot: while a phase's dependency chain (flag -> activation tiles -> MMA -> split-K reduce -> epilogue
// -> flag) resolves, the ring already fills with the next phases' weight blocks / KV slabs.
//
//   * work split ("stream-K"): a GEMM phase is the list of its 16 KB weight blocks (tile-major, k-minor); an attention
//     phase is the list of (row, head, page) units.  CTA c takes the contiguous range [c*T/G, (c+1)*T/G) of either list:
//     every SM streams the same number of bytes (+-1 block) per phase, whatever the matrix shape or the context lengths.
//   * roles: warp 0 ring producer (weights + K/V, TMA), warp 2 activation (B operand) producer -- the only one that waits
//     for the previous phase --, warp 3 L2 prefetcher, warps 4..11 workers: two warpgroups that multiply a GEMM tile
//     (wgmma, 64 features each, fp32 accumulators in registers) and run its epilogue, or do the attention math.
//   * split-K without clusters: a CTA's partial of a tile goes to an L2-resident workspace; the last CTA to arrive
//     (atomic counter) sums all partials in contributor order (deterministic) and runs the fused epilogue of
//     gemm_wgmma.cu (QKV append, residual + next LayerNorm operand and statistics, ReLU/GELU, logits).
//   * phase hand-over: one completion counter per phase (tiles done / CTAs done), release/acquire at GPU scope; data that
//     crossed CTAs is read with ld.global.cg (L1 is not coherent inside one kernel) or by TMA after fence.proxy.async.
//   * attention: same math as attn_rows_kernel (lm_kernels.cuh), but the current token's k/v come from the QKV epilogue's
//     fp32 side buffer (rounded like the cache), so the page stream has no dependency on this step at all; items split
//     between CTAs are merged flash-decoding style by the last arriver, in CTA order.
// All waits are bounded: a stuck wait records (role, phase, cta) in MegaArgs::dbg and traps instead of hanging the GPU.
#include "vcb_internal.h"

#include <algorithm>
#include <cstdio>

namespace vcb {

static constexpr int MG_THREADS = 384;
static constexpr int MG_SLOT = 16384;          // ring slot = one 128 x 64 bf16 weight block = one bf16 K (or V) slab
static constexpr int MG_POOL = 14 * 16384;     // bytes shared by the two rings: ns * 16 KB + nb * 8 KB <= MG_POOL
static constexpr int MG_BSLOT = 8192;          // 64 rows (32 hi + 32 lo) x 64 k, bf16
static constexpr int MG_NB_MIN = 3;            // activation (B operand) ring slots (MegaArgs::nb): the attention scratch
static constexpr int MG_NB_MAX = 8;            //   aliases three of them
static constexpr int MG_NS_MIN = 2;            // ring slots (MegaArgs::ns): at most what the pool leaves beside the
static constexpr int MG_NS_MAX = (MG_POOL - MG_NB_MIN * MG_BSLOT) / MG_SLOT;   //   smallest B ring (12)
static constexpr int MG_HD = 128;
static constexpr int MG_PAGE = 64;
static constexpr int MG_CHUNK = 4;             // attention: pages per work item (a chunk of one (row, head))
static constexpr int MG_MAXCH = 16;            // chunks per item the in-CTA fold can hold (4096 tokens; longer: workspace fold)
static constexpr int MG_PSTR = 132;            // floats per page partial: acc[128], m, l, pad

struct MegaSmem {
    static constexpr int RING = 0;                                  // ns slots, then the B ring (attention scratch aliases it)
    static constexpr int BAR = MG_POOL;
    static constexpr int NBAR = 2 * MG_NS_MAX + 2 * MG_NB_MAX;
    static constexpr int MISC = BAR + NBAR * 8;                    // flags, producer progress, page-count table
    static constexpr int TOTAL = MISC + 32 + 34 * 4 + 64;
    // attention scratch, aliased onto the B ring (idle during an attention phase)
    static constexpr int A_STATE = 0;                               // per-warp chunk states [8][MG_PSTR] floats
    static constexpr int A_CHUNKS = A_STATE + 8 * MG_PSTR * 4;      // chunk states of the item in flight [MG_MAXCH][MG_PSTR]
    static constexpr int A_Q = A_CHUNKS + MG_MAXCH * MG_PSTR * 4;   // q * scale * log2(e) of this / the next chunk [2][128]
    static constexpr int A_END = A_Q + 2 * MG_HD * 4;
};
static_assert(MegaSmem::A_END <= MG_NB_MIN * MG_BSLOT, "attention scratch must fit the smallest B ring");
static_assert(MegaSmem::TOTAL <= 232448, "shared memory budget of one CTA per SM");

__device__ __forceinline__ unsigned int mg_ld_acquire(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void mg_fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ unsigned long long mg_now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __noinline__ void mg_die(unsigned int* dbg, unsigned int role, unsigned int phase, unsigned int extra) {
    if (dbg) {
        if (atomicCAS(dbg, 0u, 1u) == 0u) {
            dbg[1] = role;
            dbg[2] = phase;
            dbg[3] = blockIdx.x;
            dbg[4] = extra;
        }
        __threadfence_system();
    }
    __trap();
}
// bounded mbarrier wait (2 s): a protocol bug surfaces as a CUDA error, not as a hung box
__device__ __forceinline__ void mg_wait(uint64_t* bar, uint32_t parity, unsigned int* dbg, unsigned int role, unsigned int phase) {
    if (mbar_try_wait(bar, parity)) return;
    unsigned long long t0 = 0;
    for (unsigned int spins = 1;; ++spins) {
        if (mbar_try_wait(bar, parity)) return;
        if ((spins & 0xfffu) == 0) {
            const unsigned long long t = mg_now();
            if (t0 == 0) t0 = t;
            else if (t - t0 > 2000000000ull) mg_die(dbg, role, phase, 0x100u | parity);
        }
    }
}
// Bounded wait for a phase completion counter.  The spin uses relaxed (L1-bypassing) loads and ONE acquire fence at the
// end: an ld.acquire.gpu in the loop invalidates the SM's L1 on every iteration (CCTL.IVALL), which turned every
// descriptor / bias read of the epilogue warps on the same SM into an L2 round trip.
__device__ __forceinline__ void mg_wait_flag(const unsigned int* flag, unsigned int target, unsigned int* dbg, unsigned int role,
                                             unsigned int phase) {
    unsigned long long t0 = 0;
    for (unsigned int spins = 0;; ++spins) {
        unsigned int v;
        asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
        if (v >= target) break;
        __nanosleep(32);
        if ((spins & 0x3ffu) == 0x3ffu) {
            const unsigned long long t = mg_now();
            if (t0 == 0) t0 = t;
            else if (t - t0 > 2000000000ull) mg_die(dbg, role, phase, 0x200u);
        }
    }
    asm volatile("fence.acq_rel.gpu;" ::: "memory");
}
__device__ __forceinline__ void mg_bar_workers() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
// wait until the ring producer has issued ring item `item` (s_prod = number of items issued so far)
__device__ __forceinline__ void mg_wait_issued(volatile uint32_t* s_prod, uint32_t item, unsigned int* dbg, unsigned int phase) {
    unsigned long long t0 = 0;
    for (unsigned int spins = 0; static_cast<int32_t>(*s_prod - item) <= 0; ++spins) {
        __nanosleep(20);
        if ((spins & 0xfffu) == 0xfffu) {
            const unsigned long long t = mg_now();
            if (t0 == 0) t0 = t;
            else if (t - t0 > 2000000000ull) mg_die(dbg, 8, phase, 0x300u);
        }
    }
}

// Work split of T units over the first Ge = min(G, T) CTAs (every one of them gets >= 1 unit, the others none, so the
// CTAs that share a tile / an attention item are always consecutive): range of CTA c, and the CTA that owns unit u.
// (32-bit arithmetic: the host checks T * G < 2^31; 64-bit divisions are ~10x slower and sit on every role's path)
__device__ __forceinline__ int mg_eff(long long T, int G) { return static_cast<int>(T < G ? T : G); }
__device__ __forceinline__ void mg_range(long long T, int c, int Ge, int& b0, int& b1) {
    if (c >= Ge) {
        b0 = b1 = 0;
        return;
    }
    const unsigned int t = static_cast<unsigned int>(T), g = static_cast<unsigned int>(Ge), cc = static_cast<unsigned int>(c);
    b0 = static_cast<int>(t * cc / g);
    b1 = static_cast<int>(t * (cc + 1u) / g);
}
// attention unit u -> (row, head, page) and the row's page count; units are ordered (row, head, page)
__device__ __forceinline__ void mg_locate(const int* s_cum, int H, int u, int& r, int& h, int& pg, int& npg) {
    r = 0;
    while (r < 31 && static_cast<long long>(H) * s_cum[r + 1] <= u) ++r;
    npg = s_cum[r + 1] - s_cum[r];
    const int rem = u - H * s_cum[r];
    h = npg ? rem / npg : 0;
    pg = npg ? rem - h * npg : 0;
}
// first chunk boundary at or after unit u (chunks = MG_CHUNK pages of one (row, head), the last one shorter)
__device__ __forceinline__ int mg_chunk_align(const int* s_cum, int H, int u, long long U) {
    if (u >= U) return static_cast<int>(U);
    int r, h, pg, npg;
    mg_locate(s_cum, H, u, r, h, pg, npg);
    const int m = pg % MG_CHUNK;
    return m == 0 ? u : u + min(MG_CHUNK - m, npg - pg);
}
// debug timeline: every CTA records %globaltimer at fixed (cta, phase, event) slots
__device__ __forceinline__ void mg_tl(const MegaArgs& A, int p, int ev) {
    if (A.tl != nullptr) A.tl[(static_cast<size_t>(blockIdx.x) * A.nph + p) * 16 + ev] = mg_now();
}
__device__ __forceinline__ int mg_owner(long long u, long long T, int G) {
    return static_cast<int>(((static_cast<unsigned int>(u) + 1u) * static_cast<unsigned int>(G) - 1u) / static_cast<unsigned int>(T));
}

__device__ __forceinline__ uint2 mg_pack_bf16x4(float a, float b, float c, float d) {
    const __nv_bfloat162 lo = __floats2bfloat162_rn(a, b), hi = __floats2bfloat162_rn(c, d);
    uint2 r;
    r.x = *reinterpret_cast<const uint32_t*>(&lo);
    r.y = *reinterpret_cast<const uint32_t*>(&hi);
    return r;
}
__device__ __forceinline__ float mg_bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
// Element offset of activation (k, row) in the tiled + pre-swizzled B-operand image (MegaArgs::bbase): k-block k/64 is one
// contiguous tile of rows2 = 2*bpad rows x 128 bytes; inside a row the 16-byte chunk (k%64)/8 is XORed with row % 8, which is
// exactly where TMA's SWIZZLE_128B would have put it in shared memory (rows2 is a multiple of 8).
__device__ __forceinline__ size_t mg_act_off(int k, int row, int rows2) {
    const int kk = k & 63;
    return (static_cast<size_t>(k >> 6) * rows2 + row) * 64 + ((((kk >> 3) ^ (row & 7)) << 3) | (kk & 7));
}

// ------------------------------------------------------------------------------------------------------------------------
// Split-K hand-over of one output tile, reduce-scatter through L2: every CTA that contributed a partial of the tile
// ("contributor" s = 0 .. S-1 in CTA order = ascending k) takes the token rows [s*BPAD/S, (s+1)*BPAD/S), sums the S partials
// of those rows in contributor order (deterministic) and runs the fused epilogue on them.  (A single "last arriver" would
// read all S x 16 KB partials through one SM's L2 port.)
// Thread mapping: lane -> features 4*lane .. 4*lane+3 of the tile; warp wq -> rows row_begin + wq + 8j.
// mg_epi_prefetch loads everything that does not depend on the other contributors (issued BEFORE waiting for them).
// ------------------------------------------------------------------------------------------------------------------------
template <int BPAD>
struct MgEpiRegs {
    static constexpr int MAXR = BPAD / 8;
    float bias[4], cv[4], gn[4];
    float mean[MAXR], rstd[MAXR];
    float4 xold[MAXR];
    int rpos[MAXR], rpage[MAXR];
};

template <int BPAD>
__device__ __forceinline__ void mg_epi_prefetch(const MegaArgs& A, const MegaPhase& P, const GemmEpilogue& ep, int tile, int row_begin,
                                                int row_end, int wq, int lane, MgEpiRegs<BPAD>& R) {
    constexpr int MAXR = BPAD / 8;
    const int g = tile / P.tiles_per_group, tl = tile - g * P.tiles_per_group;
    const int m0 = tl * 128 + 4 * lane;
    const int Nout = P.Nout;
    const float* bias_ptr = P.grp_bias ? P.grp_bias[g] : ep.bias;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const bool ok = m0 + i < Nout;
        R.bias[i] = ok ? bias_ptr[m0 + i] : 0.f;
        R.cv[i] = (ok && ep.ln_fold) ? ep.cvec[m0 + i] : 0.f;
        R.gn[i] = (ok && ep.emit) ? ep.next_gamma[m0 + i] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < MAXR; ++j) {
        const int row = row_begin + wq + 8 * j;
        const bool live = row < row_end && row < A.nvalid;          // warp-uniform
        R.mean[j] = 0.f;
        R.rstd[j] = 0.f;
        R.xold[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        R.rpos[j] = (live && ep.mode == EPI_QKV) ? ep.row_pos[row] : -1;
        R.rpage[j] = (live && ep.mode == EPI_QKV) ? ep.row_page[row] : 0;
        if (ep.ln_fold && live) {
            // lane t holds tile t (of each group of 32): the row sum, then the tiles' M2 about the row mean (see ln_tile_m2)
            float2 v[4];
            float s1 = 0.f, m2 = 0.f;
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                const int t = 32 * b + lane;
                v[b] = t < ep.stats_tiles ? __ldcg(reinterpret_cast<const float2*>(ep.stats + (static_cast<size_t>(t) * STATS_ROWS + row) * 2))
                                          : make_float2(0.f, 0.f);
                s1 += v[b].x;
            }
            const float mean = warp_sum(s1) * ep.inv_d;
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                const int t = 32 * b + lane;
                if (t < ep.stats_tiles) m2 += ln_tile_m2(ln_tile_n(t, ep.stats_tiles, ep.ln_d), v[b].x, v[b].y, mean);
            }
            R.mean[j] = mean;
            R.rstd[j] = 1.0f / sqrtf(warp_sum(m2) * ep.inv_d + ep.ln_eps);
        }
        if (ep.mode == EPI_RESID && live && m0 < Nout)
            R.xold[j] = __ldcg(reinterpret_cast<const float4*>(ep.x + static_cast<size_t>(row) * ep.ld_out + m0));
    }
}

template <int BPAD>
__device__ __forceinline__ void mg_epi_finish(const MegaArgs& A, const MegaPhase& P, const GemmEpilogue& ep, int p, int tile, int c_first,
                                              int ncontrib, long long T, int G, int row_begin, int row_end, int wq, int lane,
                                              const MgEpiRegs<BPAD>& R) {
    constexpr int MAXR = BPAD / 8;
    const int g = tile / P.tiles_per_group, tl = tile - g * P.tiles_per_group;
    const int m0 = tl * 128 + 4 * lane;
    const int Nout = P.Nout;
    const int col_grp = g * P.col_grp_stride;
    const int kb = P.kb;
#pragma unroll
    for (int j = 0; j < MAXR; ++j) {
        const int row = row_begin + wq + 8 * j;
        if (row >= row_end) break;                                    // warp-uniform
        const bool row_ok = row < A.nvalid;
        // ---- fixed-order sum of the S partials of this row --------------------------------------------------------------------
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int s0 = 0; s0 < ncontrib; s0 += 8) {
            float4 v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int s = s0 + u;
                if (s < ncontrib) {
                    const int c = c_first + s;
                    const int cb0 = static_cast<int>(static_cast<unsigned int>(T) * static_cast<unsigned int>(c) / static_cast<unsigned int>(G));
                    const float* src = A.part + ((static_cast<size_t>(c) * MEGA_MAXSEG + (tile - cb0 / kb)) * BPAD + row) * 128 + 4 * lane;
                    v[u] = __ldcg(reinterpret_cast<const float4*>(src));
                } else {
                    v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                acc.x += v[u].x;
                acc.y += v[u].y;
                acc.z += v[u].z;
                acc.w += v[u].w;
            }
        }
        float a[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (ep.ln_fold) a[i] = R.rstd[j] * (a[i] - R.mean[j] * R.cv[i]);
            a[i] += R.bias[i];
        }
        float xn[4] = {0.f, 0.f, 0.f, 0.f};
        if (row_ok) {
            switch (ep.mode) {
                case EPI_QKV: {
                    const int pos = R.rpos[j];
                    if (pos < 0 || m0 >= Nout) break;
                    const int part = m0 / ep.d, cc = m0 - part * ep.d;
                    if (part == 0) {
                        __stcg(reinterpret_cast<float4*>(ep.qbuf + static_cast<size_t>(row) * ep.d + cc), make_float4(a[0], a[1], a[2], a[3]));
                        break;
                    }
                    const int page = R.rpage[j];
                    const int h = cc / ep.hd, e = cc - h * ep.hd;
                    const size_t off = ((static_cast<size_t>(page) * ep.H + h) * ep.page_size + pos % ep.page_size) * ep.hd + e;
                    void* pool = (part == 1) ? ep.kpool : ep.vpool;
                    float* side = (part == 1) ? ep.knew : ep.vnew;
                    if (ep.kv_fp32) {
                        __stcg(reinterpret_cast<float4*>(static_cast<float*>(pool) + off), make_float4(a[0], a[1], a[2], a[3]));
                    } else {
                        __stcg(reinterpret_cast<uint2*>(static_cast<__nv_bfloat16*>(pool) + off), mg_pack_bf16x4(a[0], a[1], a[2], a[3]));
#pragma unroll
                        for (int i = 0; i < 4; ++i) a[i] = mg_bf16_round(a[i]);
                    }
                    __stcg(reinterpret_cast<float4*>(side + static_cast<size_t>(row) * ep.d + cc), make_float4(a[0], a[1], a[2], a[3]));
                    break;
                }
                case EPI_RESID: {
                    xn[0] = R.xold[j].x + a[0];
                    xn[1] = R.xold[j].y + a[1];
                    xn[2] = R.xold[j].z + a[2];
                    xn[3] = R.xold[j].w + a[3];
                    if (m0 < Nout)
                        __stcg(reinterpret_cast<float4*>(ep.x + static_cast<size_t>(row) * ep.ld_out + m0), make_float4(xn[0], xn[1], xn[2], xn[3]));
                    break;
                }
                case EPI_ACT: {
                    if (m0 >= Nout) break;
                    float hi[4], lo[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        float v = a[i];
                        if (ep.act_kind == 1) v = fmaxf(v, 0.f);
                        else if (ep.act_kind == 2) v = 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
                        hi[i] = mg_bf16_round(v);
                        lo[i] = v - hi[i];
                    }
                    __stcg(reinterpret_cast<uint2*>(ep.act + mg_act_off(m0, row, 2 * ep.bpad_out)), mg_pack_bf16x4(hi[0], hi[1], hi[2], hi[3]));
                    __stcg(reinterpret_cast<uint2*>(ep.act + mg_act_off(m0, row + ep.bpad_out, 2 * ep.bpad_out)),
                           mg_pack_bf16x4(lo[0], lo[1], lo[2], lo[3]));
                    break;
                }
                default: {
                    float* o = ep.out + static_cast<size_t>(row) * ep.ld_out + ep.col_off + col_grp + m0;
                    if (m0 + 3 < Nout) {
                        __stcg(reinterpret_cast<float4*>(o), make_float4(a[0], a[1], a[2], a[3]));
                    } else {
#pragma unroll
                        for (int i = 0; i < 4; ++i)
                            if (m0 + i < Nout) __stcg(o + i, a[i]);
                    }
                }
            }
        }
        if (ep.emit) {
            // next GEMM's operand gamma_next * x_new (hi/lo) and this tile's (sum x, M2 about the tile mean) of the row: a
            // warp holds exactly the 128 features of the tile for this row
            const bool mine = row_ok && m0 < Nout;
            float p1 = 0.f, p2 = 0.f;
            if (mine) {
                float hi[4], lo[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float v = R.gn[i] * xn[i];
                    hi[i] = mg_bf16_round(v);
                    lo[i] = v - hi[i];
                    p1 += xn[i];
                }
                __stcg(reinterpret_cast<uint2*>(ep.next_act + mg_act_off(m0, row, 2 * ep.next_bpad)), mg_pack_bf16x4(hi[0], hi[1], hi[2], hi[3]));
                __stcg(reinterpret_cast<uint2*>(ep.next_act + mg_act_off(m0, row + ep.next_bpad, 2 * ep.next_bpad)),
                       mg_pack_bf16x4(lo[0], lo[1], lo[2], lo[3]));
            }
            p1 = warp_sum(p1);
            const float tmean = p1 / static_cast<float>(max(1, min(128, Nout - tl * 128)));
            if (mine) {
#pragma unroll
                for (int i = 0; i < 4; ++i) p2 = fmaf(xn[i] - tmean, xn[i] - tmean, p2);
            }
            p2 = warp_sum(p2);
            if (lane == 0 && row_ok)
                __stcg(reinterpret_cast<float2*>(ep.stats_out + (static_cast<size_t>(tl) * STATS_ROWS + row) * 2), make_float2(p1, p2));
        }
    }
}

// K / V element loads from a ring slot (same conversions as lm_kernels.cuh::load_kv_vec)
template <typename KVT, int N>
__device__ __forceinline__ void mg_load_kv(const KVT* p, float (&out)[N]) {
    if constexpr (sizeof(KVT) == 2) {
        if constexpr (N == 8) {
            const uint4 u = *reinterpret_cast<const uint4*>(p);
            const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                out[2 * i] = __uint_as_float(w[i] << 16);
                out[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
            }
        } else {
            const uint2 u = *reinterpret_cast<const uint2*>(p);
            out[0] = __uint_as_float(u.x << 16);
            out[1] = __uint_as_float(u.x & 0xffff0000u);
            out[2] = __uint_as_float(u.y << 16);
            out[3] = __uint_as_float(u.y & 0xffff0000u);
        }
    } else {
#pragma unroll
        for (int i = 0; i < N; i += 4) {
            const float4 f = *reinterpret_cast<const float4*>(p + i);
            out[i] = f.x;
            out[i + 1] = f.y;
            out[i + 2] = f.z;
            out[i + 3] = f.w;
        }
    }
}

template <int BPAD, typename KVT>
__global__ void __launch_bounds__(MG_THREADS, 1) mega_step_kernel(const __grid_constant__ MegaArgs A) {
    constexpr int BN = 2 * BPAD;                          // MMA N: hi rows + lo rows
    constexpr int B_BYTES = BN * 64 * 2;
    constexpr int TPS = MG_SLOT / (MG_HD * static_cast<int>(sizeof(KVT)));   // tokens per ring slot: 64 (bf16) / 32 (fp32)
    constexpr int NSL = MG_PAGE / TPS;                    // ring slots per K (or V) slab
    using L = MegaSmem;
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t MG_NS = A.ns, MG_NB = A.nb;             // ring depths (runtime: swept by VCB_MEGA_NS / VCB_MEGA_NB)
    uint8_t* ring = smem + L::RING;
    uint8_t* bring = smem + L::RING + MG_NS * MG_SLOT;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + L::BAR);
    uint64_t* empty = full + MG_NS_MAX;
    uint64_t* bfull = empty + MG_NS_MAX;
    uint64_t* bempty = bfull + MG_NB_MAX;
    int* s_flag = reinterpret_cast<int*>(smem + L::MISC + 8);
    volatile uint32_t* s_prod = reinterpret_cast<volatile uint32_t*>(smem + L::MISC + 16);   // ring items issued so far
    int* s_cum = reinterpret_cast<int*>(smem + L::MISC + 32);           // [33] prefix sum of pages per row

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cta = blockIdx.x, G = gridDim.x;
    const MegaPhase* __restrict__ ph = A.ph;

    if (threadIdx.x == 0) {
        for (uint32_t i = 0; i < MG_NS; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], 8);          // the 8 worker warps (weights: after their MMAs; K/V slabs: after the math)
        }
        for (uint32_t i = 0; i < MG_NB; ++i) {
            mbar_init(&bfull[i], 1);
            mbar_init(&bempty[i], 8);
        }
        mbar_fence_init();
        *s_prod = 0u;
        int c = 0;
        for (int r = 0; r < 32; ++r) {
            s_cum[r] = c;
            const int pos = r < A.nvalid ? A.row_pos[r] : -1;
            c += pos >= 0 ? pos / MG_PAGE + 1 : 0;
        }
        s_cum[32] = c;
    }
    __syncthreads();
    const long long U = static_cast<long long>(A.H) * s_cum[32];     // attention units of this step
    int u0, u1;
    const int Ue = mg_eff(U, G);
    mg_range(U, cta, Ue, u0, u1);
    u0 = mg_chunk_align(s_cum, A.H, u0, U);            // a CTA owns the chunks that START in its share of the units
    u1 = mg_chunk_align(s_cum, A.H, u1, U);

    if (warp == 0) {
        // ===== ring producer: weight blocks and K/V slabs of every phase, in schedule order ==============================
        if (lane == 0) {
            const uint64_t pol = l2_policy_evict_first();
            uint32_t it = 0, landed = 0;
            const uint32_t flight = static_cast<uint32_t>(A.flight);
            auto acquire = [&](int p) -> int {
                const int s = it % MG_NS;
                if (it >= MG_NS) mg_wait(&empty[s], ((it / MG_NS) - 1) & 1, A.dbg, 0, p);
                // Bound the loads IN FLIGHT (issued, not landed), not just the ring's capacity: this SM's memory pipe serves
                // requests roughly in order, so the activation tiles / partials a phase hand-over is waiting for queue behind
                // whatever the ring still has outstanding.  `flight` x 16 KB in flight keeps HBM busy while landed slots
                // still pile up to the ring's depth during a dependency chain.
                while (it - landed >= flight) {
                    mg_wait(&full[landed % MG_NS], (landed / MG_NS) & 1, A.dbg, 9, p);
                    ++landed;
                }
                ++it;
                *s_prod = it;
                return s;
            };
            for (int p = 0; p < A.nph; ++p) {
                const MegaPhase& P = ph[p];
                if (P.type == MEGA_GEMM) {
                    const long long T = static_cast<long long>(P.groups) * P.tiles_per_group * P.kb;
                    int b0, b1;
                    const int Ge = mg_eff(T, G);
                    mg_range(T, cta, Ge, b0, b1);
                    for (int blk = b0; blk < b1; ++blk) {
                        const int tile = blk / P.kb, kbi = blk - tile * P.kb;
                        const int g = tile / P.tiles_per_group, tl = tile - g * P.tiles_per_group;
                        const int s = acquire(p);
                        mbar_arrive_expect_tx(&full[s], MG_SLOT);
                        tma_load_2d_hint(ring + s * MG_SLOT, P.tmA + g, &full[s], 0, (tl * P.kb + kbi) * 128, pol);
                    }
                } else {
                    // units are ordered (row, head, page); walk my range
                    int r = 0;
                    while (r < 31 && static_cast<long long>(A.H) * s_cum[r + 1] <= u0) ++r;
                    int npg = s_cum[r + 1] - s_cum[r];
                    int rem = u0 - A.H * s_cum[r];
                    int h = npg ? rem / npg : 0, pg = npg ? rem - h * npg : 0;
                    const KVT* kpool = static_cast<const KVT*>(P.kpool);
                    const KVT* vpool = static_cast<const KVT*>(P.vpool);
                    for (int u = u0; u < u1; ++u) {
                        const int page = A.row_pages[r * A.max_pages + pg];
                        const size_t off = (static_cast<size_t>(page) * A.H + h) * MG_PAGE * MG_HD;
#pragma unroll
                        for (int kv = 0; kv < 2; ++kv) {
                            const KVT* src = (kv == 0 ? kpool : vpool) + off;
#pragma unroll
                            for (int j = 0; j < NSL; ++j) {
                                const int s = acquire(p);
                                mbar_arrive_expect_tx(&full[s], MG_SLOT);
                                tma_bulk_g2s_hint(ring + s * MG_SLOT, src + static_cast<size_t>(j) * TPS * MG_HD, MG_SLOT, &full[s], pol);
                            }
                        }
                        if (++pg == npg) {
                            pg = 0;
                            if (++h == A.H) {
                                h = 0;
                                do {
                                    ++r;
                                    npg = r < 32 ? s_cum[r + 1] - s_cum[r] : 1;
                                } while (r < 32 && npg == 0);
                            }
                        }
                    }
                }
                mg_tl(A, p, 7);
            }
        }
    } else if (warp == 2) {
        // ===== activation (B operand) producer: the only role that waits for the previous phase ===========================
        if (lane == 0) {
            uint32_t bit = 0;
            for (int p = 0; p < A.nph; ++p) {
                const MegaPhase& P = ph[p];
                if (P.type != MEGA_GEMM) continue;
                const long long T = static_cast<long long>(P.groups) * P.tiles_per_group * P.kb;
                int b0, b1;
                const int Ge = mg_eff(T, G);
                    mg_range(T, cta, Ge, b0, b1);
                if (b0 >= b1) continue;
                if (P.dep_target > 0) mg_wait_flag(A.flags + (p - 1), P.dep_target, A.dbg, 3, p);
                mg_tl(A, p, 0);
                mg_fence_proxy_async();              // other CTAs' generic-proxy stores -> visible to my TMA loads
                for (int blk = b0; blk < b1; ++blk, ++bit) {
                    const int tile = blk / P.kb, kbi = blk - tile * P.kb;
                    const int g = tile / P.tiles_per_group;
                    const int bs = bit % MG_NB;
                    if (bit >= MG_NB) mg_wait(&bempty[bs], ((bit / MG_NB) - 1) & 1, A.dbg, 3, p);
                    mbar_arrive_expect_tx(&bfull[bs], B_BYTES);
                    const int kglob = (P.b_col_off + g * P.b_grp_stride) / 64 + kbi;            // k-block inside the operand's buffer
                    tma_bulk_g2s(bring + bs * MG_BSLOT, A.bbase[P.b_map] + static_cast<size_t>(kglob) * BN * 64, B_BYTES, &bfull[bs]);
                }
                mg_tl(A, p, 4);
            }
        }
    } else if (warp == 3) {
        // ===== L2 prefetcher: walks the same schedule `pf` items ahead of the ring producer ===============================
        // The ring holds ns * 16 KB per SM; while a dependency chain resolves and the ring is full, HBM would idle.  This
        // thread keeps pulling the items AFTER the ring's window from HBM into L2 (cp.async.bulk.prefetch.L2), so that when
        // slots free up the ring refills at L2 speed.
        if (lane == 0 && A.pf > 0) {
            uint32_t it = 0;
            auto pace = [&](int p) {
                // stay at most pf items ahead of the producer
                unsigned long long t0 = 0;
                for (unsigned int spins = 0; it >= *s_prod + MG_NS + static_cast<uint32_t>(A.pf); ++spins) {
                    __nanosleep(64);
                    if ((spins & 0xfffu) == 0xfffu) {
                        const unsigned long long t = mg_now();
                        if (t0 == 0) t0 = t;
                        else if (t - t0 > 4000000000ull) return false;      // producer stuck: its own watchdog reports
                    }
                }
                return true;
            };
            bool ok = true;
            for (int p = 0; p < A.nph && ok; ++p) {
                const MegaPhase& P = ph[p];
                if (P.type == MEGA_GEMM) {
                    const long long T = static_cast<long long>(P.groups) * P.tiles_per_group * P.kb;
                    int b0, b1;
                    const int Ge = mg_eff(T, G);
                    mg_range(T, cta, Ge, b0, b1);
                    for (int blk = b0; blk < b1 && ok; ++blk, ++it) {
                        if (it < MG_NS) continue;                            // the first window goes straight to the ring
                        ok = pace(p);
                        const int tile = blk / P.kb, kbi = blk - tile * P.kb;
                        const int g = tile / P.tiles_per_group, tl = tile - g * P.tiles_per_group;
                        tma_prefetch_l2(static_cast<const uint8_t*>(P.wptr[g]) + static_cast<size_t>(tl * P.kb + kbi) * MG_SLOT, MG_SLOT);
                    }
                } else {
                    int r = 0;
                    while (r < 31 && static_cast<long long>(A.H) * s_cum[r + 1] <= u0) ++r;
                    int npg = s_cum[r + 1] - s_cum[r];
                    int rem = u0 - A.H * s_cum[r];
                    int h = npg ? rem / npg : 0, pg = npg ? rem - h * npg : 0;
                    const KVT* kpool = static_cast<const KVT*>(P.kpool);
                    const KVT* vpool = static_cast<const KVT*>(P.vpool);
                    for (int u = u0; u < u1 && ok; ++u, it += 2 * NSL) {
                        if (it >= MG_NS) {
                            ok = pace(p);
                            const int page = A.row_pages[r * A.max_pages + pg];
                            const size_t off = (static_cast<size_t>(page) * A.H + h) * MG_PAGE * MG_HD;
                            tma_prefetch_l2(kpool + off, NSL * MG_SLOT);
                            tma_prefetch_l2(vpool + off, NSL * MG_SLOT);
                        }
                        if (++pg == npg) {
                            pg = 0;
                            if (++h == A.H) {
                                h = 0;
                                do {
                                    ++r;
                                    npg = r < 32 ? s_cum[r + 1] - s_cum[r] : 1;
                                } while (r < 32 && npg == 0);
                            }
                        }
                    }
                }
            }
        }
    } else if (warp >= 4) {
        // ===== workers: GEMM epilogues / attention ========================================================================
        const int wtid = threadIdx.x - 128;             // 0..255
        const int wq = wtid >> 5;                        // worker warp 0..7
        const int q = warp & 3;                          // warp inside its warpgroup
        const int grp = wq >> 2;                         // worker warpgroup: features [64 grp, 64 grp + 64) of a tile
        uint32_t it = 0, bit = 0;
        for (int p = 0; p < A.nph; ++p) {
            const MegaPhase& P = ph[p];
            if (P.type == MEGA_GEMM) {
                const long long T = static_cast<long long>(P.groups) * P.tiles_per_group * P.kb;
                int b0, b1;
                const int Ge = mg_eff(T, G);
                    mg_range(T, cta, Ge, b0, b1);
                const int first_tile = b0 / P.kb;
                int blk = b0;
                while (blk < b1) {
                    const int tile = blk / P.kb;
                    const int seg_end = min(b1, (tile + 1) * P.kb);
                    float acc[BN / 2];
#pragma unroll
                    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
                    for (; blk < seg_end; ++blk, ++it, ++bit) {
                        const int s = it % MG_NS, bs = bit % MG_NB;
                        mg_wait(&full[s], (it / MG_NS) & 1, A.dbg, 1, p);
                        mg_wait(&bfull[bs], (bit / MG_NB) & 1, A.dbg, 2, p);
                        wg_fence();
                        wg_mma_kblock<BN>(acc, smem_u32(ring + s * MG_SLOT) + grp * 64 * 128, smem_u32(bring + bs * MG_BSLOT));
                        wg_commit();
                        wg_wait0();
                        __syncwarp();
                        if (lane == 0) {                             // this warp's MMAs have read both slots
                            mbar_arrive(&empty[s]);
                            mbar_arrive(&bempty[bs]);
                        }
                    }
                    wg_acc_fence(acc);
                    if (wtid == 0) mg_tl(A, p, 1);
                    // ---- my partial of this tile (hi + lo columns) -> workspace [row][feature] ---------------------------------
                    float* pdst = A.part + (static_cast<size_t>(cta) * MEGA_MAXSEG + (tile - first_tile)) * BPAD * 128;
#pragma unroll
                    for (int jb = 0; jb < BPAD / 8; ++jb) {
                        const int row = 8 * jb + 2 * (lane & 3);
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int f = grp * 64 + q * 16 + (lane >> 2) + 8 * e;
                            __stcg(pdst + row * 128 + f, acc[4 * jb + 2 * e] + acc[4 * (jb + BPAD / 8) + 2 * e]);
                            __stcg(pdst + (row + 1) * 128 + f, acc[4 * jb + 2 * e + 1] + acc[4 * (jb + BPAD / 8) + 2 * e + 1]);
                        }
                    }
                    // publish my partial: the block barrier orders every worker's stores before thread 0's GPU-scope fence
                    // (fences are cumulative), then count in.  ALL my partials of the phase go out before I wait for anybody:
                    // waiting per tile would chain the tiles (tile t+1's partial stuck behind the wait for tile t's last
                    // contributor, a domino across the phase's tiles).
                    mg_bar_workers();
                    if (wtid == 0) {
                        __threadfence();
                        atomicAdd(A.tile_cnt + p * A.tile_cnt_stride + tile, 1);
                    }
                }
                if (wtid == 0) mg_tl(A, p, 3);
                // ---- second pass: my share of every tile I contributed to ----------------------------------------------------
                if (b0 < b1) {
                    const GemmEpilogue ep = P.ep;           // by value: no re-loads of its fields between the epilogue's stores
                    const int last_tile = (b1 - 1) / P.kb;
                    for (int tile = first_tile; tile <= last_tile; ++tile) {
                        const int c_first = mg_owner(static_cast<long long>(tile) * P.kb, T, Ge);
                        const int c_last = mg_owner(static_cast<long long>(tile + 1) * P.kb - 1, T, Ge);
                        const int ncontrib = c_last - c_first + 1;
                        const int sidx = cta - c_first;
                        const int row_begin = sidx * BPAD / ncontrib, row_end = (sidx + 1) * BPAD / ncontrib;
                        // operands that do not depend on the other contributors are fetched WHILE they arrive
                        MgEpiRegs<BPAD> R;
                        mg_epi_prefetch<BPAD>(A, P, ep, tile, row_begin, row_end, wq, lane, R);
                        if (wtid == 0) {
                            mg_wait_flag(reinterpret_cast<const unsigned int*>(A.tile_cnt + p * A.tile_cnt_stride + tile),
                                         static_cast<unsigned int>(ncontrib), A.dbg, 10, p);
                            mg_tl(A, p, 8);
                        }
                        mg_bar_workers();
                        mg_epi_finish<BPAD>(A, P, ep, p, tile, c_first, ncontrib, T, Ge, row_begin, row_end, wq, lane, R);
                        mg_bar_workers();
                        if (wtid == 0) {
                            __threadfence();
                            mg_fence_proxy_async();
                            atomicAdd(A.flags + p, 1u);
                            mg_tl(A, p, 2);
                        }
                    }
                }
            } else {
                // ===== attention: units [u0, u1), cut at chunk boundaries ======================================================
                // Work item = CHUNK of up to MG_CHUNK consecutive pages of one (row, head); the chunk grid depends only on the
                // row's own context length.  The 8 worker warps share every page: warp w owns keys [8w, 8w+8) of the page,
                // keeps its own online-softmax state (m, l, acc) over the chunk's pages and multiplies its 8 probabilities
                // into V -- no block barrier per page.  Per chunk the 8 warp states fold in warp order, chunks fold in chunk
                // order: every result is a fixed-order fold that depends only on the row's own context (a row's tokens do
                // not depend on what else is in the batch).
                // The page loop is issue-bound on CUDA cores rather than HBM-bound, so it is written for instruction count:
                //   * 4 lanes per key (32 dims each): one pass of 4 x LDS.128 + 32 FMA covers the warp's 8 keys, 2 shuffles
                //   * scores in the log2 domain: q is staged once per chunk as q * (scale * log2 e), probabilities are exp2
                //   * the current position's key / value (from this step's QKV epilogue, not from the page) is ONE extra key
                //     folded in by warp 0 after the last page -- no per-element selects inside the loop
                constexpr int DPT = MG_HD / 32;
                float* st_sm = reinterpret_cast<float*>(bring + L::A_STATE);         // [8 warps][MG_PSTR]
                float* cs_sm = reinterpret_cast<float*>(bring + L::A_CHUNKS);        // [MG_MAXCH chunks of one item][MG_PSTR]
                float* q_sm = reinterpret_cast<float*>(bring + L::A_Q);              // [2][MG_HD]: this / the next chunk's q'
                if (P.dep_target > 0) {
                    if (lane == 0) mg_wait_flag(A.flags + (p - 1), P.dep_target, A.dbg, 5, p);
                    __syncwarp();
                }
                if (wtid == 0) mg_tl(A, p, 4);
                const int kj = lane >> 2, qc = lane & 3;                             // my key inside the warp's slice, my dim quarter
                const uint32_t it0 = it;
                const float qscale = A.scale * 1.4426950408889634f;
                int qbuf_sel = 0;
                if (u0 < u1 && wtid < MG_HD) {                                        // first chunk's q (exposed once per phase)
                    int r, h, pg, npg;
                    mg_locate(s_cum, A.H, u0, r, h, pg, npg);
                    q_sm[wtid] = __ldcg(A.qbuf + (static_cast<size_t>(r) * A.H + h) * MG_HD + wtid) * qscale;
                }
                mg_bar_workers();
                int u = u0;
                while (u < u1) {
                    int r, h, pg, npg;
                    mg_locate(s_cum, A.H, u, r, h, pg, npg);
                    const int pe = min(npg, pg + MG_CHUNK);
                    const int pos = A.row_pos[r];
                    const int rh = r * A.H + h;
                    const bool has_self = pe == npg;                                 // the chunk ends at the current position
                    // operands fetched now, used after the page loop: next chunk's q (threads < 128), my slice of k_new / v_new
                    float q_next = 0.f;
                    const int un = u + (pe - pg);
                    if (un < u1 && wtid < MG_HD) {
                        int r2, h2, pg2, npg2;
                        mg_locate(s_cum, A.H, un, r2, h2, pg2, npg2);
                        q_next = __ldcg(A.qbuf + (static_cast<size_t>(r2) * A.H + h2) * MG_HD + wtid);
                    }
                    float4 kself4 = make_float4(0.f, 0.f, 0.f, 0.f), vself4 = kself4;
                    if (has_self && wq == 0) {
                        kself4 = __ldcg(reinterpret_cast<const float4*>(A.knew + static_cast<size_t>(rh) * MG_HD + lane * DPT));
                        vself4 = __ldcg(reinterpret_cast<const float4*>(A.vnew + static_cast<size_t>(rh) * MG_HD + lane * DPT));
                    }
                    // my 32 dims of q': dims [i*32 + qc*8, +8), i = 0..3 (the same split the K loads use: 16-byte chunks of
                    // the 4 lanes of a key are adjacent, so a quarter-warp's LDS.128 touches distinct banks)
                    float qv[32];
                    {
                        const float* qs = q_sm + qbuf_sel * MG_HD;
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const float4 a0 = *reinterpret_cast<const float4*>(qs + i * 32 + qc * 8);
                            const float4 a1 = *reinterpret_cast<const float4*>(qs + i * 32 + qc * 8 + 4);
                            qv[i * 8 + 0] = a0.x; qv[i * 8 + 1] = a0.y; qv[i * 8 + 2] = a0.z; qv[i * 8 + 3] = a0.w;
                            qv[i * 8 + 4] = a1.x; qv[i * 8 + 5] = a1.y; qv[i * 8 + 6] = a1.z; qv[i * 8 + 7] = a1.w;
                        }
                    }
                    float m_run = -INFINITY, l_run = 0.f;
                    float acc[DPT];
#pragma unroll
                    for (int i = 0; i < DPT; ++i) acc[i] = 0.f;
                    const int t_key = wq * 8 + kj;                                   // my key inside the page
                    for (int pgi = pg; pgi < pe; ++pgi) {
                        const uint32_t itu = it0 + static_cast<uint32_t>(u - u0 + (pgi - pg)) * 2 * NSL;
                        uint32_t ks[NSL], vs[NSL];
#pragma unroll
                        for (int j = 0; j < NSL; ++j) {
                            ks[j] = (itu + j) % MG_NS;
                            vs[j] = (itu + NSL + j) % MG_NS;
                        }
#pragma unroll
                        for (int j = 0; j < NSL; ++j) mg_wait(&full[ks[j]], ((itu + j) / MG_NS) & 1, A.dbg, 6, p);
                        // ---- score of my key: 32 dims per lane, reduce over the key's 4 lanes
                        float dsum = 0.f;
                        {
                            const KVT* Kp = reinterpret_cast<const KVT*>(ring + ks[t_key / TPS] * MG_SLOT) + (t_key % TPS) * MG_HD + qc * 8;
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                float kvv[8];
                                mg_load_kv<KVT, 8>(Kp + i * 32, kvv);
#pragma unroll
                                for (int e2 = 0; e2 < 8; ++e2) dsum = fmaf(qv[i * 8 + e2], kvv[e2], dsum);
                            }
                        }
                        dsum += __shfl_xor_sync(0xffffffffu, dsum, 1);
                        dsum += __shfl_xor_sync(0xffffffffu, dsum, 2);
                        const float sc = (pgi * MG_PAGE + t_key < pos) ? dsum : -INFINITY;   // cached keys only: position `pos` is k_new
                        __syncwarp();
                        if (lane == 0) {
#pragma unroll
                            for (int j = 0; j < NSL; ++j) mbar_arrive(&empty[ks[j]]);       // one of the 8 warps' arrivals
                        }
                        // ---- online softmax over my 8 keys (log2 domain)
                        float pm = sc;
                        pm = fmaxf(pm, __shfl_xor_sync(0xffffffffu, pm, 4));
                        pm = fmaxf(pm, __shfl_xor_sync(0xffffffffu, pm, 8));
                        pm = fmaxf(pm, __shfl_xor_sync(0xffffffffu, pm, 16));
                        const float m_new = fmaxf(m_run, pm);
                        float pr = 0.f, corr = 1.f;
                        if (m_new != -INFINITY) {                                   // else: every key of my slice masked so far
                            corr = exp2f(m_run - m_new);
                            pr = exp2f(sc - m_new);
                        }
                        float psum = pr;                                            // the 4 lanes of a key hold the same pr
                        psum += __shfl_xor_sync(0xffffffffu, psum, 4);
                        psum += __shfl_xor_sync(0xffffffffu, psum, 8);
                        psum += __shfl_xor_sync(0xffffffffu, psum, 16);
                        l_run = l_run * corr + psum;
                        m_run = m_new;
#pragma unroll
                        for (int i = 0; i < DPT; ++i) acc[i] *= corr;
                        // ---- PV over my 8 keys: lane owns 4 output dims
#pragma unroll
                        for (int j = 0; j < NSL; ++j) mg_wait(&full[vs[j]], ((itu + NSL + j) / MG_NS) & 1, A.dbg, 7, p);
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const float pk = __shfl_sync(0xffffffffu, pr, 4 * j);
                            const int t = wq * 8 + j;
                            float vv[DPT];
                            const KVT* Vp = reinterpret_cast<const KVT*>(ring + vs[t / TPS] * MG_SLOT) + (t % TPS) * MG_HD + lane * DPT;
                            mg_load_kv<KVT, DPT>(Vp, vv);
#pragma unroll
                            for (int i = 0; i < DPT; ++i) acc[i] = fmaf(pk, vv[i], acc[i]);
                        }
                        __syncwarp();
                        if (lane == 0) {
#pragma unroll
                            for (int j = 0; j < NSL; ++j) mbar_arrive(&empty[vs[j]]);
                        }
                    }
                    // ---- the current position: one extra key (k_new, v_new from this step's QKV epilogue), folded in by warp 0
                    if (has_self && wq == 0) {
                        const float4 q4 = *reinterpret_cast<const float4*>(q_sm + qbuf_sel * MG_HD + lane * DPT);
                        float ss = q4.x * kself4.x;
                        ss = fmaf(q4.y, kself4.y, ss);
                        ss = fmaf(q4.z, kself4.z, ss);
                        ss = fmaf(q4.w, kself4.w, ss);
                        ss = warp_sum(ss);
                        const float m_new = fmaxf(m_run, ss);
                        const float corr = exp2f(m_run - m_new), ps = exp2f(ss - m_new);
                        l_run = l_run * corr + ps;
                        m_run = m_new;
                        acc[0] = fmaf(ps, vself4.x, acc[0] * corr);
                        acc[1] = fmaf(ps, vself4.y, acc[1] * corr);
                        acc[2] = fmaf(ps, vself4.z, acc[2] * corr);
                        acc[3] = fmaf(ps, vself4.w, acc[3] * corr);
                    }
                    if (un < u1 && wtid < MG_HD) q_sm[(qbuf_sel ^ 1) * MG_HD + wtid] = q_next * qscale;   // visible after the chunk's barriers
                    qbuf_sel ^= 1;
                    // ---- chunk done: fold the 8 warp states in warp order -> chunk state ---------------------------------------
                    {
                        float* ps = st_sm + wq * MG_PSTR;
                        *reinterpret_cast<float4*>(ps + lane * DPT) = make_float4(acc[0], acc[1], acc[2], acc[3]);
                        if (lane == 0) {
                            ps[MG_HD] = m_run;
                            ps[MG_HD + 1] = l_run;
                        }
                    }
                    mg_bar_workers();
                    const int n_chunks = (npg + MG_CHUNK - 1) / MG_CHUNK, cidx = pg / MG_CHUNK;
                    const size_t ocol = static_cast<size_t>(h) * MG_HD;
                    const long long ui0 = static_cast<long long>(A.H) * s_cum[r] + static_cast<long long>(h) * npg;   // item's first unit
                    // chunks owned by other CTAs too, or more chunks than cs_sm holds (contexts over MG_MAXCH * MG_CHUNK pages):
                    // the chunk states go through the workspace, which has room for max_pages of them per (row, head)
                    const bool spans = n_chunks > MG_MAXCH || ui0 < u0 || ui0 + static_cast<long long>(n_chunks - 1) * MG_CHUNK >= u1;
                    const bool item_ends_here = pe == npg || u + (pe - pg) >= u1;   // my last chunk of this item
                    float* wsi = A.att_ws + static_cast<size_t>(rh) * A.max_pages * MG_PSTR;
                    if (wtid < MG_HD) {
                        float M = -INFINITY, Ls = 0.f, O = 0.f;
#pragma unroll
                        for (int w = 0; w < 8; ++w) {
                            const float* ps = st_sm + w * MG_PSTR;
                            const float mp = ps[MG_HD];
                            if (mp == -INFINITY) continue;                          // that warp's key slice was fully masked
                            const float Mn = fmaxf(M, mp);
                            const float c1 = exp2f(M - Mn), c2 = exp2f(mp - Mn);
                            Ls = Ls * c1 + ps[MG_HD + 1] * c2;
                            O = O * c1 + ps[wtid] * c2;
                            M = Mn;
                        }
                        if (n_chunks == 1) {
                            const float o = O / Ls;
                            __nv_bfloat16 hi, lo;
                            split_bf16(o, hi, lo);
                            A.att_out[mg_act_off(static_cast<int>(ocol) + wtid, r, 2 * A.bpad)] = hi;
                            A.att_out[mg_act_off(static_cast<int>(ocol) + wtid, r + A.bpad, 2 * A.bpad)] = lo;
                        } else if (!spans) {                                        // all chunks of the item are mine: keep it on chip
                            cs_sm[cidx * MG_PSTR + wtid] = O;
                            if (wtid == 0) {
                                cs_sm[cidx * MG_PSTR + MG_HD] = M;
                                cs_sm[cidx * MG_PSTR + MG_HD + 1] = Ls;
                            }
                        } else {
                            __stcg(wsi + static_cast<size_t>(cidx) * MG_PSTR + wtid, O);
                            if (wtid == 0) {
                                __stcg(wsi + static_cast<size_t>(cidx) * MG_PSTR + MG_HD, M);
                                __stcg(wsi + static_cast<size_t>(cidx) * MG_PSTR + MG_HD + 1, Ls);
                            }
                        }
                    }
                    if (n_chunks > 1 && item_ends_here) {
                        // fold the item's chunk states in chunk order: from shared memory if they are all mine, else the
                        // CTAs that own chunks of the item count in and the last one folds them from the workspace
                        bool do_fold = true;
                        mg_bar_workers();
                        if (spans) {
                            if (wtid == 0) {
                                int n_cta = 0, prev = -1;
                                for (int j = 0; j < n_chunks; ++j) {
                                    const int o = mg_owner(ui0 + static_cast<long long>(j) * MG_CHUNK, U, Ue);
                                    n_cta += o != prev;
                                    prev = o;
                                }
                                __threadfence();
                                *s_flag = (atomicAdd(A.att_cnt + rh, 1) == n_cta - 1);
                                __threadfence();
                            }
                            mg_bar_workers();
                            do_fold = *s_flag != 0;
                        }
                        if (do_fold && wtid < MG_HD) {
                            float M = -INFINITY, Ls = 0.f, O = 0.f;
                            for (int j = 0; j < n_chunks; ++j) {
                                float mp, lp, op;
                                if (spans) {
                                    const float* ps = wsi + static_cast<size_t>(j) * MG_PSTR;
                                    mp = __ldcg(ps + MG_HD);
                                    lp = __ldcg(ps + MG_HD + 1);
                                    op = __ldcg(ps + wtid);
                                } else {
                                    mp = cs_sm[j * MG_PSTR + MG_HD];
                                    lp = cs_sm[j * MG_PSTR + MG_HD + 1];
                                    op = cs_sm[j * MG_PSTR + wtid];
                                }
                                const float Mn = fmaxf(M, mp);
                                const float c1 = exp2f(M - Mn), c2 = exp2f(mp - Mn);
                                Ls = Ls * c1 + lp * c2;
                                O = O * c1 + op * c2;
                                M = Mn;
                            }
                            const float o = O / Ls;
                            __nv_bfloat16 hi, lo;
                            split_bf16(o, hi, lo);
                            A.att_out[mg_act_off(static_cast<int>(ocol) + wtid, r, 2 * A.bpad)] = hi;
                            A.att_out[mg_act_off(static_cast<int>(ocol) + wtid, r + A.bpad, 2 * A.bpad)] = lo;
                        }
                        if (spans && do_fold && wtid == 0) A.att_cnt[rh] = 0;
                    }
                    mg_bar_workers();                                               // warp / chunk states and s_flag are reused
                    u += pe - pg;
                }
                it = it0 + static_cast<uint32_t>(u1 - u0) * 2 * NSL;
                // this CTA's share of the phase is done (merged outputs are counted by whoever merged them)
                if (wtid == 0) mg_tl(A, p, 5);
                __threadfence();
                mg_bar_workers();
                if (wtid == 0) {
                    mg_fence_proxy_async();
                    __threadfence();
                    atomicAdd(A.flags + p, 1u);
                    mg_tl(A, p, 6);
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------------
template <int BPAD, typename KVT>
static int mega_launch_t(const MegaArgs& a, int grid, cudaStream_t st) {
    static bool attr_set = false;
    if (!attr_set) {
        VCB_CUDA_OK(cudaFuncSetAttribute(mega_step_kernel<BPAD, KVT>, cudaFuncAttributeMaxDynamicSharedMemorySize, MegaSmem::TOTAL));
        attr_set = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(MG_THREADS);
    cfg.dynamicSmemBytes = MegaSmem::TOTAL;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeCooperative;       // every CTA must be co-resident: the phase hand-over spins on peers
    at[0].val.cooperative = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    VCB_CUDA_OK(cudaLaunchKernelEx(&cfg, mega_step_kernel<BPAD, KVT>, a));
    return 0;
}

int mega_launch(const MegaArgs& a, int grid, cudaStream_t st) {
    if (a.bpad == 32) return a.kv_fp32 ? mega_launch_t<32, float>(a, grid, st) : mega_launch_t<32, __nv_bfloat16>(a, grid, st);
    if (a.bpad == 16) return a.kv_fp32 ? mega_launch_t<16, float>(a, grid, st) : mega_launch_t<16, __nv_bfloat16>(a, grid, st);
    set_error("mega_launch: unsupported bpad %d", a.bpad);
    return -1;
}

// co-resident CTAs the device offers this kernel (one per SM: the ring takes the whole shared memory)
int mega_max_grid(int bpad, int kv_fp32) {
    int dev = 0, sms = 0, per_sm = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    cudaError_t e;
    auto occ = [&](auto kern) {
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, MegaSmem::TOTAL);
        if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, MG_THREADS, MegaSmem::TOTAL);
    };
    if (bpad == 32) kv_fp32 ? occ(mega_step_kernel<32, float>) : occ(mega_step_kernel<32, __nv_bfloat16>);
    else kv_fp32 ? occ(mega_step_kernel<16, float>) : occ(mega_step_kernel<16, __nv_bfloat16>);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return sms * std::min(per_sm, 1);
}

size_t mega_part_floats(int grid, int bpad) { return static_cast<size_t>(grid) * MEGA_MAXSEG * bpad * 128; }

// The ring depths must fit the pool.  The ring producer may have at most ns loads in flight: it waits for the oldest
// in-flight load on its slot's full barrier with that load's phase parity, and with more than ns in flight the slot has
// been refilled since, so the parity names a later phase that only loads it has not issued yet can complete.
int mega_ring_config(int ns, int nb, int flight, int* out) {
    if (ns < MG_NS_MIN || ns > MG_NS_MAX || nb < MG_NB_MIN || nb > MG_NB_MAX || ns * MG_SLOT + nb * MG_BSLOT > MG_POOL) {
        set_error("VCB_MEGA_NS / VCB_MEGA_NB = %d / %d: need %d <= ns <= %d, %d <= nb <= %d and ns * 16 KB + nb * 8 KB <= %d KB", ns,
                  nb, MG_NS_MIN, MG_NS_MAX, MG_NB_MIN, MG_NB_MAX, MG_POOL / 1024);
        return -1;
    }
    out[0] = ns;
    out[1] = nb;
    out[2] = std::min(std::max(flight, 1), ns);
    return 0;
}

}  // namespace vcb
