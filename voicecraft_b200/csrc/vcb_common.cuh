// Common device helpers for the sm_90a kernels: mbarrier / TMA / wgmma PTX wrappers, small math utils.
// Everything here is hand-written PTX for Hopper (no CUTLASS dependency).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vcb {

// ------------------------------------------------------------------------------------------------
// error plumbing (host)
// ------------------------------------------------------------------------------------------------
#define VCB_CUDA_OK(expr)                                                                         \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess) {                                                                  \
            vcb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return -1;                                                                            \
        }                                                                                         \
    } while (0)

void set_error(const char* fmt, ...);
const char* get_error();

// ------------------------------------------------------------------------------------------------
// LayerNorm row statistics of the folded LayerNorm: per tile of features the producer leaves (sum x, M2 = sum (x - tile
// mean)^2); consumers combine the tiles in tile order as mean = sum / d, M2 = sum_t (M2_t + n_t (mean_t - mean)^2).
// Centred partials keep the variance exact to fp32 rounding of the spread, where E[x^2] - mean^2 loses (mean/std)^2 of it;
// the terms are independent (no dependent division chain ahead of a GEMM mainloop).
// ------------------------------------------------------------------------------------------------
// features in tile t of `tiles` tiles over d features (a single tile holds the whole row, else 128 per tile)
__device__ __forceinline__ float ln_tile_n(int t, int tiles, int d) {
    return tiles == 1 ? static_cast<float>(d) : static_cast<float>(min(128, d - 128 * t));
}
// one tile's contribution to the row's M2 given the row mean
__device__ __forceinline__ float ln_tile_m2(float n, float sum, float m2, float mean) {
    const float dm = (n == 128.f ? sum * 0.0078125f : sum / n) - mean;
    return fmaf(n * dm, dm, m2);
}

// ------------------------------------------------------------------------------------------------
// bf16 split:  x ~= hi + lo with hi = bf16(x), lo = bf16(x - hi).  Residual error <= 2^-17 |x|.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    hi = __float2bfloat16_rn(x);
    lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ------------------------------------------------------------------------------------------------
// shared-memory address, mbarrier
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// ------------------------------------------------------------------------------------------------
// TMA: tiled tensor load (2D) and plain bulk copy, both completing on an mbarrier
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// c0 = innermost coordinate (elements), c1 = row
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// contiguous global -> shared, bytes % 16 == 0, both 16B aligned
__device__ __forceinline__ void tma_bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// L2 cache policies / prefetch.  Streams that are touched once per step (KV pages, weight tiles) are loaded with
// evict_first so they do not push the *prefetched* next-kernel weights out of the 50 MB L2.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                 uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
        : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s_hint(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar,
                                                  uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
// asynchronous HBM -> L2 prefetch of a contiguous range (bytes % 16 == 0)
__device__ __forceinline__ void tma_prefetch_l2(const void* gsrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes) : "memory");
}
// this CTA's share of a [ptr, ptr+bytes) range, issued by one thread in <= 32 KB pieces
__device__ __forceinline__ void prefetch_l2_slice(const void* ptr, unsigned long long bytes, unsigned int part, unsigned int nparts) {
    if (ptr == nullptr || bytes == 0) return;
    unsigned long long chunk = ((bytes + nparts - 1) / nparts + 127ull) & ~127ull;
    unsigned long long beg = chunk * part;
    if (beg >= bytes) return;
    unsigned long long end = beg + chunk < bytes ? beg + chunk : bytes;
    const char* p = static_cast<const char*>(ptr);
    for (unsigned long long o = beg; o < end; o += 32768ull) {
        const unsigned long long n = (end - o < 32768ull ? end - o : 32768ull) & ~15ull;
        if (n) tma_prefetch_l2(p + o, static_cast<uint32_t>(n));
    }
}

// Optional device-side timeline (debug): CTA 0 of instrumented kernels appends (tag, globaltimer ns) records.
// Each translation unit has its own copy of the pointer; the host sets them through vcb_timeline_set().
static __constant__ unsigned long long* g_tl_buf = nullptr;   // constant bank: the disabled check costs no L2 round trip
static __constant__ unsigned int* g_tl_cnt = nullptr;
__device__ __forceinline__ void tl_mark(unsigned int tag) {
#ifndef VCB_TIMELINE
    (void)tag;                                   // compiled out by default: even the disabled check is a load per mark on the
    return;                                      // latency-bound decode chain; `make TIMELINE=1` builds it in
#endif
    if (g_tl_buf != nullptr && blockIdx.x == 0 && blockIdx.y == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        const unsigned int i = atomicAdd(g_tl_cnt, 1u);
        if (i < 65536u) {
            g_tl_buf[2 * i] = tag;
            g_tl_buf[2 * i + 1] = t;
        }
    }
}

// Every CTA records (vcb_timeline(2, ...)): tag | 0x8000 | cta << 16 -- used to see launch skew and stragglers.
__device__ __forceinline__ void tl_mark_all(unsigned int tag) {
#ifndef VCB_TIMELINE
    (void)tag;
    return;
#endif
    if (g_tl_buf != nullptr && g_tl_cnt[1] != 0u) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        const unsigned int i = atomicAdd(g_tl_cnt, 1u);
        if (i < 65536u) {
            g_tl_buf[2 * i] = tag | 0x8000u | ((blockIdx.x + gridDim.x * blockIdx.y) << 16);
            g_tl_buf[2 * i + 1] = t;
        }
    }
}

// Programmatic dependent launch (PDL): wait for the producer grid / let the consumer grid start.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------
// wgmma (sm_90a): one warpgroup (4 aligned warps) computes D[64 x N] += A[64 x 16] * B[N x 16]^T, both operands K-major
// in shared memory, fp32 accumulators in registers.  Accumulator fragment of thread t of the warpgroup (warp w = t / 32,
// lane l): for every 8-column block j, d[4j + 0..1] = row 16w + l/4, columns 8j + 2(l%4) + 0..1, and d[4j + 2..3] = the
// same columns of row 16w + l/4 + 8.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// all but the most recent group complete: the MMAs of k-block i run while k-block i+1 is issued
__device__ __forceinline__ void wg_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
// orders every later use of the accumulators after wg_wait0() (the asm outputs of wgmma are only valid once it returns)
template <int N>
__device__ __forceinline__ void wg_acc_fence(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ void wgmma_m64n16(float* d, uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a_desc), "l"(b_desc));
}
__device__ __forceinline__ void wgmma_m64n32(float* d, uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a_desc), "l"(b_desc));
}
__device__ __forceinline__ void wgmma_m64n64(float* d, uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc));
}

// K-major operand tile in shared memory, rows of 128 bytes (64 bf16), 128B swizzle (what TMA SWIZZLE_128B writes):
// 8-row x 128B swizzle atoms, atoms stacked every 1024 B.  sm_90 matrix descriptor:
//   [0,14) start>>4 | [16,30) LBO>>4 (unused for swizzled K-major) | [32,46) SBO>>4 | [62,64) layout (1 = SWIZZLE_128B)
// Advancing 16 K-elements inside the swizzle row is +32 B = +2 on the start field; 64 rows further is +8192 B.
__device__ __forceinline__ uint64_t gmma_desc_kmajor_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>(1) << 16;                       // LBO (ignored), canonical value 1
    d |= static_cast<uint64_t>(1024 >> 4) << 32;               // SBO: 8 rows * 128 B
    d |= static_cast<uint64_t>(1) << 62;                       // SWIZZLE_128B
    return d;
}

// D[64 x N] += A[64 rows at a_addr] * B[N rows at b_addr]^T over one 64-wide k-block (4 x k16), N issued in pieces of at
// most 64 columns.  Called by all 128 threads of a warpgroup between wg_fence() and wg_commit().
template <int N>
__device__ __forceinline__ void wg_mma_kblock(float (&d)[N / 2], uint32_t a_addr, uint32_t b_addr) {
    static_assert(N % 16 == 0 && (N <= 64 || N % 64 == 0), "N: 16, 32, 64 or a multiple of 64");
    constexpr int NC = N < 64 ? N : 64;
    const uint64_t a = gmma_desc_kmajor_sw128(a_addr), b = gmma_desc_kmajor_sw128(b_addr);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
#pragma unroll
        for (int n0 = 0; n0 < N; n0 += NC) {
            const uint64_t bk = b + static_cast<uint64_t>(n0 * 8) + 2 * k;     // n0 rows * 128 B, >> 4
            if constexpr (NC == 64) wgmma_m64n64(d + n0 / 2, a + 2 * k, bk);
            else if constexpr (NC == 32) wgmma_m64n32(d + n0 / 2, a + 2 * k, bk);
            else wgmma_m64n16(d + n0 / 2, a + 2 * k, bk);
        }
    }
}

// The same k16 step with A from registers: a[4] = the thread's bf16x2 fragment (rows 16w + l/4 and + 8; k 2(l%4), +1, +8,
// +9: a[0] row r k 2t.., a[1] row r+8, a[2] row r k 2t+8.., a[3] row r+8).  Written before the wg_fence() of the issue.
__device__ __forceinline__ void wgmma_m64n16_ra(float* d, const uint32_t (&a)[4], uint64_t b_desc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc));
}
__device__ __forceinline__ void wgmma_m64n32_ra(float* d, const uint32_t (&a)[4], uint64_t b_desc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc));
}
__device__ __forceinline__ void wgmma_m64n64_ra(float* d, const uint32_t (&a)[4], uint64_t b_desc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc));
}
// wg_mma_kblock's step k (0..3) of the 64-wide k-block at b_addr, A from registers; the same N pieces in the same order
template <int N>
__device__ __forceinline__ void wg_mma_k16_ra(float (&d)[N / 2], const uint32_t (&a)[4], uint32_t b_addr, int k) {
    constexpr int NC = N < 64 ? N : 64;
    const uint64_t b = gmma_desc_kmajor_sw128(b_addr) + 2 * k;
#pragma unroll
    for (int n0 = 0; n0 < N; n0 += NC) {
        const uint64_t bk = b + static_cast<uint64_t>(n0 * 8);
        if constexpr (NC == 64) wgmma_m64n64_ra(d + n0 / 2, a, bk);
        else if constexpr (NC == 32) wgmma_m64n32_ra(d + n0 / 2, a, bk);
        else wgmma_m64n16_ra(d + n0 / 2, a, bk);
    }
}

}  // namespace vcb
