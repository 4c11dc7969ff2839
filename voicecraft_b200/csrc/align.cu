// Text-speech alignment from the codec LM's attention (DESIGN.md section 4.6):
//   align_probe_kernel  per row that asks for it, the selected heads' softmax weights over the text keys, averaged
//   mas_kernel          monotonic alignment search (Glow-TTS) over log p [T][X] -> per-token durations
// Neither kernel is on the path of a pass that asks for no alignment.
#include "../../include/vcb200.h"
#include "vcb_internal.h"

#include <cmath>

namespace vcb {

namespace {

constexpr int PROBE_WARPS = 8;
constexpr int PROBE_UNROLL = 4;   // keys per warp in flight
constexpr int PAGE = 64;          // tokens per KV page (KV_PAGE of lm_kernels.cuh)

// N = hd / 32 (2 or 4) consecutive elements of one K row in one vector load (4 .. 16 bytes), widened to fp32 exactly
template <int N>
__device__ __forceinline__ void load_vec(const float* p, float (&o)[N]) {
    if constexpr (N == 4) {
        const float4 v = *reinterpret_cast<const float4*>(p);
        o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
    } else {
        const float2 v = *reinterpret_cast<const float2*>(p);
        o[0] = v.x; o[1] = v.y;
    }
}
template <int N>
__device__ __forceinline__ void load_vec(const __nv_bfloat16* p, float (&o)[N]) {
    uint32_t w[2];
    if constexpr (N == 4) {
        const uint2 v = *reinterpret_cast<const uint2*>(p);
        w[0] = v.x; w[1] = v.y;
    } else {
        w[0] = *reinterpret_cast<const uint32_t*>(p);
    }
#pragma unroll
    for (int i = 0; i < N / 2; ++i) {
        o[2 * i] = __uint_as_float(w[i] << 16);
        o[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
}
template <int N>
__device__ __forceinline__ void load_vec(const __nv_fp8_e4m3* p, float (&o)[N]) {
    const uint32_t w = N == 4 ? *reinterpret_cast<const uint32_t*>(p) : *reinterpret_cast<const uint16_t*>(p);
#pragma unroll
    for (int i = 0; i < N / 2; ++i) {
        const float2 f = kv_fp8_unpack2(w >> (16 * i));
        o[2 * i] = f.x;
        o[2 * i + 1] = f.y;
    }
}

// s_j = scale * q . k_j (fp8: times the token's scale): lane e multiplies its elements e*N .. e*N+N-1 in order, then a
// xor butterfly, which leaves the same bits in every lane.  Depends only on q, k_j and the code below, not on where k_j
// lives.
template <typename KVT, int HD>
__device__ __forceinline__ const KVT* key_ptr(const AlignProbeArgs& a, const int* pages, int h, int j) {
    const uint8_t* slab = static_cast<const uint8_t*>(a.kpool) +
                          (static_cast<size_t>(pages[j / PAGE]) * a.H + h) * kv_slab_bytes(sizeof(KVT) == 1 ? KV_FP8 : sizeof(KVT) == 4 ? KV_FP32 : KV_BF16, HD);
    return reinterpret_cast<const KVT*>(slab) + (j % PAGE) * HD;
}

template <typename KVT, int HD>
__device__ __forceinline__ float key_scale(const KVT* k, int j) {
    if constexpr (sizeof(KVT) == 1) {
        const KVT* slab = k - (j % PAGE) * HD;
        return reinterpret_cast<const float*>(slab + PAGE * HD)[j % PAGE];
    } else {
        return 1.f;
    }
}

template <typename KVT, int HD>
__device__ __forceinline__ void scores(const AlignProbeArgs& a, const int* pages, int h, const float (&qv)[HD / 32], int j0,
                                       int jend, int stride, float (&s)[PROBE_UNROLL]) {
    const int lane = threadIdx.x & 31;
    float kv[PROBE_UNROLL][HD / 32], ks[PROBE_UNROLL];
#pragma unroll
    for (int u = 0; u < PROBE_UNROLL; ++u) {
        const int j = j0 + u * stride;
        if (j < jend) {
            const KVT* k = key_ptr<KVT, HD>(a, pages, h, j);
#pragma unroll
            load_vec<HD / 32>(k + lane * (HD / 32), kv[u]);
            ks[u] = key_scale<KVT, HD>(k, j);
        } else {
#pragma unroll
            for (int i = 0; i < HD / 32; ++i) kv[u][i] = 0.f;
            ks[u] = 1.f;
        }
    }
#pragma unroll
    for (int u = 0; u < PROBE_UNROLL; ++u) {
        float d = 0.f;
#pragma unroll
        for (int i = 0; i < HD / 32; ++i) d = fmaf(qv[i], kv[u][i], d);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        s[u] = d * ks[u] * a.scale;
    }
}

}  // namespace

template <typename KVT, int HD>
__global__ void __launch_bounds__(PROBE_WARPS * 32) align_probe_kernel(const __grid_constant__ AlignProbeArgs a) {
    extern __shared__ float acc[];            // [x_len]: sum over the selected heads of this layer
    __shared__ float red_m[PROBE_WARPS], red_l[PROBE_WARPS];
    const int r = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int pos = a.row_pos[r];
    if (pos < 0) return;
    const int slot = a.row_slot[r];
    const uint32_t* masks = a.masks + static_cast<size_t>(slot) * a.L;
    const uint32_t mask = masks[a.layer];
    if (!mask) return;
    const int xl = min(a.slot_xlen[static_cast<size_t>(slot) * a.xlen_stride], a.cap);
    if (pos < xl) return;                     // text rows are no frame
    int first = -1, last = -1, n_heads = 0;
    for (int l = 0; l < a.L; ++l)
        if (masks[l]) {
            if (first < 0) first = l;
            last = l;
            n_heads += __popc(masks[l]);
        }
    const int* pages = a.row_pages ? a.row_pages + static_cast<size_t>(r) * a.max_pages
                                   : a.page_table + static_cast<size_t>(slot) * a.max_pages;
    for (int j = threadIdx.x; j < xl; j += blockDim.x) acc[j] = 0.f;
    __syncthreads();
    for (uint32_t hm = mask; hm; hm &= hm - 1) {
        const int h = __ffs(hm) - 1;
        float qv[HD / 32];
        const float* q = a.q + static_cast<size_t>(r) * a.q_ld + h * HD;
#pragma unroll
        for (int i = 0; i < HD / 32; ++i) qv[i] = q[lane * (HD / 32) + i];
        // pass 1: running max and sum of exp(s - max) per warp over keys warp, warp + 8, ..., then the warps in order
        float m = -INFINITY, l = 0.f;
        for (int j0 = warp; j0 <= pos; j0 += PROBE_WARPS * PROBE_UNROLL) {
            float s[PROBE_UNROLL];
            scores<KVT, HD>(a, pages, h, qv, j0, pos + 1, PROBE_WARPS, s);
#pragma unroll
            for (int u = 0; u < PROBE_UNROLL; ++u) {
                if (j0 + u * PROBE_WARPS > pos) break;
                const float mn = fmaxf(m, s[u]);
                l = l * expf(m - mn) + expf(s[u] - mn);
                m = mn;
            }
        }
        if (lane == 0) {
            red_m[warp] = m;
            red_l[warp] = l;
        }
        __syncthreads();
        float M = red_m[0];
        for (int w = 1; w < PROBE_WARPS; ++w) M = fmaxf(M, red_m[w]);
        float S = 0.f;
        for (int w = 0; w < PROBE_WARPS; ++w) S += red_l[w] * expf(red_m[w] - M);
        __syncthreads();                      // red_* are rewritten by the next head
        // pass 2: p_j = exp(s_j - M) / S over the text keys; key j's sum over heads is kept by warp j % 8, heads ascending
        for (int j0 = warp; j0 < xl; j0 += PROBE_WARPS * PROBE_UNROLL) {
            float s[PROBE_UNROLL];
            scores<KVT, HD>(a, pages, h, qv, j0, xl, PROBE_WARPS, s);
#pragma unroll
            for (int u = 0; u < PROBE_UNROLL; ++u) {
                const int j = j0 + u * PROBE_WARPS;
                if (j < xl && lane == 0) acc[j] += expf(s[u] - M) / S;
            }
        }
    }
    __syncthreads();
    float* dst = a.log ? a.log + (static_cast<size_t>(slot) * a.max_seq + pos) * a.cap : a.out + static_cast<size_t>(r) * a.cap;
    for (int j = threadIdx.x; j < xl; j += blockDim.x) {
        float v = acc[j];
        if (a.layer != first) v += dst[j];    // layers ascending: the earlier layers' sums
        if (a.layer == last) v /= static_cast<float>(n_heads);
        dst[j] = v;
    }
}

int align_probe_launch(const AlignProbeArgs& a, cudaStream_t st) {
    if (a.rows < 1) return 0;
    const size_t smem = static_cast<size_t>(std::max(a.cap, 1)) * sizeof(float);
    const dim3 grid(a.rows), block(PROBE_WARPS * 32);
    auto go = [&](auto kern) -> int {
        if (smem > 48 * 1024) VCB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        kern<<<grid, block, smem, st>>>(a);
        VCB_CUDA_OK(cudaGetLastError());
        return 0;
    };
    if (a.hd != 64 && a.hd != 128) {
        set_error("alignment probe: head dim %d (64 or 128 supported)", a.hd);
        return -1;
    }
    if (a.kv_dtype == KV_FP32) return a.hd == 128 ? go(align_probe_kernel<float, 128>) : go(align_probe_kernel<float, 64>);
    if (a.kv_dtype == KV_FP8)
        return a.hd == 128 ? go(align_probe_kernel<__nv_fp8_e4m3, 128>) : go(align_probe_kernel<__nv_fp8_e4m3, 64>);
    return a.hd == 128 ? go(align_probe_kernel<__nv_bfloat16, 128>) : go(align_probe_kernel<__nv_bfloat16, 64>);
}

// Monotonic alignment search, one CTA: Q[t][x] = max(Q[t-1][x], Q[t-1][x-1]) + lp[t][x] over the cells a path from (0, 0)
// to (T-1, X-1) can reach (x <= t), fp32, a thread per column and t ascending; the choice of each cell (1: from x - 1)
// goes to `dir`.  Backtracking from (T-1, X-1) by one thread: at x == t the path must step down, at x == 0 it stays, else
// it steps down only when Q[t-1][x-1] > Q[t-1][x] (a tie stays on the current token).
__global__ void __launch_bounds__(1024) mas_kernel(const float* __restrict__ lp, int T, int X, uint8_t* __restrict__ dir,
                                                   int* __restrict__ dur) {
    extern __shared__ float q[];              // [2][X]
    for (int x = threadIdx.x; x < X; x += blockDim.x) q[x] = x == 0 ? lp[0] : -INFINITY;
    __syncthreads();
    for (int t = 1; t < T; ++t) {
        const float* prev = q + ((t - 1) & 1) * X;
        float* cur = q + (t & 1) * X;
        for (int x = threadIdx.x; x < X; x += blockDim.x) {
            float v = -INFINITY;
            uint8_t d = 0;
            if (x <= t) {
                const float stay = x < t ? prev[x] : -INFINITY, down = x > 0 ? prev[x - 1] : -INFINITY;
                d = x == t || (x > 0 && down > stay);
                v = (d ? down : stay) + lp[static_cast<size_t>(t) * X + x];
            }
            cur[x] = v;
            dir[static_cast<size_t>(t) * X + x] = d;
        }
        __syncthreads();
    }
    for (int x = threadIdx.x; x < X; x += blockDim.x) dur[x] = 0;
    __syncthreads();
    if (threadIdx.x == 0) {
        int x = X - 1;
        for (int t = T - 1; t >= 0; --t) {
            ++dur[x];
            if (t > 0 && dir[static_cast<size_t>(t) * X + x]) --x;
        }
    }
}

}  // namespace vcb

using namespace vcb;

extern "C" {

int vcb_align_monotonic(const float* logp_dev, int32_t T, int32_t X, int32_t* durations_dev, void* stream) {
    if (!logp_dev || !durations_dev || X < 1 || T < X || X > VCB_ALIGN_MAX_TEXT) {
        set_error("vcb_align_monotonic: need 1 <= X <= %d and T >= X (T=%d X=%d) and non-null pointers", VCB_ALIGN_MAX_TEXT,
                  T, X);
        return -1;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    uint8_t* dir = nullptr;
    VCB_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&dir), static_cast<size_t>(T) * X, st));
    const size_t smem = 2 * static_cast<size_t>(X) * sizeof(float);
    if (smem > 48 * 1024) VCB_CUDA_OK(cudaFuncSetAttribute(mas_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    mas_kernel<<<1, std::min(1024, (X + 31) / 32 * 32), smem, st>>>(logp_dev, T, X, dir, durations_dev);
    const cudaError_t e = cudaGetLastError();
    cudaFreeAsync(dir, st);
    VCB_CUDA_OK(e);
    return 0;
}

int vcb_debug_align_probe(const float* q_dev, const void* kpool_dev, int32_t kv_dtype, const int32_t* row_pages_dev,
                          const int32_t* pos_dev, int32_t rows, int32_t H, int32_t hd, int32_t max_pages, uint32_t head_mask,
                          int32_t x_len, float* out_dev) {
    if (!q_dev || !kpool_dev || !row_pages_dev || !pos_dev || !out_dev || rows < 1 || H < 1 || H > 32 || max_pages < 1 ||
        (kv_dtype != KV_BF16 && kv_dtype != KV_FP32 && kv_dtype != KV_FP8) || head_mask == 0 ||
        (H < 32 && (head_mask >> H) != 0) || x_len < 1 || x_len > VCB_ALIGN_MAX_TEXT) {
        set_error("vcb_debug_align_probe: bad argument (rows=%d H=%d hd=%d max_pages=%d kv_dtype=%d mask=%#x x_len=%d)", rows,
                  H, hd, max_pages, kv_dtype, head_mask, x_len);
        return -1;
    }
    DevBuf<int> tab;                          // row_slot = r, masks [rows][1], x_len per "slot"
    if (tab.alloc(3 * static_cast<size_t>(rows))) return -1;
    std::vector<int> h(3 * static_cast<size_t>(rows));
    for (int r = 0; r < rows; ++r) {
        h[r] = r;
        h[rows + r] = static_cast<int>(head_mask);
        h[2 * rows + r] = x_len;
    }
    VCB_CUDA_OK(cudaMemcpy(tab, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice));
    AlignProbeArgs a;
    a.q = q_dev;
    a.q_ld = H * hd;
    a.kpool = kpool_dev;
    a.kv_dtype = kv_dtype;
    a.row_pages = row_pages_dev;
    a.row_slot = tab;
    a.row_pos = pos_dev;
    a.max_pages = max_pages;
    a.rows = rows;
    a.H = H;
    a.hd = hd;
    a.L = 1;
    a.layer = 0;
    a.masks = reinterpret_cast<const uint32_t*>(tab.get() + rows);
    a.slot_xlen = tab.get() + 2 * rows;
    a.xlen_stride = 1;
    a.cap = x_len;
    a.scale = 1.0f / sqrtf(static_cast<float>(hd));
    a.out = out_dev;
    if (align_probe_launch(a, nullptr)) return -1;
    VCB_CUDA_OK(cudaDeviceSynchronize());
    return 0;
}

}  // extern "C"
