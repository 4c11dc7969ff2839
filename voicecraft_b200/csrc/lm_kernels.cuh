// Device kernels of the codec-LM decode path (everything except the tensor-core GEMMs).
// All of them are HBM/L2-bound integer or fp32 work: coalesced 16-byte accesses, warp-level reductions,
// TMA bulk copies for the paged KV cache.  Included only by lm_engine.cu.
#pragma once
#include "../../include/vcb200.h"
#include "vcb_internal.h"

namespace vcb {

static constexpr int KV_PAGE = 64;          // tokens per KV page
static constexpr int ATT_CWARPS = 8;            // consumer warps per CTA
static constexpr int ATT_THREADS = ATT_CWARPS * 32;
static constexpr int ATT_STAGES = 3;
static constexpr int ATT_CHUNK_PAGES = 16;      // default pages per attention work item (VCB_ATT_CHUNK_PAGES overrides)
static constexpr int ATT_GMAX = 8;              // rows per row group of the grouped attention (larger groups are split)

__device__ __forceinline__ float block_sum_256(float v, float* red /*[8]*/) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) red[w] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i];
    return t;
}

// ---------------------------------------------------------------------------------------------------
// Prompt embedding:  text rows  x = E_text[id] + alpha_t * PE[i]          (voicecraft.py:950-951)
//                    audio rows x = sum_k E_k[tok_k] (or mask_embedding[r]) + alpha_a * PE[j]   (:978-985, 311-320)
// One CTA per row of the prefill chunk.  fp32 throughout; alpha*pe is rounded before the add, like eager torch.
// ---------------------------------------------------------------------------------------------------
struct EmbedSeq {
    const long long* text_ids;
    const long long* y_tokens;   // [y_len][K]
    const int* mask_rows;        // [y_len] or null
    int x_len, y_len;
};

__global__ void embed_rows_kernel(const EmbedSeq* __restrict__ seqs, const int* __restrict__ row_seq,
                                  const int* __restrict__ row_pos, float* __restrict__ x_rows, int d, int K,
                                  const float* __restrict__ E_text, const float* const* __restrict__ E_audio,
                                  const float* __restrict__ mask_emb, const float* __restrict__ pe, float alpha_t,
                                  float alpha_a) {
    const int r = blockIdx.x;
    const EmbedSeq s = seqs[row_seq[r]];
    const int pos = row_pos[r];
    float* out = x_rows + static_cast<size_t>(r) * d;
    if (pos < s.x_len) {
        const float* e = E_text + static_cast<size_t>(s.text_ids[pos]) * d;
        const float* p = pe + static_cast<size_t>(pos) * d;
        for (int c = threadIdx.x; c < d; c += blockDim.x) out[c] = __fadd_rn(e[c], __fmul_rn(alpha_t, p[c]));
    } else {
        const int j = pos - s.x_len;
        const float* p = pe + static_cast<size_t>(j) * d;
        const int mr = s.mask_rows ? s.mask_rows[j] : -1;
        for (int c = threadIdx.x; c < d; c += blockDim.x) {
            float acc;
            if (mr >= 0) {
                acc = mask_emb[static_cast<size_t>(mr) * d + c];
            } else {
                acc = 0.f;
                for (int k = 0; k < K; ++k) {
                    const float v = E_audio[k][static_cast<size_t>(s.y_tokens[static_cast<size_t>(j) * K + k]) * d + c];
                    acc = (k == 0) ? v : __fadd_rn(acc, v);
                }
            }
            out[c] = __fadd_rn(acc, __fmul_rn(alpha_a, p[c]));
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// LayerNorm of the fp32 residual stream -> bf16 hi / lo rows of the next GEMM's B operand.
// Replaces F.layer_norm (transformer.py:62-75); the residual adds live in the GEMM epilogue (EPI_RESID).
// One CTA per row; two-pass variance in registers.
// ---------------------------------------------------------------------------------------------------
template <int MAXV>
__global__ void __launch_bounds__(256)
ln_rows_kernel(const float* __restrict__ x_in, const int* __restrict__ src_index, const float* __restrict__ gamma,
               const float* __restrict__ beta, __nv_bfloat16* __restrict__ act, int ld_act, int bpad, int d, float eps) {
    __shared__ float red[8];
    pdl_launch_dependents();          // let the consumer GEMM start prefetching its weights right away
    if (threadIdx.x == 0) tl_mark(0x200);
    pdl_wait();
    if (threadIdx.x == 0) tl_mark(0x210);
    const int r = blockIdx.x;
    const int src = src_index ? src_index[r] : r;
    float v[MAXV];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
        const int c = threadIdx.x + j * 256;
        v[j] = (c < d) ? x_in[static_cast<size_t>(src) * d + c] : 0.f;
        s += v[j];
    }
    const float mean = block_sum_256(s, red) / d;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
        const int c = threadIdx.x + j * 256;
        if (c < d) {
            const float dv = v[j] - mean;
            q += dv * dv;
        }
    }
    const float var = block_sum_256(q, red) / d;
    const float rstd = 1.0f / sqrtf(var + eps);
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
        const int c = threadIdx.x + j * 256;
        if (c < d) {
            const float y = (v[j] - mean) * rstd * gamma[c] + beta[c];
            __nv_bfloat16 hi, lo;
            split_bf16(y, hi, lo);
            act[static_cast<size_t>(r) * ld_act + c] = hi;
            act[static_cast<size_t>(r + bpad) * ld_act + c] = lo;
        }
    }
    if (threadIdx.x == 0) tl_mark(0x230);
}

// hidden state of the last token of each utterance: out[out_index[row]] = x[row]   (prefill -> first sampling step)
__global__ void gather_rows_kernel(const float* __restrict__ x_in, float* __restrict__ out,
                                   const int* __restrict__ out_index, int d) {
    pdl_launch_dependents();
    pdl_wait();
    const int r = blockIdx.x;
    const int dst = out_index[r];
    if (dst < 0) return;
    for (int c = threadIdx.x; c < d; c += blockDim.x)
        out[static_cast<size_t>(dst) * d + c] = x_in[static_cast<size_t>(r) * d + c];
}

// Best-of-N prefill: only the group's leader runs through the layers; its members share the leader's full prompt pages
// and get a copy of what else the prefill left for the leader: the partial tail page (every layer's K and V pool) and the
// last hidden state the first sampling step reads.  Plain copies, so a member's bits are those its own prefill would write.
struct ForkPair {
    int src_slot, dst_slot;
    int src_page, dst_page;      // partial tail page, or -1: the prompt fills its last page
};

__global__ void fork_group_kernel(uint8_t* const* __restrict__ pools /*[n_pools]*/, int n_pools, int page_words,
                                  const ForkPair* __restrict__ pairs, int n_pairs, float* __restrict__ h_slot, int d) {
    const long long dw = d / 4, per_pair = static_cast<long long>(n_pools) * page_words + dw;
    const long long total = per_pair * n_pairs;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const ForkPair f = pairs[i / per_pair];
        const long long w = i % per_pair;
        if (w < per_pair - dw) {
            if (f.src_page < 0) continue;
            const long long pool = w / page_words, o = w % page_words;
            uint4* base = reinterpret_cast<uint4*>(pools[pool]);
            base[static_cast<long long>(f.dst_page) * page_words + o] = base[static_cast<long long>(f.src_page) * page_words + o];
        } else {
            const long long c = w - (per_pair - dw);
            float4* h = reinterpret_cast<float4*>(h_slot);
            h[f.dst_slot * dw + c] = h[f.src_slot * dw + c];
        }
    }
}

// Swap of one utterance's KV pages (vcb_swap_out / vcb_swap_in): the page slabs of every pool (each layer's K, then each
// layer's V) as one contiguous staging region [pool][page i][page_words], gathered from (Gather) or scattered to (!Gather)
// the pool pages pages[i].  Whole 16-byte words: a page is H slabs, and every slab size is a multiple of 16 bytes.
template <bool Gather>
__global__ void __launch_bounds__(256)
kv_pages_copy_kernel(uint8_t* const* __restrict__ pools /*[n_pools]*/, int n_pools, long long page_words,
                     const int* __restrict__ pages, int n_pages, uint4* __restrict__ stage) {
    const long long per_pool = page_words * n_pages, total = per_pool * n_pools;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long pool = i / per_pool, r = i % per_pool;
        uint4* pg = reinterpret_cast<uint4*>(pools[pool]) + static_cast<long long>(pages[r / page_words]) * page_words +
                    r % page_words;
        if (Gather)
            stage[i] = *pg;
        else
            *pg = stage[i];
    }
}

// The fp8 KV quantizer of the QKV epilogues alone (vcb_debug_kv_quantize): one CTA of hd threads per row
__global__ void kv_quantize_kernel(const float* __restrict__ x, int hd, uint8_t* __restrict__ bytes, float* __restrict__ scales) {
    __shared__ float red[4];
    const int r = blockIdx.x, i = threadIdx.x;
    const float v = x[static_cast<size_t>(r) * hd + i];
    const float am = warp_max(fabsf(v));
    if ((i & 31) == 0) red[i >> 5] = am;
    __syncthreads();
    float amax = red[0];
    for (int w = 1; w < hd / 32; ++w) amax = fmaxf(amax, red[w]);
    float inv;
    const float scale = kv_fp8_scale(amax, inv);
    bytes[static_cast<size_t>(r) * hd + i] = static_cast<uint8_t>(kv_fp8_pack2(v, 0.f, inv) & 0xff);
    if (i == 0) scales[r] = scale;
}

// fp32 rows -> bf16 hi/lo rows (bring-up hook vcb_debug_gemm only)
__global__ void split_rows_kernel(const float* __restrict__ x, int N, __nv_bfloat16* __restrict__ act, int ld_act,
                                  int bpad) {
    const int r = blockIdx.y;
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= N) return;
    __nv_bfloat16 hi, lo;
    split_bf16(x[static_cast<size_t>(r) * N + c], hi, lo);
    act[static_cast<size_t>(r) * ld_act + c] = hi;
    act[static_cast<size_t>(r + bpad) * ld_act + c] = lo;
}

// ---------------------------------------------------------------------------------------------------
// Attention over the paged KV cache, one CTA per (row, head).  q-length 1 per row (decode step, or one
// token of a prefill chunk): keys 0..pos of the row's own utterance -- the causal mask over [text;audio]
// of voicecraft.py:419-447 without ever materialising it.  K/V pages are staged with TMA bulk copies
// (cp.async.bulk -> UBLKCP) into a 2-stage shared-memory ring guarded by mbarriers; math is fp32 on CUDA
// cores (1 FLOP/byte: HBM-bound).  Replaces F.scaled_dot_product_attention at activation.py:634.
//   QK : LPT = hd/8 lanes per key, each lane one 16-byte chunk of the key row (conflict-free), xor-shuffle reduce
//   PV : warp w owns keys [16w,16w+16) of the page, lane owns hd/32 output dims
// Output: bf16 hi/lo rows for the out-projection GEMM.
// ---------------------------------------------------------------------------------------------------
// KVT: __nv_bfloat16, float, or __nv_fp8_e4m3 (fp8 slabs carry the tokens' scales after the bytes: sc = q.k * kscale * scale,
// and PV weights e^(s - m) * vscale while l sums the unscaled e^(s - m)).
template <typename KVT>
constexpr int kv_dtype_of() { return sizeof(KVT) == 1 ? KV_FP8 : sizeof(KVT) == 4 ? KV_FP32 : KV_BF16; }

template <typename KVT, int HD>
struct AttSmem {
    static constexpr int PAGE_BYTES = kv_slab_bytes(kv_dtype_of<KVT>(), HD);
    static constexpr int OFF_V = ATT_STAGES * PAGE_BYTES;
    static constexpr int OFF_SC = 2 * ATT_STAGES * PAGE_BYTES;
    static constexpr int OFF_PW = OFF_SC + 2 * KV_PAGE * 4;          // scores double-buffered by page parity
    static constexpr int OFF_RED = OFF_PW + ATT_CWARPS * KV_PAGE * 4;
    static constexpr int OFF_BAR = OFF_RED + ATT_CWARPS * HD * 4;
    static constexpr int TOTAL = OFF_BAR + 2 * ATT_STAGES * 8 + 128;
};

template <typename KVT, int N>
__device__ __forceinline__ void load_kv_vec(const KVT* p, float (&out)[N]) {
    if constexpr (sizeof(KVT) == 1) {
        uint32_t w[(N + 3) / 4];
        if constexpr (N == 8) {
            const uint2 u = *reinterpret_cast<const uint2*>(p);
            w[0] = u.x;
            w[1] = u.y;
        } else if constexpr (N == 4) {
            w[0] = *reinterpret_cast<const uint32_t*>(p);
        } else {
            w[0] = *reinterpret_cast<const uint16_t*>(p);
        }
#pragma unroll
        for (int i = 0; i < N / 2; ++i) {
            const float2 f = kv_fp8_unpack2(w[i / 2] >> (16 * (i & 1)));
            out[2 * i] = f.x;
            out[2 * i + 1] = f.y;
        }
    } else if constexpr (sizeof(KVT) == 2) {
        if constexpr (N == 8) {
            const uint4 u = *reinterpret_cast<const uint4*>(p);
            const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                out[2 * i] = __uint_as_float(w[i] << 16);
                out[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
            }
        } else if constexpr (N == 4) {
            const uint2 u = *reinterpret_cast<const uint2*>(p);
            out[0] = __uint_as_float(u.x << 16);
            out[1] = __uint_as_float(u.x & 0xffff0000u);
            out[2] = __uint_as_float(u.y << 16);
            out[3] = __uint_as_float(u.y & 0xffff0000u);
        } else {
            const uint32_t u = *reinterpret_cast<const uint32_t*>(p);
            out[0] = __uint_as_float(u << 16);
            out[1] = __uint_as_float(u & 0xffff0000u);
        }
    } else {
#pragma unroll
        for (int i = 0; i < N; i += 2) {
            const float2 f = *reinterpret_cast<const float2*>(p + i);
            out[i] = f.x;
            out[i + 1] = f.y;
        }
    }
}

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Options of attn_rows_kernel (its `opts` argument)
static constexpr int ATT_LIVE_TAIL = 1;     // copy only the token rows 0 .. pos % KV_PAGE of the page that holds pos
static constexpr int ATT_POISON = 2;        // debug: fill the K / V ring with NaN first (shows that no uncopied byte is read)

// One (page, head) slab of K and of V into one ring stage: its first ntok token rows (fp8: and their scales, whose copy
// is rounded up to 16 bytes and stays inside the slab).  The stage's full barrier expects exactly the bytes copied.
template <typename KVT, int HD>
__device__ __forceinline__ void att_issue(KVT* dK, KVT* dV, const KVT* gK, const KVT* gV, int ntok, uint64_t* bar,
                                          uint64_t pol) {
    constexpr uint32_t PAGE_BYTES = kv_slab_bytes(kv_dtype_of<KVT>(), HD);
    if (ntok == KV_PAGE) {
        mbar_arrive_expect_tx(bar, 2 * PAGE_BYTES);
        tma_bulk_g2s_hint(dK, gK, PAGE_BYTES, bar, pol);
        tma_bulk_g2s_hint(dV, gV, PAGE_BYTES, bar, pol);
        return;
    }
    const uint32_t rows = static_cast<uint32_t>(ntok) * HD * sizeof(KVT);      // a multiple of 16: HD is 64 or 128
    if constexpr (sizeof(KVT) == 1) {
        const uint32_t scb = (static_cast<uint32_t>(ntok) * 4 + 15) & ~15u;
        mbar_arrive_expect_tx(bar, 2 * (rows + scb));
        tma_bulk_g2s_hint(dK, gK, rows, bar, pol);
        tma_bulk_g2s_hint(dK + KV_PAGE * HD, gK + KV_PAGE * HD, scb, bar, pol);
        tma_bulk_g2s_hint(dV, gV, rows, bar, pol);
        tma_bulk_g2s_hint(dV + KV_PAGE * HD, gV + KV_PAGE * HD, scb, bar, pol);
    } else {
        mbar_arrive_expect_tx(bar, 2 * rows);
        tma_bulk_g2s_hint(dK, gK, rows, bar, pol);
        tma_bulk_g2s_hint(dV, gV, rows, bar, pol);
    }
}

// One page of one row's online softmax: the scores of this warp's keys (into sc, then one barrier over the consumers),
// the running max / sum, and PV for this warp's keys.  Both instantiations of attn_rows_kernel run every row through it.
// Keys past pos are never read from the stage (the producer may not have copied them, ATT_LIVE_TAIL): their score is
// -inf without a dot product and PV stops before them.  The result is that of scoring them -inf and adding their
// weight-0 products: e^-inf = 0 adds nothing to l, and fmaf(0, v, acc) == acc for the finite v a written page holds.
template <typename KVT, int HD>
__device__ __forceinline__ void att_page(const KVT* K, const KVT* V, float* sc, float* pw, const float (&q)[8], int p,
                                         int pos, float scale, float& m_run, float& l_run, float (&acc)[HD / 32]) {
    constexpr int LPT = HD / 8;          // lanes per key in QK
    constexpr int TPW = 32 / LPT;        // keys per warp iteration
    constexpr int DPT = HD / 32;         // output dims per lane in PV
    constexpr bool FP8 = sizeof(KVT) == 1;
    const float* kscale = reinterpret_cast<const float*>(K + KV_PAGE * HD);     // fp8 only: the tokens' scales
    const float* vscale = reinterpret_cast<const float*>(V + KV_PAGE * HD);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int sub = lane % LPT;
    const int last = pos - p * KV_PAGE;  // keys t <= last of this page are in the context (every key when last >= 63)
    // ---- scores for this warp's KPW keys
    constexpr int KPW = KV_PAGE / ATT_CWARPS;
#pragma unroll
    for (int itq = 0; itq < KPW / TPW; ++itq) {
        const int t = warp * KPW + itq * TPW + lane / LPT;
        float dsum = 0.f;
        if (t <= last) {
            float kv[8];
            load_kv_vec<KVT, 8>(K + t * HD + sub * 8, kv);
#pragma unroll
            for (int i = 0; i < 8; ++i) dsum = fmaf(q[i], kv[i], dsum);
        }
#pragma unroll
        for (int o = LPT / 2; o > 0; o >>= 1) dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
        if (t <= last) {
            if constexpr (FP8) dsum *= kscale[t];
            if (sub == 0) sc[t] = dsum * scale;
        } else if (sub == 0) {
            sc[t] = -INFINITY;
        }
    }
    named_bar_sync(1, ATT_THREADS);
    // ---- online softmax bookkeeping (every warp redundantly over all 64 scores: identical m, l)
    const float s0 = sc[lane], s1 = sc[lane + 32];
    const float m_new = fmaxf(m_run, warp_max(fmaxf(s0, s1)));
    const float corr = expf(m_run - m_new);
    const float e0 = expf(s0 - m_new), e1 = expf(s1 - m_new);
    float* mypw = pw + warp * KV_PAGE;
    if constexpr (FP8) {
        mypw[lane] = lane <= last ? e0 * vscale[lane] : 0.f;
        mypw[lane + 32] = lane + 32 <= last ? e1 * vscale[lane + 32] : 0.f;
    } else {
        mypw[lane] = e0;
        mypw[lane + 32] = e1;
    }
    l_run = l_run * corr + warp_sum(e0 + e1);
    m_run = m_new;
    __syncwarp();
    // ---- PV for this warp's KPW keys
#pragma unroll
    for (int i = 0; i < DPT; ++i) acc[i] *= corr;
#pragma unroll
    for (int tt = 0; tt < KPW; ++tt) {
        const int t = warp * KPW + tt;
        if (t > last) break;
        const float pt_ = mypw[t];
        float vv[DPT];
        load_kv_vec<KVT, DPT>(V + t * HD + lane * DPT, vv);
#pragma unroll
        for (int i = 0; i < DPT; ++i) acc[i] = fmaf(pt_, vv[i], acc[i]);
    }
    __syncwarp();
}

// End of one (row, head, chunk): combine the consumer warps' partial outputs; a one-chunk context writes the output rows,
// a split context publishes (o, m, l) and the last chunk to finish merges all chunks in chunk order.
template <int HD>
__device__ __forceinline__ void att_finish(const float (&acc)[HD / 32], float m_run, float l_run, int r, int h, int rh,
                                           int chunk, int nch, float* red, __nv_bfloat16* __restrict__ act, int ld_act,
                                           int bpad, float* __restrict__ ws, int* __restrict__ cnt, int maxch, int& s_last) {
    constexpr int DPT = HD / 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int i = 0; i < DPT; ++i) red[warp * HD + lane * DPT + i] = acc[i];
    named_bar_sync(1, ATT_THREADS);
    const size_t ocol = static_cast<size_t>(h) * HD;
    if (nch == 1) {
        for (int dd = threadIdx.x; dd < HD; dd += ATT_THREADS) {
            float osum = 0.f;
#pragma unroll
            for (int w = 0; w < ATT_CWARPS; ++w) osum += red[w * HD + dd];
            const float o = osum / l_run;
            __nv_bfloat16 hi, lo;
            split_bf16(o, hi, lo);
            act[static_cast<size_t>(r) * ld_act + ocol + dd] = hi;
            act[static_cast<size_t>(r + bpad) * ld_act + ocol + dd] = lo;
        }
        named_bar_sync(1, ATT_THREADS);                   // red[] is reused by the next item
        return;
    }
    float* myws = ws + (static_cast<size_t>(rh) * maxch + chunk) * (HD + 2);
    for (int dd = threadIdx.x; dd < HD; dd += ATT_THREADS) {
        float osum = 0.f;
#pragma unroll
        for (int w = 0; w < ATT_CWARPS; ++w) osum += red[w * HD + dd];
        myws[dd] = osum;
    }
    if (threadIdx.x == 0) {
        myws[HD] = m_run;
        myws[HD + 1] = l_run;
    }
    __threadfence();
    named_bar_sync(1, ATT_THREADS);
    if (threadIdx.x == 0) s_last = (atomicAdd(&cnt[rh], 1) == nch - 1);
    named_bar_sync(1, ATT_THREADS);
    if (s_last) {
        __threadfence();
        const volatile float* base = ws + static_cast<size_t>(rh) * maxch * (HD + 2);
        float M = -INFINITY;
        for (int c = 0; c < nch; ++c) M = fmaxf(M, base[c * (HD + 2) + HD]);
        for (int dd = threadIdx.x; dd < HD; dd += ATT_THREADS) {
            float Lsum = 0.f, O = 0.f;
            for (int c = 0; c < nch; ++c) {
                const float w = expf(base[c * (HD + 2) + HD] - M);
                Lsum += base[c * (HD + 2) + HD + 1] * w;
                O += base[c * (HD + 2) + dd] * w;
            }
            const float o = O / Lsum;
            __nv_bfloat16 hi, lo;
            split_bf16(o, hi, lo);
            act[static_cast<size_t>(r) * ld_act + ocol + dd] = hi;
            act[static_cast<size_t>(r + bpad) * ld_act + ocol + dd] = lo;
        }
        if (threadIdx.x == 0) cnt[rh] = 0;
    }
    named_bar_sync(1, ATT_THREADS);                       // s_last / red[] reused by the next item
}

// Decode steps: step_prep_kernel stores the step's epoch to row_epoch[r] (release) after it wrote row r's tables, and it
// writes them only after its own griddepcontrol.wait, when every kernel and copy enqueued before it has completed.  So an
// acquire load that sees this step's epoch makes row_pos[r], row_pages[r], the group table and every KV page written
// before the step readable, by the TMA too (the proxy fence), while this grid's predecessors may still be running.
__device__ __forceinline__ bool att_row_ready(const unsigned long long* row_epoch, int r, unsigned long long epoch) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(row_epoch + r) : "memory");
    if (v != epoch) return false;
    asm volatile("fence.proxy.async.global;" ::: "memory");
    return true;
}

// Persistent, warp-specialised version: grid = a few CTAs per SM; each CTA walks a static list of work items
// (row*head, context chunk).  Warp 4 is the TMA producer: it runs ahead ACROSS items, so the HBM stream never drains
// at an item boundary (short CTAs with a cold start leave HBM idle).
// Warps 0..ATT_CWARPS-1 consume pages: scores -> online softmax -> PV, release the stage through an mbarrier.
//
// GMAX > 1: row groups.  A work item is (row group, head, chunk); n_rh counts groups * heads.  Group g holds rows
// grp_first[g] .. grp_first[g+1]-1 (at most GMAX), whose positions are equal or -1 (inactive: output untouched), and whose
// first grp_shared[g] pages are the same pages (a best-of-N group's prompt).  A shared page is loaded once and the
// consumers run every active member over it in turn, each with its own q / m / l / acc; a private page is loaded per
// member.  Every row goes through att_page and att_finish in the same order as with GMAX = 1: its output is
// bit-identical.
template <typename KVT, int HD, int GMAX>
__global__ void __launch_bounds__(ATT_THREADS + 32)
attn_rows_kernel(const float* __restrict__ qbuf, const KVT* __restrict__ kpool, const KVT* __restrict__ vpool,
                 const int* __restrict__ page_table, int max_pages, const int* __restrict__ row_slot,
                 const int* __restrict__ row_pos, int H, __nv_bfloat16* __restrict__ act, int ld_act, int bpad,
                 float scale, float* __restrict__ ws, int* __restrict__ cnt, int maxch, int chunk_pages, int n_rh,
                 int n_chunks, const int* __restrict__ row_pages, const int* __restrict__ grp_first,
                 const int* __restrict__ grp_shared, const unsigned long long* __restrict__ row_epoch,
                 unsigned long long epoch, int opts) {
    using L = AttSmem<KVT, HD>;
    constexpr int LPT = HD / 8;          // lanes per key in QK
    constexpr int DPT = HD / 32;         // output dims per lane in PV
    constexpr int SLAB = L::PAGE_BYTES / sizeof(KVT);        // KVT elements of one (page, head) slab: one TMA bulk copy
    extern __shared__ __align__(128) uint8_t att_smem[];
    KVT* sK = reinterpret_cast<KVT*>(att_smem);
    KVT* sV = reinterpret_cast<KVT*>(att_smem + L::OFF_V);
    float* sc_all = reinterpret_cast<float*>(att_smem + L::OFF_SC);
    float* pw = reinterpret_cast<float*>(att_smem + L::OFF_PW);
    float* red = reinterpret_cast<float*>(att_smem + L::OFF_RED);
    uint64_t* full = reinterpret_cast<uint64_t*>(att_smem + L::OFF_BAR);
    uint64_t* empty = full + ATT_STAGES;
    __shared__ int s_last;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // row_epoch (decode steps only): the producer issues the first ring stages before griddepcontrol.wait (DESIGN.md 4.1)
    const bool early = row_epoch != nullptr;
    pdl_launch_dependents();
    if (opts & ATT_POISON) {
        uint32_t* ring = reinterpret_cast<uint32_t*>(att_smem);
        for (int i = threadIdx.x; i < 2 * ATT_STAGES * L::PAGE_BYTES / 4; i += blockDim.x) ring[i] = 0xffffffffu;
        fence_proxy_async_smem();          // the NaN lands before any copy into the ring
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < ATT_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], ATT_CWARPS);
        }
        mbar_fence_init();
        tl_mark(0x300);
        tl_mark_all(0x300);
    }
    __syncthreads();
    if (!early || warp != ATT_CWARPS) pdl_wait();
    if (threadIdx.x == 0) { tl_mark(0x310); tl_mark_all(0x310); }
    const int n_items = n_rh * n_chunks;
    // Producer before griddepcontrol.wait: it reads row r's tables and pages only once att_row_ready(r) saw this step's
    // epoch, and issues at most ATT_STAGES slabs (no wait on a consumer), all of pages strictly before the one holding
    // pos, which this layer's QKV epilogue writes.  Everything else, q included, is read after the wait.
    bool waited = !early;
    const bool live_tail = opts & ATT_LIVE_TAIL;

    if constexpr (GMAX == 1) {
        if (warp == ATT_CWARPS) {
            // ===== producer: one lane streams the K/V pages of every item of this CTA, in order ================
            if (lane == 0) {
                const uint64_t pol = l2_policy_evict_first();          // KV pages stream through L2 once per step
                int it = 0;
                for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
                    const int chunk = item / n_rh, rh = item - chunk * n_rh;
                    const int r = rh / H, h = rh - r * H;
                    if (!waited && !att_row_ready(row_epoch, r, epoch)) {
                        pdl_wait();
                        waited = true;
                    }
                    const int pos = row_pos[r];
                    if (pos < 0) continue;
                    const int npages = pos / KV_PAGE + 1;
                    const int p0 = chunk * chunk_pages;
                    if (p0 >= npages) continue;
                    const int p1 = min(npages, p0 + chunk_pages);
                    // decode steps: step_prep left a per-row copy of the slot's page list, so the first TMA issue is one
                    // L2 round trip away (row -> pages) instead of two (row -> slot -> pages)
                    const int* pt = row_pages ? row_pages + r * max_pages : page_table + row_slot[r] * max_pages;
                    for (int p = p0; p < p1; ++p, ++it) {
                        if (!waited && (it >= ATT_STAGES || p == npages - 1)) {
                            pdl_wait();
                            waited = true;
                        }
                        const int s = it % ATT_STAGES;
                        if (it >= ATT_STAGES) mbar_wait(&empty[s], ((it / ATT_STAGES) - 1) & 1);
                        const size_t off = (static_cast<size_t>(pt[p]) * H + h) * SLAB;
                        const int ntok = live_tail && p == npages - 1 ? pos % KV_PAGE + 1 : KV_PAGE;
                        att_issue<KVT, HD>(sK + s * SLAB, sV + s * SLAB, kpool + off, vpool + off, ntok, &full[s], pol);
                    }
                }
            }
            return;
        }

        // ===== consumers ================================================================================
        const int sub = lane % LPT;
        int it = 0;
        for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
            const int chunk = item / n_rh, rh = item - chunk * n_rh;
            const int r = rh / H, h = rh - r * H;
            const int pos = row_pos[r];
            if (pos < 0) continue;
            const int npages = pos / KV_PAGE + 1;
            const int p0 = chunk * chunk_pages;
            if (p0 >= npages) continue;
            const int p1 = min(npages, p0 + chunk_pages);
            const int nch = (npages + chunk_pages - 1) / chunk_pages;
            float q[8];
            {
                const float* qp = qbuf + (static_cast<size_t>(r) * H + h) * HD + sub * 8;
    #pragma unroll
                for (int i = 0; i < 8; ++i) q[i] = qp[i];
            }
            float m_run = -INFINITY, l_run = 0.f;
            float acc[DPT];
    #pragma unroll
            for (int i = 0; i < DPT; ++i) acc[i] = 0.f;

            for (int p = p0; p < p1; ++p, ++it) {
                const int s = it % ATT_STAGES;
                mbar_wait(&full[s], (it / ATT_STAGES) & 1);
                att_page<KVT, HD>(sK + s * SLAB, sV + s * SLAB, sc_all + (it & 1) * KV_PAGE, pw, q, p, pos, scale, m_run, l_run, acc);
                if (lane == 0) mbar_arrive(&empty[s]);            // this warp is done with stage s
            }
            // ---- combine the 4 warps' partial outputs of this item
    #pragma unroll
            for (int i = 0; i < DPT; ++i) red[warp * HD + lane * DPT + i] = acc[i];
            named_bar_sync(1, ATT_THREADS);
            const size_t ocol = static_cast<size_t>(h) * HD;
            if (nch == 1) {
                for (int dd = threadIdx.x; dd < HD; dd += ATT_THREADS) {
                    float osum = 0.f;
    #pragma unroll
                    for (int w = 0; w < ATT_CWARPS; ++w) osum += red[w * HD + dd];
                    const float o = osum / l_run;
                    __nv_bfloat16 hi, lo;
                    split_bf16(o, hi, lo);
                    act[static_cast<size_t>(r) * ld_act + ocol + dd] = hi;
                    act[static_cast<size_t>(r + bpad) * ld_act + ocol + dd] = lo;
                }
                named_bar_sync(1, ATT_THREADS);                   // red[] is reused by the next item
                continue;
            }
            // ---- split context: publish (o, m, l); the last chunk to finish merges all chunks in chunk order
            float* myws = ws + (static_cast<size_t>(rh) * maxch + chunk) * (HD + 2);
            for (int dd = threadIdx.x; dd < HD; dd += ATT_THREADS) {
                float osum = 0.f;
    #pragma unroll
                for (int w = 0; w < ATT_CWARPS; ++w) osum += red[w * HD + dd];
                myws[dd] = osum;
            }
            if (threadIdx.x == 0) {
                myws[HD] = m_run;
                myws[HD + 1] = l_run;
            }
            __threadfence();
            named_bar_sync(1, ATT_THREADS);
            if (threadIdx.x == 0) s_last = (atomicAdd(&cnt[rh], 1) == nch - 1);
            named_bar_sync(1, ATT_THREADS);
            if (s_last) {
                __threadfence();
                const volatile float* base = ws + static_cast<size_t>(rh) * maxch * (HD + 2);
                float M = -INFINITY;
                for (int c = 0; c < nch; ++c) M = fmaxf(M, base[c * (HD + 2) + HD]);
                for (int dd = threadIdx.x; dd < HD; dd += ATT_THREADS) {
                    float Lsum = 0.f, O = 0.f;
                    for (int c = 0; c < nch; ++c) {
                        const float w = expf(base[c * (HD + 2) + HD] - M);
                        Lsum += base[c * (HD + 2) + HD + 1] * w;
                        O += base[c * (HD + 2) + dd] * w;
                    }
                    const float o = O / Lsum;
                    __nv_bfloat16 hi, lo;
                    split_bf16(o, hi, lo);
                    act[static_cast<size_t>(r) * ld_act + ocol + dd] = hi;
                    act[static_cast<size_t>(r + bpad) * ld_act + ocol + dd] = lo;
                }
                if (threadIdx.x == 0) cnt[rh] = 0;
            }
            named_bar_sync(1, ATT_THREADS);                       // s_last / red[] reused by the next item
        }
    } else {
        // the row's page list, as in the GMAX = 1 producer
        auto pages_of = [&](int r) { return row_pages ? row_pages + r * max_pages : page_table + row_slot[r] * max_pages; };
        // the item's group: rows r0 .. r0 + size - 1, active members as a bit mask, their common position
        auto group_of = [&](int gh, int& r0, int& size, int& h, unsigned& live, int& pos) {
            const int g = gh / H;
            h = gh - g * H;
            r0 = grp_first[g];
            size = grp_first[g + 1] - r0;
            live = 0;
            pos = -1;
#pragma unroll
            for (int j = 0; j < GMAX; ++j)
                if (j < size && row_pos[r0 + j] >= 0) {
                    live |= 1u << j;
                    pos = row_pos[r0 + j];
                }
        };
        if (warp == ATT_CWARPS) {
            if (lane == 0) {
                const uint64_t pol = l2_policy_evict_first();
                int it = 0;
                for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
                    const int chunk = item / n_rh, gh = item - chunk * n_rh;
                    // row 0 published: step_prep has passed its wait, so the group table uploaded before it is in place
                    if (!waited && !att_row_ready(row_epoch, 0, epoch)) {
                        pdl_wait();
                        waited = true;
                    }
                    if (!waited) {
                        const int g = gh / H;
                        for (int r = grp_first[g]; r < grp_first[g + 1] && !waited; ++r)
                            if (!att_row_ready(row_epoch, r, epoch)) {
                                pdl_wait();
                                waited = true;
                            }
                    }
                    int r0, size, h, pos;
                    unsigned live;
                    group_of(gh, r0, size, h, live, pos);
                    if (!live) continue;
                    const int npages = pos / KV_PAGE + 1;
                    const int p0 = chunk * chunk_pages;
                    if (p0 >= npages) continue;
                    const int p1 = min(npages, p0 + chunk_pages);
                    const int S = grp_shared[gh / H];
                    const int lead = r0 + __ffs(live) - 1;
                    for (int p = p0; p < p1; ++p) {
                        for (int j = 0; j < size; ++j) {
                            if (!(live >> j & 1) || (p < S && r0 + j != lead)) continue;
                            if (!waited && (it >= ATT_STAGES || p == npages - 1)) {
                                pdl_wait();
                                waited = true;
                            }
                            const int s = it % ATT_STAGES;
                            if (it >= ATT_STAGES) mbar_wait(&empty[s], ((it / ATT_STAGES) - 1) & 1);
                            const size_t off = (static_cast<size_t>(pages_of(r0 + j)[p]) * H + h) * SLAB;
                            const int ntok = live_tail && p == npages - 1 ? pos % KV_PAGE + 1 : KV_PAGE;
                            att_issue<KVT, HD>(sK + s * SLAB, sV + s * SLAB, kpool + off, vpool + off, ntok, &full[s], pol);
                            ++it;
                        }
                    }
                }
            }
            return;
        }

        const int sub = lane % LPT;
        int it = 0, k = 0;          // k: score passes (one per member and page), the parity of the score buffer
        for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
            const int chunk = item / n_rh, gh = item - chunk * n_rh;
            int r0, size, h, pos;
            unsigned live;
            group_of(gh, r0, size, h, live, pos);
            if (!live) continue;
            const int npages = pos / KV_PAGE + 1;
            const int p0 = chunk * chunk_pages;
            if (p0 >= npages) continue;
            const int p1 = min(npages, p0 + chunk_pages);
            const int nch = (npages + chunk_pages - 1) / chunk_pages;
            const int S = grp_shared[gh / H];
            float q[GMAX][8], m_run[GMAX], l_run[GMAX], acc[GMAX][DPT];
#pragma unroll
            for (int j = 0; j < GMAX; ++j) {
                if (live >> j & 1) {
                    const float* qp = qbuf + (static_cast<size_t>(r0 + j) * H + h) * HD + sub * 8;
#pragma unroll
                    for (int i = 0; i < 8; ++i) q[j][i] = qp[i];
                }
                m_run[j] = -INFINITY;
                l_run[j] = 0.f;
#pragma unroll
                for (int i = 0; i < DPT; ++i) acc[j][i] = 0.f;
            }
            for (int p = p0; p < p1; ++p) {
                const bool shared = p < S;
#pragma unroll
                for (int j = 0; j < GMAX; ++j) {
                    if (!(live >> j & 1)) continue;
                    const int s = it % ATT_STAGES;
                    const bool first = !shared || (live & ((1u << j) - 1)) == 0;
                    const bool last = !shared || (live >> (j + 1)) == 0;
                    if (first) mbar_wait(&full[s], (it / ATT_STAGES) & 1);
                    att_page<KVT, HD>(sK + s * SLAB, sV + s * SLAB, sc_all + (k & 1) * KV_PAGE, pw, q[j], p, pos, scale,
                                      m_run[j], l_run[j], acc[j]);
                    ++k;
                    if (last) {
                        if (lane == 0) mbar_arrive(&empty[s]);
                        ++it;
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < GMAX; ++j)
                if (live >> j & 1)
                    att_finish<HD>(acc[j], m_run[j], l_run[j], r0 + j, h, (r0 + j) * H + h, chunk, nch, red, act, ld_act,
                                   bpad, ws, cnt, maxch, s_last);
        }
    }
    if (threadIdx.x == 0) { tl_mark(0x330); tl_mark_all(0x330); }
}

// ---------------------------------------------------------------------------------------------------
// Step prologue: assign each row its position, advance the per-slot counters, fetch the input embedding
// produced by the previous sampler call.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
step_prep_kernel(const int* __restrict__ slots, int n, SlotState* __restrict__ st, const GroupState* __restrict__ gr,
                 int* __restrict__ row_slot, int* __restrict__ row_pos, int* __restrict__ row_last,
                 const float* __restrict__ x_slot, float* __restrict__ x_rows, int d,
                 const float* __restrict__ gamma0, __nv_bfloat16* __restrict__ act, int bpad, float* __restrict__ stats,
                 const int* __restrict__ page_table, int max_pages, int* __restrict__ row_page,
                 int* __restrict__ row_pages, int* __restrict__ row_forced, unsigned int* __restrict__ phase_flags,
                 int n_phase_flags, unsigned int* __restrict__ tile_counters, int n_tile_counters,
                 __nv_bfloat16* __restrict__ act_tiled, unsigned long long* __restrict__ row_epoch,
                 unsigned long long epoch) {
    __shared__ float red[8];
    pdl_launch_dependents();
    pdl_wait();
    const int r = blockIdx.x;
    if (r == 0)                                  // completion counters of the persistent step kernel (mega_step.cu)
        for (int i = threadIdx.x; i < n_phase_flags; i += blockDim.x) phase_flags[i] = 0u;
    // ... and its split-K arrival counters, spread over the CTAs of this launch
    for (int i = r * blockDim.x + threadIdx.x; i < n_tile_counters; i += gridDim.x * blockDim.x) tile_counters[i] = 0u;
    const int slot = slots[r];
    __shared__ int s_pos;
    if (threadIdx.x == 0) {
        SlotState& S = st[slot];
        const bool on = S.active && !gr[S.group].done;
        s_pos = on ? S.seq_len : -1;
        row_slot[r] = slot;
        row_pos[r] = s_pos;
        row_last[r] = on ? slot : -1;
        row_page[r] = on ? page_table[slot * max_pages + s_pos / KV_PAGE] : 0;
        row_forced[r] = S.forced;           // snapshot for the sampler's K CTAs of this slot (they are not ordered)
        if (on) {
            S.seq_len += 1;
            S.y_len += 1;
        }
    }
    for (int j = threadIdx.x; j < max_pages; j += blockDim.x)       // the attention producer reads these by row
        row_pages[static_cast<size_t>(r) * max_pages + j] = page_table[slot * max_pages + j];
    __syncthreads();
    if (threadIdx.x == 0) {              // row r's tables are this step's: attention may start its K/V stream (att_row_ready)
        __threadfence();
        asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(row_epoch + r), "l"(epoch) : "memory");
    }
    if (s_pos < 0) return;
    // x row + (LayerNorm folding) gamma0 * x as hi/lo rows and the row statistics for layer 0's QKV GEMM
    float s1 = 0.f, s2 = 0.f;
    for (int c = threadIdx.x; c < d; c += blockDim.x) {
        const float v = x_slot[static_cast<size_t>(slot) * d + c];
        x_rows[static_cast<size_t>(r) * d + c] = v;
        if (gamma0) {
            __nv_bfloat16 hi, lo;
            split_bf16(gamma0[c] * v, hi, lo);
            act[static_cast<size_t>(r) * d + c] = hi;
            act[static_cast<size_t>(r + bpad) * d + c] = lo;
            if (act_tiled) {       // persistent step kernel: the same operand as the pre-swizzled image of its MMA tiles (mega_step.cu)
                const int kk = c & 63, rows2 = 2 * bpad;
                const size_t t0 = static_cast<size_t>(c >> 6) * rows2;
                act_tiled[(t0 + r) * 64 + ((((kk >> 3) ^ (r & 7)) << 3) | (kk & 7))] = hi;
                act_tiled[(t0 + r + bpad) * 64 + ((((kk >> 3) ^ ((r + bpad) & 7)) << 3) | (kk & 7))] = lo;
            }
            s1 += v;
        }
    }
    if (gamma0) {
        // one statistics tile of all d features: (sum x, M2 about the row mean), see ln_tile_m2
        s1 = block_sum_256(s1, red);
        const float mean = s1 / static_cast<float>(d);
        for (int c = threadIdx.x; c < d; c += blockDim.x) {
            const float dv = x_slot[static_cast<size_t>(slot) * d + c] - mean;
            s2 = fmaf(dv, dv, s2);
        }
        s2 = block_sum_256(s2, red);
        if (threadIdx.x == 0) {
            stats[static_cast<size_t>(r) * 2] = s1;
            stats[static_cast<size_t>(r) * 2 + 1] = s2;
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// Fused sampler: one CTA per (utterance, codebook) row of V logits.  Reproduces, without a host sync,
//   * the in-place logit edits of sample_helper (voicecraft.py:1018-1067 tts, :718-787 edit, :1269-1325 batch)
//   * temperature, top-k (strict '<' vs the k-th largest value), top-p (sorted cumulative softmax, shift by one),
//     softmax and torch.multinomial(.,1) == argmax(p / q) with caller-provided q ~ Exp(1)   (:26-86)
//   * empty-token forcing, end-token trigger (sample / argmax / length cap), silence bookkeeping, the K-1 step
//     end cascade, best-of-N `keep`, multi-span hand-over; and it emits the next input embedding
//     sum_k E_k[tok_k] + alpha * PE[t]                                                   (:1102-1116)
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t f2key(float x) {        // order-preserving float -> uint
    const uint32_t u = __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// ---------------------------------------------------------------------------------------------------
// Exp(1) noise of `torch.multinomial` generated in place (voicecraft.py:85: multinomial(p, 1) == argmax(p / q),
// q = empty_like(p).exponential_(1)).  Bit-identical to ATen's CUDA path for a draw of `numel` fp32 elements from a
// Philox generator at (seed, offset): distribution_nullary_kernel launches T = 256 * grid threads, thread `idx` runs
// curand_init(seed, idx, offset) and element li of loop iteration `it` takes component (li % 4T) / T of the it-th
// curand_uniform4 of thread (li % T); exponential_ maps u -> -log(u) with the u ~ 1 guard of
// ATen/core/TransformationHelper.h.  (offset is a multiple of 4 in torch: one 128-bit Philox counter per call.)
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u;
        k.y += 0xBB67AE85u;
    }
    return c;
}

__device__ __forceinline__ float torch_exponential_at(unsigned long long seed, unsigned long long offset,
                                                      unsigned int threads, unsigned long long li) {
    const unsigned long long per_iter = 4ull * threads;
    const unsigned long long it = li / per_iter, rem = li - it * per_iter;
    const unsigned int comp = static_cast<unsigned int>(rem / threads);
    const unsigned long long idx = rem - static_cast<unsigned long long>(comp) * threads;
    const unsigned long long ctr = offset / 4ull + it;          // curand_init skipahead(offset) + one counter per curand4
    const uint4 o = philox4x32_10(make_uint4(static_cast<uint32_t>(ctr), static_cast<uint32_t>(ctr >> 32),
                                             static_cast<uint32_t>(idx), static_cast<uint32_t>(idx >> 32)),
                                  make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32)));
    const uint32_t x = comp == 0 ? o.x : comp == 1 ? o.y : comp == 2 ? o.z : o.w;
    // curand_uniform: x * 2^-32 + 2^-33 (the product is exact, one rounding in the add), range (0, 1]
    const float u = __fadd_rn(__fmul_rn(static_cast<float>(x), 2.3283064365386963e-10f), 1.16415321826934814453e-10f);
    // at::log is __logf in device code (ATen/NumericUtils.h), which is why the transform guards u ~ 1
    const float lg = (u >= 1.0f - 1.1920928955078125e-07f / 2) ? -1.1920928955078125e-07f / 2 : __logf(u);
    return -lg;                                                 // (-1 / lambda) * log with lambda = 1
}
// philox offset consumed by one draw of numel elements (ATen calc_execution_policy: counter_offset)
__host__ __device__ inline unsigned long long torch_draw_offset(unsigned long long numel, unsigned int threads) {
    return ((numel - 1) / (4ull * threads) + 1) * 4ull;
}

__global__ void debug_exponential_kernel(float* out, unsigned long long numel, unsigned long long seed,
                                         unsigned long long offset, unsigned int threads) {
    for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < numel;
         i += static_cast<unsigned long long>(gridDim.x) * blockDim.x)
        out[i] = torch_exponential_at(seed, offset, threads, i);
}

struct SamplerArgs {
    const int* slots;
    const int* row_forced;    // per listed slot: SlotState::forced as of the step prologue (null: read the slot)
    int n;
    SlotState* st;
    GroupState* gr;
    const float* logits;      // [n][ldl] fp32 (bias included), column = k*Vpad + v
    int ldl;
    const float* noise;       // [n*K][V], or null: generated from the group's Philox stream (GroupState::rng_*)
    float* dbg_logits;        // [n*K][V] or null
    int* tok_log;             // [max_slots][max_steps][K]
    float* lp_log = nullptr;  // laid out like tok_log: log-probability of the written token under the raw row (DESIGN.md
                              // section 2.2), or null: not stored
    int max_steps, max_seq;
    float* x_slot;            // [max_slots][d]
    const float* const* E_audio;
    const float* mask_emb;
    const float* pe;
    float alpha_a;
    int d, K, V, Vpad;
    int empty_token, eog, eos, encodec_sr;
    SamplingParams sp;
    const SamplingParams* sp_tab = nullptr;   // [max_slots] by group id: each slot samples with its group's parameters; null: `sp`
    // vcb_debug_sampler_ras only: the second Exp(1) plane of a repetition-aware redraw, laid out like `noise` (used when
    // `noise` is set), and a flag per row set where the redraw fired; the engine leaves both null
    const float* noise2 = nullptr;
    int* ras_redrew = nullptr;
};

static constexpr int SAMP_THREADS = 256;
static constexpr int SAMP_MAXV = 12;       // V <= 3072
static constexpr int SAMP_SORT_N = 4096;

__device__ void sampler_finish_slot(const SamplerArgs& a, const SamplingParams& sp, int slot, float* sred);

// (max, sum of exp(u - max)) pairs of two parts of a row, merged.  A part with no entries is (-inf, 0); the part that holds
// the maximum keeps its sum unscaled, so two empty parts merge to (-inf, 0), never to NaN.
__device__ __forceinline__ void lse_merge(float& m, float& s, float om, float os) {
    const float mm = fmaxf(m, om);
    s = (m == mm ? s : s * expf(m - mm)) + (om == mm ? os : os * expf(om - mm));
    m = mm;
}

// CTL: some listed slot samples with repetition-aware sampling or a length bound (vcb_sampling.ras_window / min_frames /
// max_frames).  The instance without them is the sampler as it was before those controls, instruction for instruction:
// steps that use none of them pay nothing for them.
template <bool CTL>
__global__ void __launch_bounds__(SAMP_THREADS) sampler_kernel(const __grid_constant__ SamplerArgs a) {
    __shared__ float sred[8];
    __shared__ float s_lse_m[8], s_lse_s[8];            // per warp: (max, sum) of the raw row, for the log-probability
    __shared__ int sidx[8];
    __shared__ int hist[256];
    __shared__ uint32_t s_prefix;
    __shared__ int s_kleft;
    __shared__ int s_flag;
    extern __shared__ unsigned long long sort_buf[];     // SAMP_SORT_N entries (only used when top_p < 1)

    pdl_launch_dependents();
    if (threadIdx.x == 0) tl_mark(0x400);
    pdl_wait();
    if (threadIdx.x == 0) tl_mark(0x410);
    const int i = blockIdx.x / a.K, k = blockIdx.x % a.K;
    const int slot = a.slots[i];
    SlotState& S = a.st[slot];
    if (!S.active) return;
    GroupState& G = a.gr[S.group];
    if (G.done) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int K = a.K, V = a.V;

    // `forced` as of the start of this step: the k == 0 CTA decrements S.forced below, and the K CTAs of a slot are not
    // ordered against each other (they need not even be co-resident), so the decision is taken on a snapshot
    const int forced_now = a.row_forced ? a.row_forced[i] : S.forced;
    if (forced_now > 0) {
        // edit-mode hand-over to the next span (voicecraft.py:838-858): this forward fed a forced embedding,
        // nothing is sampled; prepare the next forced input.
        if (k != 0) return;
        const int f = forced_now;               // 2: next input = mask embedding, 1: next input = empty-token embedding
        const float* pe = a.pe + static_cast<size_t>(S.y_len) * a.d;
        for (int c = tid; c < a.d; c += SAMP_THREADS) {
            float acc;
            if (f == 2) {
                acc = a.mask_emb[static_cast<size_t>(G.more_mask[0]) * a.d + c];
            } else {
                acc = 0.f;
                for (int kk = 0; kk < K; ++kk) {
                    const float v = a.E_audio[kk][static_cast<size_t>(a.empty_token) * a.d + c];
                    acc = kk == 0 ? v : __fadd_rn(acc, v);
                }
            }
            a.x_slot[static_cast<size_t>(slot) * a.d + c] = __fadd_rn(acc, __fmul_rn(a.alpha_a, pe[c]));
        }
        __syncthreads();
        if (tid == 0) {
            if (f == 2) {                       // consume the mask row
                for (int j = 0; j < 7; ++j) G.more_mask[j] = G.more_mask[j + 1];
            }
            S.forced = f - 1;
        }
        return;
    }

    // the group's parameters or the call's; one CTA serves one (utterance, codebook), so the branches on them are uniform
    const SamplingParams& sp = a.sp_tab ? a.sp_tab[S.group] : a.sp;
    const bool tts = G.mode == 0;
    const int E = tts ? (a.eos > 0 ? a.eos : a.eog) : a.eog;
    const int n_eog = G.n_eog, cur = G.cur_num_gen;
    const int row = i * K + k;

    // ---- load logits (split-K reduce + bias), apply the reference's in-place edits -----------------
    // the edits of entry v < V with raw logit u (also applied to the full row of a repetition-aware redraw)
    auto edit = [&](int v, float u) {
        if (a.eos > 0 && v == (tts ? a.eog : a.eos)) u = -10000.f;                   // :1091-1093 / :816-818
        if (n_eog == 0) {
            if (k >= 1 && (v == E || v == a.empty_token)) u = -10000.f;                // :1021-1023
            if (k == 0 && tts && cur <= a.encodec_sr / 5 && v == E) u = -10000.f;     // :1024-1025
            if (CTL && k == 0 && cur < sp.min_frames && v == E) u = -10000.f;         // length bound, like :1024-1025
            if (k == 0 && sp.stop_repetition > 0 && v == S.prev_token && S.consec > sp.stop_repetition) {
                bool sil = false;
                for (int t = 0; t < sp.n_silence; ++t) sil |= (sp.silence_tokens[t] == v);
                if (sil) {                                                             // :1027-1031
                    const float f = static_cast<float>(S.consec - (sp.stop_repetition - 1));
                    u = (u < 0.f) ? u * f : u / f;
                }
            }
        } else {
            if (k > n_eog && (v == E || v == a.empty_token)) u = -10000.f;            // :1056-1058
        }
        return u;
    };
    float l[SAMP_MAXV], raw[SAMP_MAXV];
    float lse_m = -INFINITY;             // this thread's max of the raw (unedited) entries
#pragma unroll
    for (int j = 0; j < SAMP_MAXV; ++j) {
        const int v = tid + j * SAMP_THREADS;
        float u = -INFINITY;
        if (v < V) {
            u = a.logits[static_cast<size_t>(i) * a.ldl + k * a.Vpad + v];
            raw[j] = u;
            lse_m = fmaxf(lse_m, u);
            if (a.dbg_logits) a.dbg_logits[static_cast<size_t>(row) * V + v] = u;
            u = edit(v, u);
        }
        l[j] = u;
    }
    // log-sum-exp of the raw row, before the edits above and before temperature / top-k / top-p: this thread's entries
    // summed in index order, then merged across the warp here and across the 8 warps by thread 0 at the end (the
    // block_argmax barriers below publish s_lse_*)
    {
        float lse_s = 0.f;
#pragma unroll
        for (int j = 0; j < SAMP_MAXV; ++j)
            if (tid + j * SAMP_THREADS < V) lse_s += expf(raw[j] - lse_m);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
            lse_merge(lse_m, lse_s, __shfl_xor_sync(0xffffffffu, lse_m, o), __shfl_xor_sync(0xffffffffu, lse_s, o));
        if (lane == 0) { s_lse_m[warp] = lse_m; s_lse_s[warp] = lse_s; }
    }

    // the Exp(1) draws are independent of everything below: fetch them now, not after the softmax
    float nz[SAMP_MAXV];
    if (a.noise) {
#pragma unroll
        for (int j = 0; j < SAMP_MAXV; ++j) {
            const int v = tid + j * SAMP_THREADS;
            nz[j] = (v < V) ? a.noise[static_cast<size_t>(row) * V + v] : 1.f;
        }
    } else {
        // this group's own generator: the draw has the reference's shape [size*K, V], row = member*K + k
        const unsigned long long seed = (static_cast<unsigned long long>(G.seed_hi) << 32) | G.seed_lo;
        const unsigned long long off = (static_cast<unsigned long long>(G.off_hi) << 32) | G.off_lo;
        const unsigned long long base = (static_cast<unsigned long long>(S.member) * K + k) * V;
#pragma unroll
        for (int j = 0; j < SAMP_MAXV; ++j) {
            const int v = tid + j * SAMP_THREADS;
            nz[j] = (v < V) ? torch_exponential_at(seed, off, G.rng_threads, base + v) : 1.f;
        }
    }

    // ---- argmax of the edited logits (first index wins), needed for the end-token trigger ----------
    float bm = -INFINITY;
    int bi = 0x7fffffff;
#pragma unroll
    for (int j = 0; j < SAMP_MAXV; ++j) {
        const int v = tid + j * SAMP_THREADS;
        if (v < V && (l[j] > bm || (l[j] == bm && v < bi))) { bm = l[j]; bi = v; }
    }
    auto block_argmax = [&](float& val, int& idx) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, val, o);
            const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
            if (ov > val || (ov == val && oi < idx)) { val = ov; idx = oi; }
        }
        __syncthreads();
        if (lane == 0) { sred[warp] = val; sidx[warp] = idx; }
        __syncthreads();
        val = sred[0]; idx = sidx[0];
#pragma unroll
        for (int w = 1; w < 8; ++w)
            if (sred[w] > val || (sred[w] == val && sidx[w] < idx)) { val = sred[w]; idx = sidx[w]; }
    };
    block_argmax(bm, bi);
    const int argmax_raw = bi;

    // ---- temperature (:80-81) -----------------------------------------------------------------------
    if (sp.temperature != 1.0f) {
#pragma unroll
        for (int j = 0; j < SAMP_MAXV; ++j) l[j] = __fdiv_rn(l[j], sp.temperature);
        bm = __fdiv_rn(bm, sp.temperature);
    }

    // ---- top-k: exact k-th largest by 4-pass radix select on order-preserving keys (:38-44) ----------
    if (sp.top_k > 0) {
        const int kk = min(max(sp.top_k, 1), V);
        if (tid == 0) { s_prefix = 0; s_kleft = kk; }
        for (int pass = 0; pass < 4; ++pass) {
            const int shift = 24 - 8 * pass;
            hist[tid] = 0;
            __syncthreads();
            const uint32_t prefix = s_prefix;
            const uint32_t pmask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
#pragma unroll
            for (int j = 0; j < SAMP_MAXV; ++j) {
                const int v = tid + j * SAMP_THREADS;
                // warp-aggregated histogram update: logits share a handful of exponent bytes, so plain atomics would
                // serialise ~32-way on the same shared-memory word in the first passes
                const uint32_t key = v < V ? f2key(l[j]) : 0u;
                const bool in = v < V && (key & pmask) == prefix;
                const unsigned act = __ballot_sync(0xffffffffu, in);
                if (in) {
                    const int bin = (key >> shift) & 0xff;
                    const unsigned peers = __match_any_sync(act, bin);
                    if (lane == __ffs(peers) - 1) atomicAdd(&hist[bin], __popc(peers));
                }
            }
            __syncthreads();
            if (warp == 0) {
                // descending scan over the 256 bins: lane l owns bins [255-8l-7, 255-8l]
                int loc[8], lsum = 0;
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    loc[u] = hist[255 - 8 * lane - u];
                    lsum += loc[u];
                }
                int incl = lsum;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int t = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += t;
                }
                const int left0 = s_kleft;
                const int before = incl - lsum;                     // keys in higher bins than this lane's
                const unsigned hit = __ballot_sync(0xffffffffu, incl >= left0);
                const int owner = hit ? __ffs(hit) - 1 : 31;
                if (lane == owner) {
                    int left = left0 - before, b = 255 - 8 * lane;
                    for (int u = 0; u < 7; ++u) {
                        if (loc[u] >= left) break;
                        left -= loc[u];
                        --b;
                    }
                    s_kleft = left;
                    s_prefix = prefix | (static_cast<uint32_t>(b) << shift);
                }
            }
            __syncthreads();
        }
        const float thr = key2f(s_prefix);
#pragma unroll
        for (int j = 0; j < SAMP_MAXV; ++j)
            if (l[j] < thr) l[j] = -INFINITY;
        __syncthreads();
    }

    // ---- top-p (:46-67): sort descending, softmax, cumulative sum, keep ranks < j0 ---------------------
    if (sp.top_p < 1.0f) {
        for (int s = tid; s < SAMP_SORT_N; s += SAMP_THREADS) sort_buf[s] = 0ull;   // pads sort last (key 0 < any real key)
        __syncthreads();
#pragma unroll
        for (int j = 0; j < SAMP_MAXV; ++j) {
            const int v = tid + j * SAMP_THREADS;
            // descending by value; ties -> lower index first.  -0.0 is keyed as +0.0: f2key orders it strictly below +0.0,
            // which would rank a +0.0 at a higher index ahead of an equal -0.0
            if (v < V)
                sort_buf[v] = (static_cast<unsigned long long>(f2key(l[j] == 0.f ? 0.f : l[j])) << 32) |
                              static_cast<uint32_t>(0xffffffffu - v);
        }
        __syncthreads();
        for (int size = 2; size <= SAMP_SORT_N; size <<= 1) {
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int t = tid; t < SAMP_SORT_N / 2; t += SAMP_THREADS) {
                    const int lo = 2 * t - (t & (stride - 1));
                    const int hi = lo + stride;
                    const bool desc = ((lo & size) == 0);
                    const unsigned long long x = sort_buf[lo], y = sort_buf[hi];
                    if ((x < y) == desc) { sort_buf[lo] = y; sort_buf[hi] = x; }
                }
                __syncthreads();
            }
        }
        // softmax over the sorted row (max = first element) and inclusive scan in rank order
        const float smax = key2f(static_cast<uint32_t>(sort_buf[0] >> 32));
        constexpr int PER = SAMP_SORT_N / SAMP_THREADS;      // 16 consecutive ranks per thread
        float e[PER];
        float loc = 0.f;
#pragma unroll
        for (int j = 0; j < PER; ++j) {
            const int rnk = tid * PER + j;
            const unsigned long long ent = sort_buf[rnk];
            e[j] = (rnk < V) ? expf(key2f(static_cast<uint32_t>(ent >> 32)) - smax) : 0.f;
            loc += e[j];
        }
        const float total = block_sum_256(loc, sred);
        // exclusive prefix of `loc` across threads
        float incl = loc;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        __syncthreads();
        if (lane == 31) sred[warp] = incl;
        __syncthreads();
        float base = 0.f;
        for (int w = 0; w < warp; ++w) base += sred[w];
        float run = base + incl - loc;
        int cnt = 0;                                       // ranks j with cum_j <= top_p
#pragma unroll
        for (int j = 0; j < PER; ++j) {
            run += e[j];
            const int rnk = tid * PER + j;
            if (rnk < V && !(run / total > sp.top_p)) cnt++;
        }
        __syncthreads();
        const int j0 = static_cast<int>(block_sum_256(static_cast<float>(cnt), sred) + 0.5f) + 1;   // kept ranks: [0, j0)
        // cum is monotone, so "cum_j <= top_p" holds exactly for ranks [0, j0-1): rank of a value = its sorted position
        __syncthreads();
        // mark removed: write per-index flag through the sorted order
        // reuse hist as nothing; flags go into the low bit trick: store rank into a dense array (aliasing sort_buf upper half)
        int* rank_of = reinterpret_cast<int*>(sort_buf + SAMP_SORT_N);      // V ints after the sort area
        for (int rnk = tid; rnk < V; rnk += SAMP_THREADS) {
            const uint32_t idx = 0xffffffffu - static_cast<uint32_t>(sort_buf[rnk] & 0xffffffffull);
            rank_of[idx] = rnk;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < SAMP_MAXV; ++j) {
            const int v = tid + j * SAMP_THREADS;
            if (v < V && rank_of[v] >= j0) l[j] = -INFINITY;
        }
        __syncthreads();
    }

    // ---- softmax + multinomial == argmax(p / q)  (:85) ---------------------------------------------------
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < SAMP_MAXV; ++j) mx = fmaxf(mx, l[j]);
    mx = warp_max(mx);
    __syncthreads();
    if (lane == 0) sred[warp] = mx;
    __syncthreads();
    mx = sred[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) mx = fmaxf(mx, sred[w]);
    float ev[SAMP_MAXV];
    float esum = 0.f;
#pragma unroll
    for (int j = 0; j < SAMP_MAXV; ++j) {
        const int v = tid + j * SAMP_THREADS;
        ev[j] = (v < V) ? expf(l[j] - mx) : 0.f;
        esum += ev[j];
    }
    const float tot = block_sum_256(esum, sred);
    float best = -1.f;
    int besti = 0x7fffffff;
#pragma unroll
    for (int j = 0; j < SAMP_MAXV; ++j) {
        const int v = tid + j * SAMP_THREADS;
        if (v < V) {
            const float p = ev[j] / tot;
            const float sc = p / nz[j];
            if (sc > best || (sc == best && v < besti)) { best = sc; besti = v; }
        }
    }
    block_argmax(best, besti);
    int tok = besti;

    // ---- repetition-aware sampling (DESIGN.md section 2.2): count `tok` in the last min(W, cur) entries of this
    // codebook's column of the token log (written by earlier steps of this generation); at >= c, redraw from the full
    // tempered row with the group's second draw of this step.  The count is block-wide, so the branch is uniform.
    if (CTL && sp.ras_window > 0) {
        const int h = min(min(sp.ras_window, cur), S.n_steps);
        const int* col = a.tok_log + (static_cast<size_t>(slot) * a.max_steps + (S.n_steps - h)) * K + k;
        if (__syncthreads_count(tid < h && col[static_cast<size_t>(tid) * K] == tok) >= sp.ras_threshold) {
            const unsigned long long base = (static_cast<unsigned long long>(S.member) * K + k) * V;
            const unsigned long long seed = (static_cast<unsigned long long>(G.seed_hi) << 32) | G.seed_lo;
            const unsigned long long off = ((static_cast<unsigned long long>(G.off_hi) << 32) | G.off_lo) +
                torch_draw_offset(static_cast<unsigned long long>(G.size) * K * V, G.rng_threads);
            // exp(u / temperature - bm) of entry v < V of the edited row: p_full * sum, bm being that row's maximum.
            // Recomputed in both passes below, which are not unrolled, rather than held: the kernel's register count is
            // its maximum over all paths, and the redraw must not raise it for steps that take the others
            auto e_full = [&](int v) {
                float u = edit(v, a.logits[static_cast<size_t>(i) * a.ldl + k * a.Vpad + v]);
                if (sp.temperature != 1.0f) u = __fdiv_rn(u, sp.temperature);
                return expf(u - bm);
            };
            float es = 0.f;
#pragma unroll 1
            for (int j = 0; j < SAMP_MAXV; ++j)
                if (tid + j * SAMP_THREADS < V) es += e_full(tid + j * SAMP_THREADS);
            const float tot2 = block_sum_256(es, sred);
            best = -1.f;
            besti = 0x7fffffff;
#pragma unroll 1
            for (int j = 0; j < SAMP_MAXV; ++j) {
                const int v = tid + j * SAMP_THREADS;
                if (v < V) {
                    const float q2 = a.noise2 ? a.noise2[static_cast<size_t>(row) * V + v]
                                              : torch_exponential_at(seed, off, G.rng_threads, base + v);
                    const float sc = (e_full(v) / tot2) / q2;
                    if (sc > best || (sc == best && v < besti)) { best = sc; besti = v; }
                }
            }
            block_argmax(best, besti);
            tok = besti;
            if (a.ras_redrew && tid == 0) a.ras_redrew[row] = 1;
        }
    }

    // ---- forced values / end-token logic ----------------------------------------------------------------
    if (tid == 0) {
        if (n_eog == 0) {
            if (cur < K - 1 && k > cur) tok = a.empty_token;                                 // :1037-1039
            if (k == 0) {
                const int cap = tts ? S.x_len * (a.encodec_sr / 5) : S.x_len * 10;
                if (tok == E || argmax_raw == E || S.y_len > cap ||                          // :1041-1045
                    (CTL && sp.max_frames > 0 && cur >= sp.max_frames)) {                    // length bound
                    tok = E;
                    atomicMax(&G.trig_keep, S.member + 1);
                }
            }
        } else if (G.size == 1 || S.member == G.keep) {                                      // :1063-1066 / :1321-1323
            if (k < n_eog) tok = a.empty_token;
            else if (k == n_eog) tok = E;
        }
        const size_t at = (static_cast<size_t>(slot) * a.max_steps + S.n_steps) * K + k;
        a.tok_log[at] = tok;
        if (a.lp_log) {
            // lp = (u_tok - M) - log sum_v exp(u_v - M) of the raw row, for the written token, drawn or forced
            float m = s_lse_m[0], s = s_lse_s[0];
#pragma unroll
            for (int w = 1; w < 8; ++w) lse_merge(m, s, s_lse_m[w], s_lse_s[w]);
            a.lp_log[at] = tok < V ? (a.logits[static_cast<size_t>(i) * a.ldl + k * a.Vpad + tok] - m) - logf(s)
                                   : -INFINITY;
        }
        __threadfence();
        s_flag = (atomicAdd(&S.arrive, 1) == K - 1);
    }
    __syncthreads();
    if (!s_flag) return;
    __threadfence();
    sampler_finish_slot(a, sp, slot, sred);
    if (threadIdx.x == 0) tl_mark(0x430);
}

// Last codebook row of a slot: next input embedding + silence bookkeeping; last slot of a group: group state.
__device__ void sampler_finish_slot(const SamplerArgs& a, const SamplingParams& sp, int slot, float* sred) {
    SlotState& S = a.st[slot];
    GroupState& G = a.gr[S.group];
    const int tid = threadIdx.x, K = a.K;
    const volatile int* toks = a.tok_log + (static_cast<size_t>(slot) * a.max_steps + S.n_steps) * K;
    const float* pe = a.pe + static_cast<size_t>(S.y_len) * a.d;
    for (int c = tid; c < a.d; c += SAMP_THREADS) {
        float acc = 0.f;
        for (int kk = 0; kk < K; ++kk) {
            const float v = a.E_audio[kk][static_cast<size_t>(toks[kk]) * a.d + c];
            acc = kk == 0 ? v : __fadd_rn(acc, v);
        }
        a.x_slot[static_cast<size_t>(slot) * a.d + c] = __fadd_rn(acc, __fmul_rn(a.alpha_a, pe[c]));
    }
    __syncthreads();
    if (tid != 0) return;
    if (G.n_eog == 0) {                                                                     // :1047-1051
        const int t0 = toks[0];
        bool sil = false;
        for (int t = 0; t < sp.n_silence; ++t) sil |= (sp.silence_tokens[t] == t0);
        S.consec = (sil && t0 == S.prev_token) ? S.consec + 1 : 0;
        S.prev_token = t0;
    }
    S.n_steps += 1;
    S.arrive = 0;
    __threadfence();
    if (atomicAdd(&G.arrive, 1) != G.size - 1) return;
    __threadfence();
    // ---- group finalize
    G.arrive = 0;
    if (G.rng_threads) {                    // one draw of [size*K, V] consumed, whether or not the caller supplied noise;
        unsigned long long off = (static_cast<unsigned long long>(G.off_hi) << 32) | G.off_lo;   // two under RAS
        off += (sp.ras_window > 0 ? 2ull : 1ull) * torch_draw_offset(static_cast<unsigned long long>(G.size) * K * a.V,
                                                                     G.rng_threads);
        G.off_lo = static_cast<unsigned int>(off);
        G.off_hi = static_cast<unsigned int>(off >> 32);
    }
    if (G.n_eog == 0) {
        if (G.trig_keep > 0) {
            G.n_eog = 1;
            G.keep = G.trig_keep - 1;            // the last member that triggered wins (:1302)
        }
    } else {
        G.n_eog += 1;
    }
    G.trig_keep = 0;
    G.cur_num_gen += 1;
    if (S.n_steps >= a.max_steps - 1 || S.seq_len >= a.max_seq - 2) {     // token log / KV capacity exhausted: stop, flag it
        G.done = 2;
        return;
    }
    if (G.n_eog == K) {                                                                      // span finished
        if (G.n_spans_done < 8) G.span_ends[G.n_spans_done] = S.n_steps;
        G.n_spans_done += 1;
        if (G.mode == 1 && G.spans_left > 0) {
            G.spans_left -= 1;
            G.n_eog = 0;
            G.cur_num_gen = 0;
            for (int mI = 0; mI < G.size; ++mI) {
                SlotState& M = a.st[G.first_slot + mI];
                M.forced = 2;
                M.prev_token = -1;
                M.consec = 0;
            }
        } else {
            G.done = 1;
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// Delayed codebook pattern gather (integer): out[b,k,s] = z[b,k,s-1-k] if 0 <= s-1-k < T else special.
// codebooks_patterns.py:151-176 with the DelayedPatternProvider layout (:336-352, delays = 0..K-1).
// ---------------------------------------------------------------------------------------------------
__global__ void delay_pattern_kernel(const long long* __restrict__ z, long long* __restrict__ out, int K, int T,
                                     long long special) {
    const int S = T + K;
    const size_t bk = blockIdx.y;
    const int k = static_cast<int>(bk % K);
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < S; s += gridDim.x * blockDim.x) {
        const int t = s - 1 - k;
        out[bk * S + s] = (t >= 0 && t < T) ? z[bk * T + t] : special;
    }
}

// ---------------------------------------------------------------------------------------------------
// Streaming gather (vcb_poll_frames / vcb_poll_frames_ex): one block per listed slot.  TTS: frame t is final once the token
// log holds rows up to t+K-1 and rows[t][0] is not the end token.  Only rows [from, n_steps-K+1) are scanned: the caller's
// `from` frames are final already.  The new frames are written un-delayed as codec codes [K][max_frames] with zero padding,
// the first code outside [0, bins) (lowest frame, then codebook) is recorded, and the slot's status is copied next to the
// result.  An edit slot (a source with n_spans > 0) does the same over its output, see poll_frames_edit.
// ---------------------------------------------------------------------------------------------------
constexpr int PF_MAX_SLOTS = 128;          // listed slots per launch (the lists travel as kernel parameters)
constexpr int PF_NO_BAD = 0x7fffffff;

struct PollFramesRec {         // one listed slot: its vcb_status fields + the gather's result (copied to the host in one piece)
    int done, forced, n_steps, keep, n_spans_done;
    int span_ends[8];
    unsigned int off_lo, off_hi;
    int final_frames, bad_frame, bad_k, bad_tok;
};

struct PollFramesArgs {
    int slots[PF_MAX_SLOTS], from[PF_MAX_SLOTS];
    const SlotState* st;
    const GroupState* gr;
    const int* tok_log;        // [max_slots][max_steps][K]
    long long* codes;          // [n][K][max_frames], from this launch's first listed slot on
    PollFramesRec* rec;        // [n], same offset
    const vcb_edit_source* src;   // [n], same offset; null: every listed slot is a TTS slot
    long long code_offset, bins;
    int max_steps, K, end, eog, max_frames;
};

// listed slot i's record: its status, its final frames and the first code outside [0, bins) (frame, codebook, entry)
__device__ void pf_write_rec(const PollFramesArgs& a, int i, const SlotState& S, int fin, int bad_frame, int bad_k,
                             int bad_tok) {
    const GroupState& G = a.gr[S.group];
    PollFramesRec r;
    r.done = G.done;
    r.forced = S.forced;
    r.n_steps = S.n_steps;
    r.keep = G.keep;
    r.n_spans_done = G.n_spans_done;
    for (int j = 0; j < 8; ++j) r.span_ends[j] = G.span_ends[j];
    r.off_lo = G.off_lo;
    r.off_hi = G.off_hi;
    r.final_frames = fin;
    r.bad_frame = bad_frame;
    r.bad_k = bad_k;
    r.bad_tok = bad_tok;
    a.rec[i] = r;
}

// Edit slot i.  Its output is y0[:, 0:s1] ++ G1 ++ y0[:, e1:s2] ++ ... ++ GM ++ y0[:, eM:T] (_Prompt.result): piece p is
// original piece p/2 for even p, generated span p/2 (un-delayed token-log rows) for odd p.  With d = n_spans_done, the final
// pieces are those up to original piece d, then the frames of span d that the TTS rule (end token eog) makes final.
__device__ void poll_frames_edit(const PollFramesArgs& a, int i) {
    __shared__ int s_end, s_bad, s_np;
    __shared__ int s_ps[2 * 8 + 2], s_src[2 * 8 + 1];   // first output frame / first y0 column or token-log row of piece p
    const vcb_edit_source& E = a.src[i];
    const int slot = a.slots[i], from = a.from[i], K = a.K, tid = threadIdx.x, M = E.n_spans, T = E.T;
    const SlotState& S = a.st[slot];
    const GroupState& G = a.gr[S.group];
    const int n_steps = S.n_steps, d = min(G.n_spans_done, M);
    const int lo = d > 0 ? G.span_ends[d - 1] : 0;    // first token-log row of span d
    const int* log = a.tok_log + static_cast<size_t>(slot) * a.max_steps * K;
    const int m = d < M ? max(0, n_steps - lo - K + 1) : 0;
    if (tid == 0) {
        s_end = m;
        s_bad = PF_NO_BAD;
    }
    __syncthreads();
    for (int t = tid; t < m; t += blockDim.x)
        if (log[static_cast<size_t>(lo + t) * K] == a.eog) {
            atomicMin(&s_end, t);
            break;
        }
    __syncthreads();
    if (tid == 0) {
        int f = 0, p = 0;
        for (int j = 0;; ++j) {
            s_ps[p] = f;
            s_src[p] = j == 0 ? 0 : E.spans[j - 1][1];
            f += (j == M ? T : E.spans[j][0]) - s_src[p];
            ++p;
            if (j == M) break;
            const int r0 = j == 0 ? 0 : G.span_ends[j - 1];
            s_ps[p] = f;
            s_src[p] = r0;
            ++p;
            if (j == d) {
                f += s_end;
                break;
            }
            f += max(0, G.span_ends[j] - r0 - K);
        }
        s_ps[p] = f;
        s_np = p;
    }
    __syncthreads();
    const int fin = max(s_ps[s_np], from);
    const int n_new = min(fin - from, a.max_frames);
    auto entry = [&](int f, int k) -> long long {      // output frame f, codebook k: the y0 or token-log entry
        int p = 0;
        while (p + 1 < s_np && s_ps[p + 1] <= f) ++p;
        const int u = f - s_ps[p] + s_src[p];
        return (p & 1) ? static_cast<long long>(log[static_cast<size_t>(u + k) * K + k]) : E.orig_dev[static_cast<size_t>(k) * T + u];
    };
    long long* out = a.codes + static_cast<size_t>(i) * K * a.max_frames;
    for (int j = tid; j < K * a.max_frames; j += blockDim.x) {
        const int k = j / a.max_frames, t = j - k * a.max_frames;
        long long c = 0;
        if (t < n_new) {
            c = entry(from + t, k) - a.code_offset;
            if (c < 0 || c >= a.bins) atomicMin(&s_bad, t * K + k);
        }
        out[j] = c;
    }
    __syncthreads();
    if (tid != 0) return;
    if (s_bad == PF_NO_BAD) {
        pf_write_rec(a, i, S, fin, -1, -1, -1);
    } else {
        const int t = s_bad / K, k = s_bad - t * K;
        pf_write_rec(a, i, S, fin, from + t, k, static_cast<int>(entry(from + t, k)));
    }
}

__global__ void __launch_bounds__(256) poll_frames_kernel(const __grid_constant__ PollFramesArgs a) {
    __shared__ int s_end, s_bad;
    const int i = blockIdx.x, slot = a.slots[i], from = a.from[i], K = a.K, tid = threadIdx.x;
    if (a.src && a.src[i].n_spans > 0) {
        poll_frames_edit(a, i);
        return;
    }
    const SlotState& S = a.st[slot];
    const int n_steps = S.n_steps;
    const int* log = a.tok_log + static_cast<size_t>(slot) * a.max_steps * K;
    const int m = max(0, n_steps - K + 1);             // frames whose last codebook has been sampled
    if (tid == 0) {
        s_end = m;
        s_bad = PF_NO_BAD;
    }
    __syncthreads();
    for (int t = from + tid; t < m; t += blockDim.x)   // a thread's first hit is its lowest: the block minimum is the end
        if (log[static_cast<size_t>(t) * K] == a.end) {
            atomicMin(&s_end, t);
            break;
        }
    __syncthreads();
    const int fin = max(s_end, from);
    const int n_new = min(fin - from, a.max_frames);
    long long* out = a.codes + static_cast<size_t>(i) * K * a.max_frames;
    for (int j = tid; j < K * a.max_frames; j += blockDim.x) {
        const int k = j / a.max_frames, t = j - k * a.max_frames;
        long long c = 0;                               // padding: the codec rejects any code outside [0, bins)
        if (t < n_new) {
            c = log[static_cast<size_t>(from + t + k) * K + k] - a.code_offset;
            if (c < 0 || c >= a.bins) atomicMin(&s_bad, t * K + k);
        }
        out[j] = c;
    }
    __syncthreads();
    if (tid != 0) return;
    if (s_bad == PF_NO_BAD) {
        pf_write_rec(a, i, S, fin, -1, -1, -1);
    } else {
        const int t = s_bad / K, k = s_bad - t * K;
        pf_write_rec(a, i, S, fin, from + t, k, log[static_cast<size_t>(from + t + k) * K + k]);
    }
}

}  // namespace vcb
