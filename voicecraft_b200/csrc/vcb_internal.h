// Internal declarations shared by the .cu files of libvcb200.so (not part of the C ABI).
#pragma once
#include "vcb_common.cuh"

#include <algorithm>
#include <atomic>
#include <cstring>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

namespace vcb {

// ---------------------------------------------------------------------------------------------------
// Owners of device memory, pinned host memory and events.  Every allocation and event of the library (except the
// process-lifetime timeline buffers of vcb_timeline) lives in one of these, so whoever holds it releases it.  None of
// them synchronises: an owner whose work may still be in flight synchronises once before releasing them.
// ---------------------------------------------------------------------------------------------------
struct LiveCount {                     // process-wide: what is allocated now (vcb_counter / enc_counter "live_*")
    static inline std::atomic<long long> bytes{0}, handles{0};
    static void add(long long b, long long h) { bytes += b; handles += h; }
};

// Owner of one allocation of n elements of T: device memory (DevBuf), or pinned host memory (PinnedBuf) -- with `mapped`,
// host memory the device reaches through dev().  alloc(n, zero) releases the current allocation, then allocates at least
// one element (an allocated buffer is never null), zero-filled on request; ensure() allocates only when empty.  Both
// return 0, or -1 with the error set and the buffer empty.
template <typename T, bool Pinned>
class Buffer {
public:
    Buffer() = default;
    Buffer(Buffer&& o) noexcept { *this = std::move(o); }
    Buffer& operator=(Buffer&& o) noexcept {
        if (this != &o) {
            reset();
            p_ = std::exchange(o.p_, nullptr);
            d_ = std::exchange(o.d_, nullptr);
            n_ = std::exchange(o.n_, 0);
        }
        return *this;
    }
    ~Buffer() { reset(); }

    int alloc(size_t n, bool zero = false, bool mapped = false) {
        reset();
        const size_t bytes = std::max<size_t>(n, 1) * sizeof(T);
        void* p = nullptr;
        cudaError_t e = !Pinned ? cudaMalloc(&p, bytes) : mapped ? cudaHostAlloc(&p, bytes, cudaHostAllocMapped) : cudaMallocHost(&p, bytes);
        if (e == cudaSuccess) {
            LiveCount::add(static_cast<long long>(bytes), 1);
            p_ = d_ = static_cast<T*>(p);
            n_ = n;
            if (zero && Pinned) memset(p, 0, bytes);
            if (zero && !Pinned) e = cudaMemset(p, 0, bytes);
            if (e == cudaSuccess && mapped) e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&d_), p, 0);
        }
        if (e == cudaSuccess) return 0;
        cudaGetLastError();                 // a failed allocation leaves its error for the next cudaGetLastError()
        set_error("%s allocation of %zu bytes: %s", Pinned ? "pinned host" : "device", bytes, cudaGetErrorString(e));
        reset();
        return -1;
    }
    int ensure(size_t n, bool zero = false, bool mapped = false) { return p_ ? 0 : alloc(n, zero, mapped); }
    void reset() {
        if (!p_) return;
        Pinned ? cudaFreeHost(p_) : cudaFree(p_);
        LiveCount::add(-static_cast<long long>(std::max<size_t>(n_, 1) * sizeof(T)), -1);
        p_ = d_ = nullptr;
        n_ = 0;
    }
    T* get() const { return p_; }
    T* dev() const { return d_; }
    size_t size() const { return n_; }
    operator T*() const { return p_; }

private:
    T *p_ = nullptr, *d_ = nullptr;
    size_t n_ = 0;
};
template <typename T> using DevBuf = Buffer<T, false>;
template <typename T> using PinnedBuf = Buffer<T, true>;

class Event {
public:
    Event() = default;
    Event(Event&& o) noexcept : ev_(std::exchange(o.ev_, nullptr)) {}
    Event& operator=(Event&& o) noexcept {
        if (this != &o) {
            reset();
            ev_ = std::exchange(o.ev_, nullptr);
        }
        return *this;
    }
    ~Event() { reset(); }

    int create(unsigned flags = cudaEventDefault) {
        reset();
        const cudaError_t e = cudaEventCreateWithFlags(&ev_, flags);
        if (e == cudaSuccess) {
            LiveCount::add(0, 1);
            return 0;
        }
        ev_ = nullptr;
        set_error("event creation: %s", cudaGetErrorString(e));
        return -1;
    }
    void reset() {
        if (!ev_) return;
        cudaEventDestroy(ev_);
        LiveCount::add(0, -1);
        ev_ = nullptr;
    }
    operator cudaEvent_t() const { return ev_; }

private:
    cudaEvent_t ev_ = nullptr;
};

// Launch with the programmatic-dependent-launch attribute (when enabled): the kernel may be scheduled while its
// predecessor is still running; every such kernel orders its data accesses with griddepcontrol.wait (pdl_wait()).
template <typename... KArgs, typename... Args>
cudaError_t launch_k_pdl(int pdl, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                         Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// ---------------------------------------------------------------------------------------------------
// GEMM (gemm_wgmma.cu)
// ---------------------------------------------------------------------------------------------------
enum { EPI_QKV = 0, EPI_RESID = 1, EPI_ACT = 2, EPI_LOGITS = 3 };

// Fused epilogue of the GEMM (applied by the CTA that owns the row after the cluster reduce-scatter).
struct GemmEpilogue {
    int mode = EPI_LOGITS;
    const float* bias = nullptr;          // [Nout]
    // EPI_QKV: q -> qbuf [rows, d]; k, v -> paged KV cache at (row_slot, row_pos)
    float* qbuf = nullptr;
    void* kpool = nullptr;
    void* vpool = nullptr;
    const int* page_table = nullptr;
    const int* row_slot = nullptr;
    const int* row_pos = nullptr;
    const int* row_page = nullptr;      // optional: page index of (row_slot, row_pos), saves the dependent page-table lookup
    int kv_fp32 = 0, max_pages = 0, page_size = 64, d = 0, H = 0, hd = 0;
    // EPI_RESID: x[row, m] += y ; EPI_ACT: act hi/lo rows ; EPI_LOGITS: out[row, col_off + m]
    float* x = nullptr;
    __nv_bfloat16* act = nullptr;
    float* out = nullptr;
    int ld_out = 0, col_off = 0, act_kind = 0, bpad_out = 0;
    // LayerNorm folded into this GEMM (the B operand is gamma*x, not LN(x)):
    //   y = rstd[row] * (acc - mean[row] * cvec[m]) + bias[m]   with bias := b + W.beta, cvec := W.gamma   (DESIGN.md section 4.1)
    int ln_fold = 0, stats_tiles = 0, ln_d = 0;   // ln_d: features of a row (1 tile: all of them, else 128 per tile)
    const float* cvec = nullptr;
    const float* stats = nullptr;         // [tile][STATS_ROWS][2] (sum x, sum (x - tile mean)^2) written by the producer
    float inv_d = 0.f, ln_eps = 1e-5f;
    // EPI_RESID producer side: also emit gamma_next * x_new as hi/lo rows + this tile's row statistics
    int emit = 0, next_ld = 0, next_bpad = 0;
    const float* next_gamma = nullptr;
    __nv_bfloat16* next_act = nullptr;
    float* stats_out = nullptr;
    // EPI_QKV, persistent step kernel only: the new token's k / v (rounded like the cache) as fp32 rows [rows, d] -- the
    // attention phase takes the current position from here, so its K/V page stream never depends on this step's GEMM
    float* knew = nullptr;
    float* vnew = nullptr;
};
static constexpr int STATS_ROWS = 128;

// mean and rstd of `row` from the per-tile (sum, M2) partials a producer left (tile order, see ln_tile_m2); up to 16 tiles
// (d <= 2048) are one batch of independent loads, read once
__device__ __forceinline__ void ln_row_stats(const float* stats, int tiles, int d, int row, float inv_d, float eps, float& mean,
                                             float& rstd) {
    auto load = [&](int t) {
        return t < tiles ? *reinterpret_cast<const float2*>(stats + (static_cast<size_t>(t) * STATS_ROWS + row) * 2)
                         : make_float2(0.f, 0.f);
    };
    float2 v[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = load(i);
    float s1 = 0.f, m2 = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) s1 += v[i].x;
    for (int t0 = 16; t0 < tiles; t0 += 16)
#pragma unroll
        for (int i = 0; i < 16; ++i) s1 += load(t0 + i).x;
    mean = s1 * inv_d;
#pragma unroll
    for (int i = 0; i < 16; ++i)
        if (i < tiles) m2 += ln_tile_m2(ln_tile_n(i, tiles, d), v[i].x, v[i].y, mean);
    for (int t0 = 16; t0 < tiles; t0 += 16)
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const float2 w = load(t0 + i);
            if (t0 + i < tiles) m2 += ln_tile_m2(ln_tile_n(t0 + i, tiles, d), w.x, w.y, mean);
        }
    rstd = 1.0f / sqrtf(m2 * inv_d + eps);
}

// ---------------------------------------------------------------------------------------------------
// Persistent decode-step kernel (mega_step.cu): one launch runs every layer of a decode step.
// ---------------------------------------------------------------------------------------------------
enum { MEGA_GEMM = 0, MEGA_ATTN = 1 };
static constexpr int MEGA_MAXSEG = 8;          // output tiles a CTA's block range may touch in one GEMM phase
static constexpr int MEGA_ATT_MAXC = 16;       // CTAs that may share one (row, head) attention item
struct MegaPhase {
    int type = MEGA_GEMM;
    // GEMM: `groups` matrices of tiles_per_group x kb 16 KB weight blocks (groups > 1: the K second-stage logit heads)
    int groups = 1, tiles_per_group = 0, kb = 0, Nout = 0;
    int b_map = 0, b_col_off = 0, b_grp_stride = 0, col_grp_stride = 0;   // b_col_off / b_grp_stride in elements (multiples of 64)
    const CUtensorMap* tmA = nullptr;         // device array [groups]
    const void* const* wptr = nullptr;        // device array [groups]: packed weights (contiguous 16 KB blocks), L2 prefetch
    const float* const* grp_bias = nullptr;   // device array [groups] or null (ep.bias)
    GemmEpilogue ep;
    // ATTN: this layer's pools
    const void* kpool = nullptr;
    const void* vpool = nullptr;
    int dep_target = 0;                       // completions of the previous phase this one waits for (0: none)
    int done_target = 0;                      // completions that finish this phase (tiles, or CTAs for ATTN)
};
struct MegaArgs {
    // Activation (B) operands: 0 act_d, 1 act_d2, 2 act_f, 3 act_h, each stored as the shared-memory IMAGE of its MMA tiles:
    // [K/64 k-blocks][2*bpad rows (hi rows, then lo rows)][64] bf16 with the 128-byte swizzle already applied (16-byte chunk c
    // of row r sits at chunk c ^ (r & 7)), so a tile is one contiguous 2*bpad*128-byte bulk copy -- no tensor map, no 64
    // scattered 128-byte rows per tile (see mg_act_off in mega_step.cu).
    const __nv_bfloat16* bbase[4] = {nullptr, nullptr, nullptr, nullptr};
    const MegaPhase* ph = nullptr;      // device array
    int nph = 0, nvalid = 0, bpad = 0, kv_fp32 = 0;
    int ns = 11, nb = 6;                // ring depths: ns * 16 KB + nb * 8 KB <= 224 KB
    int pf = 0;                         // L2 prefetch distance in ring items (0 = off)
    int flight = 5;                     // ring loads in flight (issued, not landed) per SM
    unsigned int* flags = nullptr;      // [nph] completion counters (zeroed by step_prep)
    int* tile_cnt = nullptr;            // [nph][max tiles] split-K arrival counters (self-resetting)
    int tile_cnt_stride = 0;
    float* part = nullptr;              // [grid][MEGA_MAXSEG][bpad][128] split-K partials
    unsigned int* dbg = nullptr;        // watchdog record
    unsigned long long* tl = nullptr;   // debug timeline [2 CTAs][nph][8 events] of %globaltimer (null: off)
    // attention
    const float* qbuf = nullptr;
    const float* knew = nullptr;
    const float* vnew = nullptr;
    __nv_bfloat16* att_out = nullptr;   // act_d (hi/lo rows)
    float* att_ws = nullptr;            // [rows*H][max_pages][132]: page partials (acc[128], m, l) of items shared between CTAs
    int* att_cnt = nullptr;             // [nph? no: rows*H] arrival counters (self-resetting)
    const int* row_pos = nullptr;
    const int* row_pages = nullptr;
    int max_pages = 0, H = 0, d = 0;
    float scale = 0.f;
};
int mega_launch(const MegaArgs& a, int grid, cudaStream_t st);
int mega_max_grid(int bpad, int kv_fp32);
size_t mega_part_floats(int grid, int bpad);

// Grouped launch of gemm_w_xT_cluster (blockIdx.y = group): weight tensor maps in a device array, per-group bias pointers.
struct GemmGroup {
    const CUtensorMap* tmA = nullptr;     // device array [groups]; null = plain launch
    const float* const* bias = nullptr;   // device array [groups]
    int b_stride = 0, col_stride = 0;     // added per group to the activation column offset / output column offset
};

struct GemmCall {
    const CUtensorMap* tmA = nullptr;   // weights [Nout, Kdim]
    const CUtensorMap* tmB = nullptr;   // activations [2*bpad, ldx]
    const __nv_bfloat16* W = nullptr;   // raw pointers (simt cross-check path only)
    const __nv_bfloat16* X = nullptr;
    GemmEpilogue ep;
    int Nout = 0, Kdim = 0, ldx = 0, bpad = 0, splits = 1, b_col_off = 0, nvalid = 0;
    int pdl = 0, simt = 0;
    GemmGroup grp;
    int groups = 1;
    const void* pf_ptr = nullptr;       // next GEMM's weights: prefetched into L2 while this kernel runs
    size_t pf_bytes = 0;
};
int gemm_launch(const GemmCall& g, cudaStream_t st);
// What gemm_launch would launch for g: the pipeline stages and the split count after the fallback to the largest cluster
// the device can place (cluster_cap > 0: as if it could place none larger).  -1 (and the error) where gemm_launch rejects g.
int gemm_launch_shape(const GemmCall& g, int cluster_cap, int& splits, int& stages);

// Rows-as-M GEMM for prefill (gemm_rows.cu): activations [2][rcap][Kdim] (hi plane, lo plane), packed weights as above.
struct RowsGemmCall {
    const CUtensorMap* tmX = nullptr;   // activations: 2D [2*rcap rows][Kdim], box 128 rows x 64 cols
    const CUtensorMap* tmW = nullptr;   // packed weights (pack_weight)
    GemmEpilogue ep;                    // modes QKV / RESID / ACT / LOGITS; bpad_out = rows per plane of the ACT output
    int rows = 0, rcap = 0, Nout = 0, Kdim = 0, pdl = 0;
};
bool gemm_rows_supported(int Nout, int Kdim, int hd);
int gemm_rows_launch(const RowsGemmCall& g, cudaStream_t st);
// split count (= cluster size) of a decode GEMM launch of `groups` x Nout x Kdim at bpad token rows
int gemm_pick_splits(int Nout, int Kdim, int bpad, int groups);
size_t packed_weight_elems(int N, int Kdim);
int pack_weight(const float* w_f32_dev, __nv_bfloat16* out, int N, int Kdim, CUtensorMap* tm);
int ln_fold_vectors(const __nv_bfloat16* Wp, const float* gamma, const float* beta, const float* bias, float* cvec,
                    float* bprime, int N, int Kdim);
void gemm_timeline_set(unsigned long long* buf, unsigned int* cnt);
int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                      uint32_t box_rows);

// ---------------------------------------------------------------------------------------------------
// Per-utterance ("slot") and per-group device state.  A group couples the slots of one
// inference_tts_batch call (shared codebook_eog / cur_num_gen / keep, voicecraft.py:1269-1325);
// independent utterances are groups of size 1.
// ---------------------------------------------------------------------------------------------------
struct SlotState {
    int x_len;          // text tokens
    int seq_len;        // tokens already in the KV cache (text + audio columns)
    int y_len;          // audio columns embedded so far == y_input.shape[1] in the reference
    int group;          // group index
    int member;         // index of this slot inside its group
    int prev_token;     // silence bookkeeping (-1 = None)
    int consec;         // consec_silence_count
    int n_steps;        // sampling steps recorded in the token log
    int forced;         // edit mode: number of upcoming forwards that feed a forced embedding (no sampling)
    int active;         // 1 while the slot is open
    int arrive;         // scratch: codebook rows finished in this step (last-CTA-done pattern)
    int pad[5];
};

struct GroupState {
    int mode;           // 0 = tts (voicecraft.py:1018-1067), 1 = edit (:718-787)
    int size;           // number of member slots
    int n_eog;          // how many codebooks have emitted their end token (always a prefix 0..n_eog-1)
    int cur_num_gen;    // steps in the current span
    int keep;           // batch mode: member index whose tokens are returned; -1 = undecided
    int done;           // all spans finished
    int spans_left;     // edit mode: masked spans still to generate after the current one
    int trig_keep;      // scratch: 1 + max member index that triggered the end token in this step (0 = none)
    int arrive;         // scratch: member slots finished in this step
    int n_spans_done;
    int first_slot;     // slot id of member 0 (members are consecutive slots)
    // Device-side sampling noise (sampler_kernel, noise pointer null): the Philox4x32-10 stream torch's CUDA generator
    // would hand to `torch.multinomial` for a draw of shape [size*K, V] (ATen distribution_nullary_kernel + exponential_):
    // rng_threads = 256 * grid of that launch (0: this group needs caller-provided noise), offset advances per sampling step.
    unsigned int rng_threads;
    int more_mask[8];   // edit mode: mask_embedding rows of the spans still to come
    int span_ends[8];   // n_steps at which each span finished
    unsigned int seed_lo, seed_hi, off_lo, off_hi;
};
static_assert(sizeof(GroupState) == 128, "GroupState is copied in bulk by vcb_poll");

struct SamplingParams {
    int top_k;
    float top_p;
    float temperature;
    int stop_repetition;
    int silence_tokens[8];
    int n_silence;
};

struct ModelDims {
    int d, H, hd, L, F, K, V, Vpad, Hh;   // Hh = predict_layer hidden (audio_vocab_size/2); Vpad = V rounded to 4
    int n_text, empty_token, eog, eos, audio_pad, encodec_sr, max_n_spans;
    int pe_len;
};

}  // namespace vcb
