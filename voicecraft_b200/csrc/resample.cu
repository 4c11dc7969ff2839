// Band-limited sinc resampling (include/vcb200_codec.h, enc_resampler_*): torchaudio's Resample(orig, new) with its
// defaults (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99) as a polyphase FIR over ragged rows, one-shot or
// streamed with carried state.
//
// With g = gcd(orig, new), o = orig / g, n = new / g and w the filter half-width, output sample m = b*n + p is
//   y[m] = sum_{i=0}^{2w+o-1} K[p][i] * x[b*o + i - w]          (x = 0 outside [0, L)),  ceil(n*L/o) samples in all.
// The table K[n][2w+o] is built by the Python side (tokenizer.resample_table) and kept here transposed, [tap][phase], so
// the lanes of a warp (consecutive outputs, hence consecutive phases) read consecutive table words.
//
// One kernel serves both uses.  A one-shot resample is a streaming push into empty state with the final flag set.  Every
// output sums its taps in the order i = 0 .. 2w+o-1 with fp32 FMA, whatever the chunking, so a stream's concatenated
// outputs are bit-identical to the one-shot output of the whole row.
//
// Streaming rule: after L input samples of a stream, block b (outputs b*n .. b*n+n-1) is emitted once its whole window
// has arrived, b*o + w + o <= L; the final push also emits the zero-padded tail up to ceil(n*L/o).  The next block to
// emit starts its window at most 2w + o - 1 samples before L, so a stream carries its last min(L, 2w + 2o) input samples.
// The counters live on the host: output counts are known before anything is enqueued and no call waits for the device.
#include "../../include/vcb200_codec.h"
#include "vcb_internal.h"

#include <cmath>
#include <memory>
#include <numeric>
#include <vector>

namespace vcb {

static constexpr int RS_THREADS = 256;
static constexpr int RS_ROWS = 64;                          // rows per launch (per-row descriptors travel as kernel parameters)
static constexpr size_t RS_TABLE_CAP = size_t(16) << 20;    // bytes of filter table a resampler may hold
static constexpr size_t RS_SMEM_CAP = 160 * 1024;           // input window a CTA stages in shared memory
static std::atomic<long long> rs_launches{0};
long long resample_launches() { return rs_launches; }

struct RsRow {
    const float* carry;   // carried input samples of the stream (local indices [0, h)), or null when h == 0
    int h, len;           // carried samples, new samples (local [h, h + len)); zero elsewhere
    int s0;               // local index of the first tap of the row's first output block
    int n_out;            // outputs of this call
};
struct RsRows {
    RsRow r[RS_ROWS];
};
struct RsCarryRow {
    const float* cur;     // carried samples now
    float* next;          // carried samples after this push
    int row;              // input row of the call
    int h, len, hn;       // carried now, new, carried after
};
struct RsCarryRows {
    RsCarryRow r[RS_ROWS];
};

// grid (tiles, rows): a CTA produces up to `tile` consecutive outputs of one row from its input window staged in
// shared memory; each thread owns outputs k = k0 + tid, k0 + tid + 256, ...
__global__ void __launch_bounds__(RS_THREADS) resample_kernel(const float* __restrict__ in, int T, float* __restrict__ out,
                                                              int out_cap, const float* __restrict__ kt, int n, int o, int taps,
                                                              int tile, int row0, const __grid_constant__ RsRows rows) {
    extern __shared__ float sx[];
    const RsRow& r = rows.r[blockIdx.y];
    const int k0 = blockIdx.x * tile;
    if (k0 >= r.n_out) return;
    const int k1 = min(k0 + tile, r.n_out);
    const int q0 = k0 / n, q1 = (k1 - 1) / n;
    const int x0 = r.s0 + q0 * o;                 // local index of sx[0]
    const int nx = (q1 - q0) * o + taps;
    const float* x = in + static_cast<size_t>(row0 + blockIdx.y) * T - r.h;
    for (int j = threadIdx.x; j < nx; j += RS_THREADS) {
        const int g = x0 + j;
        float v = 0.f;
        if (g >= 0 && g < r.h) v = r.carry[g];
        else if (g >= r.h && g < r.h + r.len) v = __ldg(x + g);
        sx[j] = v;
    }
    __syncthreads();
    float* y = out + static_cast<size_t>(row0 + blockIdx.y) * out_cap;
    for (int k = k0 + threadIdx.x; k < k1; k += RS_THREADS) {
        const int q = k / n, p = k - q * n;
        const float* xs = sx + (q - q0) * o;
        const float* kp = kt + p;
        float acc = 0.f;
#pragma unroll 8
        for (int i = 0; i < taps; ++i) acc = fmaf(__ldg(kp + static_cast<size_t>(i) * n), xs[i], acc);
        y[k] = acc;
    }
}

// one CTA per row: the stream's next carry = the last hn samples of (carry ++ new samples)
__global__ void __launch_bounds__(RS_THREADS) resample_carry_kernel(const float* __restrict__ in, int T,
                                                                    const __grid_constant__ RsCarryRows rows) {
    const RsCarryRow& r = rows.r[blockIdx.x];
    const float* x = in + static_cast<size_t>(r.row) * T;
    const int skip = r.h + r.len - r.hn;
    for (int j = threadIdx.x; j < r.hn; j += RS_THREADS) {
        const int q = skip + j;
        r.next[j] = q < r.h ? r.cur[q] : x[q - r.h];
    }
}

}  // namespace vcb

using namespace vcb;

struct enc_resampler {
    int device = 0, orig = 0, target = 0;
    int o = 1, n = 1, w = 0, taps = 1;          // reduced rates, half-width, taps per phase (2w + o)
    int tile = RS_THREADS;                       // outputs per CTA
    size_t smem = 0;                             // dynamic shared memory of resample_kernel
    int max_streams = 0, hold = 0;               // streams; carried samples per stream (2w + 2o)
    DevBuf<float> kt;                            // [taps][n]
    DevBuf<float> carry;                         // [2][max_streams][hold]: a push reads one parity and writes the other
    std::vector<int64_t> consumed, emitted;      // per stream: input samples taken, output samples handed out
    std::vector<int> parity;
    std::vector<char> finished;                  // the final push ran; the next push needs a reset
};

namespace {

int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// outputs whose whole window lies within the first L samples (blocks b with b*o + w + o <= L)
int64_t ready_outputs(const enc_resampler* r, int64_t L) {
    return L < r->w + r->o ? 0 : ((L - r->w - r->o) / r->o + 1) * r->n;
}

size_t window_bytes(const enc_resampler* r, int tile) {
    return (static_cast<size_t>((tile - 1) / r->n + 1) * r->o + r->taps) * sizeof(float);
}

// one call over B rows: row b has carry rows[b].h samples and lens[b] new ones, emits rows[b].n_out outputs
int launch_rows(enc_resampler* r, const float* in, int T, float* out, int out_cap, const std::vector<RsRow>& rows,
                cudaStream_t st) {
    const int B = static_cast<int>(rows.size());
    for (int row0 = 0; row0 < B; row0 += RS_ROWS) {
        const int nb = std::min(RS_ROWS, B - row0);
        RsRows p{};
        int most = 0;
        for (int b = 0; b < nb; ++b) {
            p.r[b] = rows[row0 + b];
            most = std::max(most, p.r[b].n_out);
        }
        if (most == 0) continue;
        resample_kernel<<<dim3((most + r->tile - 1) / r->tile, nb), RS_THREADS, r->smem, st>>>(
            in, T, out, out_cap, r->kt, r->n, r->o, r->taps, r->tile, row0, p);
        VCB_CUDA_OK(cudaGetLastError());
        ++rs_launches;
    }
    return 0;
}

}  // namespace

extern "C" {

int enc_resampler_create(int32_t orig_sr, int32_t new_sr, const float* table_host, int32_t max_streams, int32_t device,
                         enc_resampler** out) {
    if (!out) {
        set_error("resampler: null output handle");
        return -1;
    }
    *out = nullptr;
    if (orig_sr <= 0 || new_sr <= 0 || max_streams < 0) {
        set_error("resampler: rates must be > 0 and max_streams >= 0 (got %d -> %d, %d streams)", orig_sr, new_sr, max_streams);
        return -1;
    }
    std::unique_ptr<enc_resampler> r(new enc_resampler());
    const int g = std::gcd(orig_sr, new_sr);
    r->orig = orig_sr;
    r->target = new_sr;
    r->o = orig_sr / g;
    r->n = new_sr / g;
    r->w = static_cast<int>(std::ceil(6.0 * r->o / (std::min(r->o, r->n) * 0.99)));   // torchaudio's width, same doubles
    const int64_t taps = 2 * static_cast<int64_t>(r->w) + r->o;
    const double table_bytes = static_cast<double>(taps) * r->n * sizeof(float);
    if (table_bytes > static_cast<double>(RS_TABLE_CAP)) {
        set_error("resampler: %d -> %d Hz needs a filter table of %.0f bytes (%d phases x %lld taps), over the %zu-byte cap",
                  orig_sr, new_sr, table_bytes, r->n, static_cast<long long>(taps), RS_TABLE_CAP);
        return -1;
    }
    r->taps = static_cast<int>(taps);
    while (r->tile > 1 && window_bytes(r.get(), r->tile) > RS_SMEM_CAP) r->tile /= 2;
    r->smem = window_bytes(r.get(), r->tile);
    if (r->smem > RS_SMEM_CAP) {
        set_error("resampler: %d -> %d Hz: one output's input window (%zu bytes) exceeds %zu bytes of shared memory",
                  orig_sr, new_sr, r->smem, RS_SMEM_CAP);
        return -1;
    }
    if (!table_host) {
        set_error("resampler: null filter table");
        return -1;
    }
    r->device = device;
    r->max_streams = max_streams;
    r->hold = 2 * r->w + 2 * r->o;
    VCB_CUDA_OK(cudaSetDevice(device));
    if (r->kt.alloc(static_cast<size_t>(r->taps) * r->n) || r->carry.alloc(static_cast<size_t>(2) * max_streams * r->hold))
        return -1;
    std::vector<float> kt(static_cast<size_t>(r->taps) * r->n);
    for (int p = 0; p < r->n; ++p)
        for (int i = 0; i < r->taps; ++i) kt[static_cast<size_t>(i) * r->n + p] = table_host[static_cast<size_t>(p) * r->taps + i];
    VCB_CUDA_OK(cudaMemcpy(r->kt, kt.data(), kt.size() * sizeof(float), cudaMemcpyHostToDevice));
    r->consumed.assign(max_streams, 0);
    r->emitted.assign(max_streams, 0);
    r->parity.assign(max_streams, 0);
    r->finished.assign(max_streams, 0);
    if (r->smem > 48 * 1024)
        VCB_CUDA_OK(cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(r->smem)));
    *out = r.release();
    return 0;
}

int enc_resampler_destroy(enc_resampler* r) {
    if (!r) return 0;
    cudaSetDevice(r->device);
    cudaDeviceSynchronize();
    delete r;
    return 0;
}

int enc_resampler_reset(enc_resampler* r, const int32_t* ids_host, int32_t n) {
    if (!r || (n > 0 && !ids_host)) {
        set_error("resampler: null argument");
        return -1;
    }
    for (int i = 0; i < n; ++i)
        if (ids_host[i] < 0 || ids_host[i] >= r->max_streams) {
            set_error("resampler: id %d outside [0, %d)", ids_host[i], r->max_streams);
            return -1;
        }
    for (int i = 0; i < n; ++i) {
        const int id = ids_host[i];
        r->consumed[id] = r->emitted[id] = 0;
        r->finished[id] = 0;
    }
    return 0;
}

int enc_resample(enc_resampler* r, const float* in_dev, const int32_t* lens_host, int32_t B, int32_t T, float* out_dev,
                 int32_t out_cap, int32_t* out_lens_host, void* stream) {
    if (!r || !lens_host || !out_lens_host || B < 0 || T < 0 || out_cap < 0) {
        set_error("resampler: null argument or negative size");
        return -1;
    }
    std::vector<RsRow> rows(B);
    for (int b = 0; b < B; ++b) {
        const int len = lens_host[b];
        if (len < 0 || len > T) {
            set_error("resampler: row %d: length %d outside [0, T = %d]", b, len, T);
            return -1;
        }
        const int64_t n_out = ceil_div(static_cast<int64_t>(r->n) * len, r->o);
        if (n_out > out_cap) {
            set_error("resampler: row %d gives %lld samples, the output holds %d", b, static_cast<long long>(n_out), out_cap);
            return -1;
        }
        rows[b] = RsRow{nullptr, 0, len, -r->w, static_cast<int>(n_out)};
    }
    for (int b = 0; b < B; ++b)
        if (rows[b].n_out > 0 && (!in_dev || !out_dev)) {
            set_error("resampler: null input or output");
            return -1;
        }
    for (int b = 0; b < B; ++b) out_lens_host[b] = rows[b].n_out;
    VCB_CUDA_OK(cudaSetDevice(r->device));
    return launch_rows(r, in_dev, T, out_dev, out_cap, rows, static_cast<cudaStream_t>(stream));
}

int enc_resampler_push(enc_resampler* r, const int32_t* ids_host, const int32_t* lens_host, const int32_t* final_host,
                       int32_t B, const float* in_dev, int32_t T, float* out_dev, int32_t out_cap, int32_t* out_lens_host,
                       void* stream) {
    if (!r || !ids_host || !lens_host || !out_lens_host || B < 0 || T < 0 || out_cap < 0) {
        set_error("resampler: null argument or negative size");
        return -1;
    }
    if (B > r->max_streams) {
        set_error("resampler: %d rows, %d streams", B, r->max_streams);
        return -1;
    }
    // everything is validated before any stream changes
    std::vector<char> seen(r->max_streams, 0);
    std::vector<RsRow> rows(B);
    std::vector<int64_t> total(B);
    bool any_in = false, any_out = false;
    for (int b = 0; b < B; ++b) {
        const int id = ids_host[b], len = lens_host[b];
        const bool fin = final_host && final_host[b];
        if (id < 0 || id >= r->max_streams) {
            set_error("resampler: row %d: id %d outside [0, %d)", b, id, r->max_streams);
            return -1;
        }
        if (seen[id]) {
            set_error("resampler: id %d appears twice in one call", id);
            return -1;
        }
        seen[id] = 1;
        if (len < 0 || len > T) {
            set_error("resampler: row %d: length %d outside [0, T = %d]", b, len, T);
            return -1;
        }
        if (r->finished[id]) {
            set_error("resampler: stream %d already had its final push; reset it first", id);
            return -1;
        }
        const int64_t L0 = r->consumed[id], L = L0 + len, E = r->emitted[id];
        total[b] = fin ? ceil_div(static_cast<int64_t>(r->n) * L, r->o) : ready_outputs(r, L);
        const int64_t n_out = total[b] - E;
        if (n_out > out_cap) {
            set_error("resampler: row %d gives %lld samples, the output holds %d", b, static_cast<long long>(n_out), out_cap);
            return -1;
        }
        const int h = static_cast<int>(std::min<int64_t>(L0, r->hold));
        const int64_t base = L0 - h;                         // global index of the first carried sample
        const float* cur = r->carry + (static_cast<size_t>(r->parity[id]) * r->max_streams + id) * r->hold;
        rows[b] = RsRow{cur, h, len, static_cast<int>((E / r->n) * r->o - r->w - base), static_cast<int>(n_out)};
        any_in |= len > 0;
        any_out |= n_out > 0;
    }
    if ((any_in && !in_dev) || (any_out && !out_dev)) {
        set_error("resampler: null input or output");
        return -1;
    }
    for (int b = 0; b < B; ++b) out_lens_host[b] = rows[b].n_out;
    VCB_CUDA_OK(cudaSetDevice(r->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (launch_rows(r, in_dev, T, out_dev, out_cap, rows, st)) return -1;
    // carry: after the outputs have read the old state; streams that finished or took nothing keep theirs
    std::vector<RsCarryRow> carry;
    for (int b = 0; b < B; ++b) {
        const int id = ids_host[b];
        const bool fin = final_host && final_host[b];
        if (fin || rows[b].len == 0) continue;
        const int hn = static_cast<int>(std::min<int64_t>(r->consumed[id] + rows[b].len, r->hold));
        float* next = r->carry + (static_cast<size_t>(1 - r->parity[id]) * r->max_streams + id) * r->hold;
        carry.push_back(RsCarryRow{rows[b].carry, next, b, rows[b].h, rows[b].len, hn});
    }
    for (size_t i = 0; i < carry.size(); i += RS_ROWS) {
        const int nb = static_cast<int>(std::min<size_t>(RS_ROWS, carry.size() - i));
        RsCarryRows p{};
        std::copy(carry.begin() + i, carry.begin() + i + nb, p.r);
        resample_carry_kernel<<<nb, RS_THREADS, 0, st>>>(in_dev, T, p);
        VCB_CUDA_OK(cudaGetLastError());
        ++rs_launches;
    }
    for (int b = 0; b < B; ++b) {
        const int id = ids_host[b];
        const bool fin = final_host && final_host[b];
        if (!fin && rows[b].len > 0) r->parity[id] ^= 1;
        r->consumed[id] += rows[b].len;
        r->emitted[id] = total[b];
        r->finished[id] = fin;
    }
    return 0;
}

}  // extern "C"
