// Ingest: every stream's packets at its own sample rate, resampled to 16 kHz on the device and staged until they fill
// whole chunks, which then step through oww_step_ragged.  Semantics: include/owwb200.h (oww_set_input_rates and the calls
// after it).
//
// Host state per stream: rate, S (input samples since the resampler's restart), staged (16 kHz samples not yet stepped)
// and where they start in the row (the chunks of the last call sit in front of them until the next call moves them).
// Device state per stream: the staging row [C] int16 (C = max_chunks*1280 + 1279) and the last 128 input samples [128]
// int16.  A stream with S == 0 has a zero history by definition, so restarts and resets launch nothing.
//
// One call: resample_kernel (one CTA per stream: the staged samples move to the front of the row, the new final outputs go
// behind them, the history advances), then oww_step_ragged on the rows.  Within a CTA everything it overwrites - the
// staged samples, which may overlap the new outputs, and the history - is read into shared memory before the first write.
#include <cstring>
#include <numeric>
#include "oww_internal.h"

#define ING_THREADS 256
#define ING_HIST 128                  // input samples of history per stream (a phase has at most 61 taps)
#define ING_SLOTS 4                   // pinned staging buffers of the per-call table

namespace {

const int kRates[] = {8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000};
constexpr int kNRates = sizeof(kRates) / sizeof(kRates[0]);
constexpr double kPi = 3.14159265358979323846;

int rate_index(int rate) {
    for (int i = 0; i < kNRates; ++i) if (kRates[i] == rate) return i;
    return -1;
}

void up_down(int rate, int* up, int* down) {
    const int g = std::gcd(16000, rate);
    *up = 16000 / g; *down = rate / g;
}

double bessel_i0(double x) {                              // power series; converges fast for x <= 5
    double sum = 1.0, term = 1.0;
    for (int k = 1; k < 200; ++k) {
        term *= (x / (2.0 * k)) * (x / (2.0 * k));
        sum += term;
        if (term < 1e-18 * sum) break;
    }
    return sum;
}

// scipy.signal.resample_poly's filter for `rate`, in double: firwin(N, 1/mr, window=('kaiser', 5.0)) * up
std::vector<double> design(int rate, int* up, int* down) {
    up_down(rate, up, down);
    const int mr = std::max(*up, *down), half = 10 * mr, N = 2 * half + 1;
    const double beta = 5.0, i0b = bessel_i0(beta);
    std::vector<double> h(N);
    double sum = 0.0;
    for (int k = 0; k < N; ++k) {
        const double x = (double)(k - half) / mr;
        const double sinc = x == 0.0 ? 1.0 : std::sin(kPi * x) / (kPi * x);
        const double r = 2.0 * k / (N - 1) - 1.0;
        const double w = bessel_i0(beta * std::sqrt(std::max(0.0, 1.0 - r * r))) / i0b;
        h[k] = sinc * w;
        sum += h[k];
    }
    for (double& v : h) v = v / sum * (*up);
    return h;
}

// A(S) = ceil(S * up / down): outputs that no longer depend on later input after S input samples
int64_t final_outputs(int64_t S, int up, int down) { return (S * up + down - 1) / down; }

// the arithmetic of one stream's call (oww_ingest_plan): false when n_in is over the limit (only *max_in is valid)
bool plan(int rate, int max_chunks, int64_t S, int staged, int64_t n_in, int64_t* n_out, int* chunks, int* staged_after,
          int64_t* max_in) {
    int up, down;
    up_down(rate, &up, &down);
    const int64_t cap = (int64_t)max_chunks * OWW_SAMPLES_PER_CHUNK + OWW_SAMPLES_PER_CHUNK - 1;
    // A(S + n) <= cap - staged + A(S)  <=>  (S + n) * up <= (cap - staged + A(S)) * down
    const int64_t room = cap - staged + final_outputs(S, up, down);
    *max_in = std::max<int64_t>(room * down / up - S, 0);
    if (n_in < 0 || n_in > *max_in) return false;
    *n_out = final_outputs(S + n_in, up, down) - final_outputs(S, up, down);
    const int64_t total = staged + *n_out;
    *chunks = (int)(total / OWW_SAMPLES_PER_CHUNK);
    *staged_after = (int)(total - (int64_t)*chunks * OWW_SAMPLES_PER_CHUNK);
    return true;
}

}  // namespace

// per rate of the table: up, down, taps per phase K, offset of its polyphase table (phase p, tap t at off + p*K + t:
// h[p + up*t], zero past N)
struct IngestRate { int up, down, K, off; };
struct IngestRates { IngestRate r[kNRates]; };      // the whole table, passed to the kernel by value

// per stream and call
struct IngestRow {
    int64_t in_off;                   // first new input sample in d_in
    int64_t s_prev;                   // input samples before this call since the restart (0: zero history)
    int32_t n_in;                     // new input samples
    int32_t rate;                     // index into the rate table
    int32_t rem_off;                  // where the staged samples start in the row
    int32_t rem;                      // staged samples
    int32_t n_out;                    // new final outputs
    int32_t pad;
};

struct oww_ingest_state {
    int n_streams = 0;
    int64_t cap = 0;                  // staging row, samples
    int16_t* d_stage = nullptr;       // [B][cap]
    int16_t* d_hist = nullptr;        // [B][ING_HIST]
    int* d_ids = nullptr;             // [B] id staging of export / import
    float* d_taps = nullptr;          // polyphase tables of every rate
    IngestRates rates;
    std::vector<int> rate;            // per stream, Hz
    std::vector<int64_t> S;
    std::vector<int> staged, staged_off;
    IngestRow* h_rows[ING_SLOTS] = {nullptr, nullptr, nullptr, nullptr};
    IngestRow* d_rows[ING_SLOTS] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t ev[ING_SLOTS] = {nullptr, nullptr, nullptr, nullptr};
    int next = 0;
    std::vector<int32_t> chunks;      // scratch of a call
};

// One 16 kHz output, the single definition both resamplers use: output index i0 + j of a rate whose output i0 reads input
// q00 (r0 = i0 * down - q00 * up), with q00 at position `base` of the caller's input; load(k) returns the input at
// position k.  One fp32 FMA chain over the phase's K taps (zero taps included), newest input first, from 0; then round
// half to even and saturate.
template <typename Load>
__device__ __forceinline__ int16_t resample_output(const IngestRate& rt, const float* __restrict__ taps, int r0, int base,
                                                   int j, Load load) {
    const int frac = r0 + j * rt.down;
    const int dq = frac / rt.up;
    const int p = frac - dq * rt.up;
    const int local = base + dq;                                // newest input sample the output reads
    const float* h = taps + rt.off + p * rt.K;
    float acc = 0.f;
    for (int t = 0; t < rt.K; ++t) acc = fmaf(h[t], load(local - t), acc);
    const int r = __float2int_rn(acc);                          // round half to even
    return (int16_t)max(-32768, min(32767, r));
}

// The kernels stay outside the anonymous namespace: their names in a profile do not depend on the build.
// CTA b: stream b of the call (rows[b]).
__global__ void __launch_bounds__(ING_THREADS) resample_kernel(const int16_t* __restrict__ in,
                                                               const IngestRow* __restrict__ rows, const IngestRates rates,
                                                               const float* __restrict__ taps, int16_t* __restrict__ stage,
                                                               int64_t cap, int16_t* __restrict__ hist) {
    __shared__ int16_t s_rem[OWW_SAMPLES_PER_CHUNK];
    __shared__ int16_t s_hist[ING_HIST];
    const int b = blockIdx.x;
    const IngestRow R = rows[b];
    if (R.n_in == 0 && R.rem_off == 0 && R.n_out == 0) return;
    int16_t* row = stage + (size_t)b * cap;
    int16_t* hb = hist + (size_t)b * ING_HIST;
    const IngestRate rt = rates.r[R.rate];
    const bool identity = rt.up == rt.down;
    const int16_t* x = in + R.in_off;
    // read everything this CTA overwrites before the first write
    const bool move = R.rem_off != 0;
    if (move) for (int k = threadIdx.x; k < R.rem; k += ING_THREADS) s_rem[k] = row[R.rem_off + k];
    if (!identity) for (int k = threadIdx.x; k < ING_HIST; k += ING_THREADS) s_hist[k] = R.s_prev ? hb[k] : (int16_t)0;
    __syncthreads();
    if (move) for (int k = threadIdx.x; k < R.rem; k += ING_THREADS) row[k] = s_rem[k];
    int16_t* out = row + R.rem;
    if (identity) {
        for (int j = threadIdx.x; j < R.n_out; j += ING_THREADS) out[j] = x[j];
        return;                                               // a 16 kHz stream keeps no history (a restart zeroes it)
    }
    // output i0 + j reads input q0 = floor((i0 + j) * down / up) and back, phase p = (i0 + j) * down mod up; the 64-bit
    // part is split off once per CTA, so each output needs one 32-bit division
    const int64_t i0 = (R.s_prev * rt.up + rt.down - 1) / rt.down;      // A(s_prev): global index of the first output
    const int64_t n0 = i0 * rt.down, q00 = n0 / rt.up;
    const int r0 = (int)(n0 - q00 * rt.up);
    const int base = (int)(q00 - R.s_prev);                    // >= 0: A(S) * down >= S * up
    const auto load = [&](int idx) { return (float)(idx >= 0 ? x[idx] : s_hist[ING_HIST + idx]); };
    for (int j = threadIdx.x; j < R.n_out; j += ING_THREADS) out[j] = resample_output(rt, taps, r0, base, j, load);
    // the new history: the last 128 samples of [old history | new input]
    for (int k = threadIdx.x; k < ING_HIST; k += ING_THREADS) {
        const int idx = R.n_in - ING_HIST + k;
        hb[k] = idx >= 0 ? x[idx] : s_hist[ING_HIST + idx];
    }
}

// ---- oww_resample_clips: whole clips, no state ----
// Clip c with n_in input samples and `pad` 16 kHz samples of padding has L = A(n_in) + 2*pad outputs: output i is output
// j = i - pad of upfirdn(h, clip, up, down) (pad*down/up leading zeros in front of the clip shift it by exactly pad
// outputs), and outputs with j < 0 read only those zeros, so they are 0.  The outputs are cut into tiles of CLIP_TILE; a
// CTA stages its tile's input window (the K - 1 samples before it included, zeros outside the clip) as fp32 in shared
// memory.  The window is at most (CLIP_TILE - 1) * down/up + 1 + (K - 1) samples; down/up <= 3 and K <= 61 in the table.
#define CLIP_TILE 2048
#define CLIP_WIN (3 * CLIP_TILE + 64)

struct ClipRow {                      // per clip of a call
    int64_t in_off, n_in;             // its input d_in[in_off, in_off + n_in)
    int64_t out_off, n_out;           // its outputs d_out[out_off, out_off + n_out), pads included
    int32_t rate;                     // index into the rate table
    int32_t unused;
};
struct ClipTile { int32_t clip, tile; };    // outputs [tile * CLIP_TILE, (tile + 1) * CLIP_TILE) of clip `clip`

__global__ void __launch_bounds__(ING_THREADS) resample_clips_kernel(const int16_t* __restrict__ in,
                                                                     const ClipRow* __restrict__ clips,
                                                                     const ClipTile* __restrict__ tiles,
                                                                     const IngestRates rates, const float* __restrict__ taps,
                                                                     int pad, int16_t* __restrict__ out) {
    __shared__ float s_in[CLIP_WIN];
    const ClipTile T = tiles[blockIdx.x];
    const ClipRow C = clips[T.clip];
    const IngestRate rt = rates.r[C.rate];
    const int64_t i_first = (int64_t)T.tile * CLIP_TILE;
    const int n = (int)min((int64_t)CLIP_TILE, C.n_out - i_first);
    int16_t* y = out + C.out_off + i_first;
    const int16_t* x = in + C.in_off;
    const int64_t j_first = i_first - pad;
    const int lead = (int)max((int64_t)0, min((int64_t)n, -j_first));   // outputs of the tile in the leading pad
    for (int k = threadIdx.x; k < lead; k += ING_THREADS) y[k] = 0;
    if (lead == n) return;
    const int64_t j0 = j_first + lead;                                     // >= 0
    const int m = n - lead;
    y += lead;
    if (rt.up == rt.down) {                                                // 16 kHz: a copy, zeros past the clip
        for (int k = threadIdx.x; k < m; k += ING_THREADS) y[k] = j0 + k < C.n_in ? x[j0 + k] : (int16_t)0;
        return;
    }
    // the 64-bit part split off once per tile: output j0 reads input q00, phase r0; the window starts K - 1 before it
    const int64_t n0 = j0 * rt.down, q00 = n0 / rt.up;
    const int r0 = (int)(n0 - q00 * rt.up);
    const int64_t q_lo = q00 - (rt.K - 1);
    const int w = (r0 + (m - 1) * rt.down) / rt.up + rt.K;
    for (int k = threadIdx.x; k < w; k += ING_THREADS) {
        const int64_t q = q_lo + k;
        s_in[k] = q >= 0 && q < C.n_in ? (float)x[q] : 0.f;
    }
    __syncthreads();
    const auto load = [&](int idx) { return s_in[idx]; };
    for (int k = threadIdx.x; k < m; k += ING_THREADS) y[k] = resample_output(rt, taps, r0, rt.K - 1, k, load);
}

// record i <-> stream ids[i]: the staged samples [off, off + staged) of the row (export: row i of out, zeros after them)
// and the history
__global__ void __launch_bounds__(ING_THREADS) ingest_export_kernel(const int* __restrict__ ids, const int* __restrict__ info,
                                                                    const int16_t* __restrict__ stage, int64_t cap,
                                                                    const int16_t* __restrict__ hist,
                                                                    int16_t* __restrict__ out, int64_t stride,
                                                                    int16_t* __restrict__ out_hist) {
    const int i = blockIdx.x, b = ids[i];
    const int off = info[3 * i], n = info[3 * i + 1], zero_hist = info[3 * i + 2];
    const int16_t* row = stage + (size_t)b * cap + off;
    for (int64_t k = threadIdx.x; k < stride; k += ING_THREADS) out[(size_t)i * stride + k] = k < n ? row[k] : (int16_t)0;
    for (int k = threadIdx.x; k < ING_HIST; k += ING_THREADS)
        out_hist[(size_t)i * ING_HIST + k] = zero_hist ? (int16_t)0 : hist[(size_t)b * ING_HIST + k];
}

__global__ void __launch_bounds__(ING_THREADS) ingest_import_kernel(const int* __restrict__ ids, const int* __restrict__ info,
                                                                    int16_t* __restrict__ stage, int64_t cap,
                                                                    int16_t* __restrict__ hist, const int16_t* __restrict__ in,
                                                                    int64_t stride, const int16_t* __restrict__ in_hist) {
    const int i = blockIdx.x, b = ids[i];
    const int n = info[3 * i + 1];
    int16_t* row = stage + (size_t)b * cap;
    for (int k = threadIdx.x; k < n; k += ING_THREADS) row[k] = in[(size_t)i * stride + k];
    for (int k = threadIdx.x; k < ING_HIST; k += ING_THREADS) hist[(size_t)b * ING_HIST + k] = in_hist[(size_t)i * ING_HIST + k];
}

namespace {

void free_stream_state(oww_ingest_state* g) {
    for (int j = 0; j < ING_SLOTS; ++j) {             // callers synchronise the device first
        cudaFreeHost(g->h_rows[j]); cudaFree(g->d_rows[j]); g->h_rows[j] = nullptr; g->d_rows[j] = nullptr;
    }
    cudaFree(g->d_stage); cudaFree(g->d_hist); cudaFree(g->d_ids);
    g->d_stage = nullptr; g->d_hist = nullptr; g->d_ids = nullptr;
    g->n_streams = 0;
    g->rate.clear(); g->S.clear(); g->staged.clear(); g->staged_off.clear();
}

void ingest_free(oww_ctx* ctx) {
    oww_ingest_state* g = ctx->ingest;
    if (!g) return;
    free_stream_state(g);
    cudaFree(g->d_taps);
    for (auto e : g->ev) if (e) cudaEventDestroy(e);
    delete g;
    ctx->ingest = nullptr;
}

// every stream at 16000 with nothing staged, for ctx->n_streams streams; the device is idle
int alloc_stream_state(oww_ctx* ctx) {
    oww_ingest_state* g = ctx->ingest;
    free_stream_state(g);
    const int B = ctx->n_streams;
    if (B <= 0) return OWW_OK;
    g->cap = (int64_t)ctx->cfg.max_chunks * OWW_SAMPLES_PER_CHUNK + OWW_SAMPLES_PER_CHUNK - 1;
    OWW_CUDA(ctx, cudaMalloc(&g->d_stage, (size_t)B * g->cap * sizeof(int16_t)));
    OWW_CUDA(ctx, cudaMalloc(&g->d_hist, (size_t)B * ING_HIST * sizeof(int16_t)));
    OWW_CUDA(ctx, cudaMalloc(&g->d_ids, (size_t)B * (sizeof(int) + 3 * sizeof(int))));
    for (int j = 0; j < ING_SLOTS; ++j) {
        OWW_CUDA(ctx, cudaMallocHost(&g->h_rows[j], (size_t)B * sizeof(IngestRow)));
        OWW_CUDA(ctx, cudaMalloc(&g->d_rows[j], (size_t)B * sizeof(IngestRow)));
        if (!g->ev[j]) OWW_CUDA(ctx, cudaEventCreateWithFlags(&g->ev[j], cudaEventDisableTiming));
    }
    g->rate.assign(B, 16000);
    g->S.assign(B, 0);
    g->staged.assign(B, 0);
    g->staged_off.assign(B, 0);
    g->n_streams = B;
    return OWW_OK;
}

// the polyphase tables of every rate, uploaded to *d_taps
int upload_taps(oww_ctx* ctx, IngestRates* rates, float** d_taps) {
    std::vector<float> all;
    for (int r = 0; r < kNRates; ++r) {
        IngestRate& R = rates->r[r];
        R.off = (int)all.size();
        if (kRates[r] == 16000) { R.up = R.down = 1; R.K = 0; continue; }
        const std::vector<double> h = design(kRates[r], &R.up, &R.down);
        const int N = (int)h.size();
        R.K = (N + R.up - 1) / R.up;
        all.resize(all.size() + (size_t)R.up * R.K, 0.f);
        for (int p = 0; p < R.up; ++p)
            for (int t = 0; t < R.K; ++t)
                if (p + R.up * t < N) all[R.off + (size_t)p * R.K + t] = (float)h[p + R.up * t];
    }
    OWW_CUDA(ctx, cudaMalloc(d_taps, all.size() * sizeof(float)));
    OWW_CUDA(ctx, cudaMemcpy(*d_taps, all.data(), all.size() * sizeof(float), cudaMemcpyHostToDevice));
    return OWW_OK;
}

// n_in samples at `rate` with `pad` 16 kHz samples of padding -> outputs (A(n_in) + 2*pad); false for arguments
// oww_resample_clip_plan refuses
bool clip_plan(int rate, int64_t n_in, int pad, int64_t* n_out) {
    if (rate_index(rate) < 0 || n_in < 0 || pad < 0) return false;
    int up, down;
    up_down(rate, &up, &down);
    if (pad % up) return false;
    *n_out = final_outputs(n_in, up, down) + 2 * (int64_t)pad;
    return true;
}

}  // namespace

// The clip resampler's own taps and tables: kept apart from oww_ingest_state, whose existence means "the handle's
// streams take ingest" to oww_set_input_rates.
struct oww_clip_resampler {
    IngestRates rates;
    float* d_taps = nullptr;
    void* h_tab = nullptr;            // pinned: ClipRow [n_clips], then ClipTile [n_tiles]
    void* d_tab = nullptr;
    size_t tab_bytes = 0;
    cudaEvent_t done = nullptr;       // after the last launch: the tables may be rewritten once it has completed
};

namespace {

void clip_free(oww_ctx* ctx) {
    oww_clip_resampler* c = ctx->clip_rs;
    if (!c) return;
    cudaFree(c->d_taps); cudaFreeHost(c->h_tab); cudaFree(c->d_tab);
    if (c->done) cudaEventDestroy(c->done);
    delete c;
    ctx->clip_rs = nullptr;
}

int check_ids(oww_ctx* ctx, const int32_t* h_ids, int n, bool distinct) {
    const int B = ctx->n_streams;
    if (n < 0 || n > B) return oww_fail(ctx, OWW_EINVAL, "n=%d outside [0,%d]", n, B);
    if (n && !h_ids) return oww_fail(ctx, OWW_EINVAL, "null argument");
    std::vector<uint8_t> hit(B, 0);
    for (int i = 0; i < n; ++i) {
        if (h_ids[i] < 0 || h_ids[i] >= B) return oww_fail(ctx, OWW_EINVAL, "stream id %d out of range", h_ids[i]);
        if (distinct && hit[h_ids[i]]++) return oww_fail(ctx, OWW_EINVAL, "stream id %d given twice", h_ids[i]);
    }
    return OWW_OK;
}

int need_state(oww_ctx* ctx) {
    if (!ctx->ingest || !ctx->ingest->d_stage)
        return oww_fail(ctx, OWW_EINVAL, "no ingest state (oww_set_input_rates after oww_set_streams)");
    return OWW_OK;
}

}  // namespace

void oww_ingest_free(oww_ctx* ctx) { ingest_free(ctx); clip_free(ctx); }

void oww_ingest_free_streams(oww_ctx* ctx) { if (ctx->ingest) free_stream_state(ctx->ingest); }

int oww_ingest_alloc_streams(oww_ctx* ctx) { return ctx->ingest ? alloc_stream_state(ctx) : OWW_OK; }

void oww_ingest_reset(oww_ctx* ctx, const int32_t* h_ids, int n) {
    oww_ingest_state* g = ctx->ingest;
    if (!g || !g->d_stage) return;
    for (int i = 0; i < n; ++i) {
        const int b = h_ids ? h_ids[i] : i;
        g->S[b] = 0; g->staged[b] = 0; g->staged_off[b] = 0;
    }
}

int oww_ingest_check(oww_ctx* ctx, const int64_t* h_offsets) {
    int rc = need_state(ctx);
    if (rc) return rc;
    const oww_ingest_state* g = ctx->ingest;
    if (!h_offsets) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (!ctx->mel_loaded || !ctx->emb_loaded) return oww_fail(ctx, OWW_EINVAL, "weights not loaded");
    if (h_offsets[0] < 0) return oww_fail(ctx, OWW_EINVAL, "offsets[0]=%lld is negative", (long long)h_offsets[0]);
    for (int b = 0; b < g->n_streams; ++b) {
        const int64_t n = h_offsets[b + 1] - h_offsets[b];
        if (n < 0) return oww_fail(ctx, OWW_EINVAL, "offsets decrease at stream %d", b);
        int64_t n_out, max_in;
        int c, after;
        if (!plan(g->rate[b], ctx->cfg.max_chunks, g->S[b], g->staged[b], n, &n_out, &c, &after, &max_in))
            return oww_fail(ctx, OWW_EINVAL, "stream %d: %lld input samples, its capacity is %lld (oww_ingest_capacity)", b,
                            (long long)n, (long long)max_in);
    }
    return OWW_OK;
}

extern "C" {

int oww_resampler_taps(int rate, float* h_taps, int max, int* up, int* down) {
    if (rate_index(rate) < 0) return OWW_EINVAL;
    int u, d;
    if (rate == 16000) { u = d = 1; }
    else {
        const std::vector<double> h = design(rate, &u, &d);
        for (int k = 0; h_taps && k < std::min(max, (int)h.size()); ++k) h_taps[k] = (float)h[k];
        if (up) *up = u;
        if (down) *down = d;
        return (int)h.size();
    }
    if (up) *up = u;
    if (down) *down = d;
    return 0;
}

int oww_ingest_plan(int rate, int max_chunks, int64_t n_before, int staged, int64_t n_in, int64_t* n_out, int32_t* chunks,
                    int32_t* staged_after, int64_t* max_in) {
    if (rate_index(rate) < 0 || max_chunks < 1 || n_before < 0 || staged < 0) return OWW_EINVAL;
    int64_t no = 0, mi = 0;
    int c = 0, sa = 0;
    const bool ok = plan(rate, max_chunks, n_before, staged, n_in, &no, &c, &sa, &mi);
    if (max_in) *max_in = mi;
    if (!ok) return OWW_EINVAL;
    if (n_out) *n_out = no;
    if (chunks) *chunks = c;
    if (staged_after) *staged_after = sa;
    return OWW_OK;
}

int oww_set_input_rates(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const int32_t* h_rates, void* stream) {
    (void)stream;                                     // host state only: it applies to the calls enqueued after it
    if (!ctx) return OWW_EINVAL;
    if (ctx->n_streams <= 0) return oww_fail(ctx, OWW_EINVAL, "oww_set_streams has not been called");
    if (!h_stream_ids) n = ctx->n_streams;
    int rc = check_ids(ctx, h_stream_ids, h_stream_ids ? n : 0, false);
    if (rc) return rc;
    if (n && !h_rates) return oww_fail(ctx, OWW_EINVAL, "null argument");
    for (int i = 0; i < n; ++i)
        if (rate_index(h_rates[i]) < 0) return oww_fail(ctx, OWW_EINVAL, "input rate %d is not in the rate table", h_rates[i]);
    if (!ctx->ingest) {
        OWW_CUDA(ctx, cudaSetDevice(ctx->device));
        OWW_CUDA(ctx, cudaDeviceSynchronize());
        ctx->ingest = new (std::nothrow) oww_ingest_state();
        if (!ctx->ingest) return oww_fail(ctx, OWW_ENOMEM, "out of host memory");
        oww_ingest_state* g = ctx->ingest;
        if ((rc = upload_taps(ctx, &g->rates, &g->d_taps)) || (rc = alloc_stream_state(ctx))) { ingest_free(ctx); return rc; }
    }
    oww_ingest_state* g = ctx->ingest;
    for (int i = 0; i < n; ++i) {
        const int b = h_stream_ids ? h_stream_ids[i] : i;
        g->rate[b] = h_rates[i];
        g->S[b] = 0;
    }
    return OWW_OK;
}

int oww_ingest_capacity(oww_ctx* ctx, int64_t* h_max_in) {
    if (!ctx) return OWW_EINVAL;
    int rc = need_state(ctx);
    if (rc) return rc;
    if (!h_max_in) return oww_fail(ctx, OWW_EINVAL, "null argument");
    const oww_ingest_state* g = ctx->ingest;
    for (int b = 0; b < g->n_streams; ++b) {
        int64_t no; int c, sa;
        plan(g->rate[b], ctx->cfg.max_chunks, g->S[b], g->staged[b], 0, &no, &c, &sa, &h_max_in[b]);
    }
    return OWW_OK;
}

int oww_ingest(oww_ctx* ctx, const int16_t* d_in, const int64_t* h_offsets, int32_t* h_chunks_out, int32_t* h_prepared_out,
               float* d_scores, void* stream) {
    if (!ctx) return OWW_EINVAL;
    int rc = need_state(ctx);
    if (rc) return rc;
    oww_ingest_state* g = ctx->ingest;
    const int B = g->n_streams;
    if (!h_offsets || !d_scores) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (!ctx->mel_loaded || !ctx->emb_loaded) return oww_fail(ctx, OWW_EINVAL, "weights not loaded");
    if (h_offsets[0] < 0) return oww_fail(ctx, OWW_EINVAL, "offsets[0]=%lld is negative", (long long)h_offsets[0]);
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    const int j = g->next;
    OWW_CUDA(ctx, cudaEventSynchronize(g->ev[j]));             // the table copy of the call ING_SLOTS back has run
    IngestRow* rows = g->h_rows[j];
    g->chunks.resize(B);
    bool any = false;
    for (int b = 0; b < B; ++b) {
        const int64_t n = h_offsets[b + 1] - h_offsets[b];
        if (n < 0) return oww_fail(ctx, OWW_EINVAL, "offsets decrease at stream %d", b);
        int64_t n_out, max_in;
        int c, after;
        if (!plan(g->rate[b], ctx->cfg.max_chunks, g->S[b], g->staged[b], n, &n_out, &c, &after, &max_in))
            return oww_fail(ctx, OWW_EINVAL, "stream %d: %lld input samples, its capacity is %lld (oww_ingest_capacity)", b,
                            (long long)n, (long long)max_in);
        rows[b] = IngestRow{h_offsets[b], g->S[b], (int32_t)n, rate_index(g->rate[b]), g->staged_off[b], g->staged[b],
                            (int32_t)n_out, 0};
        g->chunks[b] = c;
        any = any || n > 0 || g->staged_off[b] != 0;
    }
    if (h_offsets[B] > h_offsets[0] && !d_in) return oww_fail(ctx, OWW_EINVAL, "null argument");
    cudaStream_t s = (cudaStream_t)stream;
    if (any) {
        g->next = (j + 1) % ING_SLOTS;
        OWW_CUDA(ctx, cudaMemcpyAsync(g->d_rows[j], rows, (size_t)B * sizeof(IngestRow), cudaMemcpyHostToDevice, s));
        OWW_CUDA(ctx, cudaEventRecord(g->ev[j], s));
        resample_kernel<<<B, ING_THREADS, 0, s>>>(d_in, g->d_rows[j], g->rates, g->d_taps, g->d_stage, g->cap, g->d_hist);
        OWW_LAUNCH_CHECK(ctx);
    }
    if ((rc = oww_step_ragged(ctx, g->d_stage, g->cap, g->chunks.data(), d_scores, stream))) return rc;
    for (int b = 0; b < B; ++b) {
        const IngestRow& R = rows[b];
        const int total = R.rem + R.n_out, c = g->chunks[b];
        g->S[b] += R.n_in;
        g->staged[b] = total - c * OWW_SAMPLES_PER_CHUNK;
        g->staged_off[b] = c * OWW_SAMPLES_PER_CHUNK;
        if (h_chunks_out) h_chunks_out[b] = c;
        if (h_prepared_out) h_prepared_out[b] = c ? c * OWW_SAMPLES_PER_CHUNK : total;
    }
    return OWW_OK;
}

int oww_ingest_export(oww_ctx* ctx, const int32_t* h_stream_ids, int n, int32_t* h_rates, int64_t* h_consumed,
                      int32_t* h_staged, int16_t* d_staged, int64_t staged_stride, int16_t* d_hist, void* stream) {
    if (!ctx) return OWW_EINVAL;
    int rc = need_state(ctx);
    if (rc || (rc = check_ids(ctx, h_stream_ids, n, false))) return rc;
    const oww_ingest_state* g = ctx->ingest;
    const bool device = d_staged || d_hist;
    if (device && (!d_staged || !d_hist)) return oww_fail(ctx, OWW_EINVAL, "null argument");
    std::vector<int> info(3 * (size_t)n);
    for (int i = 0; i < n; ++i) {
        const int b = h_stream_ids[i];
        if (device && g->staged[b] > staged_stride)
            return oww_fail(ctx, OWW_EINVAL, "stream %d holds %d staged samples, staged_stride is %lld", b, g->staged[b],
                            (long long)staged_stride);
        // no history before the first input, and none at 16 kHz (the kernel keeps no filter state for a copy): zeros
        info[3 * i] = g->staged_off[b]; info[3 * i + 1] = g->staged[b]; info[3 * i + 2] = g->S[b] == 0 || g->rate[b] == 16000;
    }
    for (int i = 0; i < n; ++i) {
        const int b = h_stream_ids[i];
        if (h_rates) h_rates[i] = g->rate[b];
        if (h_consumed) h_consumed[i] = g->S[b];
        if (h_staged) h_staged[i] = g->staged[b];
    }
    if (!device || n == 0) return OWW_OK;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    // pageable sources: staged by the driver before the call returns; stream-ordered on the device
    OWW_CUDA(ctx, cudaMemcpyAsync(g->d_ids, h_stream_ids, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    OWW_CUDA(ctx, cudaMemcpyAsync(g->d_ids + g->n_streams, info.data(), info.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    // the staged rows as the host counters describe them: after the detect calls submitted so far
    if ((rc = oww_order_begin(ctx, s))) return rc;
    ingest_export_kernel<<<n, ING_THREADS, 0, s>>>(g->d_ids, g->d_ids + g->n_streams, g->d_stage, g->cap, g->d_hist, d_staged,
                                                   staged_stride, d_hist);
    OWW_LAUNCH_CHECK(ctx);
    return oww_order_end(ctx, s);
}

int oww_ingest_import(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const int32_t* h_rates, const int64_t* h_consumed,
                      const int32_t* h_staged, const int16_t* d_staged, int64_t staged_stride, const int16_t* d_hist,
                      void* stream) {
    if (!ctx) return OWW_EINVAL;
    int rc = need_state(ctx);
    if (rc || (rc = check_ids(ctx, h_stream_ids, n, true))) return rc;
    if (n == 0) return OWW_OK;
    if (!h_rates || !h_consumed || !h_staged || !d_staged || !d_hist) return oww_fail(ctx, OWW_EINVAL, "null argument");
    oww_ingest_state* g = ctx->ingest;
    std::vector<int> info(3 * (size_t)n);
    for (int i = 0; i < n; ++i) {
        if (rate_index(h_rates[i]) < 0) return oww_fail(ctx, OWW_EINVAL, "input rate %d is not in the rate table", h_rates[i]);
        if (h_staged[i] < 0 || h_staged[i] > g->cap || h_staged[i] > staged_stride)
            return oww_fail(ctx, OWW_EINVAL, "staged count %d outside [0,%lld]", h_staged[i],
                            (long long)std::min(g->cap, staged_stride));
        if (h_consumed[i] < 0) return oww_fail(ctx, OWW_EINVAL, "negative input count");
        info[3 * i + 1] = h_staged[i];
    }
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    OWW_CUDA(ctx, cudaMemcpyAsync(g->d_ids, h_stream_ids, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    OWW_CUDA(ctx, cudaMemcpyAsync(g->d_ids + g->n_streams, info.data(), info.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    if ((rc = oww_order_begin(ctx, s))) return rc;
    ingest_import_kernel<<<n, ING_THREADS, 0, s>>>(g->d_ids, g->d_ids + g->n_streams, g->d_stage, g->cap, g->d_hist, d_staged,
                                                   staged_stride, d_hist);
    OWW_LAUNCH_CHECK(ctx);
    if ((rc = oww_order_end(ctx, s))) return rc;
    for (int i = 0; i < n; ++i) {
        const int b = h_stream_ids[i];
        g->rate[b] = h_rates[i]; g->S[b] = h_consumed[i]; g->staged[b] = h_staged[i]; g->staged_off[b] = 0;
    }
    return OWW_OK;
}

int oww_resample_clip_plan(int rate, int64_t n_in, int pad_samples, int64_t* n_out) {
    int64_t n = 0;
    if (!clip_plan(rate, n_in, pad_samples, &n)) return OWW_EINVAL;
    if (n_out) *n_out = n;
    return OWW_OK;
}

int oww_resample_clips(oww_ctx* ctx, const int16_t* d_in, const int64_t* h_in_offsets, const int32_t* h_rates, int n_clips,
                       int pad_samples, int16_t* d_out, const int64_t* h_out_offsets, void* stream) {
    if (!ctx) return OWW_EINVAL;
    if (n_clips < 0) return oww_fail(ctx, OWW_EINVAL, "n_clips=%d is negative", n_clips);
    if (pad_samples < 0) return oww_fail(ctx, OWW_EINVAL, "pad_samples=%d is negative", pad_samples);
    if (n_clips == 0) return OWW_OK;
    if (!h_in_offsets || !h_rates || !h_out_offsets) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (h_in_offsets[0] < 0 || h_out_offsets[0] < 0) return oww_fail(ctx, OWW_EINVAL, "negative first offset");
    int64_t n_tiles = 0;
    for (int i = 0; i < n_clips; ++i) {
        const int64_t n_in = h_in_offsets[i + 1] - h_in_offsets[i];
        if (n_in < 0) return oww_fail(ctx, OWW_EINVAL, "input offsets decrease at clip %d", i);
        if (rate_index(h_rates[i]) < 0)
            return oww_fail(ctx, OWW_EINVAL, "clip %d: rate %d is not in the rate table", i, h_rates[i]);
        int64_t L;
        if (!clip_plan(h_rates[i], n_in, pad_samples, &L))
            return oww_fail(ctx, OWW_EINVAL, "clip %d: pad_samples=%d is not a multiple of %d Hz's up factor", i,
                            pad_samples, h_rates[i]);
        if (h_out_offsets[i + 1] - h_out_offsets[i] != L)
            return oww_fail(ctx, OWW_EINVAL, "clip %d: output offsets give %lld samples, oww_resample_clip_plan %lld", i,
                            (long long)(h_out_offsets[i + 1] - h_out_offsets[i]), (long long)L);
        n_tiles += (L + CLIP_TILE - 1) / CLIP_TILE;
    }
    if (n_tiles > INT32_MAX) return oww_fail(ctx, OWW_EINVAL, "%lld tiles in one call", (long long)n_tiles);
    if (h_in_offsets[n_clips] > h_in_offsets[0] && !d_in) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (n_tiles == 0) return OWW_OK;
    if (!d_out) return oww_fail(ctx, OWW_EINVAL, "null argument");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->clip_rs) {
        ctx->clip_rs = new (std::nothrow) oww_clip_resampler();
        if (!ctx->clip_rs) return oww_fail(ctx, OWW_ENOMEM, "out of host memory");
        int rc = upload_taps(ctx, &ctx->clip_rs->rates, &ctx->clip_rs->d_taps);
        if (!rc && cudaEventCreateWithFlags(&ctx->clip_rs->done, cudaEventDisableTiming) != cudaSuccess)
            rc = oww_fail(ctx, OWW_ECUDA, "cudaEventCreate failed");
        if (rc) { clip_free(ctx); return rc; }
    }
    oww_clip_resampler* c = ctx->clip_rs;
    OWW_CUDA(ctx, cudaEventSynchronize(c->done));              // the previous call's tables have been read
    const size_t tile_off = (size_t)n_clips * sizeof(ClipRow);
    const size_t bytes = tile_off + (size_t)n_tiles * sizeof(ClipTile);
    if (bytes > c->tab_bytes) {
        cudaFreeHost(c->h_tab); cudaFree(c->d_tab);
        c->h_tab = nullptr; c->d_tab = nullptr; c->tab_bytes = 0;
        const size_t want = std::max(bytes, 2 * c->tab_bytes);
        OWW_CUDA(ctx, cudaMallocHost(&c->h_tab, want));
        OWW_CUDA(ctx, cudaMalloc(&c->d_tab, want));
        c->tab_bytes = want;
    }
    ClipRow* rows = (ClipRow*)c->h_tab;
    ClipTile* tiles = (ClipTile*)((char*)c->h_tab + tile_off);
    int64_t t = 0;
    for (int i = 0; i < n_clips; ++i) {
        const int64_t L = h_out_offsets[i + 1] - h_out_offsets[i];
        rows[i] = ClipRow{h_in_offsets[i], h_in_offsets[i + 1] - h_in_offsets[i], h_out_offsets[i], L, rate_index(h_rates[i]), 0};
        for (int64_t k = 0; k * CLIP_TILE < L; ++k) tiles[t++] = ClipTile{i, (int32_t)k};
    }
    cudaStream_t s = (cudaStream_t)stream;
    OWW_CUDA(ctx, cudaMemcpyAsync(c->d_tab, c->h_tab, bytes, cudaMemcpyHostToDevice, s));
    resample_clips_kernel<<<(unsigned)n_tiles, ING_THREADS, 0, s>>>(d_in, (const ClipRow*)c->d_tab,
                                                                   (const ClipTile*)((char*)c->d_tab + tile_off), c->rates,
                                                                   c->d_taps, pad_samples, d_out);
    OWW_LAUNCH_CHECK(ctx);
    OWW_CUDA(ctx, cudaEventRecord(c->done, s));
    return OWW_OK;
}

}  // extern "C"
