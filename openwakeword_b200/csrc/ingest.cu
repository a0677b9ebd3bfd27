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
    for (int j = threadIdx.x; j < R.n_out; j += ING_THREADS) {
        const int frac = r0 + j * rt.down;
        const int dq = frac / rt.up;
        const int p = frac - dq * rt.up;
        const int local = base + dq;                            // newest input sample the output reads
        const float* h = taps + rt.off + p * rt.K;
        float acc = 0.f;
        for (int t = 0; t < rt.K; ++t) {
            const int idx = local - t;
            const int16_t v = idx >= 0 ? x[idx] : s_hist[ING_HIST + idx];
            acc = fmaf(h[t], (float)v, acc);
        }
        const int r = __float2int_rn(acc);                      // round half to even
        out[j] = (int16_t)max(-32768, min(32767, r));
    }
    // the new history: the last 128 samples of [old history | new input]
    for (int k = threadIdx.x; k < ING_HIST; k += ING_THREADS) {
        const int idx = R.n_in - ING_HIST + k;
        hb[k] = idx >= 0 ? x[idx] : s_hist[ING_HIST + idx];
    }
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

// the polyphase tables of every rate, once per handle
int upload_taps(oww_ctx* ctx) {
    oww_ingest_state* g = ctx->ingest;
    std::vector<float> all;
    for (int r = 0; r < kNRates; ++r) {
        IngestRate& R = g->rates.r[r];
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
    OWW_CUDA(ctx, cudaMalloc(&g->d_taps, all.size() * sizeof(float)));
    OWW_CUDA(ctx, cudaMemcpy(g->d_taps, all.data(), all.size() * sizeof(float), cudaMemcpyHostToDevice));
    return OWW_OK;
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

void oww_ingest_free(oww_ctx* ctx) { ingest_free(ctx); }

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
        if ((rc = upload_taps(ctx)) || (rc = alloc_stream_state(ctx))) { ingest_free(ctx); return rc; }
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
        info[3 * i] = g->staged_off[b]; info[3 * i + 1] = g->staged[b]; info[3 * i + 2] = g->S[b] == 0;
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
    ingest_export_kernel<<<n, ING_THREADS, 0, s>>>(g->d_ids, g->d_ids + g->n_streams, g->d_stage, g->cap, g->d_hist, d_staged,
                                                   staged_stride, d_hist);
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
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
    ingest_import_kernel<<<n, ING_THREADS, 0, s>>>(g->d_ids, g->d_ids + g->n_streams, g->d_stage, g->cap, g->d_hist, d_staged,
                                                   staged_stride, d_hist);
    OWW_LAUNCH_CHECK(ctx);
    for (int i = 0; i < n; ++i) {
        const int b = h_stream_ids[i];
        g->rate[b] = h_rates[i]; g->S[b] = h_consumed[i]; g->staged[b] = h_staged[i]; g->staged_off[b] = 0;
    }
    return OWW_OK;
}

}  // extern "C"
