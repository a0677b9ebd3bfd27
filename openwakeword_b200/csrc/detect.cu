// Detections on the device: the half of Model.predict that turns a step's scores into detections (openwakeword/model.py:
// 303-363) - per-stream prediction history, zeroing of the first five predictions, patience, debounce, the "repeat the
// previous prediction below 1280 samples" rule and the threshold - for every (stream, label) in one kernel, and the
// detections returned as a compact, ordered event list.  Semantics: include/owwb200.h (oww_set_detector, oww_detect);
// restated per stream in oracle/detect.py.
//
// State: hist [30][B * n_labels] fp32 (ring slot s of pair p = stream * n_labels + label at hist[s * P + p]: the threads of
// a warp read one slot of neighbouring pairs, so every history pass is coalesced) and count [B] int32 (predictions
// appended since the stream's reset; ring slot = count % 30).  Per-stream settings (oww_set_stream_detection): ovr
// [B * n_labels] records at pair p and ovr_deb [B] doubles, read only while some stream has an override; the host keeps
// the table and uploads it whole, so the device copy never needs a scatter or a clear.
//
// Event compaction is two launches rather than one pass with decoupled look-back: detect_kernel leaves each CTA's event
// count and each pair's fired score, detect_events_kernel sums the counts of the CTAs before it (a few hundred ints at
// 8192 streams) and writes its events behind them.  No CTA ever waits for another, so nothing can spin on a device that
// is shared, and the order - ascending (stream, label) - follows from the thread mapping alone.
#include <cmath>
#include <cstring>
#include "oww_internal.h"

#define DET_HIST 30
#define DET_THREADS 256
#define DET_MAX_LABELS 256
// count is rebased by a multiple of 30 past 2^30 (2.7 years at 12.5 predictions/s): the ring slot and min(count, 30) stay
#define DET_COUNT_REBASE (35791392 * 30)

struct oww_detector {
    std::vector<oww_detect_label> labels;
    double debounce = 0.0;
    oww_detect_label* d_labels = nullptr;
    int n_streams = 0;                 // streams the state below is allocated for
    float* d_hist = nullptr;           // [30][B * L]
    int* d_count = nullptr;            // [B]
    float* d_fire = nullptr;           // [B * L] final score of the pairs that fired in the last call, NaN elsewhere
    int* d_cta = nullptr;              // [CTAs] events per CTA of the last call
    int* d_ids = nullptr;              // [B] staging of export / import ids
    std::vector<oww_stream_detect> ovr;   // [B * L] per-stream settings (host copy of d_ovr); kNoOverride: the handle's
    std::vector<double> ovr_deb;          // [B] per-stream debounce, NaN: the handle's
    int n_ovr = 0;                        // streams with an override; 0: oww_detect passes no table
    oww_stream_detect* d_ovr = nullptr;
    double* d_ovr_deb = nullptr;
    // per-stream `prepared` of a call, staged like the counts of oww_step_ragged
    static constexpr int kSlots = 4;
    int32_t* h_prep[kSlots] = {nullptr, nullptr, nullptr, nullptr};
    int32_t* d_prep[kSlots] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t ev[kSlots] = {nullptr, nullptr, nullptr, nullptr};
    int next = 0;
};

static const oww_stream_detect kNoOverride = {NAN, -1, 0};

static __device__ __forceinline__ int det_wrap(int c) { return c >= OWW_COUNT_WRAP ? c - DET_COUNT_REBASE : c; }

// streams per CTA: whole streams only, so that the one count of a stream is read by all its threads before it is written
static inline int det_streams_per_cta(int L) { return DET_THREADS / L; }

// The rule of one prediction of one (stream or clip, label), model.py:303-363.  stepped: the call stepped at least one
// chunk, and `score` is its score; prep: the samples it prepared; c: the predictions appended before it (only c > 0,
// c < 5 and min(c, 30) matter); hist(i): the prediction appended i + 1 calls ago, i < min(c, 30).  p (NaN: none): a
// verifier's p on the call's newest window, which a repeated prediction >= vthr becomes (Model.predict re-verifies it).
template <class Hist>
static __device__ __forceinline__ float det_rule(const oww_detect_label& lab, bool stepped, float score, float p, float vthr,
                                                 int c, int prep, double debounce, Hist hist) {
    const int n = min(c, DET_HIST);
    float pred = 0.f;
    if (stepped) pred = score;
    else if (lab.repeats && c > 0) pred = hist(0);
    if (!stepped && !isnan(p) && pred >= vthr) pred = p;
    if (c < 5) pred = 0.f;
    if (lab.patience > 0) {
        if (pred != 0.f) {
            const int k = min(lab.patience, n);
            int ge = 0;
            for (int i = 0; i < k; ++i) ge += hist(i) >= lab.threshold;
            if (ge < lab.patience) pred = 0.f;
        }
    } else if (debounce > 0.0 && !isnan(lab.threshold) && pred != 0.f && pred >= lab.threshold) {
        int k = n;
        if (prep > 0) {
            const double nf = ceil(debounce / ((double)prep / 16000.0));
            if (nf < (double)k) k = (int)nf;
        }
        bool hit = false;
        for (int i = 0; i < k; ++i) hit = hit || hist(i) >= lab.threshold;
        if (hit) pred = 0.f;
    }
    return pred;
}

// The kernels stay outside the anonymous namespace: their names in a profile do not depend on the build.
// One thread per (stream, label); CTA `blockIdx.x` owns streams [blockIdx.x * S, +S).
__global__ void __launch_bounds__(DET_THREADS) detect_kernel(const float* __restrict__ scores, int n_out, int B, int L, int S,
                                                             const oww_detect_label* __restrict__ labels, double debounce,
                                                             const oww_stream_detect* __restrict__ ovr,
                                                             const double* __restrict__ ovr_deb, int prepared_all, const int* __restrict__ prepared,
                                                             float* __restrict__ hist, int* __restrict__ count,
                                                             float* __restrict__ d_final, float* __restrict__ fire,
                                                             int* __restrict__ cta_events) {
    const int sl = threadIdx.x / L, j = threadIdx.x - sl * L;
    const int b = blockIdx.x * S + sl;
    const bool live = sl < S && b < B;
    const size_t P = (size_t)B * L, p = (size_t)b * L + j;
    int prep = -1, c = 0;
    if (live) {
        prep = prepared ? prepared[b] : prepared_all;
        c = count[b];
    }
    bool fired = false;
    float pred = 0.f;
    if (prep >= 0) {
        oww_detect_label lab = labels[j];
        if (ovr) {                                           // this stream's settings (oww_set_stream_detection)
            const oww_stream_detect o = ovr[p];
            if (o.flags & OWW_DETECT_NO_THRESHOLD) lab.threshold = __int_as_float(0x7fc00000);
            else if (!isnan(o.threshold)) lab.threshold = o.threshold;
            if (o.patience >= 0) lab.patience = o.patience;
            if (!isnan(ovr_deb[b])) debounce = ovr_deb[b];
        }
        const bool stepped = prep >= OWW_SAMPLES_PER_CHUNK;
        const float score = stepped && lab.column >= 0 ? scores[(size_t)b * n_out + lab.column] : 0.f;
        pred = det_rule(lab, stepped, score, __int_as_float(0x7fc00000), 0.f, c, prep, debounce,
                        [&](int i) { return hist[(size_t)((c - 1 - i) % DET_HIST) * P + p]; });
        fired = !isnan(lab.threshold) && pred >= lab.threshold;
        hist[(size_t)(c % DET_HIST) * P + p] = pred;
        if (d_final) d_final[p] = pred;
    }
    if (live) fire[p] = fired ? pred : __int_as_float(0x7fc00000);
    const int n_fired = __syncthreads_count(fired);          // also: every thread of a stream has read its count
    if (prep >= 0 && j == 0) count[b] = det_wrap(c + 1);
    if (threadIdx.x == 0) cta_events[blockIdx.x] = n_fired;
}

// Same grid and thread mapping.  Events of this CTA start behind those of the CTAs before it.
__global__ void __launch_bounds__(DET_THREADS) detect_events_kernel(const float* __restrict__ fire, const int* __restrict__ count,
                                                                    const int* __restrict__ cta_events, int B, int L, int S,
                                                                    oww_event* __restrict__ events, int max_events,
                                                                    int* __restrict__ n_events) {
    __shared__ int s_sum[DET_THREADS / 32];
    __shared__ int s_fired[DET_THREADS / 32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int part = 0;
    for (int i = threadIdx.x; i < (int)blockIdx.x; i += DET_THREADS) part += cta_events[i];
    for (int o = 16; o; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    const int sl = threadIdx.x / L, j = threadIdx.x - sl * L;
    const int b = blockIdx.x * S + sl;
    const bool live = sl < S && b < B;
    const float sc = live ? fire[(size_t)b * L + j] : __int_as_float(0x7fc00000);
    const bool f = !isnan(sc);
    const unsigned m = __ballot_sync(0xffffffffu, f);
    if (lane == 0) { s_sum[warp] = part; s_fired[warp] = __popc(m); }
    __syncthreads();
    int base = 0, before = 0;
    for (int w = 0; w < DET_THREADS / 32; ++w) {
        base += s_sum[w];
        if (w < warp) before += s_fired[w];
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0 && n_events) *n_events = base + cta_events[blockIdx.x];
    const int pos = base + before + __popc(m & ((1u << lane) - 1u));
    if (f && events && pos < max_events) events[pos] = oww_event{b, j, sc, count[b] - 1};
}

// The delivery of oww_detect_host_submit: the count, the first k = min(count, max_events) events and, with capture > 0,
// their ends and clip rows, from the device buffers of the call (oww_detect_layout) into its mapped host buffer, so that
// PCIe carries only what was found.  CTA 0 writes the count.  Without capture thread t of the grid writes event t; with
// capture CTA i writes event i, its end and its clip row.  CTAs past the count exit at once, as in audio_capture_kernel.
__global__ void __launch_bounds__(DET_THREADS) detect_deliver_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                                     DetectLayout lay, int max_events, int capture) {
    const int n = *reinterpret_cast<const int*>(src);
    const int k = min(n, max_events);
    if (blockIdx.x == 0 && threadIdx.x == 0) *reinterpret_cast<int*>(dst) = n;
    const uint4* ev = reinterpret_cast<const uint4*>(src + lay.events);     // oww_event: 16 bytes
    uint4* ev_out = reinterpret_cast<uint4*>(dst + lay.events);
    if (capture == 0) {
        const int i = blockIdx.x * DET_THREADS + threadIdx.x;
        if (i < k) ev_out[i] = ev[i];
        return;
    }
    const int i = blockIdx.x;
    if (i >= k) return;
    if (threadIdx.x == 0) {
        ev_out[i] = ev[i];
        reinterpret_cast<int64_t*>(dst + lay.ends)[i] = reinterpret_cast<const int64_t*>(src + lay.ends)[i];
    }
    const int16_t* row = reinterpret_cast<const int16_t*>(src + lay.clips) + (size_t)i * capture;
    int16_t* out = reinterpret_cast<int16_t*>(dst + lay.clips) + (size_t)i * capture;
    int j0 = 0;
    if (((reinterpret_cast<uintptr_t>(row) | reinterpret_cast<uintptr_t>(out)) & 15) == 0) {   // 8 samples per store
        const int nv = capture / 8;
        for (int j = threadIdx.x; j < nv; j += DET_THREADS)
            reinterpret_cast<uint4*>(out)[j] = reinterpret_cast<const uint4*>(row)[j];
        j0 = nv * 8;
    }
    for (int j = j0 + threadIdx.x; j < capture; j += DET_THREADS) out[j] = row[j];
}

// streams ids[0..n) (nullptr: stream blockIdx.x) start afresh: an empty history
__global__ void detect_clear_kernel(const int* ids, int B, int L, float* hist, int* count) {
    const int b = ids ? ids[blockIdx.x] : blockIdx.x;
    const size_t P = (size_t)B * L;
    for (int i = threadIdx.x; i < DET_HIST * L; i += blockDim.x) hist[(size_t)(i / L) * P + (size_t)b * L + i % L] = 0.f;
    if (threadIdx.x == 0) count[b] = 0;
}

// record i <-> stream ids[i]: [L][30] oldest first (entry k = the prediction 30 - k appends ago; zeros before the first)
__global__ void detect_export_kernel(const int* ids, int B, int L, const float* hist, const int* count, float* out, int* out_count) {
    const int b = ids[blockIdx.x], c = count[b];
    const size_t P = (size_t)B * L;
    for (int i = threadIdx.x; i < DET_HIST * L; i += blockDim.x) {
        const int j = i / DET_HIST, k = i - j * DET_HIST;
        out[(size_t)blockIdx.x * L * DET_HIST + i] = hist[(size_t)((c % DET_HIST + k) % DET_HIST) * P + (size_t)b * L + j];
    }
    if (threadIdx.x == 0) out_count[blockIdx.x] = c;
}

__global__ void detect_import_kernel(const int* ids, int B, int L, float* hist, int* count, const float* in, const int* in_count) {
    const int b = ids[blockIdx.x];
    const int c = det_wrap(max(in_count[blockIdx.x], 0));
    const size_t P = (size_t)B * L;
    for (int i = threadIdx.x; i < DET_HIST * L; i += blockDim.x) {
        const int j = i / DET_HIST, k = i - j * DET_HIST;
        hist[(size_t)((c % DET_HIST + k) % DET_HIST) * P + (size_t)b * L + j] = in[(size_t)blockIdx.x * L * DET_HIST + i];
    }
    if (threadIdx.x == 0) count[b] = c;
}

// ---- the bulk clip path (oww_detect_clips) ----
// One thread per (clip, label), CTA `blockIdx.x` owns clips [blockIdx.x * S, +S).  Each thread walks its clip's rows in
// call order from an empty history, kept as a ring in shared memory (ring[slot][threadIdx.x]: no bank conflicts, no
// local memory).  Two passes, as detect_kernel / detect_events_kernel: detect_clips_kernel writes the final rows and
// counts each thread's events, detect_clips_events_kernel walks again and writes the events behind those of the threads
// before it - ascending (clip, label, call) - so no CTA ever waits for another.
struct DetClips {
    const float* scores; int n_out;             // [rows][n_out]
    const float* verified; float vthr;          // [rows][L] or nullptr
    const int64_t* row_off; int n_clips;        // [n_clips + 1]
    int chunk;
    const oww_detect_label* labels; int L, S;
    double debounce;
    float* final;                               // [rows][L] or nullptr
    int* thread_events;                         // [n_clips * L] or nullptr (no event list)
    int* cta_events;                            // [CTAs]
    oww_event* events; int max_events; int* n_events;
};

// emit(row, call, pred, fired) for every call of `clip`, in call order
template <class F>
static __device__ __forceinline__ void clip_walk(const DetClips& a, float (*ring)[DET_THREADS], int clip, int j, F emit) {
    const oww_detect_label lab = a.labels[j];
    const int64_t r0 = a.row_off[clip], n = a.row_off[clip + 1] - r0;
    const int t = threadIdx.x;
    int slot = 0;                                                  // c % 30
    for (int64_t c = 0; c < n; ++c) {
        const int64_t row = r0 + c;
        const int64_t k = oww_call_first_step(c + 1, a.chunk) - oww_call_first_step(c, a.chunk);   // chunks stepped
        const int prep = k > 0 ? (int)(k * OWW_SAMPLES_PER_CHUNK) : (int)((c + 1) * a.chunk % OWW_SAMPLES_PER_CHUNK);
        const bool stepped = k > 0;
        const float score = stepped && lab.column >= 0 ? a.scores[row * a.n_out + lab.column] : 0.f;
        const float p = !stepped && a.verified ? a.verified[row * a.L + j] : __int_as_float(0x7fc00000);
        const float pred = det_rule(lab, stepped, score, p, a.vthr, (int)min(c, (int64_t)DET_HIST), prep, a.debounce,
                                    [&](int i) { return ring[(slot + DET_HIST - 1 - i) % DET_HIST][t]; });
        ring[slot][t] = pred;
        slot = slot == DET_HIST - 1 ? 0 : slot + 1;
        emit(row, c, pred, !isnan(lab.threshold) && pred >= lab.threshold);
    }
}

__global__ void __launch_bounds__(DET_THREADS) detect_clips_kernel(const DetClips a) {
    __shared__ float ring[DET_HIST][DET_THREADS];
    __shared__ int s_events;
    const int sl = threadIdx.x / a.L, j = threadIdx.x - sl * a.L;
    const int clip = blockIdx.x * a.S + sl;
    const bool live = sl < a.S && clip < a.n_clips;
    if (threadIdx.x == 0) s_events = 0;
    __syncthreads();
    int ev = 0;
    if (live)
        clip_walk(a, ring, clip, j, [&](int64_t row, int64_t, float pred, bool fired) {
            if (a.final) a.final[row * a.L + j] = pred;
            ev += fired;
        });
    if (!a.thread_events) return;
    if (live) a.thread_events[(size_t)clip * a.L + j] = ev;
    if (ev) atomicAdd(&s_events, ev);
    __syncthreads();
    if (threadIdx.x == 0) a.cta_events[blockIdx.x] = s_events;
}

// Same grid and thread mapping.  A thread's events start behind those of the CTAs and threads before it.
__global__ void __launch_bounds__(DET_THREADS) detect_clips_events_kernel(const DetClips a) {
    __shared__ float ring[DET_HIST][DET_THREADS];
    __shared__ int s_sum[DET_THREADS / 32];
    __shared__ int s_warp[DET_THREADS / 32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int part = 0;
    for (int i = threadIdx.x; i < (int)blockIdx.x; i += DET_THREADS) part += a.cta_events[i];
    for (int o = 16; o; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    const int sl = threadIdx.x / a.L, j = threadIdx.x - sl * a.L;
    const int clip = blockIdx.x * a.S + sl;
    const bool live = sl < a.S && clip < a.n_clips;
    const int mine = live ? a.thread_events[(size_t)clip * a.L + j] : 0;
    int incl = mine;                                               // inclusive scan over the warp
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) s_warp[warp] = incl;
    if (lane == 0) s_sum[warp] = part;
    __syncthreads();
    int base = 0, before = 0;
    for (int w = 0; w < DET_THREADS / 32; ++w) {
        base += s_sum[w];
        if (w < warp) before += s_warp[w];
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *a.n_events = base + a.cta_events[blockIdx.x];
    int pos = base + before + incl - mine;
    if (!mine || !a.events || pos >= a.max_events) return;
    clip_walk(a, ring, clip, j, [&](int64_t, int64_t c, float pred, bool fired) {
        if (fired && pos < a.max_events) a.events[pos] = oww_event{clip, j, pred, (int)c};
        pos += fired;
    });
}

namespace {

void free_stream_state(oww_detector* d) {
    cudaFree(d->d_hist); cudaFree(d->d_count); cudaFree(d->d_fire); cudaFree(d->d_cta); cudaFree(d->d_ids);
    cudaFree(d->d_ovr); cudaFree(d->d_ovr_deb);
    d->d_hist = d->d_fire = nullptr;
    d->d_count = d->d_cta = d->d_ids = nullptr;
    d->d_ovr = nullptr;
    d->d_ovr_deb = nullptr;
    for (int j = 0; j < oww_detector::kSlots; ++j) {
        cudaFreeHost(d->h_prep[j]); cudaFree(d->d_prep[j]);
        d->h_prep[j] = d->d_prep[j] = nullptr;
    }
    d->n_streams = 0;
}

bool is_override(const oww_stream_detect& o) { return !std::isnan(o.threshold) || o.patience != -1 || o.flags != 0; }

// n_ovr from the host table, and the table to the device on `s` while some stream has an override
int sync_overrides(oww_ctx* ctx, cudaStream_t s) {
    oww_detector* d = ctx->det;
    const size_t L = d->labels.size();
    d->n_ovr = 0;
    for (size_t b = 0; b < d->ovr_deb.size(); ++b) {
        bool any = !std::isnan(d->ovr_deb[b]);
        for (size_t j = 0; j < L && !any; ++j) any = is_override(d->ovr[b * L + j]);
        d->n_ovr += any;
    }
    if (d->n_ovr && d->d_ovr) {                          // pageable sources: staged by the driver before the call returns
        OWW_CUDA(ctx, cudaMemcpyAsync(d->d_ovr, d->ovr.data(), d->ovr.size() * sizeof(oww_stream_detect),
                                      cudaMemcpyHostToDevice, s));
        OWW_CUDA(ctx, cudaMemcpyAsync(d->d_ovr_deb, d->ovr_deb.data(), d->ovr_deb.size() * sizeof(double),
                                      cudaMemcpyHostToDevice, s));
    }
    return OWW_OK;
}

// the detector's per-stream state for ctx->n_streams streams, every history empty, the settings of the streams below
// that count kept; the device is idle
int alloc_stream_state(oww_ctx* ctx) {
    oww_detector* d = ctx->det;
    free_stream_state(d);
    const int B = std::max(ctx->n_streams, 0), L = (int)d->labels.size();
    d->ovr.resize((size_t)B * L, kNoOverride);          // stream-major: the first streams keep their rows
    d->ovr_deb.resize((size_t)B, NAN);
    if (B == 0) { d->n_ovr = 0; return OWW_OK; }
    const size_t P = (size_t)B * L;
    const int ctas = (B + det_streams_per_cta(L) - 1) / det_streams_per_cta(L);
    OWW_CUDA(ctx, cudaMalloc(&d->d_hist, DET_HIST * P * sizeof(float)));
    OWW_CUDA(ctx, cudaMalloc(&d->d_count, (size_t)B * sizeof(int)));
    OWW_CUDA(ctx, cudaMalloc(&d->d_fire, P * sizeof(float)));
    OWW_CUDA(ctx, cudaMalloc(&d->d_cta, (size_t)ctas * sizeof(int)));
    OWW_CUDA(ctx, cudaMalloc(&d->d_ids, (size_t)B * sizeof(int)));
    OWW_CUDA(ctx, cudaMalloc(&d->d_ovr, P * sizeof(oww_stream_detect)));
    OWW_CUDA(ctx, cudaMalloc(&d->d_ovr_deb, (size_t)B * sizeof(double)));
    OWW_CUDA(ctx, cudaMemset(d->d_hist, 0, DET_HIST * P * sizeof(float)));
    OWW_CUDA(ctx, cudaMemset(d->d_count, 0, (size_t)B * sizeof(int)));
    for (int j = 0; j < oww_detector::kSlots; ++j) {
        OWW_CUDA(ctx, cudaMallocHost(&d->h_prep[j], (size_t)B * sizeof(int32_t)));
        OWW_CUDA(ctx, cudaMalloc(&d->d_prep[j], (size_t)B * sizeof(int32_t)));
        if (!d->ev[j]) OWW_CUDA(ctx, cudaEventCreateWithFlags(&d->ev[j], cudaEventDisableTiming));
    }
    d->n_streams = B;
    return sync_overrides(ctx, nullptr);
}

// checks shared by export and import; stages the ids on `s`
int stage_ids(oww_ctx* ctx, const int32_t* h_ids, int n, bool distinct, cudaStream_t s) {
    const oww_detector* d = ctx->det;
    if (!d || !d->d_hist) return oww_fail(ctx, OWW_EINVAL, "no detector configured (oww_set_detector, oww_set_streams)");
    const int B = ctx->n_streams;
    if (n < 0 || n > B) return oww_fail(ctx, OWW_EINVAL, "n=%d outside [0,%d]", n, B);
    if (n && !h_ids) return oww_fail(ctx, OWW_EINVAL, "null argument");
    std::vector<uint8_t> hit(distinct ? B : 0, 0);
    for (int i = 0; i < n; ++i) {
        if (h_ids[i] < 0 || h_ids[i] >= B) return oww_fail(ctx, OWW_EINVAL, "stream id %d out of range", h_ids[i]);
        if (distinct && hit[h_ids[i]]++) return oww_fail(ctx, OWW_EINVAL, "stream id %d imported twice", h_ids[i]);
    }
    // pageable source: staged by the driver before the call returns; stream-ordered on the device
    if (n) OWW_CUDA(ctx, cudaMemcpyAsync(d->d_ids, h_ids, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    return OWW_OK;
}

// checks of the settings calls: a detector with streams, ids in range (NULL: every stream), distinct if asked
int check_settings_ids(oww_ctx* ctx, const int32_t* h_ids, int n, bool distinct) {
    const oww_detector* d = ctx->det;
    if (!d || !d->d_hist) return oww_fail(ctx, OWW_EINVAL, "no detector configured (oww_set_detector, oww_set_streams)");
    const int B = ctx->n_streams;
    if (n < 0 || n > B || (!h_ids && n != B)) return oww_fail(ctx, OWW_EINVAL, "n=%d outside [0,%d] (or not %d without ids)", n, B, B);
    std::vector<uint8_t> hit(h_ids && distinct ? B : 0, 0);
    for (int i = 0; h_ids && i < n; ++i) {
        if (h_ids[i] < 0 || h_ids[i] >= B) return oww_fail(ctx, OWW_EINVAL, "stream id %d out of range", h_ids[i]);
        if (distinct && hit[h_ids[i]]++) return oww_fail(ctx, OWW_EINVAL, "stream id %d given twice", h_ids[i]);
    }
    return OWW_OK;
}

}  // namespace

void oww_detect_free(oww_ctx* ctx) {
    oww_detector* d = ctx->det;
    if (!d) return;
    free_stream_state(d);
    for (auto e : d->ev) if (e) cudaEventDestroy(e);
    cudaFree(d->d_labels);
    delete d;
    ctx->det = nullptr;
}

void oww_detect_free_streams(oww_ctx* ctx) { if (ctx->det) free_stream_state(ctx->det); }

int oww_detect_alloc_streams(oww_ctx* ctx) { return ctx->det ? alloc_stream_state(ctx) : OWW_OK; }

int oww_detect_reset(oww_ctx* ctx, const int* d_ids, int n, cudaStream_t s) {
    const oww_detector* d = ctx->det;
    if (!d || !d->d_hist || n <= 0) return OWW_OK;
    detect_clear_kernel<<<n, DET_THREADS, 0, s>>>(d_ids, ctx->n_streams, (int)d->labels.size(), d->d_hist, d->d_count);
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

int oww_detect_n_labels(const oww_ctx* ctx) { return ctx->det && ctx->det->d_hist ? (int)ctx->det->labels.size() : 0; }

DetectLayout oww_detect_layout(int max_events, int capture, int n_streams, int n_labels) {
    const auto up16 = [](size_t x) { return (x + 15) & ~(size_t)15; };
    DetectLayout l;
    const size_t m = (size_t)std::max(max_events, 0);
    l.events = 16;
    l.ends = up16(l.events + m * sizeof(oww_event));
    l.clips = up16(l.ends + (capture > 0 ? m * sizeof(int64_t) : 0));
    l.final = up16(l.clips + (capture > 0 ? m * (size_t)capture * sizeof(int16_t) : 0));
    l.bytes = l.final + (size_t)n_streams * n_labels * sizeof(float);
    return l;
}

int oww_detect_deliver(oww_ctx* ctx, const uint8_t* d_out, uint8_t* h_out, int max_events, int capture, cudaStream_t s) {
    const DetectLayout lay = oww_detect_layout(max_events, capture, 0, 0);
    const int ctas = capture > 0 ? std::max(max_events, 1) : std::max((max_events + DET_THREADS - 1) / DET_THREADS, 1);
    detect_deliver_kernel<<<ctas, DET_THREADS, 0, s>>>(d_out, h_out, lay, max_events, capture);
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

extern "C" {

int oww_set_detector(oww_ctx* ctx, const oww_detect_label* h_labels, int n_labels, double debounce_time) {
    if (!ctx) return OWW_EINVAL;
    if (n_labels < 0 || n_labels > DET_MAX_LABELS) return oww_fail(ctx, OWW_EINVAL, "n_labels=%d outside [0,%d]", n_labels, DET_MAX_LABELS);
    if (n_labels && !h_labels) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (!(debounce_time >= 0.0) || !std::isfinite(debounce_time)) return oww_fail(ctx, OWW_EINVAL, "debounce_time must be finite and >= 0");
    for (int j = 0; j < n_labels; ++j) {
        const oww_detect_label& l = h_labels[j];
        if (l.column < -1 || l.column >= ctx->n_out_total)
            return oww_fail(ctx, OWW_EINVAL, "label %d: column %d outside [-1,%d)", j, l.column, ctx->n_out_total);
        if (l.patience < 0 || l.patience > DET_HIST) return oww_fail(ctx, OWW_EINVAL, "label %d: patience %d outside [0,%d]", j, l.patience, DET_HIST);
        if (l.patience > 0 && std::isnan(l.threshold)) return oww_fail(ctx, OWW_EINVAL, "label %d: patience needs a threshold", j);
        if (l.patience > 0 && debounce_time > 0.0) return oww_fail(ctx, OWW_EINVAL, "patience and debounce_time cannot be used together");
    }
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaDeviceSynchronize());              // detect calls may be in flight on any stream
    if (n_labels == 0) { oww_detect_free(ctx); return OWW_OK; }
    oww_detector* d = ctx->det;
    bool same = d && (int)d->labels.size() == n_labels;
    for (int j = 0; same && j < n_labels; ++j)
        same = d->labels[j].column == h_labels[j].column && (d->labels[j].repeats != 0) == (h_labels[j].repeats != 0);
    if (!same) {                                         // another label set: the histories mean nothing under it
        oww_detect_free(ctx);
        d = ctx->det = new (std::nothrow) oww_detector();
        if (!d) return oww_fail(ctx, OWW_ENOMEM, "out of host memory");
        OWW_CUDA(ctx, cudaMalloc(&d->d_labels, (size_t)n_labels * sizeof(oww_detect_label)));
    }
    d->labels.assign(h_labels, h_labels + n_labels);
    d->debounce = debounce_time;
    d->ovr.assign(d->ovr.size(), kNoOverride);           // every stream back to the handle's settings
    d->ovr_deb.assign(d->ovr_deb.size(), NAN);
    d->n_ovr = 0;
    OWW_CUDA(ctx, cudaMemcpy(d->d_labels, h_labels, (size_t)n_labels * sizeof(oww_detect_label), cudaMemcpyHostToDevice));
    return same ? OWW_OK : alloc_stream_state(ctx);
}

int oww_detect(oww_ctx* ctx, const float* d_scores, int prepared_all, const int32_t* h_prepared, float* d_final,
               oww_event* d_events, int max_events, int32_t* d_n_events, void* stream) {
    if (!ctx) return OWW_EINVAL;
    oww_detector* d = ctx->det;
    if (!d || !d->d_hist) return oww_fail(ctx, OWW_EINVAL, "no detector configured (oww_set_detector, oww_set_streams)");
    if (!d_scores) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (max_events < 0) return oww_fail(ctx, OWW_EINVAL, "max_events=%d is negative", max_events);
    if (!d_final && !d_n_events && !d_events) return oww_fail(ctx, OWW_EINVAL, "no output: d_final and the event list are both NULL");
    if (max_events > 0 && !d_events) return oww_fail(ctx, OWW_EINVAL, "max_events=%d without d_events", max_events);
    if (d_events && !d_n_events) return oww_fail(ctx, OWW_EINVAL, "d_events without d_n_events");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    const int B = ctx->n_streams, L = (int)d->labels.size(), S = det_streams_per_cta(L);
    const int ctas = (B + S - 1) / S;
    const int* d_prep = nullptr;
    if (h_prepared) {
        const int j = d->next;
        d->next = (j + 1) % oww_detector::kSlots;
        OWW_CUDA(ctx, cudaEventSynchronize(d->ev[j]));   // the copy of the call kSlots calls back has run
        std::memcpy(d->h_prep[j], h_prepared, (size_t)B * sizeof(int32_t));
        OWW_CUDA(ctx, cudaMemcpyAsync(d->d_prep[j], d->h_prep[j], (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        OWW_CUDA(ctx, cudaEventRecord(d->ev[j], s));
        d_prep = d->d_prep[j];
    }
    detect_kernel<<<ctas, DET_THREADS, 0, s>>>(d_scores, ctx->n_out_total, B, L, S, d->d_labels, d->debounce,
                                               d->n_ovr ? d->d_ovr : nullptr, d->d_ovr_deb, prepared_all, d_prep, d->d_hist, d->d_count, d_final, d->d_fire, d->d_cta);
    OWW_LAUNCH_CHECK(ctx);
    if (d_n_events) {
        detect_events_kernel<<<ctas, DET_THREADS, 0, s>>>(d->d_fire, d->d_count, d->d_cta, B, L, S, d_events, max_events, d_n_events);
        OWW_LAUNCH_CHECK(ctx);
    }
    return OWW_OK;
}

int oww_detect_clips(oww_ctx* ctx, const oww_detect_label* h_labels, int n_labels, double debounce_time,
                     const float* d_scores, const float* d_verified, float verifier_threshold, const int64_t* h_row_offsets,
                     int n_clips, int chunk_size, float* d_final, oww_event* d_events, int max_events, int32_t* d_n_events,
                     void* stream) {
    if (!ctx) return OWW_EINVAL;
    if (n_labels < 1 || n_labels > DET_MAX_LABELS) return oww_fail(ctx, OWW_EINVAL, "n_labels=%d outside [1,%d]", n_labels, DET_MAX_LABELS);
    if (!h_labels || !h_row_offsets) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (!(debounce_time >= 0.0) || !std::isfinite(debounce_time)) return oww_fail(ctx, OWW_EINVAL, "debounce_time must be finite and >= 0");
    for (int j = 0; j < n_labels; ++j) {
        const oww_detect_label& l = h_labels[j];
        if (l.column < -1 || l.column >= ctx->n_out_total)
            return oww_fail(ctx, OWW_EINVAL, "label %d: column %d outside [-1,%d)", j, l.column, ctx->n_out_total);
        if (l.patience < 0 || l.patience > DET_HIST) return oww_fail(ctx, OWW_EINVAL, "label %d: patience %d outside [0,%d]", j, l.patience, DET_HIST);
        if (l.patience > 0 && std::isnan(l.threshold)) return oww_fail(ctx, OWW_EINVAL, "label %d: patience needs a threshold", j);
        if (l.patience > 0 && debounce_time > 0.0) return oww_fail(ctx, OWW_EINVAL, "patience and debounce_time cannot be used together");
    }
    if (n_clips < 0) return oww_fail(ctx, OWW_EINVAL, "n_clips=%d is negative", n_clips);
    if (chunk_size < 1) return oww_fail(ctx, OWW_EINVAL, "chunk_size=%d < 1", chunk_size);
    if (h_row_offsets[0] != 0) return oww_fail(ctx, OWW_EINVAL, "row offsets must start at 0");
    for (int i = 0; i < n_clips; ++i)
        if (h_row_offsets[i + 1] < h_row_offsets[i]) return oww_fail(ctx, OWW_EINVAL, "row offsets decrease at clip %d", i);
    const int64_t rows = h_row_offsets[n_clips];
    if (rows > 0 && !d_scores) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (max_events < 0) return oww_fail(ctx, OWW_EINVAL, "max_events=%d is negative", max_events);
    if (!d_final && !d_n_events && !d_events) return oww_fail(ctx, OWW_EINVAL, "no output: d_final and the event list are both NULL");
    if (max_events > 0 && !d_events) return oww_fail(ctx, OWW_EINVAL, "max_events=%d without d_events", max_events);
    if (d_events && !d_n_events) return oww_fail(ctx, OWW_EINVAL, "d_events without d_n_events");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    if (n_clips == 0) {
        if (d_n_events) OWW_CUDA(ctx, cudaMemsetAsync(d_n_events, 0, sizeof(int32_t), s));
        return OWW_OK;
    }
    const int L = n_labels, S = det_streams_per_cta(L), ctas = (n_clips + S - 1) / S;
    // one allocation: the row offsets and the labels (uploaded), then the event counts of the threads and the CTAs
    const size_t off_bytes = (size_t)(n_clips + 1) * sizeof(int64_t), lab_bytes = (size_t)L * sizeof(oww_detect_label);
    const size_t cnt_bytes = d_n_events ? ((size_t)n_clips * L + ctas) * sizeof(int) : 0;
    std::vector<uint8_t> tab(off_bytes + lab_bytes);
    std::memcpy(tab.data(), h_row_offsets, off_bytes);
    std::memcpy(tab.data() + off_bytes, h_labels, lab_bytes);
    uint8_t* d_tab = nullptr;
    OWW_CUDA(ctx, cudaMallocAsync(&d_tab, tab.size() + cnt_bytes, s));
    int* d_counts = d_n_events ? reinterpret_cast<int*>(d_tab + tab.size()) : nullptr;
    cudaError_t e = cudaMemcpyAsync(d_tab, tab.data(), tab.size(), cudaMemcpyHostToDevice, s);   // pageable: staged before return
    DetClips a{d_scores, ctx->n_out_total, d_verified, verifier_threshold, reinterpret_cast<const int64_t*>(d_tab), n_clips,
               chunk_size, reinterpret_cast<const oww_detect_label*>(d_tab + off_bytes), L, S, debounce_time, d_final,
               d_counts, d_counts ? d_counts + (size_t)n_clips * L : nullptr, d_events, max_events, d_n_events};
    if (e == cudaSuccess) {
        detect_clips_kernel<<<ctas, DET_THREADS, 0, s>>>(a);
        ctx->launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && d_n_events) {
        detect_clips_events_kernel<<<ctas, DET_THREADS, 0, s>>>(a);
        ctx->launches++;
        e = cudaGetLastError();
    }
    cudaFreeAsync(d_tab, s);
    if (e != cudaSuccess) return oww_fail(ctx, OWW_ECUDA, "detect_clips: %s (%s:%d)", cudaGetErrorString(e), __FILE__, __LINE__);
    return OWW_OK;
}

int oww_detector_export(oww_ctx* ctx, const int32_t* h_stream_ids, int n, float* d_hist, int32_t* d_counts, void* stream) {
    if (!ctx) return OWW_EINVAL;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n > 0 && (!d_hist || !d_counts)) return oww_fail(ctx, OWW_EINVAL, "null argument");
    int rc = stage_ids(ctx, h_stream_ids, n, false, (cudaStream_t)stream);
    if (rc || n == 0) return rc;
    const oww_detector* d = ctx->det;
    if ((rc = oww_order_begin(ctx, (cudaStream_t)stream))) return rc;     // between the detect calls submitted around it
    detect_export_kernel<<<n, DET_THREADS, 0, (cudaStream_t)stream>>>(d->d_ids, ctx->n_streams, (int)d->labels.size(), d->d_hist,
                                                                      d->d_count, d_hist, d_counts);
    OWW_LAUNCH_CHECK(ctx);
    return oww_order_end(ctx, (cudaStream_t)stream);
}

int oww_detector_import(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const float* d_hist, const int32_t* d_counts, void* stream) {
    if (!ctx) return OWW_EINVAL;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n > 0 && (!d_hist || !d_counts)) return oww_fail(ctx, OWW_EINVAL, "null argument");
    int rc = stage_ids(ctx, h_stream_ids, n, true, (cudaStream_t)stream);
    if (rc || n == 0) return rc;
    const oww_detector* d = ctx->det;
    if ((rc = oww_order_begin(ctx, (cudaStream_t)stream))) return rc;
    detect_import_kernel<<<n, DET_THREADS, 0, (cudaStream_t)stream>>>(d->d_ids, ctx->n_streams, (int)d->labels.size(), d->d_hist,
                                                                      d->d_count, d_hist, d_counts);
    OWW_LAUNCH_CHECK(ctx);
    return oww_order_end(ctx, (cudaStream_t)stream);
}

int oww_set_stream_detection(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const oww_stream_detect* h_overrides,
                             const double* h_debounce, void* stream) {
    if (!ctx) return OWW_EINVAL;
    int rc = check_settings_ids(ctx, h_stream_ids, n, true);
    if (rc) return rc;
    oww_detector* d = ctx->det;
    const int L = (int)d->labels.size();
    for (int i = 0; h_overrides && i < n; ++i) {         // every stream's resulting values, before anything changes
        const int b = h_stream_ids ? h_stream_ids[i] : i;
        const double deb = h_debounce ? h_debounce[i] : NAN;
        if (!std::isnan(deb) && !(deb >= 0.0 && std::isfinite(deb)))
            return oww_fail(ctx, OWW_EINVAL, "stream %d: debounce_time must be finite and >= 0 (NaN: the handle's)", b);
        const double eff_deb = std::isnan(deb) ? d->debounce : deb;
        for (int j = 0; j < L; ++j) {
            const oww_stream_detect& o = h_overrides[(size_t)i * L + j];
            if (o.flags & ~OWW_DETECT_NO_THRESHOLD) return oww_fail(ctx, OWW_EINVAL, "stream %d label %d: flags 0x%x", b, j, o.flags);
            if (o.patience < -1 || o.patience > DET_HIST)
                return oww_fail(ctx, OWW_EINVAL, "stream %d label %d: patience %d outside [-1,%d]", b, j, o.patience, DET_HIST);
            const bool thr = !(o.flags & OWW_DETECT_NO_THRESHOLD) && !std::isnan(std::isnan(o.threshold) ? d->labels[j].threshold : o.threshold);
            const int pat = o.patience >= 0 ? o.patience : d->labels[j].patience;
            if (pat > 0 && !thr) return oww_fail(ctx, OWW_EINVAL, "stream %d label %d: patience needs a threshold", b, j);
            if (pat > 0 && eff_deb > 0.0)
                return oww_fail(ctx, OWW_EINVAL, "stream %d: patience and debounce_time cannot be used together", b);
        }
    }
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    for (int i = 0; i < n; ++i) {
        const int b = h_stream_ids ? h_stream_ids[i] : i;
        for (int j = 0; j < L; ++j) d->ovr[(size_t)b * L + j] = h_overrides ? h_overrides[(size_t)i * L + j] : kNoOverride;
        d->ovr_deb[b] = h_overrides && h_debounce ? h_debounce[i] : NAN;
    }
    // the table is one device buffer: the upload waits for the detect calls submitted so far, which read the old one,
    // and those submitted later wait for it
    if ((rc = oww_order_begin(ctx, (cudaStream_t)stream)) || (rc = sync_overrides(ctx, (cudaStream_t)stream))) return rc;
    return oww_order_end(ctx, (cudaStream_t)stream);
}

int oww_get_stream_detection(oww_ctx* ctx, const int32_t* h_stream_ids, int n, oww_stream_detect* h_overrides,
                             double* h_debounce) {
    if (!ctx) return OWW_EINVAL;
    int rc = check_settings_ids(ctx, h_stream_ids, n, false);
    if (rc) return rc;
    const oww_detector* d = ctx->det;
    const size_t L = d->labels.size();
    for (int i = 0; i < n; ++i) {
        const size_t b = h_stream_ids ? h_stream_ids[i] : i;
        if (h_overrides) std::memcpy(h_overrides + i * L, d->ovr.data() + b * L, L * sizeof(oww_stream_detect));
        if (h_debounce) h_debounce[i] = d->ovr_deb[b];
    }
    return OWW_OK;
}

}  // extern "C"
