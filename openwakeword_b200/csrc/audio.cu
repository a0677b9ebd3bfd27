// Stream audio on the device: the last H samples every stream stepped (the reference's AudioFeatures.raw_data_buffer,
// openwakeword/utils.py:164,403-430), so that a serving loop can read the audio of a detection without keeping its own
// host copy of every stream.  Semantics: include/owwb200.h (oww_set_audio_history and the calls after it).
//
// State: audio [B][H] int16 (a ring per stream; sample p of a stream at audio[b][p % H]) and pos [B] int64 (samples the
// stream has stepped since its reset).  The ring holds samples [max(0, pos - H), pos).  H is a multiple of 1280, so a
// stream's appends start at a multiple of 8 samples unless an import stored another pos.
//
// The append is a launch of its own at each step entry point, before the frontend: the fused step kernel is untouched and
// a handle without history launches nothing for it.
#include <cstring>
#include "oww_internal.h"

#define AUD_THREADS 256
#define AUD_SPAN 4096                 // samples of a gathered row per CTA
#define AUD_MAX_SAMPLES (60 * 16000)

struct oww_audio {
    int H = 0;                          // samples per stream
    int n_streams = 0;                  // streams the state below is allocated for
    int16_t* d_audio = nullptr;         // [B][H]
    int64_t* d_pos = nullptr;           // [B]
    int* d_ids = nullptr;               // [cap] staging of stream ids
    int64_t* d_end = nullptr;           // [cap] staging of oww_get_audio's ends
    int cap = 0;
    cudaEvent_t ev[2] = {nullptr, nullptr};   // orders the calls with own_stream (the host-buffer steps)
};

// The kernels stay outside the anonymous namespace: their names in a profile do not depend on the build.
// One warp per stream: its cnt * 1280 samples go behind sample pos.  cnt = counts[b] (nullptr: n_all for every stream).
__global__ void __launch_bounds__(AUD_THREADS) audio_append_kernel(const int16_t* __restrict__ pcm, int64_t stride, int B,
                                                                   int n_all, const int* __restrict__ counts, int H,
                                                                   int16_t* __restrict__ audio, int64_t* __restrict__ pos) {
    oww_pdl_sync();
    const int b = blockIdx.x * (AUD_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= B) return;
    const int n = (counts ? counts[b] : n_all) * OWW_SAMPLES_PER_CHUNK;
    if (n <= 0) return;
    const int64_t p0 = pos[b];
    const int16_t* src = pcm + (int64_t)b * stride;
    int16_t* ring = audio + (size_t)b * H;
    const int r0 = (int)((uint64_t)p0 % (uint64_t)H);      // any stored pos stays in bounds
    if ((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (r0 & 7) == 0) {
        // 8 samples per access, four loads in flight per lane; H and r0 are multiples of 8, so no group straddles the
        // end of the ring
        const uint4* s4 = reinterpret_cast<const uint4*>(src);
        const int nv = n / 8;
        for (int i0 = lane; i0 < nv; i0 += 4 * 32) {
            uint4 v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) if (i0 + 32 * u < nv) v[u] = s4[i0 + 32 * u];
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (i0 + 32 * u < nv) *reinterpret_cast<uint4*>(ring + (r0 + 8 * (i0 + 32 * u)) % H) = v[u];
        }
    } else {
        for (int i = lane; i < n; i += 32) ring[(r0 + i) % H] = src[i];
    }
    __syncwarp();                                             // every lane has read pos
    if (lane == 0) pos[b] = p0 + n;
}

// out[0..n) of a row <- samples [e - n, e) of stream b, the part [k0, k1) of it in this CTA; zeros where the ring does
// not hold them
static __device__ __forceinline__ void audio_window(const int16_t* __restrict__ audio, int64_t p, int H, int b, int64_t e,
                                                    int n, int k0, int k1, int16_t* __restrict__ out) {
    const int64_t lo = max(p - (int64_t)H, (int64_t)0);
    const int16_t* ring = audio + (size_t)b * H;
    const int64_t s0 = e - n;
    const int base = (int)(lo % H);                           // q in [lo, p): ring slot (q - lo) + base, less than 2H
    for (int k = k0 + threadIdx.x; k < k1; k += blockDim.x) {
        const int64_t q = s0 + k;
        int16_t v = 0;
        if (q >= lo && q < p) {
            const int r = (int)(q - lo) + base;
            v = ring[r >= H ? r - H : r];
        }
        out[k] = v;
    }
}

// row i <- stream ids[i], ending at ends[i] (ends nullptr or < 0: the stream's pos); CTA (i, y) writes samples
// [y * AUD_SPAN, +AUD_SPAN) of the row
__global__ void __launch_bounds__(AUD_THREADS) audio_get_kernel(const int* __restrict__ ids, const int64_t* __restrict__ ends,
                                                                int n, int H, const int16_t* __restrict__ audio,
                                                                const int64_t* __restrict__ pos, int16_t* __restrict__ out,
                                                                int64_t* __restrict__ out_pos) {
    const int i = blockIdx.x, b = ids[i];
    const int64_t p = pos[b];
    const int64_t e = (ends && ends[i] >= 0) ? ends[i] : p;
    const int k0 = blockIdx.y * AUD_SPAN;
    audio_window(audio, p, H, b, e, n, k0, min(k0 + AUD_SPAN, n), out + (size_t)i * n);
    if (blockIdx.y == 0 && threadIdx.x == 0 && out_pos) out_pos[i] = p;
}

// row i < min(*n_events, max_events) <- the last n samples of stream events[i].stream; CTAs past the count exit
__global__ void __launch_bounds__(AUD_THREADS) audio_capture_kernel(const oww_event* __restrict__ events,
                                                                    const int32_t* __restrict__ n_events, int B, int n, int H,
                                                                    const int16_t* __restrict__ audio,
                                                                    const int64_t* __restrict__ pos, int16_t* __restrict__ out,
                                                                    int64_t* __restrict__ out_pos) {
    const int i = blockIdx.x;
    if (i >= *n_events) return;
    const int b = events[i].stream;
    if (b < 0 || b >= B) return;
    const int64_t p = pos[b];
    const int k0 = blockIdx.y * AUD_SPAN;
    audio_window(audio, p, H, b, p, n, k0, min(k0 + AUD_SPAN, n), out + (size_t)i * n);
    if (blockIdx.y == 0 && threadIdx.x == 0 && out_pos) out_pos[i] = p;
}

// streams ids[0..n) (nullptr: stream blockIdx.x) start with an empty history
__global__ void audio_clear_kernel(const int* ids, int n, int64_t* pos) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pos[ids ? ids[i] : i] = 0;
}

// record i <-> stream ids[i]: [H] oldest first (entry k = sample pos - H + k, zeros before sample 0) and pos.  Entry k
// sits at ring slot (pos + k) % H.
__global__ void __launch_bounds__(AUD_THREADS) audio_export_kernel(const int* __restrict__ ids, int H,
                                                                   const int16_t* __restrict__ audio,
                                                                   const int64_t* __restrict__ pos, int16_t* __restrict__ out,
                                                                   int64_t* __restrict__ out_pos) {
    const int b = ids[blockIdx.x];
    const int64_t p = pos[b];
    const int16_t* ring = audio + (size_t)b * H;
    int16_t* o = out + (size_t)blockIdx.x * H;
    for (int k = threadIdx.x; k < H; k += AUD_THREADS) o[k] = p - H + k >= 0 ? ring[(p + k) % H] : (int16_t)0;
    if (threadIdx.x == 0) out_pos[blockIdx.x] = p;
}

__global__ void __launch_bounds__(AUD_THREADS) audio_import_kernel(const int* __restrict__ ids, int H,
                                                                   int16_t* __restrict__ audio, int64_t* __restrict__ pos,
                                                                   const int16_t* __restrict__ in,
                                                                   const int64_t* __restrict__ in_pos) {
    const int b = ids[blockIdx.x];
    const int64_t p = max(in_pos[blockIdx.x], (int64_t)0);
    int16_t* ring = audio + (size_t)b * H;
    const int16_t* r = in + (size_t)blockIdx.x * H;
    for (int k = threadIdx.x; k < H; k += AUD_THREADS) ring[(p + k) % H] = r[k];
    if (threadIdx.x == 0) pos[b] = p;
}

namespace {

void free_stream_state(oww_audio* a) {
    cudaFree(a->d_audio); cudaFree(a->d_pos); cudaFree(a->d_ids); cudaFree(a->d_end);
    a->d_audio = nullptr; a->d_pos = nullptr; a->d_ids = nullptr; a->d_end = nullptr;
    a->cap = 0;
    a->n_streams = 0;
}

void audio_free(oww_ctx* ctx) {
    oww_audio* a = ctx->audio;
    if (!a) return;
    free_stream_state(a);
    for (auto e : a->ev) if (e) cudaEventDestroy(e);
    delete a;
    ctx->audio = nullptr;
}

// the history of ctx->n_streams streams, every one empty; the device is idle.  A failed allocation turns history off.
int alloc_stream_state(oww_ctx* ctx) {
    oww_audio* a = ctx->audio;
    free_stream_state(a);
    const int B = ctx->n_streams;
    if (B <= 0) return OWW_OK;
    cudaError_t e = cudaMalloc(&a->d_audio, (size_t)B * a->H * sizeof(int16_t));
    if (e == cudaSuccess) e = cudaMalloc(&a->d_pos, (size_t)B * sizeof(int64_t));
    if (e == cudaSuccess) e = cudaMalloc(&a->d_ids, (size_t)B * sizeof(int));
    if (e == cudaSuccess) e = cudaMalloc(&a->d_end, (size_t)B * sizeof(int64_t));
    if (e == cudaSuccess) e = cudaMemset(a->d_pos, 0, (size_t)B * sizeof(int64_t));
    for (int j = 0; j < 2 && e == cudaSuccess; ++j)
        if (!a->ev[j]) e = cudaEventCreateWithFlags(&a->ev[j], cudaEventDisableTiming);
    if (e != cudaSuccess) {
        cudaGetLastError();
        const int H = a->H;
        audio_free(ctx);
        return oww_fail(ctx, e == cudaErrorMemoryAllocation ? OWW_ENOMEM : OWW_ECUDA,
                        "audio history of %d samples x %d streams: %s (history is off)", H, B, cudaGetErrorString(e));
    }
    a->cap = B;
    a->n_streams = B;
    return OWW_OK;
}

// checks shared by the calls; stages the ids (and ends) on `s`
int stage(oww_ctx* ctx, const int32_t* h_ids, const int64_t* h_end, int n, bool distinct, cudaStream_t s) {
    oww_audio* a = ctx->audio;
    if (!a || !a->d_audio) return oww_fail(ctx, OWW_EINVAL, "no audio history (oww_set_audio_history, oww_set_streams)");
    const int B = ctx->n_streams;
    if (n < 0 || (distinct && n > B)) return oww_fail(ctx, OWW_EINVAL, "n=%d outside [0,%d]", n, distinct ? B : INT32_MAX);
    if (n && !h_ids) return oww_fail(ctx, OWW_EINVAL, "null argument");
    std::vector<uint8_t> hit(distinct ? B : 0, 0);
    for (int i = 0; i < n; ++i) {
        if (h_ids[i] < 0 || h_ids[i] >= B) return oww_fail(ctx, OWW_EINVAL, "stream id %d out of range", h_ids[i]);
        if (distinct && hit[h_ids[i]]++) return oww_fail(ctx, OWW_EINVAL, "stream id %d imported twice", h_ids[i]);
    }
    if (n > a->cap) {                                   // more rows than streams (duplicate ids): grow the staging
        OWW_CUDA(ctx, cudaDeviceSynchronize());
        cudaFree(a->d_ids); cudaFree(a->d_end); a->d_ids = nullptr; a->d_end = nullptr; a->cap = 0;
        OWW_CUDA(ctx, cudaMalloc(&a->d_ids, (size_t)n * sizeof(int)));
        OWW_CUDA(ctx, cudaMalloc(&a->d_end, (size_t)n * sizeof(int64_t)));
        a->cap = n;
    }
    // pageable sources: staged by the driver before the call returns; stream-ordered on the device
    if (n) OWW_CUDA(ctx, cudaMemcpyAsync(a->d_ids, h_ids, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    if (n && h_end) OWW_CUDA(ctx, cudaMemcpyAsync(a->d_end, h_end, (size_t)n * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    return OWW_OK;
}

// the host-buffer steps append on the handle's own stream: a call on `s` runs after the steps submitted there so far
// (begin) and before the later ones (end)
int order_begin(oww_ctx* ctx, cudaStream_t s) {
    if (s == ctx->own_stream) return OWW_OK;
    OWW_CUDA(ctx, cudaEventRecord(ctx->audio->ev[0], ctx->own_stream));
    OWW_CUDA(ctx, cudaStreamWaitEvent(s, ctx->audio->ev[0], 0));
    return OWW_OK;
}

int order_end(oww_ctx* ctx, cudaStream_t s) {
    if (s == ctx->own_stream) return OWW_OK;
    OWW_CUDA(ctx, cudaEventRecord(ctx->audio->ev[1], s));
    OWW_CUDA(ctx, cudaStreamWaitEvent(ctx->own_stream, ctx->audio->ev[1], 0));
    return OWW_OK;
}

}  // namespace

void oww_audio_free(oww_ctx* ctx) { audio_free(ctx); }

void oww_audio_free_streams(oww_ctx* ctx) { if (ctx->audio) free_stream_state(ctx->audio); }

int oww_audio_alloc_streams(oww_ctx* ctx) { return ctx->audio ? alloc_stream_state(ctx) : OWW_OK; }

int oww_audio_history_samples(const oww_ctx* ctx) { return ctx->audio && ctx->audio->d_audio ? ctx->audio->H : 0; }

int oww_audio_reset(oww_ctx* ctx, const int* d_ids, int n, cudaStream_t s) {
    const oww_audio* a = ctx->audio;
    if (!a || !a->d_audio || n <= 0) return OWW_OK;
    audio_clear_kernel<<<(n + 255) / 256, 256, 0, s>>>(d_ids, n, a->d_pos);
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

int oww_audio_append(oww_ctx* ctx, const int16_t* d_pcm, int64_t pcm_stride, int n_chunks, const int* d_counts,
                     cudaStream_t s) {
    const oww_audio* a = ctx->audio;
    if (!a || !a->d_audio) return OWW_OK;
    const int B = ctx->n_streams, per_cta = AUD_THREADS / 32;
    OWW_CUDA(ctx, oww_launch_pdl(ctx->late_pdl, audio_append_kernel, dim3((B + per_cta - 1) / per_cta), dim3(AUD_THREADS), 0,
                                 s, d_pcm, pcm_stride, B, n_chunks, d_counts, a->H, a->d_audio, a->d_pos));
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

extern "C" {

int oww_set_audio_history(oww_ctx* ctx, int n_samples) {
    if (!ctx) return OWW_EINVAL;
    if (n_samples < 0 || n_samples > AUD_MAX_SAMPLES || n_samples % OWW_SAMPLES_PER_CHUNK)
        return oww_fail(ctx, OWW_EINVAL, "n_samples=%d: 0, or a multiple of %d up to %d", n_samples, OWW_SAMPLES_PER_CHUNK,
                        AUD_MAX_SAMPLES);
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaDeviceSynchronize());              // steps and reads may be in flight on any stream
    audio_free(ctx);
    if (n_samples == 0) return OWW_OK;
    oww_audio* a = ctx->audio = new (std::nothrow) oww_audio();
    if (!a) return oww_fail(ctx, OWW_ENOMEM, "out of host memory");
    a->H = n_samples;
    return alloc_stream_state(ctx);
}

int oww_get_audio(oww_ctx* ctx, const int32_t* h_stream_ids, const int64_t* h_end, int n, int n_samples, int16_t* d_out,
                  int64_t* d_pos, void* stream) {
    if (!ctx) return OWW_EINVAL;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    if (ctx->audio && (n_samples < 1 || n_samples > ctx->audio->H))
        return oww_fail(ctx, OWW_EINVAL, "n_samples=%d outside [1,%d]", n_samples, ctx->audio->H);
    if (n > 0 && !d_out) return oww_fail(ctx, OWW_EINVAL, "null argument");
    cudaStream_t s = (cudaStream_t)stream;
    int rc = stage(ctx, h_stream_ids, h_end, n, false, s);
    if (rc || n == 0) return rc;
    const oww_audio* a = ctx->audio;
    if ((rc = order_begin(ctx, s))) return rc;
    const dim3 grid(n, (n_samples + AUD_SPAN - 1) / AUD_SPAN);
    audio_get_kernel<<<grid, AUD_THREADS, 0, s>>>(a->d_ids, h_end ? a->d_end : nullptr, n_samples, a->H, a->d_audio, a->d_pos,
                                                  d_out, d_pos);
    OWW_LAUNCH_CHECK(ctx);
    return order_end(ctx, s);
}

int oww_capture_events(oww_ctx* ctx, const oww_event* d_events, const int32_t* d_n_events, int max_events, int n_samples,
                       int16_t* d_out, int64_t* d_pos, void* stream) {
    if (!ctx) return OWW_EINVAL;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    const oww_audio* a = ctx->audio;
    if (!a || !a->d_audio) return oww_fail(ctx, OWW_EINVAL, "no audio history (oww_set_audio_history, oww_set_streams)");
    if (n_samples < 1 || n_samples > a->H) return oww_fail(ctx, OWW_EINVAL, "n_samples=%d outside [1,%d]", n_samples, a->H);
    if (max_events < 0) return oww_fail(ctx, OWW_EINVAL, "max_events=%d is negative", max_events);
    if (max_events == 0) return OWW_OK;
    if (!d_events || !d_n_events || !d_out) return oww_fail(ctx, OWW_EINVAL, "null argument");
    cudaStream_t s = (cudaStream_t)stream;
    int rc = order_begin(ctx, s);
    if (rc) return rc;
    const dim3 grid(max_events, (n_samples + AUD_SPAN - 1) / AUD_SPAN);
    audio_capture_kernel<<<grid, AUD_THREADS, 0, s>>>(d_events, d_n_events, ctx->n_streams, n_samples, a->H, a->d_audio,
                                                      a->d_pos, d_out, d_pos);
    OWW_LAUNCH_CHECK(ctx);
    return order_end(ctx, s);
}

int oww_audio_export(oww_ctx* ctx, const int32_t* h_stream_ids, int n, int16_t* d_audio, int64_t* d_pos, void* stream) {
    if (!ctx) return OWW_EINVAL;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n > 0 && (!d_audio || !d_pos)) return oww_fail(ctx, OWW_EINVAL, "null argument");
    cudaStream_t s = (cudaStream_t)stream;
    int rc = stage(ctx, h_stream_ids, nullptr, n, false, s);
    if (rc || n == 0) return rc;
    const oww_audio* a = ctx->audio;
    if ((rc = order_begin(ctx, s))) return rc;
    audio_export_kernel<<<n, AUD_THREADS, 0, s>>>(a->d_ids, a->H, a->d_audio, a->d_pos, d_audio, d_pos);
    OWW_LAUNCH_CHECK(ctx);
    return order_end(ctx, s);
}

int oww_audio_import(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const int16_t* d_audio, const int64_t* d_pos,
                     void* stream) {
    if (!ctx) return OWW_EINVAL;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n > 0 && (!d_audio || !d_pos)) return oww_fail(ctx, OWW_EINVAL, "null argument");
    cudaStream_t s = (cudaStream_t)stream;
    int rc = stage(ctx, h_stream_ids, nullptr, n, true, s);
    if (rc || n == 0) return rc;
    const oww_audio* a = ctx->audio;
    if ((rc = order_begin(ctx, s))) return rc;
    audio_import_kernel<<<n, AUD_THREADS, 0, s>>>(a->d_ids, a->H, a->d_audio, a->d_pos, d_audio, d_pos);
    OWW_LAUNCH_CHECK(ctx);
    return order_end(ctx, s);
}

}  // extern "C"
