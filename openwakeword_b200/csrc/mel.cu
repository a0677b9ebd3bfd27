// K1: int16 PCM -> log-mel rows, one CTA per (stream, call).
//
// Replaces the melspectrogram.onnx session of the reference
// (openwakeword/utils.py:84-87,180-208; graph spec
// notebooks/converting_google_speech_embedding_model.ipynb:426-477): frames of 512 samples every
// 160, periodic Hann(400) zero-padded to 512, |rFFT|^2, 32 Slaney mel filters (60-3800 Hz),
// 10*log10(max(.,1e-10)), clamp at (max over the call) - 80 dB, then x/10+2.
//
// The reference graph evaluates the STFT as a dense 512x514 conv; here each warp runs a 256-point
// complex radix-4 Stockham FFT in shared memory on the even/odd-packed real frame and unpacks only
// the bins the filterbank touches.  One CTA owns one call of one stream, so the per-call dB
// maximum (SURVEY.md F7) is a block reduction; the CTA also advances the stream's PCM tail and mel
// ring, so the whole frontend is one launch with no host round trip.
//
// The frame routine is mel_frames_db (mel_device.cuh), the one the full-depth fused step kernel runs, so rows are
// bit-identical between the two.  A CTA takes 4 KB of work buffer per warp plus the 6 KB twiddle / window tables, so
// five CTAs (40 warps) share an SM: the one-chunk step's frontend (8 frames per stream) runs as a single launch at
// that occupancy instead of on the 16 warps of the step kernel.
// Dependent launch (MelLaunch::pdl): every CTA lets its successor start at once, computes its frames, and only then
// waits for the predecessor grid before its first store.  What it reads before that wait - PCM, PCM tail, `seen`,
// the ring count - is written only by kernels that are complete by then: the previous frontend, reset and import
// kernels all finish before the step kernel that follows them (launched without an early trigger) ends.
#include "oww_internal.h"
#include "tc_common.cuh"
#include "mel_device.cuh"
#include <climits>
#include <cmath>
#include <cstring>

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;

struct MelDev {
    const float* window;       // [512]
    const float2* twiddle;     // [512]
    const int* mel_start;      // [32]
    const int* mel_len;        // [32]
    const float* mel_w;        // [32][OWW_MEL_MAXSUPPORT]
    int kmax;
};

__global__ void __launch_bounds__(kThreads, 5) mel_kernel(MelLaunch p, MelDev c) {
    __shared__ __align__(16) uint8_t s_work[kWarps][kMelFrameScratch];
    __shared__ float2 s_tw[512];
    __shared__ float s_win[512];
    __shared__ float s_red[kWarps];

    pdl_trigger();
    const int clip = p.ids ? p.ids[blockIdx.x] : blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (p.live && p.live[clip] < p.live_min) {       // dead slot of a ragged step: no trace
        pdl_wait();
        return;
    }

    for (int i = tid; i < 512; i += kThreads) { s_tw[i] = c.twiddle[i]; s_win[i] = c.window[i]; }

    const bool streaming = p.tail != nullptr;
    const int prefix = streaming ? OWW_TAIL : 0;
    const int seen0 = streaming ? p.seen[clip] : 0;
    const bool fresh = streaming && seen0 == 0;
    const int total = prefix + p.n_body;
    const int T = (total - OWW_FFT_N) / OWW_HOP + 1;
    const int f0 = fresh ? 3 : 0;                 // frames 0..2 would read the (absent) prefix
    const int nrows = T - f0;
    const bool one_pass = nrows <= kWarps;        // every frame's row stays in a register until the clamp
    const int16_t* body = p.body + (int64_t)clip * p.body_stride;
    const int16_t* tail = streaming ? p.tail + (int64_t)clip * OWW_TAIL : nullptr;
    const int row0 = p.out_count ? p.out_count[clip] : 0;
    float* out = p.out + (int64_t)clip * p.out_stride;
    __syncthreads();

    const int my_start = c.mel_start[lane];
    const int my_len = c.mel_len[lane];
    const float* my_w = c.mel_w + lane * OWW_MEL_MAXSUPPORT;
    float vmax = -INFINITY, kept = 0.f;

    for (int f = f0 + warp; f < T; f += kWarps) {
        float db;
        mel_frames_db<1>(&tail, prefix, &body, &f, s_work[warp], s_tw, s_win, c.kmax, my_start, my_len, my_w, lane, &db);
        vmax = fmaxf(vmax, db);
        if (one_pass) { kept = db; continue; }
        pdl_wait();
        const int r = f - f0;
        const int slot = p.out_rows_mask >= 0 ? ((row0 + r) & p.out_rows_mask) : r;
        out[(int64_t)slot * OWW_MEL_BINS + lane] = db;
    }
    // per-call maximum -> clamp -> affine
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    if (lane == 0) s_red[warp] = vmax;
    __syncthreads();                              // also: every frame has read the old tail
    float m = s_red[0];
#pragma unroll
    for (int w = 1; w < kWarps; ++w) m = fmaxf(m, s_red[w]);
    const float floor_db = m - 80.0f;
    // the stream's new tail = the last 480 samples of this call: loaded now, stored behind the wait
    int16_t tv[(OWW_TAIL + kThreads - 1) / kThreads];
#pragma unroll
    for (int u = 0; u < (OWW_TAIL + kThreads - 1) / kThreads; ++u) {
        const int i = tid + u * kThreads;
        tv[u] = streaming && i < OWW_TAIL ? __ldg(body + (p.n_body - OWW_TAIL + i)) : (int16_t)0;
    }
    pdl_wait();
    if (one_pass) {
        if (warp < nrows) {
            float v = fmaxf(kept, floor_db);
            if (p.affine) v = v / 10.0f + 2.0f;
            const int slot = p.out_rows_mask >= 0 ? ((row0 + warp) & p.out_rows_mask) : warp;
            out[(int64_t)slot * OWW_MEL_BINS + lane] = v;
        }
    } else {
        for (int i = tid; i < nrows * OWW_MEL_BINS; i += kThreads) {
            const int r = i >> 5, col = i & 31;
            const int slot = p.out_rows_mask >= 0 ? ((row0 + r) & p.out_rows_mask) : r;
            float* q = out + (int64_t)slot * OWW_MEL_BINS + col;
            float v = fmaxf(__ldcg(q), floor_db);
            if (p.affine) v = v / 10.0f + 2.0f;
            *q = v;
        }
    }
    if (streaming) {
        int16_t* tw = p.tail + (int64_t)clip * OWW_TAIL;
#pragma unroll
        for (int u = 0; u < (OWW_TAIL + kThreads - 1) / kThreads; ++u)
            if (tid + u * kThreads < OWW_TAIL) tw[tid + u * kThreads] = tv[u];
        if (tid == 0) {
            p.out_count[clip] = oww_wrap_count(row0 + nrows);
            const int sn = seen0 + p.n_chunks;
            p.seen[clip] = sn > (1 << 30) ? (1 << 30) : sn;
        }
    }
}

// Bulk path (predict_clip over many clips, SURVEY.md F10): one CTA per clip computes the mel rows of the WHOLE padded clip
// exactly as the streaming calls would have produced them and lays them out as the virtual history the fully
// convolutional CNN pass needs:  out[clip] = [ones x 71 | frames 0..4 of step 0 | 8 frames of step 1 | ...],
// 76 + 8 (steps - 1) rows.  The -80 dB clamp is per CALL (F7): a call that steps k chunks clamps its 8 k frames (5 + 8 (k - 1)
// for the first call of the clip) against their own maximum; with 1280-sample calls the groups are [0,5), [5,13), ...
// pad_samples zeros are virtual (nothing is copied), as is everything after the clip's own samples.
// A launch covers the steps [k0, k1), k1 on a call boundary: virtual rows [8 k0, 76 + 8 (k1 - 1)), i.e. frames up to
// 8 k1 - 3 and, at k0 > 0, from 8 k0 - 71 on.  When that first frame lies inside its call's group, the kernel computes the
// group's earlier frames for its maximum and does not write them.
__host__ __device__ __forceinline__ int clip_frame_step(int f) { return f < 5 ? 0 : (f - 5) / 8 + 1; }   // the step of frame f
// the group of frame f: the first step of the call that steps it
__host__ __device__ __forceinline__ int clip_group(int f, int chunk) {
    return (int)oww_call_first_step(oww_call_of_step(clip_frame_step(f), chunk), chunk);
}
__host__ __device__ __forceinline__ int clip_first_group(int k0, int chunk) { return clip_group(8 * k0 > 71 ? 8 * k0 - 71 : 0, chunk); }

__global__ void __launch_bounds__(kThreads) mel_clip_kernel(const int16_t* pcm, const int64_t* clip_off, const int* clip_len, int pad,
                                                            int chunk, int k0, int k1, float* out, int64_t out_stride, MelDev c) {
    extern __shared__ __align__(16) uint8_t dyn[];
    float2 (*s_buf)[2][256] = reinterpret_cast<float2 (*)[2][256]>(dyn);               // [kWarps][2][256]
    float2* s_tw = reinterpret_cast<float2*>(dyn + kWarps * 2 * 256 * sizeof(float2));
    float* s_win = reinterpret_cast<float*>(s_tw + 512);
    float (*s_pow)[264] = reinterpret_cast<float (*)[264]>(s_win + 512);
    int16_t (*s_frame)[512] = reinterpret_cast<int16_t (*)[512]>(s_pow + kWarps);       // [kWarps][512] padded-clip samples of a frame
    int* s_gmax = reinterpret_cast<int*>(s_frame + kWarps);                              // [k1 - g0] per-call maxima (ordered-int encoding)
    const int clip = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int v0 = 8 * k0;                                   // first virtual row written (output row 0)
    const int g0 = clip_first_group(k0, chunk);
    const int f0 = g0 == 0 ? 0 : 8 * g0 - 3;                 // first frame of group g0
    const int n_frames = 8 * k1 - 3;
    for (int i = tid; i < 512; i += kThreads) { s_tw[i] = c.twiddle[i]; s_win[i] = c.window[i]; }
    for (int i = tid; i < k1 - g0; i += kThreads) s_gmax[i] = INT_MIN;
    const int16_t* body = pcm + clip_off[clip];
    const int n_samples = clip_len[clip];
    float* o = out + (int64_t)clip * out_stride;
    for (int i = tid; i < (71 - v0) * 32; i += kThreads) o[i] = 1.0f;
    __syncthreads();
    const int my_start = c.mel_start[lane];
    const int my_len = c.mel_len[lane];
    const float* my_w = c.mel_w + lane * OWW_MEL_MAXSUPPORT;
    auto enc = [](float v) { int i = __float_as_int(v); return i >= 0 ? i : i ^ 0x7FFFFFFF; };   // order-preserving float -> int
    for (int f = f0 + warp; f < n_frames; f += kWarps) {
        // stage the frame's 512 samples of the zero-padded clip, then run the ordinary frame routine on them
        for (int j = lane; j < 512; j += 32) {
            const int64_t p = (int64_t)f * OWW_HOP + j - pad;
            s_frame[warp][j] = (p >= 0 && p < n_samples) ? body[p] : (int16_t)0;
        }
        __syncwarp();
        const float db = mel_frame_db<false>(nullptr, 0, s_frame[warp], 0, s_buf[warp][0], s_buf[warp][1], s_pow[warp], s_tw, s_win, c.kmax,
                                      my_start, my_len, my_w, lane);
        if (71 + f >= v0) o[(int64_t)(71 + f - v0) * 32 + lane] = db;
        float m = db;
#pragma unroll
        for (int k = 16; k > 0; k >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, k));
        if (lane == 0) atomicMax(&s_gmax[clip_group(f, chunk) - g0], enc(m));
        __syncwarp();
    }
    __syncthreads();
    const int fw = max(f0, v0 - 71);                         // first frame written
    for (int i = tid; i < (n_frames - fw) * 32; i += kThreads) {
        const int f = fw + (i >> 5);
        const int e = s_gmax[clip_group(f, chunk) - g0];
        const float gmax = __int_as_float(e >= 0 ? e : e ^ 0x7FFFFFFF);
        float* q = o + (int64_t)(71 + f - v0) * 32 + (i & 31);
        *q = fmaxf(*q, gmax - 80.0f) / 10.0f + 2.0f;
    }
}

// ---- host-side constants (double precision), SURVEY.md Appendix A ---------------------------
double hz_to_mel(double f) {
    const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp;
    const double logstep = std::log(6.4) / 27.0;
    return f >= min_log_hz ? min_log_mel + std::log(f / min_log_hz) / logstep : f / f_sp;
}
double mel_to_hz(double m) {
    const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp;
    const double logstep = std::log(6.4) / 27.0;
    return m >= min_log_mel ? min_log_hz * std::exp(logstep * (m - min_log_mel)) : f_sp * m;
}

}  // namespace

int oww_mel_launch(oww_ctx* ctx, const MelLaunch& p, cudaStream_t s) {
    if (!ctx->mel_loaded) return oww_fail(ctx, OWW_EINVAL, "mel constants not loaded");
    const int prefix = p.tail ? OWW_TAIL : 0;
    if (prefix + p.n_body < OWW_FFT_N) return oww_fail(ctx, OWW_EINVAL, "clip shorter than 512 samples");
    if (p.n_clips <= 0) return OWW_OK;
    MelDev c{ctx->d_window, ctx->d_twiddle, ctx->d_mel_start, ctx->d_mel_len, ctx->d_mel_w, ctx->mel_kmax};
    OWW_CUDA(ctx, oww_launch_pdl(p.pdl, mel_kernel, dim3(p.n_clips), dim3(kThreads), 0, s, p, c));
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

int oww_mel_clips_launch(oww_ctx* ctx, const int16_t* d_pcm, const int64_t* d_off, const int* d_len, int n_clips, int pad,
                         int chunk, int k0, int k1, float* d_out, int64_t out_stride, cudaStream_t s) {
    if (!ctx->mel_loaded) return oww_fail(ctx, OWW_EINVAL, "mel constants not loaded");
    if (n_clips <= 0 || k1 <= k0) return OWW_OK;
    if (k0 < 0 || k1 - k0 > 8192 || chunk < 1 || oww_call_first_step(oww_call_of_step(k1, chunk), chunk) != k1)
        return oww_fail(ctx, OWW_EINVAL, "step range [%d,%d) is not a bulk frontend segment", k0, k1);
    MelDev c{ctx->d_window, ctx->d_twiddle, ctx->d_mel_start, ctx->d_mel_len, ctx->d_mel_w, ctx->mel_kmax};
    const size_t smem = (size_t)kWarps * 2 * 256 * sizeof(float2) + 512 * sizeof(float2) + 512 * sizeof(float) +
                        (size_t)kWarps * 264 * sizeof(float) + (size_t)kWarps * 512 * sizeof(int16_t) +
                        (size_t)(k1 - clip_first_group(k0, chunk)) * sizeof(int);
    if (!ctx->mel_clip_attr_set) {
        OWW_CUDA(ctx, cudaFuncSetAttribute(mel_clip_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        ctx->mel_clip_attr_set = true;
    }
    mel_clip_kernel<<<n_clips, kThreads, smem, s>>>(d_pcm, d_off, d_len, pad, chunk, k0, k1, d_out, out_stride, c);
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

extern "C" int oww_load_mel(oww_ctx* ctx, const float* h_window512, const float* h_mel_fb) {
    if (!ctx) return OWW_EINVAL;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    const double kPi = 3.14159265358979323846;
    std::vector<float> win(512, 0.f);
    if (h_window512) {
        std::memcpy(win.data(), h_window512, 512 * sizeof(float));
    } else {
        for (int n = 0; n < 400; ++n) win[56 + n] = (float)(0.5 - 0.5 * std::cos(2.0 * kPi * n / 400.0));
    }
    std::vector<float2> tw(512);
    for (int k = 0; k < 512; ++k) {
        const double a = -2.0 * kPi * k / 512.0;
        tw[k] = make_float2((float)std::cos(a), (float)std::sin(a));
    }
    std::vector<float> fb(OWW_N_BINS * OWW_MEL_BINS);
    if (h_mel_fb) {
        std::memcpy(fb.data(), h_mel_fb, fb.size() * sizeof(float));
    } else {
        const int n_mels = OWW_MEL_BINS;
        std::vector<double> mel_f(n_mels + 2);
        const double m0 = hz_to_mel(60.0), m1 = hz_to_mel(3800.0);
        for (int i = 0; i < n_mels + 2; ++i) mel_f[i] = mel_to_hz(m0 + (m1 - m0) * i / (n_mels + 1));
        for (int k = 0; k < OWW_N_BINS; ++k) {
            const double ff = 8000.0 * k / 256.0;
            for (int i = 0; i < n_mels; ++i) {
                const double lower = (ff - mel_f[i]) / (mel_f[i + 1] - mel_f[i]);
                const double upper = (mel_f[i + 2] - ff) / (mel_f[i + 2] - mel_f[i + 1]);
                double w = lower < upper ? lower : upper;
                if (w < 0) w = 0;
                w *= 2.0 / (mel_f[i + 2] - mel_f[i]);
                fb[k * n_mels + i] = (float)w;
            }
        }
    }
    std::vector<int> st(OWW_MEL_BINS, 0), ln(OWW_MEL_BINS, 0);
    std::vector<float> mw(OWW_MEL_BINS * OWW_MEL_MAXSUPPORT, 0.f);
    int kmax = 0;
    for (int i = 0; i < OWW_MEL_BINS; ++i) {
        int lo = -1, hi = -1;
        for (int k = 0; k < OWW_N_BINS; ++k)
            if (fb[k * OWW_MEL_BINS + i] != 0.f) { if (lo < 0) lo = k; hi = k; }
        if (lo < 0) { st[i] = 0; ln[i] = 0; continue; }
        if (hi - lo + 1 > OWW_MEL_MAXSUPPORT)
            return oww_fail(ctx, OWW_EUNSUPPORTED, "mel filter %d spans %d FFT bins (max %d)", i, hi - lo + 1,
                            OWW_MEL_MAXSUPPORT);
        st[i] = lo; ln[i] = hi - lo + 1;
        for (int k = lo; k <= hi; ++k) mw[i * OWW_MEL_MAXSUPPORT + (k - lo)] = fb[k * OWW_MEL_BINS + i];
        if (hi + 1 > kmax) kmax = hi + 1;
    }
    ctx->mel_kmax = kmax;
    ctx->mel_key = oww_fnv1a(fb.data(), fb.size() * sizeof(float), oww_fnv1a(win.data(), win.size() * sizeof(float)));
    auto up = [&](void** d, const void* h, size_t bytes) -> cudaError_t {
        if (!*d) { cudaError_t e = cudaMalloc(d, bytes); if (e != cudaSuccess) return e; }
        return cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice);
    };
    OWW_CUDA(ctx, up((void**)&ctx->d_window, win.data(), 512 * sizeof(float)));
    OWW_CUDA(ctx, up((void**)&ctx->d_twiddle, tw.data(), 512 * sizeof(float2)));
    OWW_CUDA(ctx, up((void**)&ctx->d_mel_start, st.data(), OWW_MEL_BINS * sizeof(int)));
    OWW_CUDA(ctx, up((void**)&ctx->d_mel_len, ln.data(), OWW_MEL_BINS * sizeof(int)));
    OWW_CUDA(ctx, up((void**)&ctx->d_mel_w, mw.data(), mw.size() * sizeof(float)));
    ctx->mel_loaded = true;
    return OWW_OK;
}
