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
#include "oww_internal.h"
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

__global__ void __launch_bounds__(kThreads) mel_kernel(MelLaunch p, MelDev c) {
    __shared__ float2 s_buf[kWarps][2][256];
    __shared__ float2 s_tw[512];
    __shared__ float s_win[512];
    __shared__ float s_pow[kWarps][264];
    __shared__ float s_red[kWarps];

    const int clip = p.ids ? p.ids[blockIdx.x] : blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    for (int i = tid; i < 512; i += kThreads) { s_tw[i] = c.twiddle[i]; s_win[i] = c.window[i]; }

    const bool streaming = p.tail != nullptr;
    const int prefix = streaming ? OWW_TAIL : 0;
    const bool fresh = streaming && p.seen[clip] == 0;
    const int total = prefix + p.n_body;
    const int T = (total - OWW_FFT_N) / OWW_HOP + 1;
    const int f0 = fresh ? 3 : 0;                 // frames 0..2 would read the (absent) prefix
    const int16_t* body = p.body + (int64_t)clip * p.body_stride;
    const int16_t* tail = streaming ? p.tail + (int64_t)clip * OWW_TAIL : nullptr;
    const int row0 = p.out_count ? p.out_count[clip] : 0;
    float* out = p.out + (int64_t)clip * p.out_stride;
    __syncthreads();

    const int my_start = c.mel_start[lane];
    const int my_len = c.mel_len[lane];
    const float* my_w = c.mel_w + lane * OWW_MEL_MAXSUPPORT;
    float vmax = -INFINITY;

    for (int f = f0 + warp; f < T; f += kWarps) {
        const float db = mel_frame_db(tail, prefix, body, f, s_buf[warp][0], s_buf[warp][1], s_pow[warp], s_tw, s_win, c.kmax,
                                      my_start, my_len, my_w, lane);
        vmax = fmaxf(vmax, db);
        const int r = f - f0;
        const int slot = p.out_rows_mask >= 0 ? ((row0 + r) & p.out_rows_mask) : r;
        out[(int64_t)slot * OWW_MEL_BINS + lane] = db;
        __syncwarp();
    }
    // per-call maximum -> clamp -> affine
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    if (lane == 0) s_red[warp] = vmax;
    __syncthreads();
    float m = s_red[0];
#pragma unroll
    for (int w = 1; w < kWarps; ++w) m = fmaxf(m, s_red[w]);
    const float floor_db = m - 80.0f;
    const int nrows = T - f0;
    for (int i = tid; i < nrows * OWW_MEL_BINS; i += kThreads) {
        const int r = i >> 5, col = i & 31;
        const int slot = p.out_rows_mask >= 0 ? ((row0 + r) & p.out_rows_mask) : r;
        float* q = out + (int64_t)slot * OWW_MEL_BINS + col;
        float v = fmaxf(__ldcg(q), floor_db);
        if (p.affine) v = v / 10.0f + 2.0f;
        *q = v;
    }
    if (streaming) {
        __syncthreads();                       // every frame has read the old tail
        int16_t* tw = p.tail + (int64_t)clip * OWW_TAIL;
        for (int i = tid; i < OWW_TAIL; i += kThreads) tw[i] = __ldg(body + (p.n_body - OWW_TAIL + i));
        if (tid == 0) {
            p.out_count[clip] = oww_wrap_count(row0 + nrows);
            const int sn = p.seen[clip] + p.n_chunks;
            p.seen[clip] = sn > (1 << 30) ? (1 << 30) : sn;
        }
    }
}

// Bulk path (predict_clip over many clips, SURVEY.md F10): one CTA per clip computes the mel rows of the WHOLE padded clip
// exactly as the streaming calls would have produced them and lays them out as the virtual history the fully
// convolutional CNN pass needs:  out[clip] = [ones x 71 | frames 0..4 of call 0 | 8 frames of call 1 | ...],
// 76 + 8 (steps - 1) rows.  The -80 dB clamp is per CALL (F7): frames are grouped [0,5), [5,13), [13,21), ... and each
// group is clamped against its own maximum.  pad_samples zeros are virtual (nothing is copied).
__global__ void __launch_bounds__(kThreads) mel_clip_kernel(const int16_t* pcm, int64_t clip_stride, int n_samples, int pad, int steps,
                                                            float* out, int64_t out_stride, MelDev c) {
    extern __shared__ __align__(16) uint8_t dyn[];
    float2 (*s_buf)[2][256] = reinterpret_cast<float2 (*)[2][256]>(dyn);               // [kWarps][2][256]
    float2* s_tw = reinterpret_cast<float2*>(dyn + kWarps * 2 * 256 * sizeof(float2));
    float* s_win = reinterpret_cast<float*>(s_tw + 512);
    float (*s_pow)[264] = reinterpret_cast<float (*)[264]>(s_win + 512);
    int16_t (*s_frame)[512] = reinterpret_cast<int16_t (*)[512]>(s_pow + kWarps);       // [kWarps][512] padded-clip samples of a frame
    int* s_gmax = reinterpret_cast<int*>(s_frame + kWarps);                              // [steps] per-call maxima (ordered-int encoding)
    const int clip = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < 512; i += kThreads) { s_tw[i] = c.twiddle[i]; s_win[i] = c.window[i]; }
    for (int i = tid; i < steps; i += kThreads) s_gmax[i] = INT_MIN;
    const int16_t* body = pcm + (int64_t)clip * clip_stride;
    float* o = out + (int64_t)clip * out_stride;
    const int n_frames = 8 * steps - 3;
    for (int i = tid; i < 71 * 32; i += kThreads) o[i] = 1.0f;
    __syncthreads();
    const int my_start = c.mel_start[lane];
    const int my_len = c.mel_len[lane];
    const float* my_w = c.mel_w + lane * OWW_MEL_MAXSUPPORT;
    auto enc = [](float v) { int i = __float_as_int(v); return i >= 0 ? i : i ^ 0x7FFFFFFF; };   // order-preserving float -> int
    for (int f = warp; f < n_frames; f += kWarps) {
        // stage the frame's 512 samples of the zero-padded clip, then run the ordinary frame routine on them
        for (int j = lane; j < 512; j += 32) {
            const int64_t p = (int64_t)f * OWW_HOP + j - pad;
            s_frame[warp][j] = (p >= 0 && p < n_samples) ? body[p] : (int16_t)0;
        }
        __syncwarp();
        const float db = mel_frame_db<false>(nullptr, 0, s_frame[warp], 0, s_buf[warp][0], s_buf[warp][1], s_pow[warp], s_tw, s_win, c.kmax,
                                      my_start, my_len, my_w, lane);
        o[(int64_t)(71 + f) * 32 + lane] = db;
        float m = db;
#pragma unroll
        for (int k = 16; k > 0; k >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, k));
        if (lane == 0) atomicMax(&s_gmax[f < 5 ? 0 : (f - 5) / 8 + 1], enc(m));
        __syncwarp();
    }
    __syncthreads();
    for (int i = tid; i < n_frames * 32; i += kThreads) {
        const int f = i >> 5;
        const int e = s_gmax[f < 5 ? 0 : (f - 5) / 8 + 1];
        const float gmax = __int_as_float(e >= 0 ? e : e ^ 0x7FFFFFFF);
        float* q = o + (int64_t)(71 + f) * 32 + (i & 31);
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
    mel_kernel<<<p.n_clips, kThreads, 0, s>>>(p, c);
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

int oww_mel_clips_launch(oww_ctx* ctx, const int16_t* d_pcm, int64_t clip_stride, int n_clips, int n_samples, int pad, int steps,
                         float* d_out, int64_t out_stride, cudaStream_t s) {
    if (!ctx->mel_loaded) return oww_fail(ctx, OWW_EINVAL, "mel constants not loaded");
    if (n_clips <= 0 || steps <= 0) return OWW_OK;
    if (steps > 8192) return oww_fail(ctx, OWW_EUNSUPPORTED, "clip of %d steps is too long for the one-pass bulk frontend", steps);
    MelDev c{ctx->d_window, ctx->d_twiddle, ctx->d_mel_start, ctx->d_mel_len, ctx->d_mel_w, ctx->mel_kmax};
    const size_t smem = (size_t)kWarps * 2 * 256 * sizeof(float2) + 512 * sizeof(float2) + 512 * sizeof(float) +
                        (size_t)kWarps * 264 * sizeof(float) + (size_t)kWarps * 512 * sizeof(int16_t) + (size_t)steps * sizeof(int);
    if (!ctx->mel_clip_attr_set) {
        OWW_CUDA(ctx, cudaFuncSetAttribute(mel_clip_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        ctx->mel_clip_attr_set = true;
    }
    mel_clip_kernel<<<n_clips, kThreads, smem, s>>>(d_pcm, clip_stride, n_samples, pad, steps, d_out, out_stride, c);
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
