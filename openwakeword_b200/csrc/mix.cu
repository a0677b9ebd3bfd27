// Mixing clean clips with background noise and room impulse responses (RIRs) on the device: the test clips of a
// false-reject evaluation (openwakeword/data.py:294-527, mix_clips_batch / mix_clip / truncate_clip, and speechbrain's
// reverberate).  The per-mixture transform is stated in include/owwb200.h (oww_mix_clips); three launches per call:
//
//   mix_kernel     one CTA per mixture: both squared norms in float64, then m = (b + g f) / 2 stored as float32 and
//                  sum |m| (the reverb's target amplitude).  HBM bound.
//   reverb_kernel  the circular convolution with the RIR, aligned on its direct path, as a banded circulant GEMM on the
//                  tensor cores.  Output sample n = 64 s + c of a mixture is row s, column c of Y = A T: A's row s holds the
//                  mixture's samples around 64 s, T is Toeplitz in (c - t) and made of the RIR's taps.  Cut into K-blocks
//                  of 64, block b of T is T_b[t][c] = h[64 b + 63 + c - t], the same for every row, and A_b's row s is the
//                  64 mixture samples from 64 (s - b) + d - 63 (mod N): consecutive blocks are the same window shifted by
//                  one row.  A CTA (one warpgroup) owns 64 rows (4096 outputs) of one mixture and visits only the
//                  floor((L - 1) / 64) + 2 blocks that hold taps.  Operands are fp16 hi/lo splits (hi*hi + hi*lo + lo*hi
//                  into fp32, as the CNN's split layers); the taps are scaled by a power of two so the largest is in
//                  [0.5, 1), and the outputs scaled back exactly.  The epilogue sums |y| per tile for the rescale.
//   finish_kernel  one CTA per mixture: the reverb's rescale, the level (signed maximum with a volume, |y| <= 1
//                  without), int16 conversion with saturation, and the valid flag.
#include "oww_internal.h"
#include "tc_common.cuh"

#include <algorithm>
#include <cmath>
#include <new>
#include <numeric>
#include <vector>

namespace {

constexpr int MIX_THREADS = 256;
constexpr int RV_THREADS = 128;                  // one warpgroup
constexpr int RV_KB = 16;                        // K-blocks of 64 staged per chunk
constexpr int RV_Q = 63 + RV_KB;                 // A rows of a chunk: the 64 output rows and the shifts of its blocks
constexpr int RV_GCH = 8 * RV_KB + 7;            // 16-byte tap groups of each of the 8 shifted copies
constexpr int RV_TAPS = 64 * RV_KB + 63;         // taps a chunk reads
constexpr uint32_t RV_A_BYTES = 8u * RV_Q * 16u;           // 8 K-strips of RV_Q rows x 16 B
constexpr uint32_t RV_G_BYTES = RV_GCH * 128u;
constexpr uint32_t RV_SMEM = 2 * RV_A_BYTES + 2 * RV_G_BYTES + ((RV_TAPS * 4 + 127) & ~127) + 128;

struct MixRow {                   // per mixture of a call
    int64_t fg_off, fg_len;       // foreground window in d_fg
    int64_t bg_off, bg_len;       // background clip in d_bg
    int64_t bg_pos, start;
    double snr_amp;               // 10^(snr_db / 20)
    double volume;
    int64_t rir_off;              // RIR in d_rir
    int32_t rir_len;
    int32_t slot;                 // row of the reverb buffer, -1: no reverb
    int32_t tile0, n_tiles;       // its reverb tiles
};
struct MixTile { int32_t row, s0; };     // output rows (64-sample segments) s0 .. s0 + 63 of mixture `row`

template <typename T>
__device__ __forceinline__ T block_sum(T v, T* red) {          // fixed-order tree: the same sum on every run
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[w] = v;
    __syncthreads();
    T s = 0;
    for (int i = 0; i < nw; ++i) s += red[i];
    return s;
}

__device__ __forceinline__ float block_max(float v, float* red) {
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[w] = v;
    __syncthreads();
    float s = red[0];
    for (int i = 1; i < nw; ++i) s = fmaxf(s, red[i]);
    return s;
}

__global__ void __launch_bounds__(MIX_THREADS) mix_kernel(const int16_t* __restrict__ fg, const int16_t* __restrict__ bg,
                                                          const MixRow* __restrict__ rows, int64_t N, float* __restrict__ m,
                                                          double* __restrict__ sum_abs, uint8_t* __restrict__ bad) {
    __shared__ double red[MIX_THREADS / 32];
    const MixRow R = rows[blockIdx.x];
    const int16_t* f = fg + R.fg_off;
    const int16_t* b = bg + R.bg_off;
    const int64_t step = MIX_THREADS % R.bg_len;
    double ff = 0.0, bb = 0.0;
    for (int64_t k = threadIdx.x; k < R.fg_len; k += MIX_THREADS) { const double x = f[k]; ff += x * x; }
    int64_t j = (R.bg_pos + threadIdx.x) % R.bg_len;
    for (int64_t n = threadIdx.x; n < N; n += MIX_THREADS) {
        const double x = b[j];
        bb += x * x;
        j += step; if (j >= R.bg_len) j -= R.bg_len;
    }
    ff = block_sum(ff, red);
    bb = block_sum(bb, red);
    const bool invalid = ff == 0.0 || bb == 0.0;
    const double g = invalid ? 0.0 : R.snr_amp * sqrt(bb) / sqrt(ff);     // the 1/32768 of both norms cancels
    float* out = m + (int64_t)blockIdx.x * N;
    double sa = 0.0;
    j = (R.bg_pos + threadIdx.x) % R.bg_len;
    for (int64_t n = threadIdx.x; n < N; n += MIX_THREADS) {
        double v = (double)b[j] * (1.0 / 32768.0);
        const int64_t k = n - R.start;
        if (k >= 0 && k < R.fg_len) v += g * ((double)f[k] * (1.0 / 32768.0));
        const float mv = invalid ? 0.0f : (float)(0.5 * v);
        out[n] = mv;
        sa += fabs((double)mv);
        j += step; if (j >= R.bg_len) j -= R.bg_len;
    }
    sa = block_sum(sa, red);
    if (threadIdx.x == 0) { sum_abs[blockIdx.x] = sa; bad[blockIdx.x] = invalid; }
}

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

// hi = fp16(x), lo = fp16(x - hi) for 8 values, stored as one 16-byte row of a core matrix each
__device__ __forceinline__ void store_split8(const float* x, unsigned char* hi, unsigned char* lo) {
    float h[8], l[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        h[e] = __half2float(__float2half_rn(x[e]));
        l[e] = x[e] - h[e];
    }
    *reinterpret_cast<uint4*>(hi) = make_uint4(pack_h2(h[0], h[1]), pack_h2(h[2], h[3]), pack_h2(h[4], h[5]), pack_h2(h[6], h[7]));
    *reinterpret_cast<uint4*>(lo) = make_uint4(pack_h2(l[0], l[1]), pack_h2(l[2], l[3]), pack_h2(l[4], l[5]), pack_h2(l[6], l[7]));
}

__global__ void __launch_bounds__(RV_THREADS) reverb_kernel(const float* __restrict__ m, const float* __restrict__ rir,
                                                            const MixRow* __restrict__ rows, const MixTile* __restrict__ tiles,
                                                            int64_t N, float* __restrict__ y, double* __restrict__ partial) {
    extern __shared__ __align__(128) unsigned char smem[];
    unsigned char* a_hi = smem;
    unsigned char* a_lo = a_hi + RV_A_BYTES;
    unsigned char* g_hi = a_lo + RV_A_BYTES;
    unsigned char* g_lo = g_hi + RV_G_BYTES;
    float* tw = reinterpret_cast<float*>(g_lo + RV_G_BYTES);
    __shared__ float red_v[RV_THREADS / 32];
    __shared__ int red_i[RV_THREADS / 32];
    __shared__ double red_d[RV_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const MixTile T = tiles[blockIdx.x];
    const MixRow R = rows[T.row];
    const float* h = rir + R.rir_off;
    const int L = R.rir_len;
    const float* x = m + (int64_t)T.row * N;

    // direct path: the first index of the largest |h|
    float best = -1.0f;
    int bi = 0;
    for (int k = tid; k < L; k += RV_THREADS) {
        const float a = fabsf(h[k]);
        if (a > best) { best = a; bi = k; }
    }
    for (int o = 16; o; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) { red_v[warp] = best; red_i[warp] = bi; }
    __syncthreads();
    best = red_v[0]; bi = red_i[0];
    for (int w = 1; w < RV_THREADS / 32; ++w)
        if (red_v[w] > best || (red_v[w] == best && red_i[w] < bi)) { best = red_v[w]; bi = red_i[w]; }
    const int64_t d = bi;
    int ex = 0;
    frexpf(best, &ex);                               // best = 0: ex = 0
    const float tap_scale = ldexpf(1.0f, -ex), out_scale = ldexpf(1.0f, ex);

    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.0f;
    const int b_max = (L - 1) / 64;
    const int64_t s0 = T.s0;
    const uint32_t sa_hi = smem_u32(a_hi), sa_lo = smem_u32(a_lo), sg_hi = smem_u32(g_hi), sg_lo = smem_u32(g_lo);
    for (int b_lo = -1; b_lo <= b_max; b_lo += RV_KB) {
        const int kb = min(RV_KB, b_max - b_lo + 1), b_top = b_lo + kb - 1;
        __syncthreads();                             // the previous chunk's operands have been read
        for (int u = tid; u < 64 * kb + 63; u += RV_THREADS) {
            const int k = 64 * b_lo + u;
            tw[u] = (k >= 0 && k < L) ? h[k] * tap_scale : 0.0f;
        }
        // A rows q < 63 + kb: W[q][t] = x[(64 (s0 + q - b_top) + d - 63 + t) mod N], K-strip t / 8 of RV_Q rows
        for (int it = tid; it < (63 + kb) * 8; it += RV_THREADS) {
            const int q = it >> 3, gs = it & 7;
            int64_t p = (64 * (s0 + q - b_top) + d - 63 + 8 * gs) % N;
            if (p < 0) p += N;
            float v[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                v[e] = x[p];
                if (++p >= N) p -= N;
                if (p >= N) p %= N;                  // N < 8
            }
            const uint32_t off = (uint32_t)gs * (RV_Q * 16u) + (uint32_t)q * 16u;
            store_split8(v, a_hi + off, a_lo + off);
        }
        __syncthreads();                             // tw complete
        // B: 8 copies of the reversed taps shifted by one sample each, so that block b's T_b is the K-major matrix at
        // 16-byte group 8 (b_top - b) with LBO = SBO = 128 B: G[q][sg][e] = tw[126 + 64 (kb - 1) - 8 q - e - sg]
        for (int it = tid; it < (8 * kb + 7) * 8; it += RV_THREADS) {
            const int q = it >> 3, sg = it & 7;
            const int base = 126 + 64 * (kb - 1) - 8 * q - sg;
            float v[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = tw[base - e];
            const uint32_t off = (uint32_t)q * 128u + (uint32_t)sg * 16u;
            store_split8(v, g_hi + off, g_lo + off);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to the tensor core
        __syncthreads();
        wg_fence();
        for (int b = b_lo; b <= b_top; ++b) {
            const uint32_t q0 = (uint32_t)(b_top - b), c0 = 8u * (uint32_t)(b_top - b);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t ao = (uint32_t)(2 * kk) * (RV_Q * 16u) + q0 * 16u;
                const uint32_t bo = (c0 + 2u * kk) * 128u;
                const uint64_t ah = make_desc(sa_hi + ao, RV_Q * 16u, 128u), al = make_desc(sa_lo + ao, RV_Q * 16u, 128u);
                const uint64_t bh = make_desc(sg_hi + bo, 128u, 128u), bl = make_desc(sg_lo + bo, 128u, 128u);
                wg_mma<64>(acc, ah, bh, 1u);
                wg_mma<64>(acc, ah, bl, 1u);
                wg_mma<64>(acc, al, bh, 1u);
            }
        }
        wg_commit();
        wg_wait_all();
    }
    // D fragment: acc[4 j + 2 i + e] is row 16 warp + lane / 4 + 8 i, column n = 8 j + 2 (lane % 4) + e, output c = 63 - n
    float* out = y + (int64_t)R.slot * N;
    double sa = 0.0;
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int64_t s = s0 + 16 * warp + (lane >> 2) + 8 * i;
                const int64_t pos = 64 * s + 63 - (8 * j + 2 * (lane & 3) + e);
                if (pos < N) {
                    const float v = acc[4 * j + 2 * i + e] * out_scale;
                    out[pos] = v;
                    sa += fabs((double)v);
                }
            }
    sa = block_sum(sa, red_d);
    if (tid == 0) partial[blockIdx.x] = sa;
}

__global__ void __launch_bounds__(MIX_THREADS) finish_kernel(const float* __restrict__ m, const float* __restrict__ y,
                                                             const MixRow* __restrict__ rows, const double* __restrict__ sum_abs,
                                                             const uint8_t* __restrict__ bad, const double* __restrict__ partial,
                                                             int64_t N, int16_t* __restrict__ out, uint8_t* __restrict__ valid) {
    __shared__ float red_f[MIX_THREADS / 32];
    __shared__ int red_i[MIX_THREADS / 32];
    const int r = blockIdx.x;
    const MixRow R = rows[r];
    int16_t* o = out + (int64_t)r * N;
    const float* src = R.slot >= 0 ? y + (int64_t)R.slot * N : m + (int64_t)r * N;
    double f0 = 1.0;                                 // the reverb's rescale a0 / (mean |y| + 1e-14)
    if (R.slot >= 0) {
        double sy = 0.0;
        for (int t = 0; t < R.n_tiles; ++t) sy += partial[R.tile0 + t];
        f0 = (sum_abs[r] / (double)N) / (sy / (double)N + 1e-14);
    }
    float mx = -INFINITY, amx = 0.0f;
    for (int64_t n = threadIdx.x; n < N; n += MIX_THREADS) {
        const float v = src[n];
        mx = fmaxf(mx, v);
        amx = fmaxf(amx, fabsf(v));
    }
    mx = block_max(mx, red_f);
    amx = block_max(amx, red_f);
    bool zero = bad[r] != 0;
    double F;
    if (R.volume >= 0.0) {
        zero = zero || !((double)mx * f0 > 0.0);
        F = zero ? 0.0 : R.volume / (double)mx;      // (y f0) * volume / max(y f0)
    } else {
        F = f0 / fmax((double)amx * f0, 1.0);
    }
    int top = -32768;
    for (int64_t n = threadIdx.x; n < N; n += MIX_THREADS) {
        int q = 0;
        if (!zero) {
            const double v = trunc((double)src[n] * F * 32767.0);
            q = (int)fmin(fmax(v, -32768.0), 32767.0);
        }
        o[n] = (int16_t)q;
        top = max(top, q);
    }
    for (int s = 16; s; s >>= 1) top = max(top, __shfl_xor_sync(0xffffffffu, top, s));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red_i[threadIdx.x >> 5] = top;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < MIX_THREADS / 32; ++w) top = max(top, red_i[w]);
        top = max(top, red_i[0]);
        valid[r] = (!zero && top != 0) ? 1 : 0;
    }
}

int check_offsets(oww_ctx* ctx, const int64_t* off, int n, const char* what) {
    if (n < 0) return oww_fail(ctx, OWW_EINVAL, "n_%s=%d is negative", what, n);
    if (!off) return n ? oww_fail(ctx, OWW_EINVAL, "null argument") : OWW_OK;
    if (off[0] < 0) return oww_fail(ctx, OWW_EINVAL, "%s offsets: first offset %lld is negative", what, (long long)off[0]);
    for (int i = 0; i < n; ++i)
        if (off[i + 1] < off[i]) return oww_fail(ctx, OWW_EINVAL, "%s offsets decrease at clip %d", what, i);
    return OWW_OK;
}

}  // namespace

struct oww_mixer {
    void* h_tab = nullptr;            // pinned: MixRow [n_mix], then MixTile [n_tiles]
    void* d_tab = nullptr;
    size_t tab_bytes = 0;
    float* d_m = nullptr;             // mixtures before reverb, [n_mix][N]
    size_t m_bytes = 0;
    float* d_y = nullptr;             // reverberated mixtures, [n_reverb][N]
    size_t y_bytes = 0;
    void* d_stats = nullptr;          // sum |m| (double) [n_mix], partial sums |y| (double) [n_tiles], invalid (u8) [n_mix]
    size_t stats_bytes = 0;
    cudaEvent_t done = nullptr;       // after the last launch: tables and scratch are free once it has completed
};

namespace {

int grow(oww_ctx* ctx, void** p, size_t* cap, size_t need) {
    if (need <= *cap) return OWW_OK;
    cudaFree(*p);
    *p = nullptr; *cap = 0;
    if (cudaMalloc(p, need) != cudaSuccess) {
        cudaGetLastError();
        *p = nullptr;
        return oww_fail(ctx, OWW_ENOMEM, "cudaMalloc of %zu bytes for the mixer failed", need);
    }
    *cap = need;
    return OWW_OK;
}

}  // namespace

void oww_mix_free(oww_ctx* ctx) {
    oww_mixer* c = ctx->mixer;
    if (!c) return;
    cudaFreeHost(c->h_tab); cudaFree(c->d_tab); cudaFree(c->d_m); cudaFree(c->d_y); cudaFree(c->d_stats);
    if (c->done) cudaEventDestroy(c->done);
    delete c;
    ctx->mixer = nullptr;
}

extern "C" {

int oww_mix_clips(oww_ctx* ctx, const int16_t* d_fg, const int64_t* h_fg_off, int n_fg,
                  const int16_t* d_bg, const int64_t* h_bg_off, int n_bg,
                  const float* d_rir, const int64_t* h_rir_off, int n_rir,
                  const oww_mix_params* h_params, int n_mix, int64_t n_samples,
                  int16_t* d_out, uint8_t* d_valid, void* stream) {
    if (!ctx) return OWW_EINVAL;
    const int64_t N = n_samples;
    if (N <= 0) return oww_fail(ctx, OWW_EINVAL, "n_samples=%lld is not positive", (long long)N);
    if (n_mix < 0) return oww_fail(ctx, OWW_EINVAL, "n_mix=%d is negative", n_mix);
    int rc;
    if ((rc = check_offsets(ctx, h_fg_off, n_fg, "fg")) || (rc = check_offsets(ctx, h_bg_off, n_bg, "bg")) ||
        (rc = check_offsets(ctx, h_rir_off, n_rir, "rir")))
        return rc;
    if (n_mix == 0) return OWW_OK;
    if (!h_params || !d_out || !d_valid) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if ((n_fg && h_fg_off[n_fg] > h_fg_off[0] && !d_fg) || (n_bg && h_bg_off[n_bg] > h_bg_off[0] && !d_bg) ||
        (n_rir && h_rir_off[n_rir] > h_rir_off[0] && !d_rir))
        return oww_fail(ctx, OWW_EINVAL, "null argument");
    const int64_t tiles_per_row = (N + 4095) / 4096;
    int64_t n_rev = 0;
    for (int i = 0; i < n_mix; ++i) {
        const oww_mix_params& p = h_params[i];
        if (p.fg < 0 || p.fg >= n_fg) return oww_fail(ctx, OWW_EINVAL, "mixture %d: foreground %d out of range", i, p.fg);
        if (p.bg < 0 || p.bg >= n_bg) return oww_fail(ctx, OWW_EINVAL, "mixture %d: background %d out of range", i, p.bg);
        if (p.rir < -1 || p.rir >= n_rir) return oww_fail(ctx, OWW_EINVAL, "mixture %d: rir %d out of range", i, p.rir);
        const int64_t fl = h_fg_off[p.fg + 1] - h_fg_off[p.fg], bl = h_bg_off[p.bg + 1] - h_bg_off[p.bg];
        if (p.fg_start < 0 || p.fg_len < 0 || p.fg_start > fl - p.fg_len)
            return oww_fail(ctx, OWW_EINVAL, "mixture %d: foreground window [%lld, +%lld) outside its %lld samples", i,
                            (long long)p.fg_start, (long long)p.fg_len, (long long)fl);
        if (bl <= 0) return oww_fail(ctx, OWW_EINVAL, "mixture %d: background %d is empty", i, p.bg);
        if (p.bg_offset < 0 || p.bg_offset >= bl)
            return oww_fail(ctx, OWW_EINVAL, "mixture %d: bg_offset %lld outside [0, %lld)", i, (long long)p.bg_offset,
                            (long long)bl);
        if (p.start < 0 || p.start > N - p.fg_len)
            return oww_fail(ctx, OWW_EINVAL, "mixture %d: start %lld + %lld foreground samples exceed N=%lld", i,
                            (long long)p.start, (long long)p.fg_len, (long long)N);
        if (!std::isfinite(p.snr_db) || !std::isfinite(p.volume))
            return oww_fail(ctx, OWW_EINVAL, "mixture %d: snr_db and volume must be finite", i);
        if (p.rir >= 0) {
            const int64_t L = h_rir_off[p.rir + 1] - h_rir_off[p.rir];
            if (L <= 0) return oww_fail(ctx, OWW_EINVAL, "mixture %d: rir %d is empty", i, p.rir);
            if (L > N) return oww_fail(ctx, OWW_EINVAL, "mixture %d: rir %d has %lld taps, more than N=%lld", i, p.rir,
                                       (long long)L, (long long)N);
            ++n_rev;
        }
    }
    const int64_t n_tiles = n_rev * tiles_per_row;
    if (n_tiles > INT32_MAX) return oww_fail(ctx, OWW_EINVAL, "%lld reverb tiles in one call", (long long)n_tiles);
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->mixer) {
        ctx->mixer = new (std::nothrow) oww_mixer();
        if (!ctx->mixer) return oww_fail(ctx, OWW_ENOMEM, "out of host memory");
        if (cudaEventCreateWithFlags(&ctx->mixer->done, cudaEventDisableTiming) != cudaSuccess ||
            cudaFuncSetAttribute(reverb_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RV_SMEM) != cudaSuccess) {
            oww_mix_free(ctx);
            return oww_fail(ctx, OWW_ECUDA, "mixer set-up failed");
        }
    }
    oww_mixer* c = ctx->mixer;
    OWW_CUDA(ctx, cudaEventSynchronize(c->done));              // the previous call's tables and scratch are free
    const size_t tile_off = ((size_t)n_mix * sizeof(MixRow) + 15) & ~(size_t)15;
    const size_t bytes = tile_off + (size_t)n_tiles * sizeof(MixTile);
    if (bytes > c->tab_bytes) {
        cudaFreeHost(c->h_tab); cudaFree(c->d_tab);
        c->h_tab = nullptr; c->d_tab = nullptr; c->tab_bytes = 0;
        const size_t want = std::max(bytes, 2 * c->tab_bytes);
        OWW_CUDA(ctx, cudaMallocHost(&c->h_tab, want));
        OWW_CUDA(ctx, cudaMalloc(&c->d_tab, want));
        c->tab_bytes = want;
    }
    const size_t sum_off = 0, part_off = (size_t)n_mix * 8, bad_off = part_off + (size_t)n_tiles * 8;
    if ((rc = grow(ctx, (void**)&c->d_m, &c->m_bytes, (size_t)n_mix * N * sizeof(float))) ||
        (rc = grow(ctx, (void**)&c->d_y, &c->y_bytes, (size_t)std::max<int64_t>(n_rev, 1) * N * sizeof(float))) ||
        (rc = grow(ctx, &c->d_stats, &c->stats_bytes, bad_off + (size_t)n_mix)))
        return rc;
    MixRow* rows = (MixRow*)c->h_tab;
    MixTile* tiles = (MixTile*)((char*)c->h_tab + tile_off);
    // reverb rows grouped by RIR (stable), so the CTAs that read one RIR's taps run next to each other
    std::vector<int> order;
    order.reserve((size_t)n_rev);
    for (int i = 0; i < n_mix; ++i) if (h_params[i].rir >= 0) order.push_back(i);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return h_params[a].rir < h_params[b].rir; });
    for (int i = 0; i < n_mix; ++i) {
        const oww_mix_params& p = h_params[i];
        MixRow& R = rows[i];
        R.fg_off = h_fg_off[p.fg] + p.fg_start;
        R.fg_len = p.fg_len;
        R.bg_off = h_bg_off[p.bg];
        R.bg_len = h_bg_off[p.bg + 1] - h_bg_off[p.bg];
        R.bg_pos = p.bg_offset;
        R.start = p.start;
        R.snr_amp = std::pow(10.0, p.snr_db / 20.0);
        R.volume = p.volume;
        R.rir_off = p.rir >= 0 ? h_rir_off[p.rir] : 0;
        R.rir_len = p.rir >= 0 ? (int32_t)(h_rir_off[p.rir + 1] - h_rir_off[p.rir]) : 0;
        R.slot = -1;
        R.tile0 = 0; R.n_tiles = 0;
    }
    int32_t t = 0;
    for (size_t k = 0; k < order.size(); ++k) {
        MixRow& R = rows[order[k]];
        R.slot = (int32_t)k;
        R.tile0 = t;
        R.n_tiles = (int32_t)tiles_per_row;
        for (int64_t s = 0; s < tiles_per_row; ++s) tiles[t++] = MixTile{order[k], (int32_t)(64 * s)};
    }
    cudaStream_t s = (cudaStream_t)stream;
    double* d_sum = (double*)((char*)c->d_stats + sum_off);
    double* d_part = (double*)((char*)c->d_stats + part_off);
    uint8_t* d_bad = (uint8_t*)c->d_stats + bad_off;
    const MixRow* d_rows = (const MixRow*)c->d_tab;
    OWW_CUDA(ctx, cudaMemcpyAsync(c->d_tab, c->h_tab, bytes, cudaMemcpyHostToDevice, s));
    mix_kernel<<<(unsigned)n_mix, MIX_THREADS, 0, s>>>(d_fg, d_bg, d_rows, N, c->d_m, d_sum, d_bad);
    OWW_LAUNCH_CHECK(ctx);
    if (n_tiles) {
        reverb_kernel<<<(unsigned)n_tiles, RV_THREADS, RV_SMEM, s>>>(c->d_m, d_rir, d_rows,
                                                                    (const MixTile*)((char*)c->d_tab + tile_off), N, c->d_y, d_part);
        OWW_LAUNCH_CHECK(ctx);
    }
    finish_kernel<<<(unsigned)n_mix, MIX_THREADS, 0, s>>>(c->d_m, c->d_y, d_rows, d_sum, d_bad, d_part, N, d_out, d_valid);
    OWW_LAUNCH_CHECK(ctx);
    OWW_CUDA(ctx, cudaEventRecord(c->done, s));
    return OWW_OK;
}

}  // extern "C"
