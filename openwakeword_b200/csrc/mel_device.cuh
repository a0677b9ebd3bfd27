// Warp-level log-mel frame routine shared by mel.cu (stand-alone frontend kernel) and cnn_tc_inc.cu (fused step).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "oww_internal.h"

namespace {

// Explicit rounding intrinsics: the compiler may not re-associate or contract these differently in different inlined
// contexts, so the stand-alone frontend kernel and the fused step kernel produce bit-identical mel rows.
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
    return make_float2(__fmaf_rn(a.x, b.x, -__fmul_rn(a.y, b.y)), __fmaf_rn(a.x, b.y, __fmul_rn(a.y, b.x)));
}

// One warp computes frame f (512 samples at hop 160) of the virtual clip [tail (prefix samples) | body]:
// window, 256-point complex radix-4 Stockham FFT of the even/odd-packed frame in the two 256-entry buffers a/b,
// real-spectrum unpack of the bins the filterbank reads (into pw), sparse mel projection (lane = mel bin) and
// 10*log10(max(.,1e-10)).  Returns this lane's dB value (before the per-call clamp and the x/10+2 affine).
template <bool kBodyGlobal = true>     // false: `body` points into shared memory (plain loads instead of ld.global.nc)
__device__ __forceinline__ float mel_frame_db(const int16_t* tail, int prefix, const int16_t* body, int f, float2* a, float2* b,
                                              float* pw_buf, const float2* s_tw, const float* s_win, int kmax, int my_start,
                                              int my_len, const float* my_w, int lane) {
        // windowed frame, packed z[n] = x[2n] + i x[2n+1]
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = lane + 32 * j;
            const int s0 = f * OWW_HOP + 2 * n;
            float x0, x1;
            if (s0 + 1 < prefix) { x0 = (float)tail[s0]; x1 = (float)tail[s0 + 1]; }
            else if (s0 >= prefix) {
                if (kBodyGlobal) { x0 = (float)__ldg(body + (s0 - prefix)); x1 = (float)__ldg(body + (s0 + 1 - prefix)); }
                else { x0 = (float)body[s0 - prefix]; x1 = (float)body[s0 + 1 - prefix]; }
            }
            else { x0 = (float)tail[s0]; x1 = kBodyGlobal ? (float)__ldg(body) : (float)body[0]; }
            a[n] = make_float2(__fmul_rn(x0, s_win[2 * n]), __fmul_rn(x1, s_win[2 * n + 1]));
        }
        __syncwarp();
        // 256-point complex FFT, radix-4 Stockham autosort, 4 passes
#pragma unroll
        for (int Ns = 1; Ns < 256; Ns *= 4) {
            const int tstep = 128 / Ns;
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
                const int j = lane + 32 * jj;
                const int k = j & (Ns - 1);
                float2 v0 = a[j];
                float2 v1 = cmul(a[j + 64], s_tw[k * tstep]);
                float2 v2 = cmul(a[j + 128], s_tw[2 * k * tstep]);
                float2 v3 = cmul(a[j + 192], s_tw[3 * k * tstep]);
                float2 a0 = make_float2(v0.x + v2.x, v0.y + v2.y);
                float2 a1 = make_float2(v0.x - v2.x, v0.y - v2.y);
                float2 a2 = make_float2(v1.x + v3.x, v1.y + v3.y);
                float2 d = make_float2(v1.x - v3.x, v1.y - v3.y);
                float2 a3 = make_float2(d.y, -d.x);          // -i * (v1 - v3)
                const int dst = (j / Ns) * Ns * 4 + k;
                b[dst] = make_float2(a0.x + a2.x, a0.y + a2.y);
                b[dst + Ns] = make_float2(a1.x + a3.x, a1.y + a3.y);
                b[dst + 2 * Ns] = make_float2(a0.x - a2.x, a0.y - a2.y);
                b[dst + 3 * Ns] = make_float2(a1.x - a3.x, a1.y - a3.y);
            }
            __syncwarp();
            float2* t = a; a = b; b = t;
        }
        // unpack the real spectrum, power of the bins the filterbank reads
        for (int k = lane; k < kmax; k += 32) {
            float pw;
            if (k == 256) {
                const float x = a[0].x - a[0].y;
                pw = __fmul_rn(x, x);
            } else {
                const float2 zk = a[k & 255];
                const float2 zc = a[(256 - k) & 255];
                const float2 xe = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y - zc.y));
                const float2 dd = make_float2(zk.x - zc.x, zk.y + zc.y);   // Zk - conj(Zc')
                const float2 xo = make_float2(0.5f * dd.y, -0.5f * dd.x);  // -i/2 * dd
                const float2 t2 = cmul(s_tw[k], xo);
                const float re = __fadd_rn(xe.x, t2.x), im = __fadd_rn(xe.y, t2.y);
                pw = __fmaf_rn(re, re, __fmul_rn(im, im));
            }
            pw_buf[k] = pw;
        }
        __syncwarp();
        float acc = 0.f;
        for (int i = 0; i < my_len; ++i) acc = fmaf(pw_buf[my_start + i], my_w[i], acc);
        const float db = 10.0f * logf(fmaxf(acc, 1e-10f)) / logf(10.0f);
    return db;
}

// Same arithmetic as mel_frame_db for NF frames at once: the NF instruction streams are interleaved stage by stage, so
// a lone warp (the fused step kernel runs only 16 of them per SM) has NF independent dependency chains in flight.
// Frame i: clip pointers tail[i]/body[i], frame index f[i], work buffers bufs + i*kMelFrameScratch bytes laid out as
// a[256] float2 | b[256] float2; the bin powers pw[<= 257] reuse b, which is free once the last FFT pass has read it.
// db[i] receives this lane's dB value.
// Index swizzle of the FFT work buffers in mel_frames_db: the radix-4 Stockham stores of the first two passes are strided by
// 4 and 16 elements (8- and 4-way bank conflicts on 8-byte elements); XOR-ing bits 4..5 of the index into bits 0..1 and 2..3
// makes every access pattern of the four passes conflict-free per half-warp.  Pure layout: the arithmetic is unchanged.
#ifndef OWW_FFT_SWZ
#define OWW_FFT_SWZ 1
#endif
__device__ __forceinline__ int fswz(int e) {
#if OWW_FFT_SWZ
    return e ^ (((e >> 4) & 3) * 5);
#else
    return e;
#endif
}

constexpr int kMelFrameScratch = 2048 + 2048;
template <int NF>
__device__ __forceinline__ void mel_frames_db(const int16_t* const* tail, int prefix, const int16_t* const* body, const int* f,
                                              uint8_t* bufs, const float2* s_tw, const float* s_win, int kmax, int my_start,
                                              int my_len, const float* my_w, int lane, float* db, long long* stamps = nullptr) {
    float2* a[NF]; float2* b[NF]; float* pw[NF];
    if (stamps && lane == 0) stamps[0] = clock64();
#pragma unroll
    for (int i = 0; i < NF; ++i) {
        a[i] = reinterpret_cast<float2*>(bufs + i * kMelFrameScratch);
        b[i] = a[i] + 256;
        pw[i] = reinterpret_cast<float*>(b[i]);            // four passes (even): the spectrum ends in a, b is free
    }
    // sample pairs (x[2n], x[2n+1]) never straddle the tail / body boundary (s0 and prefix are even), so each pair is one
    // 32-bit load when the clip is 4-byte aligned (it is for every contiguous int16 batch); all 8 x NF loads are in flight
    // before the first use
    bool al[NF];
#pragma unroll
    for (int i = 0; i < NF; ++i) al[i] = (((size_t)body[i] | (size_t)tail[i]) & 3) == 0 && (prefix & 1) == 0;
    uint32_t raw[8][NF];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int n = lane + 32 * j;
#pragma unroll
        for (int i = 0; i < NF; ++i) {
            const int s0 = f[i] * OWW_HOP + 2 * n;
            if (al[i]) {
                raw[j][i] = s0 + 1 < prefix ? *reinterpret_cast<const uint32_t*>(tail[i] + s0)
                                            : __ldg(reinterpret_cast<const uint32_t*>(body[i] + (s0 - prefix)));
            } else {
                unsigned short u0, u1;
                if (s0 + 1 < prefix) { u0 = (unsigned short)tail[i][s0]; u1 = (unsigned short)tail[i][s0 + 1]; }
                else if (s0 >= prefix) { u0 = (unsigned short)__ldg(body[i] + (s0 - prefix)); u1 = (unsigned short)__ldg(body[i] + (s0 + 1 - prefix)); }
                else { u0 = (unsigned short)tail[i][s0]; u1 = (unsigned short)__ldg(body[i]); }
                raw[j][i] = (uint32_t)u0 | ((uint32_t)u1 << 16);
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int n = lane + 32 * j;
        const float2 wn = *reinterpret_cast<const float2*>(s_win + 2 * n);
#pragma unroll
        for (int i = 0; i < NF; ++i) {
            const float x0 = (float)(short)(raw[j][i] & 0xFFFFu), x1 = (float)(short)(raw[j][i] >> 16);
            a[i][fswz(n)] = make_float2(__fmul_rn(x0, wn.x), __fmul_rn(x1, wn.y));
        }
    }
    __syncwarp();
    if (stamps && lane == 0) stamps[1] = clock64();
#pragma unroll
    for (int Ns = 1; Ns < 256; Ns *= 4) {
        const int tstep = 128 / Ns;
        // k = j & (Ns - 1) does not depend on jj while Ns <= 32: one set of twiddles per pass; in the first pass they are 1
        // (cmul by (1, 0) returns its argument bit for bit, so skipping it changes nothing)
        float2 t1 = make_float2(1.f, 0.f), t2 = t1, t3 = t1;
        if (Ns > 1 && Ns <= 32) { const int k = lane & (Ns - 1); t1 = s_tw[k * tstep]; t2 = s_tw[2 * k * tstep]; t3 = s_tw[3 * k * tstep]; }
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
            const int j = lane + 32 * jj;
            const int k = j & (Ns - 1);
            if (Ns > 32) { t1 = s_tw[k * tstep]; t2 = s_tw[2 * k * tstep]; t3 = s_tw[3 * k * tstep]; }
            const int dst = (j / Ns) * Ns * 4 + k;
            // the swizzle only touches bits 0..3 and reads bits 4..5: adding multiples of 64 commutes with it
            const int sj = fswz(j);
            const int d0 = fswz(dst), d1 = fswz(dst + Ns), d2 = fswz(dst + 2 * Ns), d3 = fswz(dst + 3 * Ns);
#pragma unroll
            for (int i = 0; i < NF; ++i) {
                const float2 v0 = a[i][sj];
                float2 v1 = a[i][sj + 64], v2 = a[i][sj + 128], v3 = a[i][sj + 192];
                if (Ns > 1) { v1 = cmul(v1, t1); v2 = cmul(v2, t2); v3 = cmul(v3, t3); }
                float2 a0 = make_float2(v0.x + v2.x, v0.y + v2.y);
                float2 a1 = make_float2(v0.x - v2.x, v0.y - v2.y);
                float2 a2 = make_float2(v1.x + v3.x, v1.y + v3.y);
                float2 d = make_float2(v1.x - v3.x, v1.y - v3.y);
                float2 a3 = make_float2(d.y, -d.x);
                b[i][d0] = make_float2(a0.x + a2.x, a0.y + a2.y);
                b[i][d1] = make_float2(a1.x + a3.x, a1.y + a3.y);
                b[i][d2] = make_float2(a0.x - a2.x, a0.y - a2.y);
                b[i][d3] = make_float2(a1.x - a3.x, a1.y - a3.y);
            }
        }
        __syncwarp();
#pragma unroll
        for (int i = 0; i < NF; ++i) { float2* t = a[i]; a[i] = b[i]; b[i] = t; }
    }
    if (stamps && lane == 0) stamps[2] = clock64();
    for (int k = lane; k < kmax; k += 32) {
#pragma unroll
        for (int i = 0; i < NF; ++i) {
            float p;
            if (k == 256) {
                const float x = a[i][fswz(0)].x - a[i][fswz(0)].y;
                p = __fmul_rn(x, x);
            } else {
                const float2 zk = a[i][fswz(k & 255)];
                const float2 zc = a[i][fswz((256 - k) & 255)];
                const float2 xe = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y - zc.y));
                const float2 dd = make_float2(zk.x - zc.x, zk.y + zc.y);
                const float2 xo = make_float2(0.5f * dd.y, -0.5f * dd.x);
                const float2 t2 = cmul(s_tw[k], xo);
                const float re = __fadd_rn(xe.x, t2.x), im = __fadd_rn(xe.y, t2.y);
                p = __fmaf_rn(re, re, __fmul_rn(im, im));
            }
            pw[i][k] = p;
        }
    }
    __syncwarp();
    if (stamps && lane == 0) stamps[3] = clock64();
    float acc[NF];
#pragma unroll
    for (int i = 0; i < NF; ++i) acc[i] = 0.f;
    // four filter taps per trip: one 16-byte weight load (rows of the table are 128 bytes), the FMA order stays q = 0, 1, 2 ...
    for (int q = 0; q < my_len; q += 4) {
        const float4 w4 = __ldg(reinterpret_cast<const float4*>(my_w + q));
        const float w[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
        for (int e = 0; e < 4; ++e)
            if (q + e < my_len) {
#pragma unroll
                for (int i = 0; i < NF; ++i) acc[i] = fmaf(pw[i][my_start + q + e], w[e], acc[i]);
            }
    }
#pragma unroll
    for (int i = 0; i < NF; ++i) db[i] = 10.0f * logf(fmaxf(acc[i], 1e-10f)) / logf(10.0f);
    __syncwarp();
    if (stamps && lane == 0) stamps[4] = clock64();
}

}  // namespace
