// Later layers of a wake-word head on a 64-stream tile, shared by the tensor-core head kernels (heads_tc.cu, heads_grp.cu).
//
// One warpgroup holds the accumulators of a Linear layer for 64 streams in registers (wgmma fragment, tc_common.cuh).
// Per layer they are written to shared memory as fp32 rows (x 2^-s, + bias); thread r < 64 of the warpgroup
// then runs the row-wise part in heads.cu's fp32 arithmetic order ([LayerNorm], ReLU or the final activation) and
// writes the next GEMM's A tile as fp16 hi + lo in the no-swizzle K-major core-matrix order ([octet][64 rows][16 B]).
// The next layer's weights (packed [hi | lo][Kp/8][NP][8] by oww_heads_tc_pack) arrive in `w_next` from the CTA's
// producer warp; the three MMA terms per K step are hi*hi + lo*hi + hi*lo (n_terms = 1: hi*hi).
#pragma once
#include "tc_common.cuh"

namespace {

constexpr int kHmRows = 64;                          // streams per tile = wgmma M
constexpr int kHmAPlane = kHmRows * 16;              // bytes per k-octet plane of a 64-row A tile (LBO)
constexpr int kHmPitch = 129;                        // fp32 row pitch of the hidden-activation buffer (layers <= 128 wide)
constexpr int kHmHBytes = (kHmRows * kHmPitch * 4 + 127) & ~127;
constexpr int kHmABytes = 2 * 16 * kHmAPlane;        // next A tile: [hi | lo] x 16 octets (K <= 128)
constexpr int kHmPBytes = 3 * 128 * 4;               // bias | gamma | beta of the layer in hand
constexpr int kHmBufBytes = kHmHBytes + kHmABytes + kHmPBytes;   // per warpgroup

struct HmLayer { int K, D, Kp, NP; uint32_t w_off, w_bytes; float unscale; };     // packed weights of one Linear layer

// eight fp32 values -> one 16-byte unit of fp16 hi parts and one of lo parts
__device__ __forceinline__ void hm_split8(const float* x, uint4& hi, uint4& lo) {
    __half2 h[4], l[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const __half h0 = __float2half_rn(x[2 * e]), h1 = __float2half_rn(x[2 * e + 1]);
        h[e] = __halves2half2(h0, h1);
        l[e] = __floats2half2_rn(x[2 * e] - __half2float(h0), x[2 * e + 1] - __half2float(h1));
    }
    hi = *reinterpret_cast<uint4*>(h);
    lo = *reinterpret_cast<uint4*>(l);
}

// acc: this thread's fragment of layer 0's accumulators (n0 columns).  buf: this warpgroup's hbuf | A tile | parameters
// (kHmBufBytes); w_next: the later layers' weight slot (shared by the CTA's warpgroups); wn_full completes once per
// later layer (phase l - 1 for layer l); acc_done receives one arrival per warp after every later GEMM; bar: named
// barrier of this warpgroup.  o: this row's first output column (thread r < 64 of the warpgroup; nullptr = no output),
// combine_max: keep the maximum with what o holds.
__device__ __forceinline__ void hm_layers(float* acc, int n0, const HeadDev& H, const HmLayer* L, int n_terms, uint8_t* buf,
                                          uint32_t w_next, uint32_t wn_full, uint32_t acc_done, int bar, float* o, int combine_max) {
    const int tid = threadIdx.x & 127, wq = tid >> 5, lane = tid & 31, q = lane & 3;
    float* hbuf = reinterpret_cast<float*>(buf);
    uint8_t* a_next = buf + kHmHBytes;
    float* prm = reinterpret_cast<float*>(buf + kHmHBytes + kHmABytes);
    const int n_layers = H.n_layers;
    int ncols = n0;
    for (int l = 0; l < n_layers; ++l) {
        const int D = L[l].D;
        const float us = L[l].unscale;
        // the layer's bias [gamma, beta] -> shared memory (the previous layer's readers are past the last barrier)
        if (tid < D) {
            prm[tid] = __ldg(H.blob + H.b_off[l] + tid);
            if (H.layernorm && l < n_layers - 1) {
                prm[128 + tid] = __ldg(H.blob + H.g_off[l] + tid);
                prm[256 + tid] = __ldg(H.blob + H.h_off[l] + tid);
            }
        }
        named_bar_sync(bar, 128);
        // accumulators -> fp32 rows: exact 2^-s, bias
#pragma unroll
        for (int k = 0; k < 64; ++k) {
            const int j = k >> 2, i = (k >> 1) & 1, e = k & 1;
            const int col = 8 * j + 2 * q + e, row = 16 * wq + (lane >> 2) + 8 * i;
            if (8 * j < ncols && col < D) hbuf[row * kHmPitch + col] = fmaf(acc[k], us, prm[col]);
        }
        named_bar_sync(bar, 128);
        float* hrow = hbuf + tid * kHmPitch;
        if (l == n_layers - 1) {
            // final activation + store
            if (tid < kHmRows && o) {
                const int n_out = D;
                if (H.final_act == 4) {
                    for (int d = 0; d < n_out; ++d) hrow[d] = fmaxf(hrow[d], 0.f);
                } else if (H.final_act == 1) {
                    for (int d = 0; d < n_out; ++d) hrow[d] = 1.0f / (1.0f + expf(-hrow[d]));
                } else if (H.final_act == 2 || H.final_act == 3) {
                    float m = -INFINITY;
                    for (int d = 0; d < n_out; ++d) {
                        if (H.final_act == 3) hrow[d] = fmaxf(hrow[d], 0.f);
                        m = fmaxf(m, hrow[d]);
                    }
                    float sum = 0.f;
                    for (int d = 0; d < n_out; ++d) { hrow[d] = expf(hrow[d] - m); sum += hrow[d]; }
                    for (int d = 0; d < n_out; ++d) hrow[d] = hrow[d] / sum;
                }
                for (int d = 0; d < n_out; ++d) o[d] = combine_max ? fmaxf(o[d], hrow[d]) : hrow[d];
            }
            break;
        }
        // [LayerNorm] + ReLU in fp32 (same arithmetic as heads.cu), then the next GEMM's A tile as fp16 hi/lo
        const HmLayer& N = L[l + 1];
        if (tid < kHmRows) {
            float mu = 0.f, rstd = 1.f;
            if (H.layernorm) {
                float sum = 0.f;
                for (int d = 0; d < D; ++d) sum += hrow[d];
                mu = sum / (float)D;
                float sq = 0.f;
                for (int d = 0; d < D; ++d) { const float c = hrow[d] - mu; sq = fmaf(c, c, sq); }
                rstd = 1.0f / sqrtf(sq / (float)D + 1e-5f);
            }
            const float* g = prm + 128;
            const float* hb = prm + 256;
            for (int j = 0; j < N.Kp / 8; ++j) {
                float x[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const int d = j * 8 + e;
                    float v = 0.f;
                    if (d < D) {
                        v = hrow[d];
                        if (H.layernorm) v = (v - mu) * rstd * g[d] + hb[d];
                        v = fmaxf(v, 0.f);
                    }
                    x[e] = v;
                }
                uint4 hi, lo;
                hm_split8(x, hi, lo);
                *reinterpret_cast<uint4*>(a_next + j * kHmAPlane + tid * 16) = hi;
                if (n_terms >= 2) *reinterpret_cast<uint4*>(a_next + 16 * kHmAPlane + j * kHmAPlane + tid * 16) = lo;
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy stores -> visible to the tensor core
        named_bar_sync(bar, 128);
        // ---- layer l+1: D[64 x NP] = A[64 x Kp] * W[Kp x NP] ----
        mbar_wait(wn_full, (uint32_t)(l & 1));
        const uint32_t a_lo = smem_u32(a_next);
        const uint32_t a_unit[2] = {a_lo, a_lo + 16u * kHmAPlane};
        const uint32_t w_unit[2] = {w_next, w_next + N.w_bytes / 2};
        // N, the K steps and the term count as compile-time constants: one unrolled chain of MMAs
        wg_dispatch_n(N.NP, [&](auto nc) {
            dispatch_int<8, 4, 2, 6, 1, 3, 5, 7>(N.Kp / 16, [&](auto kc) {
                dispatch_int<3, 1>(n_terms, [&](auto tc) {
                    constexpr int NN = decltype(nc)::value, NK = decltype(kc)::value, NT = decltype(tc)::value;
                    float d[NN / 2];                                   // this chain's own registers (no aliasing with other N)
                    wg_fence();
#pragma unroll
                    for (int s = 0; s < NT * NK; ++s) {
                        const int t = s / NK, kq = s - t * NK;
                        const uint32_t au = a_unit[t == 1 ? 1 : 0], wu = w_unit[t == 2 ? 1 : 0];
                        const uint64_t ad = make_desc(au + (uint32_t)(2 * kq) * kHmAPlane, kHmAPlane, 128u);
                        const uint64_t bd = make_desc(wu + (uint32_t)(2 * kq * NN) * 16u, (uint32_t)NN * 16u, 128u);
                        wg_mma<NN>(d, ad, bd, s > 0);
                    }
                    wg_commit();
                    wg_wait_all();
#pragma unroll
                    for (int k = 0; k < NN / 2; ++k) acc[k] = d[k];
                });
            });
        });
        __syncwarp();
        if (lane == 0) mbar_arrive(acc_done);                          // the weight slot may be refilled
        ncols = N.NP;
    }
}

}  // namespace
