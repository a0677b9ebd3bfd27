// K3: wake-word classifier heads, one CTA per (tile of 32 streams, head).
//
// Replaces the per-head onnxruntime sessions of the reference
// (openwakeword/model.py:137-138,153-159,287-302) for the DNN family of
// openwakeword/train.py:56-83,144-165: Flatten([n_in,96]) -> Linear -> [LayerNorm]
// -> ReLU -> n x (Linear -> [LayerNorm] -> ReLU) -> Linear -> Sigmoid | (ReLU+)Softmax.
// The input window is gathered straight from the per-stream feature ring (AudioFeatures.get_features,
// utils.py:454-460), so predict() needs no host copy of the embeddings.  All loaded heads run in the
// same launch (blockIdx.y = head), each reading the same ring rows - "one embedding, every head".
#include "oww_internal.h"

namespace {

constexpr int KC = 96;          // K chunk of the first (wide) layer = one 96-wide feature row
constexpr int NTHREADS = 256;
constexpr int HMAX = 256;       // widest hidden / output layer supported
constexpr int kMaxStages = 4;   // cp.async ring depth of the first layer: 2..4, chosen per launch to fit shared memory
constexpr int XS_LD = KC + 4;   // x tile row pitch (floats): 16-byte aligned rows, conflict-light

struct HeadsArgs {
    HeadDev head[16];
    FeatSrc src;
    int n; float* out; int out_stride; int combine_max;
    int dmax;                       // widest layer over the heads of this launch (power of two >= 32)
    int stages;                     // cp.async ring depth
};

__device__ __forceinline__ int next_pow2_32(int d) { int p = 32; while (p < d) p <<= 1; return p; }

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    const int sz = valid ? 16 : 0;                      // src-size 0 -> 16 bytes of zeros
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_dyn(int n) {       // wait until at most n groups are pending
    switch (n) {
        case 0: asm volatile("cp.async.wait_group 0;" ::: "memory"); break;
        case 1: asm volatile("cp.async.wait_group 1;" ::: "memory"); break;
        case 2: asm volatile("cp.async.wait_group 2;" ::: "memory"); break;
        default: asm volatile("cp.async.wait_group 3;" ::: "memory"); break;
    }
}

// First (wide) layer: out[tb][d] = b[d] + sum_k x[tb][k] W[k][d], K = n_in*96, x gathered from the feature ring.
// K is consumed in chunks of KC=32 through a kStages-deep cp.async ring (x tile + W tile per stage) so the
// global/L2 latency of chunk c+2 hides under the FMAs of chunk c.  Register tiling: the 256 threads are
// 4 K-slices x 64; a thread owns RPT = TB/4 rows x CPT = DP/16 columns and walks 8 of the chunk's 32 k values,
// so one broadcast x load + one vector W load feed RPT*CPT FMAs; the 4 slices are summed through hout at the end.
template <int TB, int DP>
__device__ __forceinline__ void dense_gather(const HeadDev& H, const FeatSrc& src, int s0, int n, float* xs_all,
                                             float* ws_all, int ws_stage, int kStages, float (*hout)[HMAX + 1]) {
    constexpr int CPT = DP / 16, RPT = TB / 4;
    const int tid = threadIdx.x, slice = tid >> 6, t = tid & 63, rq = t >> 4, cq = t & 15;
    const int D = H.dims[1], K = H.dims[0];
    const float* W = H.blob + H.w_off[0];
    const int n_chunks = K / KC;
    float acc[RPT][CPT];
#pragma unroll
    for (int i = 0; i < RPT; ++i)
#pragma unroll
        for (int j = 0; j < CPT; ++j) acc[i][j] = 0.f;
    auto issue = [&](int c) {
        if (c < n_chunks) {
            const int k0 = c * KC;
            const int frow = k0 / 96, fcol = k0 % 96;
            float* xs = xs_all + (c % kStages) * (TB * XS_LD);
            float* ws = ws_all + (c % kStages) * ws_stage;
            for (int q = tid; q < TB * (KC / 4); q += NTHREADS) {
                const int tb = q / (KC / 4), k4 = (q % (KC / 4)) * 4;
                const int s = s0 + tb;
                const float* g = src.base;
                bool ok = s < n;
                if (ok) {
                    if (src.count) {
                        const int r = src.count[s] - src.back - H.n_in + frow;
                        ok = r >= 0;
                        g = src.base + (int64_t)s * src.stride + (int64_t)(r & src.rows_mask) * 96 + fcol + k4;
                    } else {
                        g = src.base + (int64_t)s * src.stride + (int64_t)frow * 96 + fcol + k4;
                    }
                }
                cp_async16(xs + tb * XS_LD + k4, g, ok);
            }
            // W tile: [KC][DP] in smem; DP is a power of two so the item -> (row, column) split is shifts; columns
            // beyond the real width D are zero-filled by cp.async (src-size 0)
            constexpr int CQ = DP / 4;
            if ((D & 3) == 0) {
#pragma unroll
                for (int it = 0; it < (KC * CQ + NTHREADS - 1) / NTHREADS; ++it) {
                    const int q = tid + it * NTHREADS;
                    if (q < KC * CQ) {
                        const int kk = q / CQ, c4 = (q % CQ) * 4;
                        const bool ok = c4 < D;
                        cp_async16(ws + kk * DP + c4, W + (int64_t)(k0 + kk) * D + (ok ? c4 : 0), ok);
                    }
                }
            } else {                                   // odd widths: plain loads (visible after the next __syncthreads)
                for (int q = tid; q < KC * DP; q += NTHREADS) {
                    const int kk = q / DP, cc = q % DP;
                    ws[q] = cc < D ? __ldg(W + (int64_t)(k0 + kk) * D + cc) : 0.f;
                }
            }
        }
        cp_async_commit();
    };
    for (int c = 0; c < kStages - 1; ++c) issue(c);
    for (int c = 0; c < n_chunks; ++c) {
        cp_async_wait_dyn(kStages - 2);
        __syncthreads();                                   // chunk c landed for everyone; stage (c-1)%S is free
        issue(c + kStages - 1);
        const float* xs = xs_all + (c % kStages) * (TB * XS_LD);
        const float* ws = ws_all + (c % kStages) * ws_stage;
#pragma unroll
        for (int k8 = 0; k8 < KC / 4; ++k8) {
            const int kk = slice * (KC / 4) + k8;
            float wv[CPT];
#pragma unroll
            for (int j = 0; j < CPT; ++j) wv[j] = ws[kk * DP + cq * CPT + j];
#pragma unroll
            for (int i = 0; i < RPT; ++i) {
                const float x = xs[(rq * RPT + i) * XS_LD + kk];
#pragma unroll
                for (int j = 0; j < CPT; ++j) acc[i][j] = fmaf(x, wv[j], acc[i][j]);
            }
        }
    }
    cp_async_wait_dyn(0);
    __syncthreads();
    // sum the 4 K-slices in a fixed order (deterministic) through hout, slice 0 seeds with the bias
    const float* bias = H.blob + H.b_off[0];
    for (int sl = 0; sl < 4; ++sl) {
        if (slice == sl) {
#pragma unroll
            for (int i = 0; i < RPT; ++i)
#pragma unroll
                for (int j = 0; j < CPT; ++j) {
                    const int d = cq * CPT + j;
                    if (d < D) {
                        float* o = &hout[rq * RPT + i][d];
                        *o = (sl == 0 ? __ldg(bias + d) : *o) + acc[i][j];
                    }
                }
        }
        __syncthreads();
    }
}

template <int TB, int DP>
__device__ __forceinline__ void dense_smem(const float* __restrict__ W, int K, int D, const float (*hin)[HMAX + 1],
                                           float* acc) {
    constexpr int R = NTHREADS / DP, NR = TB / R;
    const int tid = threadIdx.x, d = tid % DP, rgrp = tid / DP;
#pragma unroll
    for (int i = 0; i < NR; ++i) acc[i] = 0.f;
    if (d < D) {
        for (int k = 0; k < K; ++k) {
            const float w = __ldg(W + (int64_t)k * D + d);
#pragma unroll
            for (int i = 0; i < NR; ++i) acc[i] = fmaf(hin[rgrp + R * i][k], w, acc[i]);
        }
    }
}

template <int TB, int DP>
__device__ __forceinline__ void store_acc(const float* acc, const float* bias, int D, float (*hout)[HMAX + 1]) {
    constexpr int R = NTHREADS / DP, NR = TB / R;
    const int tid = threadIdx.x, d = tid % DP, rgrp = tid / DP;
    if (d < D) {
        const float b = __ldg(bias + d);
#pragma unroll
        for (int i = 0; i < NR; ++i) hout[rgrp + R * i][d] = acc[i] + b;
    }
}

template <int TB>
__global__ void __launch_bounds__(NTHREADS) heads_kernel(HeadsArgs a) {
    extern __shared__ __align__(16) float smem_dyn[];
    const int kStages = a.stages;
    float* xs = smem_dyn;                                          // [stages][TB][XS_LD]
    float* ws = xs + kStages * TB * XS_LD;                         // [stages][KC][dmax]
    const int ws_stage = KC * a.dmax;
    float (*hA)[HMAX + 1] = reinterpret_cast<float (*)[HMAX + 1]>(ws + kStages * ws_stage);
    float (*hB)[HMAX + 1] = reinterpret_cast<float (*)[HMAX + 1]>(ws + kStages * ws_stage + TB * (HMAX + 1));
    const HeadDev& H = a.head[blockIdx.y];
    const int s0 = blockIdx.x * TB;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float acc[TB];

    float (*cur)[HMAX + 1] = hA;
    float (*nxt)[HMAX + 1] = hB;
    for (int l = 0; l < H.n_layers; ++l) {
        const int D = H.dims[l + 1], K = H.dims[l];
        const int DP = next_pow2_32(D);
        if (l == 0) {
            switch (DP) {
                case 32: dense_gather<TB, 32>(H, a.src, s0, a.n, xs, ws, ws_stage, kStages, cur); break;
                case 64: dense_gather<TB, 64>(H, a.src, s0, a.n, xs, ws, ws_stage, kStages, cur); break;
                case 128: dense_gather<TB, 128>(H, a.src, s0, a.n, xs, ws, ws_stage, kStages, cur); break;
                default:
                    if constexpr (TB <= 8) dense_gather<TB, 256>(H, a.src, s0, a.n, xs, ws, ws_stage, kStages, cur);
                    else __trap();                    // the host never launches 32-row tiles for layers wider than 128
                    break;
            }
        } else {
            const float* W = H.blob + H.w_off[l];
            switch (DP) {
                case 32: dense_smem<TB, 32>(W, K, D, cur, acc); store_acc<TB, 32>(acc, H.blob + H.b_off[l], D, nxt); break;
                case 64: dense_smem<TB, 64>(W, K, D, cur, acc); store_acc<TB, 64>(acc, H.blob + H.b_off[l], D, nxt); break;
                case 128: dense_smem<TB, 128>(W, K, D, cur, acc); store_acc<TB, 128>(acc, H.blob + H.b_off[l], D, nxt); break;
                default: dense_smem<TB, 256>(W, K, D, cur, acc); store_acc<TB, 256>(acc, H.blob + H.b_off[l], D, nxt); break;
            }
            float (*t)[HMAX + 1] = cur; cur = nxt; nxt = t;
        }
        __syncthreads();
        const bool last = l == H.n_layers - 1;
        if (!last) {
            // [LayerNorm] + ReLU, one warp per row
            for (int r = warp; r < TB; r += NTHREADS / 32) {
                if (H.layernorm) {
                    float sum = 0.f;
                    for (int d = lane; d < D; d += 32) sum += cur[r][d];
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
                    const float mu = sum / (float)D;
                    float sq = 0.f;
                    for (int d = lane; d < D; d += 32) { const float c = cur[r][d] - mu; sq = fmaf(c, c, sq); }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
                    const float rstd = 1.0f / sqrtf(sq / (float)D + 1e-5f);
                    const float* g = H.blob + H.g_off[l];
                    const float* hb = H.blob + H.h_off[l];
                    for (int d = lane; d < D; d += 32)
                        cur[r][d] = fmaxf((cur[r][d] - mu) * rstd * __ldg(g + d) + __ldg(hb + d), 0.f);
                } else {
                    for (int d = lane; d < D; d += 32) cur[r][d] = fmaxf(cur[r][d], 0.f);
                }
            }
            __syncthreads();
        }
    }
    // final activation + store: one thread per row
    const int n_out = H.dims[H.n_layers];
    if (tid < TB && s0 + tid < a.n) {
        float* row = cur[tid];
        if (H.final_act == 4) {
            for (int d = 0; d < n_out; ++d) row[d] = fmaxf(row[d], 0.f);
        } else if (H.final_act == 1) {
            for (int d = 0; d < n_out; ++d) row[d] = 1.0f / (1.0f + expf(-row[d]));
        } else if (H.final_act == 2 || H.final_act == 3) {
            float m = -INFINITY;
            for (int d = 0; d < n_out; ++d) {
                if (H.final_act == 3) row[d] = fmaxf(row[d], 0.f);
                m = fmaxf(m, row[d]);
            }
            float sum = 0.f;
            for (int d = 0; d < n_out; ++d) { row[d] = expf(row[d] - m); sum += row[d]; }
            for (int d = 0; d < n_out; ++d) row[d] = row[d] / sum;
        }
        float* o = a.out + (int64_t)(s0 + tid) * a.out_stride + H.col0;
        for (int d = 0; d < n_out; ++d) o[d] = a.combine_max ? fmaxf(o[d], row[d]) : row[d];
    }
}

}  // namespace

// head_id < 0: all heads (blockIdx.y = head), score columns at each head's col0 (+out_col0).
int oww_heads_launch(oww_ctx* ctx, int head_id, const FeatSrc& src, int n, float* d_out, int out_stride,
                     int out_col0, int combine_max, cudaStream_t s, uint32_t head_mask) {
    if (n <= 0) return OWW_OK;
    int sel[16], nh = 0;
    if (head_id >= 0) sel[nh++] = head_id;
    else {
        if (ctx->heads.size() > 16) return oww_fail(ctx, OWW_EUNSUPPORTED, "at most 16 heads per launch");
        for (int i = 0; i < (int)ctx->heads.size(); ++i) if (head_mask >> i & 1u) sel[nh++] = i;
    }
    if (nh == 0) return OWW_OK;
    if (src.steps > 0) return oww_fail(ctx, OWW_EUNSUPPORTED, "sliding feature windows need the tensor-core heads kernel");
    HeadsArgs a;
    for (int i = 0; i < nh; ++i) {
        const Head& h = ctx->heads[sel[i]];
        HeadDev& d = a.head[i];
        d.blob = h.d_blob;
        d.n_in = h.desc.n_in; d.n_layers = h.desc.n_layers; d.layernorm = h.desc.layernorm; d.final_act = h.desc.final_act;
        for (int l = 0; l <= h.desc.n_layers; ++l) d.dims[l] = h.desc.dims[l];
        for (int l = 0; l < h.desc.n_layers; ++l) {
            d.w_off[l] = (int)h.w_off[l]; d.b_off[l] = (int)h.b_off[l];
            d.g_off[l] = (int)h.g_off[l]; d.h_off[l] = (int)h.h_off[l];
        }
        d.col0 = (head_id < 0 ? h.col0 : 0) + out_col0;
    }
    a.src = src; a.n = n; a.out = d_out; a.out_stride = out_stride; a.combine_max = combine_max;
    int dmax = 4;
    for (int i = 0; i < nh; ++i)
        for (int l = 1; l <= a.head[i].n_layers; ++l) dmax = a.head[i].dims[l] > dmax ? a.head[i].dims[l] : dmax;
    { int p2 = 32; while (p2 < dmax) p2 <<= 1; dmax = p2; }   // the first layer pads its W tile to the power-of-two width
    a.dmax = dmax;
    // small batches: 8 samples per CTA so that the grid still covers the SMs; wide layers: register budget
    auto smem_of = [&](int tb, int st) { return sizeof(float) * (size_t)(st * tb * XS_LD + st * KC * dmax + 2 * tb * (HMAX + 1)); };
    const size_t kLimit = 224 * 1024;
    // 8 samples per CTA for small batches (grid covers the SMs) and whenever the 32-row tile does not fit
    bool small = (n + 31) / 32 * nh < 2 * ctx->sm_count || dmax > 128 || smem_of(32, 2) > kLimit;
    const int tb = small ? 8 : 32;
    int stages = kMaxStages;
    while (stages > 2 && smem_of(tb, stages) > kLimit) --stages;
    if (smem_of(tb, stages) > kLimit)
        return oww_fail(ctx, OWW_EUNSUPPORTED, "head layer width %d needs too much shared memory", dmax);
    a.stages = stages;
    if (!ctx->heads_attr_set) {      // the attribute is per (function, device): tracked per handle, not per process
        OWW_CUDA(ctx, cudaFuncSetAttribute(heads_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
        OWW_CUDA(ctx, cudaFuncSetAttribute(heads_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
        ctx->heads_attr_set = true;
    }
    if (small) {
        dim3 grid((n + 7) / 8, nh);
        heads_kernel<8><<<grid, NTHREADS, smem_of(8, stages), s>>>(a);
    } else {
        dim3 grid((n + 31) / 32, nh);
        heads_kernel<32><<<grid, NTHREADS, smem_of(32, stages), s>>>(a);
    }
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}
