// K3 (tensor-core path, per head): the wake-word heads as a chain of wgmma GEMMs, one CTA per (64 samples, head).
// Streaming steps and bulk clips run heads_grp.cu (A operand from the fp16 mirror of the feature rings); this kernel
// serves stateless calls on caller-supplied features and the heads the mirror path does not cover.
//
// Same graphs as heads.cu (reference: <head>.onnx sessions, openwakeword/model.py:137-138,153-159,287-302 of the
// original project; family openwakeword/train.py:56-83,144-165).  heads.cu tiles 8 or 32 streams per CTA and runs every
// layer on CUDA cores.  Here a CTA owns 64 streams of one head and every Linear layer is an MMA:
//   layer 0:  D[64 x D1] (fp32, registers of one warpgroup) = sum over the n_in feature rows c of X_c[64 x 96] * W1_c[96 x D1]
//             X_c is gathered from the per-stream feature rings (fp32) by 8 converter warps, split into fp16 hi + lo
//             (x = hi + lo, |lo| <= ulp(hi)/2) and written to shared memory in the no-swizzle K-major core-matrix
//             order ([k-octet][64 rows][16 B]; LBO = 1024 B, SBO = 128 B); W1_c is pre-packed on the host as fp16
//             hi + lo of W * 2^s in the same order and arrives by one cp.async.bulk per feature row (3-stage ring).
//   layer l:  heads_mma.cuh: the accumulators get the exact 2^-s, the bias, [LayerNorm] and ReLU in fp32, are split into
//             hi + lo again and become the A tile of the next GEMM (W_l pre-packed the same way, one bulk copy per layer).
// Three MMA terms per K step (hi*hi + lo*hi + hi*lo, fp32 accumulate) reproduce the fp32 product to ~2^-21 relative, so
// the scores stay within a few 1e-5 of heads.cu / the oracle; n_terms = 1 is plain fp16 operands.  Sigmoid / softmax /
// relu of the last layer and the store (with the max over chunk windows of a multi-chunk call) finish the CTA.
// Warp roles: 0-3 MMA warpgroup + epilogue, 4 = weight producer, 5-12 converters.  Heads are launched heaviest first
// (blockIdx.y) so the long CTAs do not form the tail.
#include "oww_internal.h"
#include "heads_mma.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace {

constexpr int kHtWorkers = 8;                        // converter warps
constexpr int kHtProducer = 4;                       // warp index of the weight producer
constexpr int kHtThreads = (kHtProducer + 1 + kHtWorkers) * 32;   // 416
constexpr int kHtTile = kHmRows;                     // streams per CTA = MMA M
constexpr int kHtMaxStages = 3;
constexpr int kHtAPlane = kHmAPlane;                 // bytes per k-octet plane of an A tile (LBO)
constexpr int kHtABytes = 12 * kHtAPlane;            // one 64 x 96 fp16 tile: 12 KB
constexpr int kHtSmem = 227 * 1024;

// one lane polls, the warp follows
__device__ __forceinline__ void ht_warp_wait(uint32_t bar, uint32_t parity, int lane) {
    if (lane == 0) mbar_wait(bar, parity);
    __syncwarp();
}

using HtLayer = HmLayer;
struct HtHead {
    HeadDev dev;                    // fp32 blob: biases, LayerNorm parameters
    const uint8_t* w;               // packed fp16 hi/lo weights of every layer
    HtLayer L[OWW_MAX_HEAD_LAYERS];
};
struct HeadsTcArgs {
    HtHead head[16];
    FeatSrc src;
    int n; float* out; int out_stride; int combine_max;
    int n_terms;                  // 1: hi*hi   3: + lo*hi + hi*lo (default)
    int stages, stage_bytes;
};

// Where sample s's window starts: row index r0 of feature row 0 (rows r0 + c, c = 0..n_in-1; negative = not available ->
// zeros), the row mask (ring) or -1 (linear), and the sample's base pointer.
struct HtRows { const float* base; int r0, mask; };
__device__ __forceinline__ HtRows ht_rows(const FeatSrc& src, int n_in, int s, int n) {
    HtRows w{nullptr, 0, -1};
    if (s >= n) return w;
    if (src.count) {                                       // per-stream ring
        w.base = src.base + (int64_t)s * src.stride;
        w.r0 = src.count[s] - src.back - n_in; w.mask = src.rows_mask;
    } else if (src.steps > 0) {                            // sliding windows over per-clip linear feature rows (bulk path)
        const int clip = s / src.steps, st = s - clip * src.steps;
        w.base = src.base + (int64_t)clip * src.stride;
        w.r0 = src.row0 + st + 1 - n_in;
    } else {                                               // linear [n][n_in][96]
        w.base = src.base + (int64_t)s * src.stride;
    }
    return w;
}

__global__ void __launch_bounds__(kHtThreads, 1) heads_tc_kernel(const __grid_constant__ HeadsTcArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    const HtHead& HH = a.head[blockIdx.y];
    const HeadDev& H = HH.dev;
    const int NP = HH.L[0].NP;
    const int n_in = H.n_in, n_layers = H.n_layers;
    const int s0 = blockIdx.x * kHtTile;
    const int S = a.stages;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem);
    uint8_t* stage0 = smem + 1024;
    // after the mainloop the stage ring is dead and is reused as: hidden activations fp32 | next A tile (hi, lo) | W slot
    uint8_t* w_next = stage0 + kHmBufBytes;                                  // [hi | lo] x [Kp/8][NP][16 B], <= 64 KB
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;
    const uint32_t bar0 = smem_u32(bars);
    auto a_full = [&](int s) { return bar0 + 8u * s; };
    auto w_full = [&](int s) { return bar0 + 8u * (kHtMaxStages + s); };
    auto empty = [&](int s) { return bar0 + 8u * (2 * kHtMaxStages + s); };
    const uint32_t acc_done = bar0 + 8u * (3 * kHtMaxStages);          // a GEMM's operands have been read (one arrival per MMA warp)
    const uint32_t wn_full = acc_done + 8u;                            // next layer's weights landed

    if (threadIdx.x == 0) {
        for (int s = 0; s < kHtMaxStages; ++s) { mbar_init(a_full(s), kHtWorkers); mbar_init(w_full(s), 1); mbar_init(empty(s), 4); }
        mbar_init(acc_done, 4);
        mbar_init(wn_full, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t w_term_bytes = 12u * (uint32_t)NP * 16u;

    if (warp == kHtProducer) {
        // ===================== weight producer =====================
        if (lane == 0) {
            const uint32_t bytes = w_term_bytes * (a.n_terms >= 3 ? 2u : 1u);
            for (int c = 0; c < n_in; ++c) {                         // layer 0: one bulk copy per feature row
                const int s = c % S;
                mbar_wait(empty(s), (((uint32_t)(c / S)) & 1u) ^ 1u);
                mbar_expect_tx(w_full(s), bytes);
                bulk_g2s(smem_u32(stage0 + s * a.stage_bytes + 2 * kHtABytes), HH.w + (size_t)c * 2u * w_term_bytes, bytes, w_full(s));
            }
            for (int l = 1; l < n_layers; ++l) {                     // later layers: the whole matrix, once the slot is free
                mbar_wait(acc_done, (uint32_t)((l - 1) & 1));        // layer l-1's MMAs are done: ring / previous W dead
                const uint32_t wb = a.n_terms >= 3 ? HH.L[l].w_bytes : HH.L[l].w_bytes / 2;
                mbar_expect_tx(wn_full, wb);
                bulk_g2s(smem_u32(w_next), HH.w + HH.L[l].w_off, wb, wn_full);
            }
        }
    } else if (warp < 4) {
        // ===================== MMA warpgroup: layer 0 mainloop, then the later layers and the store =====================
        float acc[64];
        // N and the term count as compile-time constants: one unrolled chain of MMAs per feature row
        wg_dispatch_n(NP, [&](auto nc) { dispatch_int<3, 1>(a.n_terms, [&](auto tc) {
            constexpr int NN = decltype(nc)::value, NT = decltype(tc)::value;
            float d[NN / 2];                                             // this chain's own registers (no aliasing with other N)
            for (int c = 0; c < n_in; ++c) {
                const int s = c % S;
                const uint32_t par = ((uint32_t)(c / S)) & 1u;
                ht_warp_wait(a_full(s), par, lane);
                ht_warp_wait(w_full(s), par, lane);
                const uint32_t st_addr = smem_u32(stage0 + s * a.stage_bytes);
                wg_fence();
#pragma unroll
                for (int k = 0; k < NT * 6; ++k) {
                    const int t = k / 6, q = k - t * 6;
                    const uint32_t au = st_addr + (t == 1 ? (uint32_t)kHtABytes : 0u);                       // term 1 = x_lo * w_hi
                    const uint32_t wu = st_addr + 2 * kHtABytes + (t == 2 ? w_term_bytes : 0u);             // term 2 = x_hi * w_lo
                    const uint64_t ad = make_desc(au + (uint32_t)(2 * q) * kHtAPlane, kHtAPlane, 128u);
                    const uint64_t bd = make_desc(wu + (uint32_t)(2 * q * NN) * 16u, (uint32_t)NN * 16u, 128u);
                    wg_mma<NN>(d, ad, bd, (c | k) != 0);
                }
                wg_commit();
                wg_wait_all();
                __syncwarp();
                if (lane == 0) mbar_arrive(empty(s));                     // stage free once these MMAs have read it
            }
#pragma unroll
            for (int k = 0; k < NN / 2; ++k) acc[k] = d[k];
        }); });
        __syncwarp();
        if (lane == 0) mbar_arrive(acc_done);
        const int r = threadIdx.x;
        float* o = (r < kHtTile && s0 + r < a.n) ? a.out + (int64_t)(s0 + r) * a.out_stride + H.col0 : nullptr;
        // the ring is dead once every stage has been consumed by the MMAs above (all of this warpgroup's)
        named_bar_sync(1, 128);
        hm_layers(acc, NP, H, HH.L, a.n_terms, stage0, smem_u32(w_next), wn_full, acc_done, 1, o, a.combine_max);
    } else {
        // ===================== converters: fp32 ring rows -> fp16 hi/lo A tiles =====================
        // thread = (row 8*w + lane%8, octet quad lane/8): three octets (32 B of fp32 each) per feature row
        const int row = 8 * (warp - kHtProducer - 1) + (lane & 7), jq = lane >> 3;
        const int s = s0 + row;
        float4 buf[2][6];
        const HtRows rows_of = ht_rows(a.src, n_in, s, a.n);
        auto load = [&](int c, float4* v) {
            const float* p = nullptr;
            if (c < n_in && rows_of.base) {
                const int r = rows_of.r0 + c;
                if (r >= 0) p = rows_of.base + (int64_t)(rows_of.mask >= 0 ? (r & rows_of.mask) : r) * 96;
            }
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                if (p) {
                    const float4* q = reinterpret_cast<const float4*>(p + (4 * i + jq) * 8);
                    v[2 * i] = __ldcg(q); v[2 * i + 1] = __ldcg(q + 1);
                } else {
                    v[2 * i] = make_float4(0.f, 0.f, 0.f, 0.f); v[2 * i + 1] = v[2 * i];
                }
            }
        };
        auto convert_store = [&](int c, const float4* v) {
            const int st = c % S;
            ht_warp_wait(empty(st), (((uint32_t)(c / S)) & 1u) ^ 1u, lane);
            uint8_t* A = stage0 + st * a.stage_bytes;
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                const float x[8] = {v[2 * i].x, v[2 * i].y, v[2 * i].z, v[2 * i].w, v[2 * i + 1].x, v[2 * i + 1].y, v[2 * i + 1].z, v[2 * i + 1].w};
                uint4 hi, lo;
                hm_split8(x, hi, lo);
                const int off = (4 * i + jq) * kHtAPlane + row * 16;
                *reinterpret_cast<uint4*>(A + off) = hi;
                if (a.n_terms >= 2) *reinterpret_cast<uint4*>(A + kHtABytes + off) = lo;
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy stores -> visible to the tensor core
            __syncwarp();
            if (lane == 0) mbar_arrive(a_full(st));
        };
        load(0, buf[0]);
        load(1, buf[1]);
        for (int c = 0; c < n_in; c += 2) {
            convert_store(c, buf[0]);
            load(c + 2, buf[0]);
            if (c + 1 < n_in) {
                convert_store(c + 1, buf[1]);
                load(c + 3, buf[1]);
            }
        }
    }
}

// exponent s with amax * 2^s in [2^13, 2^14): the fp16 lo parts of W * 2^s stay in the normal range
int scale_exponent(const float* w, size_t n) {
    float amax = 0.f;
    for (size_t i = 0; i < n; ++i) amax = std::fmax(amax, std::fabs(w[i]));
    if (!(amax > 0.f) || !std::isfinite(amax)) return 0;
    int e;
    std::frexp(amax, &e);                                          // amax = m * 2^e, m in [0.5, 1)
    return std::min(24, std::max(-8, 14 - e));
}

// fp16 hi/lo of rows [k0, k0 + Kp) of w[K][D] * 2^s in K-major core-matrix order: [term][octet Kp/8][NP][8]
void pack_block(const float* w, int K, int D, int k0, int Kp, int NP, float sc, __half* out) {
    const size_t term = (size_t)(Kp / 8) * NP * 8;
    for (int j = 0; j < Kp / 8; ++j)
        for (int n = 0; n < NP; ++n)
            for (int e = 0; e < 8; ++e) {
                const int k = k0 + j * 8 + e;
                const float v = (k < K && n < D) ? w[(size_t)k * D + n] * sc : 0.f;
                const __half hi = __float2half_rn(v);
                const size_t at = ((size_t)j * NP + n) * 8 + e;
                out[at] = hi;
                out[at + term] = __float2half_rn(v - __half2float(hi));
            }
}

}  // namespace

// Host side: pack every Linear layer of a head for the tensor-core kernel (layer 0 in blocks of one feature row).
int oww_heads_tc_pack(oww_ctx* ctx, Head& h, const float* blob /* staging in device layout: tensors at h.w_off[] */) {
    const int n_in = h.desc.n_in, nl = h.desc.n_layers;
    h.tc_ok = false;
    for (int l = 1; l <= nl; ++l) if (h.desc.dims[l] > 128) return OWW_OK;     // hidden buffers / register accumulators are 128 wide
    std::vector<__half> packed;
    h.tc_layers.assign(nl, Head::TcLayer{});
    for (int l = 0; l < nl; ++l) {
        const int K = h.desc.dims[l], D = h.desc.dims[l + 1];
        Head::TcLayer& T = h.tc_layers[l];
        T.K = K; T.D = D; T.NP = (D + 15) & ~15;
        T.Kp = l == 0 ? 96 : (K + 15) & ~15;
        const float* w = blob + h.w_off[l];
        const int s = scale_exponent(w, (size_t)K * D);
        const float sc = std::ldexp(1.0f, s);
        T.unscale = std::ldexp(1.0f, -s);
        T.w_off = (uint32_t)(packed.size() * sizeof(__half));
        const int n_blocks = l == 0 ? n_in : 1;
        const size_t per = (size_t)2 * (T.Kp / 8) * T.NP * 8;          // halves per block (hi + lo)
        packed.resize(packed.size() + (size_t)n_blocks * per);
        __half* base = packed.data() + T.w_off / sizeof(__half);
        for (int c = 0; c < n_blocks; ++c) pack_block(w, K, D, c * T.Kp, T.Kp, T.NP, sc, base + (size_t)c * per);
        T.w_bytes = (uint32_t)(n_blocks * per * sizeof(__half));
        while (packed.size() % 64) packed.push_back(__float2half(0.f));    // 128-byte aligned blocks for the bulk copies
    }
    cudaFree(h.d_w1_tc); h.d_w1_tc = nullptr;
    OWW_CUDA(ctx, cudaMalloc(&h.d_w1_tc, packed.size() * sizeof(__half)));
    OWW_CUDA(ctx, cudaMemcpy(h.d_w1_tc, packed.data(), packed.size() * sizeof(__half), cudaMemcpyHostToDevice));
    h.tc_w0_host.assign(blob + h.w_off[0], blob + h.w_off[0] + (size_t)h.desc.dims[0] * h.desc.dims[1]);
    h.tc_ok = true;
    return OWW_OK;
}

bool oww_heads_tc_supported(const oww_ctx* ctx, int head_id) {
    if (!ctx->tc_heads || ctx->cfg.cnn_mode == OWW_CNN_FP32_WINDOW) return false;     // mode 0 stays fp32 end to end
    return head_id >= 0 && head_id < (int)ctx->heads.size() && ctx->heads[head_id].tc_ok;
}

// Every head of the handle on the same samples: the tensor-core kernel for the heads it covers, heads.cu for the rest,
// then the conditional verifier pairs (applied to THIS call's scores, i.e. per chunk - model.py runs the whole gated
// graph per chunk and takes the max over chunks afterwards).
namespace {
__global__ void gate_kernel(float* scores, int n, int stride, const Gate* gates, int n_gates) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    oww_pdl_sync();
    if (i >= n * n_gates) return;
    const int s = i / n_gates;
    const Gate g = gates[i - s * n_gates];
    float* o = scores + (int64_t)s * stride;
    if (o[g.main_col] > g.thr) o[g.main_col] = o[g.ver_col];
}
__global__ void max_combine_kernel(float* dst, const float* src, int n, int cols, int dst_stride) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * cols) return;
    const int s = i / cols, c = i - s * cols;
    float* d = dst + (int64_t)s * dst_stride + c;
    *d = fmaxf(*d, src[i]);
}
}  // namespace

int oww_heads_all(oww_ctx* ctx, const FeatSrc& src, int n, float* d_out, int out_stride, int combine_max, cudaStream_t s) {
    if (ctx->heads.empty() || n <= 0) return OWW_OK;
    uint32_t tc_mask = 0, cc_mask = 0;
    for (int i = 0; i < (int)ctx->heads.size(); ++i) {
        if (oww_heads_tc_supported(ctx, i)) tc_mask |= 1u << i; else cc_mask |= 1u << i;
    }
    float* out = d_out; int stride = out_stride; int comb = combine_max;
    const bool via_tmp = combine_max && !ctx->gates.empty();       // gate this chunk's raw scores before the max
    if (via_tmp) {
        const size_t need = (size_t)n * ctx->n_out_total;
        if (ctx->scores_tmp_floats < need) {
            cudaFree(ctx->d_scores_tmp); ctx->d_scores_tmp = nullptr; ctx->scores_tmp_floats = 0;
            OWW_CUDA(ctx, cudaMalloc(&ctx->d_scores_tmp, need * sizeof(float)));
            ctx->scores_tmp_floats = need;
        }
        out = ctx->d_scores_tmp; stride = ctx->n_out_total; comb = 0;
    }
    int rc;
    // streaming ring of the handle: the heads the groups cover run in one CTA per 128 streams (heads_grp.cu)
    if (src.count && src.base == ctx->d_feat_ring && n == ctx->n_streams) {
        const uint32_t grp_mask = oww_heads_grp_covered(ctx) & tc_mask;
        if (grp_mask) {
            if ((rc = oww_heads_grp_launch(ctx, src.back, n, out, stride, comb, s))) return rc;
            tc_mask &= ~grp_mask;
        }
    }
    if (!src.count && src.steps > 0 && !combine_max) {     // bulk clips: every sliding window of every clip, same kernel
        const uint32_t grp_mask = oww_heads_grp_bulk(ctx, src, n, out, stride, s, &rc) & tc_mask;
        if (rc) return rc;
        tc_mask &= ~grp_mask;
    }
    if (tc_mask && (rc = oww_heads_tc_launch(ctx, -1, src, n, out, stride, 0, comb, s, tc_mask))) return rc;
    if (cc_mask && (rc = oww_heads_launch(ctx, -1, src, n, out, stride, 0, comb, s, cc_mask))) return rc;
    if (!ctx->gates.empty()) {
        const int total = n * (int)ctx->gates.size();
        OWW_CUDA(ctx, oww_launch_pdl(ctx->late_pdl, gate_kernel, dim3((total + 255) / 256), dim3(256), 0, s, out, n, stride,
                                     (const Gate*)ctx->d_gates, (int)ctx->gates.size()));
        OWW_LAUNCH_CHECK(ctx);
    }
    if (via_tmp) {
        const int total = n * ctx->n_out_total;
        max_combine_kernel<<<(total + 255) / 256, 256, 0, s>>>(d_out, ctx->d_scores_tmp, n, ctx->n_out_total, out_stride);
        OWW_LAUNCH_CHECK(ctx);
    }
    return OWW_OK;
}

// Same contract as oww_heads_launch (heads.cu).
int oww_heads_tc_launch(oww_ctx* ctx, int head_id, const FeatSrc& src, int n, float* d_out, int out_stride,
                        int out_col0, int combine_max, cudaStream_t s, uint32_t head_mask) {
    if (n <= 0) return OWW_OK;
    int sel[16], nh = 0;
    if (head_id >= 0) sel[nh++] = head_id;
    else {
        if (ctx->heads.size() > 16) return oww_fail(ctx, OWW_EUNSUPPORTED, "at most 16 heads per launch");
        for (int i = 0; i < (int)ctx->heads.size(); ++i) if (head_mask >> i & 1u) sel[nh++] = i;
    }
    if (nh == 0) return OWW_OK;
    // heaviest heads first: their CTAs start in the first wave instead of forming the tail
    std::sort(sel, sel + nh, [&](int x, int y) {
        const Head& p = ctx->heads[x]; const Head& q = ctx->heads[y];
        const int64_t wp = (int64_t)p.desc.n_in * p.desc.dims[1], wq = (int64_t)q.desc.n_in * q.desc.dims[1];
        return wp != wq ? wp > wq : x < y;
    });
    HeadsTcArgs a;
    std::memset(&a, 0, sizeof(a));
    int np_max = 16;
    for (int i = 0; i < nh; ++i) {
        const Head& h = ctx->heads[sel[i]];
        if (!h.tc_ok) return oww_fail(ctx, OWW_EUNSUPPORTED, "head %d has no tensor-core packing", sel[i]);
        HeadDev& d = a.head[i].dev;
        d.blob = h.d_blob;
        d.n_in = h.desc.n_in; d.n_layers = h.desc.n_layers; d.layernorm = h.desc.layernorm; d.final_act = h.desc.final_act;
        for (int l = 0; l <= h.desc.n_layers; ++l) d.dims[l] = h.desc.dims[l];
        for (int l = 0; l < h.desc.n_layers; ++l) {
            d.w_off[l] = (int)h.w_off[l]; d.b_off[l] = (int)h.b_off[l];
            d.g_off[l] = (int)h.g_off[l]; d.h_off[l] = (int)h.h_off[l];
            const Head::TcLayer& T = h.tc_layers[l];
            a.head[i].L[l] = HtLayer{T.K, T.D, T.Kp, T.NP, T.w_off, T.w_bytes, T.unscale};
        }
        d.col0 = (head_id < 0 ? h.col0 : 0) + out_col0;
        a.head[i].w = reinterpret_cast<const uint8_t*>(h.d_w1_tc);
        if (h.tc_layers[0].NP > np_max) np_max = h.tc_layers[0].NP;
    }
    a.src = src; a.n = n; a.out = d_out; a.out_stride = out_stride; a.combine_max = combine_max;
    a.n_terms = ctx->tc_heads_terms;
    a.stage_bytes = 2 * kHtABytes + 2 * 12 * np_max * 16;
    a.stages = (kHtSmem - 1024) / a.stage_bytes;
    if (a.stages > kHtMaxStages) a.stages = kHtMaxStages;
    if (a.stages < 2) return oww_fail(ctx, OWW_EUNSUPPORTED, "tensor-core heads: stage of %d bytes does not fit twice", a.stage_bytes);
    if (!ctx->heads_tc_attr_set) {
        OWW_CUDA(ctx, cudaFuncSetAttribute(heads_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kHtSmem));
        ctx->heads_tc_attr_set = true;
    }
    dim3 grid((n + kHtTile - 1) / kHtTile, nh);
    heads_tc_kernel<<<grid, kHtThreads, kHtSmem, s>>>(a);
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}
