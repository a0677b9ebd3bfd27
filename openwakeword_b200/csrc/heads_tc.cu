// K3 (tensor-core path, per head): the wake-word heads as a chain of wgmma GEMMs, one CTA per (64 samples, head).
// Streaming steps and bulk clips run heads_grp.cu (A operand from the fp16 mirror of the feature rings); this kernel
// serves stateless calls on caller-supplied features, the heads the mirror path does not cover and the per-stream head
// banks (heads_tc_kernel<true>: one CTA per work item of up to 64 streams that share a slot; bottom of this file).
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
    // head bank (heads_tc_kernel<true>): CTA i runs item items[i] = {slot, first, rows}, the streams perm[first ..
    // first + rows) with the head slots[slot]; slot -1 only stores zeros in the columns of head[0] (the bank's shape).
    // step != nullptr: streams with step[b] == 0 are not written.
    const int4* items; const int* perm; const HtHead* slots; const int* step;
};

template <bool kBank>
__global__ void __launch_bounds__(kHtThreads, 1) heads_tc_kernel(const __grid_constant__ HeadsTcArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    const HtHead* hp = &a.head[blockIdx.y];
    int s0 = blockIdx.x * kHtTile, n_rows = 0;
    if constexpr (kBank) {
        const int4 it = a.items[blockIdx.x];
        s0 = it.y; n_rows = it.z;
        if (it.x < 0) {
            const HeadDev& D0 = a.head[0].dev;
            const int n_out = D0.dims[D0.n_layers];
            for (int i = threadIdx.x; i < n_rows * n_out; i += blockDim.x) {
                const int r = i / n_out, b = a.perm[s0 + r];
                if (!a.step || a.step[b] != 0) a.out[(int64_t)b * a.out_stride + D0.col0 + (i - r * n_out)] = 0.f;
            }
            return;
        }
        hp = a.slots + it.x;
    }
    const HtHead& HH = *hp;
    const HeadDev& H = HH.dev;
    const int NP = HH.L[0].NP;
    const int n_in = H.n_in, n_layers = H.n_layers;
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
        float* o = nullptr;
        if constexpr (kBank) {
            const int b = r < n_rows ? a.perm[s0 + r] : -1;
            if (b >= 0 && (!a.step || a.step[b] != 0)) o = a.out + (int64_t)b * a.out_stride + H.col0;
        } else {
            o = (r < kHtTile && s0 + r < a.n) ? a.out + (int64_t)(s0 + r) * a.out_stride + H.col0 : nullptr;
        }
        // the ring is dead once every stage has been consumed by the MMAs above (all of this warpgroup's)
        named_bar_sync(1, 128);
        hm_layers(acc, NP, H, HH.L, a.n_terms, stage0, smem_u32(w_next), wn_full, acc_done, 1, o, a.combine_max);
    } else {
        // ===================== converters: fp32 ring rows -> fp16 hi/lo A tiles =====================
        // thread = (row 8*w + lane%8, octet quad lane/8): three octets (32 B of fp32 each) per feature row
        const int row = 8 * (warp - kHtProducer - 1) + (lane & 7), jq = lane >> 3;
        float4 buf[2][6];
        FeatRows rows_of{nullptr, 0, -1};
        if constexpr (kBank) {
            if (row < n_rows) rows_of = feat_rows(a.src, n_in, a.perm[s0 + row]);
        } else {
            const int s = s0 + row;
            if (s < a.n) rows_of = feat_rows(a.src, n_in, s);
        }
        auto load = [&](int c, float4* v) {
            const float* p = (c < n_in && rows_of.base) ? feat_row(rows_of, c) : nullptr;
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

// a head the tensor-core kernel covers: every Linear layer at most 128 wide (hidden buffers / register accumulators)
bool tc_covers(const oww_head_desc& d) {
    for (int l = 1; l <= d.n_layers; ++l) if (d.dims[l] > 128) return false;
    return true;
}

// pack every Linear layer of a head the kernel covers (layer 0 in blocks of one feature row) -> packed, h.tc_layers
void pack_layers(Head& h, const float* blob, std::vector<__half>& packed) {
    const int n_in = h.desc.n_in, nl = h.desc.n_layers;
    h.tc_layers.assign(nl, Head::TcLayer{});
    for (int l = 0; l < nl; ++l) {
        const int K = h.desc.dims[l], D = h.desc.dims[l + 1];
        Head::TcLayer& T = h.tc_layers[l];
        T.K = K; T.D = D; T.NP = (D + 15) & ~15;
        T.Kp = l == 0 ? 96 : (K + 15) & ~15;
        const float* w = blob + h.w_off[l];
        const int s = oww_weight_scale_exponent(w, (size_t)K * D);
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
}

}  // namespace

// Host side: pack every Linear layer of a head for the tensor-core kernel.
int oww_heads_tc_pack(oww_ctx* ctx, Head& h, const float* blob /* staging in device layout: tensors at h.w_off[] */) {
    h.tc_ok = false;
    if (!tc_covers(h.desc)) return OWW_OK;
    std::vector<__half> packed;
    pack_layers(h, blob, packed);
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

int oww_heads_all(oww_ctx* ctx, const FeatSrc& src, int n, float* d_out, int out_stride, int combine_max, cudaStream_t s,
                  const BankRows* bank_rows) {
    if (ctx->heads.empty() || n <= 0) {
        return n > 0 ? oww_head_banks_launch(ctx, src, n, d_out, out_stride, combine_max, s, nullptr, bank_rows) : OWW_OK;
    }
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
    if ((rc = oww_head_banks_launch(ctx, src, n, out, stride, comb, s, nullptr, bank_rows))) return rc;
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

// stage ring for first-layer tiles of up to np_max columns, then the launch
template <bool kBank>
static int ht_run(oww_ctx* ctx, HeadsTcArgs& a, int np_max, dim3 grid, cudaStream_t s) {
    a.n_terms = ctx->tc_heads_terms;
    a.stage_bytes = 2 * kHtABytes + 2 * 12 * np_max * 16;
    a.stages = (kHtSmem - 1024) / a.stage_bytes;
    if (a.stages > kHtMaxStages) a.stages = kHtMaxStages;
    if (a.stages < 2) return oww_fail(ctx, OWW_EUNSUPPORTED, "tensor-core heads: stage of %d bytes does not fit twice", a.stage_bytes);
    if (!ctx->heads_tc_attr_set) {
        OWW_CUDA(ctx, cudaFuncSetAttribute(heads_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kHtSmem));
        OWW_CUDA(ctx, cudaFuncSetAttribute(heads_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kHtSmem));
        ctx->heads_tc_attr_set = true;
    }
    heads_tc_kernel<kBank><<<grid, kHtThreads, kHtSmem, s>>>(a);
    OWW_LAUNCH_CHECK(ctx);
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
    return ht_run<false>(ctx, a, np_max, dim3((n + kHtTile - 1) / kHtTile, nh), s);
}

// ================================ head banks ================================
namespace {

// the kernel descriptor of slot k (its unscale factors: per layer, from that slot's weights)
HtHead bank_slot_head(const HeadBank& b, int k, const float* unscale) {
    HtHead t;
    std::memset(&t, 0, sizeof(t));
    const oww_head_desc& d = b.shape.desc;
    HeadDev& H = t.dev;
    H.blob = b.d_p + (size_t)k * b.p_floats;
    H.n_in = d.n_in; H.n_layers = d.n_layers; H.layernorm = d.layernorm; H.final_act = d.final_act;
    for (int l = 0; l <= d.n_layers; ++l) H.dims[l] = d.dims[l];
    for (int l = 0; l < d.n_layers; ++l) {
        H.b_off[l] = b.p_off[3 * l]; H.g_off[l] = b.p_off[3 * l + 1]; H.h_off[l] = b.p_off[3 * l + 2];
        const Head::TcLayer& T = b.shape.tc_layers[l];
        t.L[l] = HtLayer{T.K, T.D, T.Kp, T.NP, T.w_off, T.w_bytes, unscale ? unscale[l] : 1.f};
    }
    H.col0 = b.shape.col0;
    t.w = b.d_w + (size_t)k * b.w_bytes;
    return t;
}

const HtHead& host_slot(const HeadBank& b, int k) { return reinterpret_cast<const HtHead*>(b.h_slots.data())[k]; }

// items of at most kHtTile streams per slot, streams ordered by slot (-1 first) -> h[0 .. 4B) items, h[4B .. 5B) ids,
// h[5B .. 6B) the slot of each stream
int build_items(const std::vector<int>& assign, int* h) {
    const int B = (int)assign.size();
    int* perm = h + 4 * B;
    for (int b = 0; b < B; ++b) perm[b] = b;
    std::copy(assign.begin(), assign.end(), h + 5 * B);
    std::stable_sort(perm, perm + B, [&](int x, int y) { return assign[x] < assign[y]; });
    int n = 0;
    for (int i = 0; i < B;) {
        int j = i;
        while (j < B && assign[perm[j]] == assign[perm[i]] && j - i < kHtTile) ++j;
        h[4 * n] = assign[perm[i]]; h[4 * n + 1] = i; h[4 * n + 2] = j - i; h[4 * n + 3] = 0;
        ++n; i = j;
    }
    return n;
}

// upload the item table of b.assign on s through the pinned staging (the copy of the previous upload has run)
int upload_items(oww_ctx* ctx, HeadBank& b, cudaStream_t s) {
    const int B = (int)b.assign.size();
    OWW_CUDA(ctx, cudaEventSynchronize(b.stage_ev));
    b.n_items = build_items(b.assign, b.h_stage);
    OWW_CUDA(ctx, cudaMemcpyAsync(b.d_table, b.h_stage, (size_t)6 * B * sizeof(int), cudaMemcpyHostToDevice, s));
    OWW_CUDA(ctx, cudaEventRecord(b.stage_ev, s));
    return OWW_OK;
}

void bank_free_streams(HeadBank& b) {
    if (b.stage_ev) cudaEventSynchronize(b.stage_ev);
    cudaFree(b.d_table); cudaFreeHost(b.h_stage);
    b.d_table = nullptr; b.h_stage = nullptr; b.assign.clear(); b.n_items = 0;
}

int bank_alloc_streams(oww_ctx* ctx, HeadBank& b) {
    bank_free_streams(b);
    const int B = ctx->n_streams;
    if (B <= 0) return OWW_OK;
    if (!b.stage_ev) OWW_CUDA(ctx, cudaEventCreateWithFlags(&b.stage_ev, cudaEventDisableTiming));
    OWW_CUDA(ctx, cudaMalloc(&b.d_table, (size_t)6 * B * sizeof(int)));
    OWW_CUDA(ctx, cudaMallocHost(&b.h_stage, (size_t)6 * B * sizeof(int)));
    b.assign.assign(B, -1);
    int rc = upload_items(ctx, b, nullptr);
    if (rc) return rc;
    OWW_CUDA(ctx, cudaEventSynchronize(b.stage_ev));
    return OWW_OK;
}

int check_bank(oww_ctx* ctx, int bank) {
    if (!ctx) return OWW_EINVAL;
    if (bank < 0 || bank >= (int)ctx->head_banks.size()) return oww_fail(ctx, OWW_EINVAL, "bad head bank %d", bank);
    return OWW_OK;
}

int check_slot(oww_ctx* ctx, const HeadBank& b, int slot, bool none_ok) {
    if (none_ok && slot == -1) return OWW_OK;
    if (slot < 0 || slot >= b.capacity)
        return oww_fail(ctx, OWW_EINVAL, "slot %d outside [%d,%d)", slot, none_ok ? -1 : 0, b.capacity);
    if (!b.loaded[slot]) return oww_fail(ctx, OWW_EINVAL, "slot %d holds no head (oww_load_bank_head)", slot);
    return OWW_OK;
}

}  // namespace

int oww_head_banks_launch(oww_ctx* ctx, const FeatSrc& src, int n, float* d_out, int out_stride, int combine_max,
                          cudaStream_t s, const int* d_step, const BankRows* rows) {
    if (n <= 0) return OWW_OK;
    const bool streams = src.count && src.base == ctx->d_feat_ring && n == ctx->n_streams;
    for (size_t i = 0; i < ctx->head_banks.size(); ++i) {
        const HeadBank& b = ctx->head_banks[i];
        const int np = std::max(16, b.shape.tc_layers[0].NP);
        HeadsTcArgs a;
        std::memset(&a, 0, sizeof(a));
        a.src = src; a.n = n; a.out = d_out; a.out_stride = out_stride; a.combine_max = combine_max;
        int rc;
        if (streams) {
            // one CTA per item; head[0] carries the bank's columns for the items of unassigned streams
            a.head[0] = bank_slot_head(b, 0, nullptr);
            a.items = reinterpret_cast<const int4*>(b.d_table);
            a.perm = b.d_table + 4 * ctx->n_streams;
            a.slots = reinterpret_cast<const HtHead*>(b.d_slots);
            a.step = d_step;
            rc = ht_run<true>(ctx, a, np, dim3(b.n_items), s);
        } else if (rows) {                   // rows of the bulk path, each on the slot of its clip's stream
            a.head[0] = bank_slot_head(b, 0, nullptr);
            a.items = rows[i].items;
            a.perm = rows[i].perm;
            a.slots = reinterpret_cast<const HtHead*>(b.d_slots);
            rc = rows[i].n_items > 0 ? ht_run<true>(ctx, a, np, dim3(rows[i].n_items), s) : OWW_OK;
        } else if (b.clip_slot >= 0) {       // rows of the bulk path: every row on the clip slot
            a.head[0] = host_slot(b, b.clip_slot);
            rc = ht_run<false>(ctx, a, np, dim3((n + kHtTile - 1) / kHtTile), s);
        } else {
            OWW_CUDA(ctx, cudaMemset2DAsync(d_out + b.shape.col0, (size_t)out_stride * sizeof(float), 0,
                                            (size_t)b.shape.n_out * sizeof(float), n, s));
            rc = OWW_OK;
        }
        if (rc) return rc;
    }
    return OWW_OK;
}

const int* oww_head_bank_stream_slots(const oww_ctx* ctx, int bank) {
    const HeadBank& b = ctx->head_banks[bank];
    return b.d_table ? b.d_table + 5 * ctx->n_streams : nullptr;
}

int oww_head_banks_alloc_streams(oww_ctx* ctx) {
    for (HeadBank& b : ctx->head_banks) {
        int rc = bank_alloc_streams(ctx, b);
        if (rc) return rc;
    }
    return OWW_OK;
}

void oww_head_banks_free(oww_ctx* ctx) {
    for (HeadBank& b : ctx->head_banks) {
        bank_free_streams(b);
        if (b.stage_ev) cudaEventDestroy(b.stage_ev);
        cudaFree(b.d_w); cudaFree(b.d_p); cudaFree(b.d_slots);
    }
    ctx->head_banks.clear();
}

extern "C" {

int oww_add_head_bank(oww_ctx* ctx, const oww_head_desc* desc, int capacity, int* bank_id) {
    if (!ctx || !desc) return oww_fail(ctx, OWW_EINVAL, "null argument");
    int rc = oww_check_head_desc(ctx, desc);
    if (rc) return rc;
    if (ctx->cfg.cnn_mode == OWW_CNN_FP32_WINDOW)
        return oww_fail(ctx, OWW_EUNSUPPORTED, "head banks run on the tensor cores: not in cnn_mode 0");
    if (!tc_covers(*desc)) return oww_fail(ctx, OWW_EUNSUPPORTED, "head banks cover layers up to 128 wide");
    if (capacity < 1 || capacity > (1 << 20)) return oww_fail(ctx, OWW_EINVAL, "capacity %d outside [1, 2^20]", capacity);
    HeadBank b;
    b.capacity = capacity;
    // the packing layout from a zero blob of the shape (every slot's packing has the same layout)
    size_t n_floats = 0;
    for (int l = 0; l < desc->n_layers; ++l) {
        const size_t dout = (size_t)desc->dims[l + 1];
        n_floats += (size_t)desc->dims[l] * dout + dout + (desc->layernorm && l < desc->n_layers - 1 ? 2 * dout : 0);
    }
    {
        std::vector<float> zeros(n_floats, 0.f), staged;
        if ((rc = oww_stage_head(ctx, desc, zeros.data(), n_floats, b.shape, staged))) return rc;
        std::vector<__half> packed;
        pack_layers(b.shape, staged.data(), packed);
        b.w_bytes = packed.size() * sizeof(__half);
    }
    for (int l = 0; l < desc->n_layers; ++l) {     // bias | gamma | beta per layer, each on a 16-byte boundary
        const int D = desc->dims[l + 1], Dp = (D + 3) & ~3;
        const bool ln = desc->layernorm && l < desc->n_layers - 1;
        b.p_off.push_back((int)b.p_floats); b.p_floats += Dp;
        b.p_off.push_back(ln ? (int)b.p_floats : 0); b.p_floats += ln ? Dp : 0;
        b.p_off.push_back(ln ? (int)b.p_floats : 0); b.p_floats += ln ? Dp : 0;
    }
    b.shape.n_out = desc->dims[desc->n_layers];
    b.shape.col0 = ctx->n_out_total;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    auto fail = [&](cudaError_t e) {
        cudaFree(b.d_w); cudaFree(b.d_p); cudaFree(b.d_slots);
        return oww_fail(ctx, OWW_ENOMEM, "head bank of %d slots: %s", capacity, cudaGetErrorString(e));
    };
    cudaError_t e;
    if ((e = cudaMalloc(&b.d_w, (size_t)capacity * b.w_bytes)) != cudaSuccess) return fail(e);
    if ((e = cudaMalloc(&b.d_p, (size_t)capacity * b.p_floats * sizeof(float))) != cudaSuccess) return fail(e);
    if ((e = cudaMalloc(&b.d_slots, (size_t)capacity * sizeof(HtHead))) != cudaSuccess) return fail(e);
    for (auto& ev : ctx->ver_ev)     // orders oww_assign_bank_head with own_stream, as for the verifier banks
        if (!ev && (e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)) != cudaSuccess) return fail(e);
    b.h_slots.assign((size_t)capacity * sizeof(HtHead), 0);
    b.loaded.assign(capacity, 0);
    ctx->head_banks.push_back(b);
    ctx->n_out_total += b.shape.n_out;
    if ((rc = bank_alloc_streams(ctx, ctx->head_banks.back()))) return rc;
    if (bank_id) *bank_id = (int)ctx->head_banks.size() - 1;
    return OWW_OK;
}

int oww_load_bank_head(oww_ctx* ctx, int bank, int slot, const float* h_blob, size_t n_floats) {
    int rc = check_bank(ctx, bank);
    if (rc) return rc;
    if (!h_blob) return oww_fail(ctx, OWW_EINVAL, "null argument");
    HeadBank& b = ctx->head_banks[bank];
    if (slot < 0 || slot >= b.capacity) return oww_fail(ctx, OWW_EINVAL, "slot %d outside [0,%d)", slot, b.capacity);
    Head h;
    std::vector<float> staged;
    if ((rc = oww_stage_head(ctx, &b.shape.desc, h_blob, n_floats, h, staged))) return rc;
    std::vector<__half> packed;
    pack_layers(h, staged.data(), packed);
    std::vector<float> prm(b.p_floats, 0.f), unscale(h.desc.n_layers);
    for (int l = 0; l < h.desc.n_layers; ++l) {
        const int D = h.desc.dims[l + 1];
        std::memcpy(prm.data() + b.p_off[3 * l], staged.data() + h.b_off[l], D * sizeof(float));
        if (h.desc.layernorm && l < h.desc.n_layers - 1) {
            std::memcpy(prm.data() + b.p_off[3 * l + 1], staged.data() + h.g_off[l], D * sizeof(float));
            std::memcpy(prm.data() + b.p_off[3 * l + 2], staged.data() + h.h_off[l], D * sizeof(float));
        }
        unscale[l] = h.tc_layers[l].unscale;
    }
    const HtHead t = bank_slot_head(b, slot, unscale.data());
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaDeviceSynchronize());           // steps in flight on any stream finish with the old contents
    OWW_CUDA(ctx, cudaMemcpy(b.d_w + (size_t)slot * b.w_bytes, packed.data(), b.w_bytes, cudaMemcpyHostToDevice));
    OWW_CUDA(ctx, cudaMemcpy(b.d_p + (size_t)slot * b.p_floats, prm.data(), b.p_floats * sizeof(float), cudaMemcpyHostToDevice));
    OWW_CUDA(ctx, cudaMemcpy(reinterpret_cast<HtHead*>(b.d_slots) + slot, &t, sizeof(t), cudaMemcpyHostToDevice));
    std::memcpy(b.h_slots.data() + (size_t)slot * sizeof(HtHead), &t, sizeof(t));
    b.loaded[slot] = 1;
    return OWW_OK;
}

int oww_assign_bank_head(oww_ctx* ctx, int bank, const int32_t* h_stream_ids, int n, const int32_t* h_slots, void* stream) {
    int rc = check_bank(ctx, bank);
    if (rc) return rc;
    if (!h_slots) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (ctx->n_streams <= 0) return oww_fail(ctx, OWW_EINVAL, "oww_set_streams has not been called");
    HeadBank& b = ctx->head_banks[bank];
    if (!h_stream_ids) n = ctx->n_streams;
    if (n <= 0) return OWW_OK;
    if (n > ctx->n_streams) return oww_fail(ctx, OWW_EINVAL, "more stream ids (%d) than streams (%d)", n, ctx->n_streams);
    for (int i = 0; i < n; ++i) {
        if (h_stream_ids && (h_stream_ids[i] < 0 || h_stream_ids[i] >= ctx->n_streams))
            return oww_fail(ctx, OWW_EINVAL, "stream id %d out of range", h_stream_ids[i]);
        if ((rc = check_slot(ctx, b, h_slots[i], true))) return rc;
    }
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    // the host-buffer steps run on the handle's own stream: order the new table after the steps already submitted there
    // and before the ones submitted later, as on `stream` itself
    const bool other = s != ctx->own_stream;
    if (other) {
        OWW_CUDA(ctx, cudaEventRecord(ctx->ver_ev[0], ctx->own_stream));
        OWW_CUDA(ctx, cudaStreamWaitEvent(s, ctx->ver_ev[0], 0));
    }
    for (int i = 0; i < n; ++i) b.assign[h_stream_ids ? h_stream_ids[i] : i] = h_slots[i];
    if ((rc = upload_items(ctx, b, s))) return rc;
    if (other) {
        OWW_CUDA(ctx, cudaEventRecord(ctx->ver_ev[1], s));
        OWW_CUDA(ctx, cudaStreamWaitEvent(ctx->own_stream, ctx->ver_ev[1], 0));
    }
    return OWW_OK;
}

int oww_set_head_bank_clip_slot(oww_ctx* ctx, int bank, int slot) {
    int rc = check_bank(ctx, bank);
    if (rc) return rc;
    if ((rc = check_slot(ctx, ctx->head_banks[bank], slot, true))) return rc;
    ctx->head_banks[bank].clip_slot = slot;
    return OWW_OK;
}

int oww_bank_head_predict(oww_ctx* ctx, int bank, int slot, const float* d_feats, int n, float* d_out, void* stream) {
    int rc = check_bank(ctx, bank);
    if (rc) return rc;
    if (!d_feats || !d_out) return oww_fail(ctx, OWW_EINVAL, "null argument");
    const HeadBank& b = ctx->head_banks[bank];
    if ((rc = check_slot(ctx, b, slot, false))) return rc;
    if (n < 0) return oww_fail(ctx, OWW_EINVAL, "n=%d", n);
    if (n == 0) return OWW_OK;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    HeadsTcArgs a;
    std::memset(&a, 0, sizeof(a));
    a.head[0] = host_slot(b, slot);
    a.head[0].dev.col0 = 0;
    a.src = FeatSrc{d_feats, (int64_t)b.shape.desc.n_in * 96, nullptr, -1, 0};
    a.n = n; a.out = d_out; a.out_stride = b.shape.n_out; a.combine_max = 0;
    return ht_run<false>(ctx, a, std::max(16, b.shape.tc_layers[0].NP), dim3((n + kHtTile - 1) / kHtTile), (cudaStream_t)stream);
}

}  // extern "C"
