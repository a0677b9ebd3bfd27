// K3 (tensor-core path, streaming and bulk clips): the heads on the fp16 mirror of the feature rings.
//
// Same graphs as heads.cu / heads_tc.cu (reference: <head>.onnx sessions, openwakeword/model.py:137-138,153-159,287-302
// of the original project; family openwakeword/train.py:56-83,144-165).  heads_tc.cu converts the fp32 feature window to
// fp16 hi/lo again in every CTA.  Here
//   * the feature rings have an fp16 hi/lo MIRROR in HBM, already in the no-swizzle K-major core-matrix order and
//     addressed by a slot counter shared by all streams ([slot][tile of 128 streams][K chunk of 32][hi|lo][4 octets]
//     [128 rows][8 halves]): the A operand of (tile, feature row, chunk) is one contiguous 16 KB block that arrives by
//     ONE cp.async.bulk - no converter warps.  feat16_sync_kernel appends the rows each step added (and rewrites the window of a
//     stream that was reset) from the fp32 ring, which stays the state the API reads;
//   * a CTA owns a tile of 128 streams and one head: two warpgroups (64 streams each) accumulate the first layer in
//     registers (N = the head's widest layer, <= 128) while the producer warp streams A chunks and first-layer weight
//     blocks through a ring; the later layers and the store are heads_mma.cuh.
// Three MMA terms per K step (hi*hi + lo*hi + hi*lo, fp32 accumulate), as in heads_tc.cu.
#include "oww_internal.h"
#include "heads_mma.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace {

constexpr int kHgThreads = 9 * 32;                    // two MMA warpgroups + producer warp
constexpr int kHgTile = 128;                          // streams per mirror tile
constexpr int kHgMaxStages = 6;
constexpr int kHgChunkK = 32;                         // K per pipeline stage (4 octets)
constexpr int kHgAPlane = 4 * kHgTile * 16;           // one hi or lo plane of a mirror A chunk: 8 KB
constexpr int kHgABytes = 2 * kHgAPlane;              // hi + lo: 16 KB
constexpr int kHgTileBytes = 3 * kHgABytes;           // one feature row of one tile: 48 KB
constexpr int kHgSmem = 227 * 1024;
constexpr int kHgRing0 = 1024;                        // ring offset in shared memory (barriers below)

__device__ __forceinline__ void hg_warp_wait(uint32_t bar, uint32_t parity, int lane) {
    if (lane == 0) mbar_wait(bar, parity);
    __syncwarp();
}
__device__ __forceinline__ void hg_split8(const float* x, uint4& hi, uint4& lo) { hm_split8(x, hi, lo); }

// ---------------------------------------------------------------- fp16 mirror of the feature rings
// Rows count[b]-1-k (k = 0..depth-1) of stream b's fp32 ring -> slots (pos - k) mod NS of the mirror (zeros where the
// stream has no such row yet).  ids == nullptr: all n streams.
__global__ void __launch_bounds__(256) feat16_sync_kernel(const float* __restrict__ ring, int64_t ring_stride, int rows_mask,
                                                          const int* __restrict__ count, const int* __restrict__ ids, int n,
                                                          int depth, int pos, int NS, int n_tiles, uint8_t* __restrict__ out) {
    const int64_t total = (int64_t)n * 12 * depth;
    oww_pdl_sync();
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        const int lb = (int)(i % n);
        const int j = (int)((i / n) % 12);
        const int k = (int)(i / ((int64_t)n * 12));
        const int b = ids ? ids[lb] : lb;
        const int row = count[b] - 1 - k;
        float x[8];
        if (row >= 0) {
            const float4* p = reinterpret_cast<const float4*>(ring + (int64_t)b * ring_stride + (int64_t)(row & rows_mask) * 96 + j * 8);
            const float4 u = __ldcg(p), v = __ldcg(p + 1);
            x[0] = u.x; x[1] = u.y; x[2] = u.z; x[3] = u.w; x[4] = v.x; x[5] = v.y; x[6] = v.z; x[7] = v.w;
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e) x[e] = 0.f;
        }
        uint4 hi, lo;
        hg_split8(x, hi, lo);
        int slot = (pos - k) % NS;
        if (slot < 0) slot += NS;
        const int tile = b >> 7, r = b & 127, q = j >> 2, o = j & 3;
        uint8_t* t = out + ((int64_t)slot * n_tiles + tile) * kHgTileBytes + q * kHgABytes + (o * kHgTile + r) * 16;
        *reinterpret_cast<uint4*>(t) = hi;
        *reinterpret_cast<uint4*>(t + kHgAPlane) = lo;
    }
}

// Bulk clips: row t of clip b's linear feature rows [n_rows][96] -> slot pad + t of a mirror whose first `pad` slots are zero
// (a window that starts before the clip's first row reads zeros there, like FeatSrc's negative rows).
__global__ void __launch_bounds__(256) feat16_linear_kernel(const float* __restrict__ feats, int64_t clip_stride, int n_clips,
                                                            int n_rows, int pad, int n_tiles, uint8_t* __restrict__ out) {
    const int64_t total = (int64_t)n_clips * 12 * n_rows;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        const int b = (int)(i % n_clips);
        const int j = (int)((i / n_clips) % 12);
        const int t = (int)(i / ((int64_t)n_clips * 12));
        const float4* p = reinterpret_cast<const float4*>(feats + (int64_t)b * clip_stride + (int64_t)t * 96 + j * 8);
        const float4 u = __ldcg(p), v = __ldcg(p + 1);
        const float x[8] = {u.x, u.y, u.z, u.w, v.x, v.y, v.z, v.w};
        uint4 hi, lo;
        hg_split8(x, hi, lo);
        const int tile = b >> 7, r = b & 127, q = j >> 2, o = j & 3;
        uint8_t* d = out + ((int64_t)(pad + t) * n_tiles + tile) * kHgTileBytes + q * kHgABytes + (o * kHgTile + r) * 16;
        *reinterpret_cast<uint4*>(d) = hi;
        *reinterpret_cast<uint4*>(d + kHgAPlane) = lo;
    }
}

// ---------------------------------------------------------------- kernel arguments
using HgLayer = HmLayer;
struct HgHead {
    HeadDev dev;                    // fp32 blob: biases, LayerNorm parameters
    const uint8_t* w;               // per-head packed fp16 hi/lo weights (layers >= 1 are read from here)
    HgLayer L[OWW_MAX_HEAD_LAYERS];
};
struct HgGroup {                    // one head on the mirror
    int head, n_in, n_tot;          // index into HeadsGrpArgs::head; window rows; first-layer N (the head's widest layer)
    const uint8_t* w0;              // [n_in][3][hi|lo][4][n_tot][8] halves
    uint32_t w0_bytes;              // one (feature row, chunk) block, hi + lo
    int stages; uint32_t stage_bytes;
    int cpr;                        // K chunks of 32 per pipeline stage: 3 (a whole feature row) when two such stages fit, else 1
};
struct HeadsGrpArgs {
    HgHead head[16];
    HgGroup grp[8];
    const uint8_t* f16; int n_tiles, NS, slot_end;     // slot_end: mirror slot of the newest row of the window
    int steps;                      // > 0: bulk clips, blockIdx.z = step: window ends at slot_end + z, output row = clip * steps + z
    int n; float* out; int out_stride, combine_max, n_terms;
    long long* dbg;                 // [8 per group] clock64 stamps of CTA 0 (oww_debug_heads_clocks)
};

__global__ void __launch_bounds__(kHgThreads, 1) heads_grp_kernel(const __grid_constant__ HeadsGrpArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    const HgGroup& G = a.grp[blockIdx.y];
    const int tile = blockIdx.x, s0 = tile * kHgTile;
    const int S = G.stages;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem);
    uint8_t* ring = smem + kHgRing0;
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;
    const uint32_t bar0 = smem_u32(bars);
    auto full = [&](int s) { return bar0 + 8u * s; };
    auto empty = [&](int s) { return bar0 + 8u * (kHgMaxStages + s); };
    const uint32_t acc_done = bar0 + 8u * (2 * kHgMaxStages);          // a GEMM's operands have been read (one arrival per MMA warp)
    const uint32_t wn_full = acc_done + 8u;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kHgMaxStages; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), 8); }
        mbar_init(acc_done, 8);
        mbar_init(wn_full, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const bool split = a.n_terms >= 3;
    const int cpr = G.cpr;
    const int n_in = G.n_in, n_tot = G.n_tot, n_terms = a.n_terms;
    const int n_it = n_in * 3 / cpr;
    const HgHead& HH = a.head[G.head];
    const uint32_t stage_bytes = G.stage_bytes, w0_bytes = G.w0_bytes;
    const uint32_t ring_u = smem_u32(ring);
    // after the first-layer mainloop the ring is dead: per warpgroup hidden rows | next A tile, then the later-layer weight slot
    const uint32_t w_next = ring_u + 2 * kHmBufBytes;
    long long* dbg = (a.dbg && blockIdx.x == 0) ? a.dbg + 8 * blockIdx.y : nullptr;
    if (dbg && threadIdx.x == 0) dbg[0] = clock64();
    pdl_trigger();              // dependent launch chain of a step (tc_common.cuh): barriers are set up, now the
    pdl_wait();                 // predecessor's feature rows are needed

    if (warp == 8) {
        // ===================== producer =====================
        if (lane == 0) {
            const int NS = a.NS, n_tiles = a.n_tiles;
            int slot = (a.slot_end + (a.steps > 0 ? (int)blockIdx.z : 0) - n_in + 1) % NS;
            if (slot < 0) slot += NS;
            const uint8_t* f16 = a.f16 + (int64_t)tile * kHgTileBytes;
            const uint8_t* w0 = G.w0;
            const int64_t slot_pitch = (int64_t)n_tiles * kHgTileBytes;
            uint32_t stage = 0, par = 1, st = ring_u;
            const uint32_t a_off = (uint32_t)cpr * kHgABytes;            // stage: cpr A chunks (hi|lo each), then cpr W blocks
            const uint32_t a_bytes = split ? kHgABytes : kHgAPlane, w_bytes = split ? w0_bytes : w0_bytes / 2;
            for (int c = 0; c < n_in; ++c) {
                const uint8_t* arow = f16 + (int64_t)slot * slot_pitch;
                for (int q = 0; q < 3; q += cpr) {
                    mbar_wait(empty(stage), par);
                    mbar_expect_tx(full(stage), (uint32_t)cpr * (a_bytes + w_bytes));
                    for (int k = 0; k < cpr; ++k) {                      // plain fp16 operands: the hi planes only
                        bulk_g2s(st + k * kHgABytes, arow + (q + k) * kHgABytes, a_bytes, full(stage));
                        bulk_g2s(st + a_off + k * w0_bytes, w0 + (size_t)k * w0_bytes, w_bytes, full(stage));
                    }
                    w0 += (size_t)cpr * w0_bytes;
                    st += stage_bytes;
                    if (++stage == (uint32_t)S) { stage = 0; par ^= 1u; st = ring_u; }
                }
                if (++slot == NS) slot = 0;
            }
            if (dbg) dbg[1] = clock64();
            for (int l = 1; l < HH.dev.n_layers; ++l) {                  // later layers: the whole matrix, once the slot is free
                mbar_wait(acc_done, (uint32_t)((l - 1) & 1));
                const uint32_t wb = split ? HH.L[l].w_bytes : HH.L[l].w_bytes / 2;
                mbar_expect_tx(wn_full, wb);
                bulk_g2s(w_next, HH.w + HH.L[l].w_off, wb, wn_full);
            }
        }
    } else {
        // ===================== MMA warpgroups (streams 64 wg ..): first layer over the ring, later layers, store =====================
        const int wg = warp >> 2;
        float acc[64];
        const uint32_t w_plane = (uint32_t)n_tot * 64u;                  // 4 octets x n_tot rows x 16 B
        // N, the chunks per stage and the term count as compile-time constants: one unrolled chain of MMAs per stage
        wg_dispatch_n(n_tot, [&](auto nc) { dispatch_int<3, 1>(cpr, [&](auto cc) { dispatch_int<3, 1>(n_terms, [&](auto tc) {
            constexpr int NN = decltype(nc)::value, CPR = decltype(cc)::value, PER_CHUNK = 2 * decltype(tc)::value;
            float d[NN / 2];                                             // this chain's own registers (no aliasing with other N)
            uint32_t stage = 0, par = 0, st = ring_u;
            for (int it = 0; it < n_it; ++it) {
                hg_warp_wait(full(stage), par, lane);
                wg_fence();
#pragma unroll
                for (int s = 0; s < CPR * PER_CHUNK; ++s) {
                    const int k = s / PER_CHUNK, r = s - k * PER_CHUNK, t = r >> 1, ks = r & 1;
                    const uint32_t ab = st + (uint32_t)k * kHgABytes + (uint32_t)wg * kHmAPlane, wb = st + (uint32_t)cpr * kHgABytes + (uint32_t)k * w0_bytes;
                    const uint32_t au = ab + (t == 1 ? (uint32_t)kHgAPlane : 0u);         // term 1 = x_lo * w_hi
                    const uint32_t wu = wb + (t == 2 ? w_plane : 0u);                     // term 2 = x_hi * w_lo
                    const uint64_t ad = make_desc(au + (uint32_t)(2 * ks) * (kHgTile * 16), kHgTile * 16, 128u);
                    const uint64_t bd = make_desc(wu + (uint32_t)(2 * ks) * (uint32_t)NN * 16u, (uint32_t)NN * 16u, 128u);
                    wg_mma<NN>(d, ad, bd, (it | s) != 0);                               // the very first K step overwrites
                }
                wg_commit();
                wg_wait_all();
                __syncwarp();
                if (lane == 0) mbar_arrive(empty(stage));
                st += stage_bytes;
                if (++stage == (uint32_t)S) { stage = 0; par ^= 1u; st = ring_u; }
            }
#pragma unroll
            for (int k = 0; k < NN / 2; ++k) acc[k] = d[k];
        }); }); });
        __syncwarp();
        if (lane == 0) mbar_arrive(acc_done);
        if (dbg && threadIdx.x == 0) dbg[2] = clock64();
        const int r = threadIdx.x & 127, sr = s0 + wg * kHmRows + r;
        float* o = nullptr;
        if (r < kHmRows && sr < a.n) {
            const int64_t orow = a.steps > 0 ? (int64_t)sr * a.steps + blockIdx.z : (int64_t)sr;
            o = a.out + orow * a.out_stride + HH.dev.col0;
        }
        named_bar_sync(3, 256);                                          // both warpgroups are done with the ring
        hm_layers(acc, n_tot, HH.dev, HH.L, n_terms, ring + wg * kHmBufBytes, w_next, wn_full, acc_done, 1 + wg, o,
                  a.combine_max);
        if (dbg && threadIdx.x == 0) dbg[4] = clock64();
    }
}

}  // namespace

// Per-handle state of the grouped path (built lazily, dropped when the head set or the stream set changes).
struct oww_heads_grp {
    HeadsGrpArgs args;
    int n_groups = 0;
    uint32_t covered = 0;                // heads the groups cover
    std::vector<void*> d_w0;             // group-packed first-layer matrices
    long long* d_dbg = nullptr;          // clock stamps (debug)
    uint8_t* d_f16_bulk = nullptr; size_t bulk_bytes = 0;   // mirror of one slab of bulk clips (grow-only)
    uint8_t* d_f16 = nullptr;            // the mirror
    int NS = 0, n_tiles = 0, depth = 0;
    long pos = 0;                        // slot counter of the newest row
    bool mirror_valid = false;
    size_t n_heads_built = 0;
};

void oww_heads_grp_free(oww_ctx* ctx) {
    oww_heads_grp* g = ctx->heads_grp;
    if (!g) return;
    for (void* p : g->d_w0) cudaFree(p);
    cudaFree(g->d_f16); cudaFree(g->d_dbg); cudaFree(g->d_f16_bulk);
    delete g;
    ctx->heads_grp = nullptr;
}

// the stream set changed: the mirror is rebuilt at the next step
void oww_heads_grp_drop_mirror(oww_ctx* ctx) {
    oww_heads_grp* g = ctx->heads_grp;
    if (!g) return;
    cudaFree(g->d_f16); g->d_f16 = nullptr; g->mirror_valid = false;
}

void oww_feat16_invalidate(oww_ctx* ctx) {
    if (ctx->heads_grp) ctx->heads_grp->mirror_valid = false;
}

static int hg_build(oww_ctx* ctx) {
    oww_heads_grp_free(ctx);
    oww_heads_grp* g = new oww_heads_grp();
    ctx->heads_grp = g;
    g->n_heads_built = ctx->heads.size();
    HeadsGrpArgs& a = g->args;
    std::memset(&a, 0, sizeof(a));
    const int nh = (int)ctx->heads.size();
    if (nh > 16) return OWW_OK;
    // candidates: tensor-core packable heads, heaviest first
    std::vector<int> cand;
    for (int i = 0; i < nh; ++i)
        if (oww_heads_tc_supported(ctx, i) && !ctx->heads[i].tc_w0_host.empty()) cand.push_back(i);
    auto colw = [&](int i) { int w = 16; for (const auto& T : ctx->heads[i].tc_layers) w = std::max(w, T.NP); return w; };
    std::sort(cand.begin(), cand.end(), [&](int x, int y) {
        const int nx = ctx->heads[x].desc.n_in, ny = ctx->heads[y].desc.n_in;
        if (nx != ny) return nx > ny;
        const int cx = colw(x), cy = colw(y);
        return cx != cy ? cx > cy : x < y;
    });
    // one head per group: its first-layer accumulators fill the registers of the CTA's two MMA warpgroups (2 x 64 x <= 128)
    for (int i : cand) {
        if (g->n_groups >= 8) break;
        HgGroup& G = a.grp[g->n_groups];
        std::memset(&G, 0, sizeof(G));
        const Head& h = ctx->heads[i];
        G.head = i;
        G.n_in = h.desc.n_in;
        HgHead& HH = a.head[i];
        HeadDev& d = HH.dev;
        d.blob = h.d_blob;
        d.n_in = h.desc.n_in; d.n_layers = h.desc.n_layers; d.layernorm = h.desc.layernorm; d.final_act = h.desc.final_act;
        uint32_t wn_max = 0;
        for (int l = 0; l <= h.desc.n_layers; ++l) d.dims[l] = h.desc.dims[l];
        for (int l = 0; l < h.desc.n_layers; ++l) {
            d.w_off[l] = (int)h.w_off[l]; d.b_off[l] = (int)h.b_off[l];
            d.g_off[l] = (int)h.g_off[l]; d.h_off[l] = (int)h.h_off[l];
            const Head::TcLayer& T = h.tc_layers[l];
            HH.L[l] = HgLayer{T.K, T.D, T.Kp, T.NP, T.w_off, T.w_bytes, T.unscale};
            if (l >= 1) wn_max = std::max(wn_max, T.w_bytes);
        }
        d.col0 = h.col0;
        HH.w = reinterpret_cast<const uint8_t*>(h.d_w1_tc);
        G.n_tot = colw(i);
        G.w0_bytes = (uint32_t)(2 * 4 * G.n_tot * 16);
        // a stage carries a whole feature row (3 chunks: 18 MMAs between two barrier round trips) when two such stages
        // fit, else one chunk
        G.cpr = 2 * 3 * (kHgABytes + (int)G.w0_bytes) <= kHgSmem - kHgRing0 ? 3 : 1;
        G.stage_bytes = (uint32_t)(G.cpr * (kHgABytes + (int)G.w0_bytes));
        G.stages = std::min(kHgMaxStages, (kHgSmem - kHgRing0) / (int)G.stage_bytes);
        const bool fits = G.stages >= 2 && 2 * (size_t)kHmBufBytes + ((wn_max + 127u) & ~127u) <= (size_t)(kHgSmem - kHgRing0);
        if (!fits) continue;                                         // this head stays with heads_tc.cu
        // first-layer matrix: [feature row][chunk][hi|lo][4 octets][n_tot][8]
        const size_t blk = (size_t)G.w0_bytes / 2;                   // halves per (row, chunk) block
        std::vector<__half> packed((size_t)G.n_in * 3 * blk, __float2half(0.f));
        const int D = h.desc.dims[1];
        const float sc = 1.0f / h.tc_layers[0].unscale;
        const float* w = h.tc_w0_host.data();
        for (int c = 0; c < G.n_in; ++c)
            for (int q = 0; q < 3; ++q) {
                __half* dst = packed.data() + ((size_t)c * 3 + q) * blk;
                for (int o = 0; o < 4; ++o)
                    for (int n = 0; n < D; ++n)
                        for (int e = 0; e < 8; ++e) {
                            const int kk = c * 96 + q * kHgChunkK + o * 8 + e;
                            const float v = w[(size_t)kk * D + n] * sc;
                            const __half hi = __float2half_rn(v);
                            const size_t at = ((size_t)o * G.n_tot + n) * 8 + e;
                            dst[at] = hi;
                            dst[at + blk / 2] = __float2half_rn(v - __half2float(hi));
                        }
            }
        void* dw = nullptr;
        OWW_CUDA(ctx, cudaMalloc(&dw, packed.size() * sizeof(__half)));
        g->d_w0.push_back(dw);
        OWW_CUDA(ctx, cudaMemcpy(dw, packed.data(), packed.size() * sizeof(__half), cudaMemcpyHostToDevice));
        G.w0 = reinterpret_cast<const uint8_t*>(dw);
        g->covered |= 1u << i;
        g->depth = std::max(g->depth, G.n_in);
        ++g->n_groups;
    }
    // heaviest groups first (blockIdx.y order = launch order of the CTAs)
    std::sort(a.grp, a.grp + g->n_groups, [](const HgGroup& x, const HgGroup& y) {
        return (int64_t)x.n_in * x.n_tot > (int64_t)y.n_in * y.n_tot;
    });
    if (g->n_groups) OWW_CUDA(ctx, cudaFuncSetAttribute(heads_grp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kHgSmem));
    return OWW_OK;
}

static int hg_ensure(oww_ctx* ctx) {
    if (!ctx->heads_grp || ctx->heads_grp->n_heads_built != ctx->heads.size()) return hg_build(ctx);
    return OWW_OK;
}

static int hg_sync(oww_ctx* ctx, const int* d_ids, int n, int depth, cudaStream_t s) {
    oww_heads_grp* g = ctx->heads_grp;
    const int64_t total = (int64_t)n * 12 * depth;
    if (total <= 0) return OWW_OK;
    const unsigned grid = (unsigned)std::min<int64_t>((total + 255) / 256, (int64_t)ctx->sm_count * 16);
    OWW_CUDA(ctx, oww_launch_pdl(ctx->late_pdl, feat16_sync_kernel, dim3(grid), dim3(256), 0, s, (const float*)ctx->d_feat_ring,
                                 (int64_t)ctx->feat_rows * 96, ctx->feat_rows - 1, (const int*)ctx->d_feat_count, d_ids, n, depth,
                                 (int)(g->pos % g->NS), g->NS, g->n_tiles, g->d_f16));
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

// Every stream's ring has just gained n_chunks rows: append them to the mirror (or build it).
int oww_feat16_advance(oww_ctx* ctx, int n_chunks, cudaStream_t s) {
    if (!ctx->tc_heads || ctx->cfg.cnn_mode == OWW_CNN_FP32_WINDOW || ctx->heads.empty() || !ctx->grp_heads) return OWW_OK;
    int rc = hg_ensure(ctx);
    if (rc) return rc;
    oww_heads_grp* g = ctx->heads_grp;
    if (!g->n_groups) return OWW_OK;
    const int need_ns = g->depth + ctx->cfg.max_chunks;
    if (!g->d_f16 || g->NS < need_ns) {
        cudaFree(g->d_f16); g->d_f16 = nullptr;
        g->NS = need_ns;
        g->n_tiles = (ctx->n_streams + kHgTile - 1) / kHgTile;
        const size_t bytes = (size_t)g->NS * g->n_tiles * kHgTileBytes;
        OWW_CUDA(ctx, cudaMalloc(&g->d_f16, bytes));
        OWW_CUDA(ctx, cudaMemsetAsync(g->d_f16, 0, bytes, s));
        g->mirror_valid = false;
    }
    if (!g->mirror_valid) {
        g->pos = g->NS;                                               // any position: the whole window depth is rewritten
        g->mirror_valid = true;
        return hg_sync(ctx, nullptr, ctx->n_streams, g->depth + ctx->cfg.max_chunks - 1, s);
    }
    g->pos += n_chunks;
    if (g->pos > (1L << 40)) g->pos = g->pos % g->NS + g->NS;
    return hg_sync(ctx, nullptr, ctx->n_streams, n_chunks, s);
}

// The listed streams were reset (rings refilled, counts changed): rewrite their windows in the mirror.
int oww_feat16_resync(oww_ctx* ctx, const int* d_ids, int n, cudaStream_t s) {
    oww_heads_grp* g = ctx->heads_grp;
    if (!g || !g->d_f16 || !g->mirror_valid) return OWW_OK;
    return hg_sync(ctx, d_ids, n, g->depth + ctx->cfg.max_chunks - 1, s);
}

uint32_t oww_heads_grp_covered(oww_ctx* ctx) {
    oww_heads_grp* g = ctx->heads_grp;
    if (!g || !g->mirror_valid || !g->n_groups || g->n_heads_built != ctx->heads.size()) return 0;
    return g->covered;
}

// The grouped heads on every stream's window ending `back` rows before the newest (FeatSrc ring semantics).
int oww_heads_grp_launch(oww_ctx* ctx, int back, int n, float* d_out, int out_stride, int combine_max, cudaStream_t s) {
    oww_heads_grp* g = ctx->heads_grp;
    HeadsGrpArgs& a = g->args;
    a.f16 = g->d_f16; a.n_tiles = g->n_tiles; a.NS = g->NS;
    a.slot_end = (int)((g->pos - back) % g->NS);
    a.n = n; a.out = d_out; a.out_stride = out_stride; a.combine_max = combine_max;
    a.n_terms = ctx->tc_heads_terms;
    a.dbg = g->d_dbg;
    a.steps = 0;
    dim3 grid((n + kHgTile - 1) / kHgTile, g->n_groups);
    OWW_CUDA(ctx, oww_launch_pdl(ctx->late_pdl, heads_grp_kernel, grid, dim3(kHgThreads), kHgSmem, s, a));
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

// Bulk clips (FeatSrc sliding mode): the same kernel over every window position of every clip.  The clips' feature rows
// are mirrored once per call ([pad zero slots | rows]); returns the mask of heads it ran (0: the caller keeps its path).
uint32_t oww_heads_grp_bulk(oww_ctx* ctx, const FeatSrc& src, int n, float* d_out, int out_stride, cudaStream_t s, int* rc_out) {
    *rc_out = OWW_OK;
    if (!ctx->tc_heads || !ctx->grp_heads || ctx->cfg.cnn_mode == OWW_CNN_FP32_WINDOW || src.count || src.steps <= 0) return 0;
    if ((*rc_out = hg_ensure(ctx))) return 0;
    oww_heads_grp* g = ctx->heads_grp;
    if (!g->n_groups || src.steps > 65535 || n % src.steps) return 0;
    const int m = n / src.steps, n_rows = (int)(src.stride / 96), pad = g->depth;
    if (src.row0 + src.steps > n_rows) return 0;
    const int n_tiles = (m + kHgTile - 1) / kHgTile;
    const size_t bytes = (size_t)(pad + n_rows) * n_tiles * kHgTileBytes;
    auto fail = [&](cudaError_t e) { *rc_out = oww_fail(ctx, OWW_ECUDA, "bulk feature mirror: %s", cudaGetErrorString(e)); return 0u; };
    cudaError_t e;
    if (g->bulk_bytes < bytes) {
        cudaFree(g->d_f16_bulk); g->d_f16_bulk = nullptr; g->bulk_bytes = 0;
        if ((e = cudaMalloc(&g->d_f16_bulk, bytes)) != cudaSuccess) return fail(e);
        g->bulk_bytes = bytes;
    }
    // rows of clips beyond m in the last tile and the pad slots read as zeros
    if ((e = cudaMemsetAsync(g->d_f16_bulk, 0, bytes, s)) != cudaSuccess) return fail(e);
    {
        const int64_t total = (int64_t)m * 12 * n_rows;
        const unsigned grid = (unsigned)std::min<int64_t>((total + 255) / 256, (int64_t)ctx->sm_count * 32);
        feat16_linear_kernel<<<grid, 256, 0, s>>>(src.base, src.stride, m, n_rows, pad, n_tiles, g->d_f16_bulk);
        ctx->launches++;
    }
    HeadsGrpArgs& a = g->args;
    a.f16 = g->d_f16_bulk; a.n_tiles = n_tiles; a.NS = pad + n_rows;
    a.slot_end = pad + src.row0;
    a.steps = src.steps;
    a.n = m; a.out = d_out; a.out_stride = out_stride; a.combine_max = 0;
    a.n_terms = ctx->tc_heads_terms;
    a.dbg = nullptr;
    dim3 grid(n_tiles, g->n_groups, src.steps);
    heads_grp_kernel<<<grid, kHgThreads, kHgSmem, s>>>(a);
    ctx->launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return fail(e);
    return g->covered;
}

// debug: clock64 stamps of the last mirror-path launch (CTA 0 of each head): [0] start, [1] producer done, [2] first-layer
// accumulators complete, [4] scores stored.  First call arms the stamps.
extern "C" int oww_debug_heads_clocks(oww_ctx* ctx, int64_t* h_out64) {
    oww_heads_grp* g = ctx ? ctx->heads_grp : nullptr;
    if (!g) return OWW_EINVAL;
    if (!g->d_dbg) {
        OWW_CUDA(ctx, cudaMalloc(&g->d_dbg, 256 * sizeof(long long)));
        OWW_CUDA(ctx, cudaMemset(g->d_dbg, 0, 256 * sizeof(long long)));
        return OWW_OK;
    }
    OWW_CUDA(ctx, cudaDeviceSynchronize());
    OWW_CUDA(ctx, cudaMemcpy(h_out64, g->d_dbg, 256 * sizeof(long long), cudaMemcpyDeviceToHost));
    return OWW_OK;
}
