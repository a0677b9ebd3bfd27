// K2 (tensor-core path): the speech-embedding CNN as warpgroup-MMA (wgmma) implicit GEMMs for sm_90a.
//
// Same graph as cnn_fp32.cu (reference: embedding_model.onnx, openwakeword/utils.py:90-93 of the original project;
// spec notebooks/converting_google_speech_embedding_model.ipynb:871-951).  Layers 1..19 are dense
// (1,3)/(3,1) convolutions: M = output positions, N = Cout, K = 3 taps x Cin.
//
// Layout.  Activations live in HBM/L2 as fp16 "channel-group planes": plane g holds channels
// 8g..8g+7 of every position as one 16-byte unit, positions ordered (window, t, f) with ONE zero pad
// column per row (f = W), i.e. exactly the canonical no-swizzle K-major core-matrix order of a wgmma
// operand (8 consecutive positions x 16 B = one 8x8 core matrix, SBO = 128 B, LBO = plane pitch).  Hence
//   * an A tile (128 positions + halo, all planes) is CG contiguous runs -> CG 1-D bulk copies
//     (cp.async.bulk, mbarrier complete_tx), no im2col, no tensor map;
//   * a conv tap is just a 16-byte-granular shift of the A descriptor's start address:
//     (1,3) taps shift by -1/0/+1 positions (the pad column supplies the "same" zeros),
//     (3,1) taps shift by 0/Wp/2Wp positions; one smem tile feeds all three taps.
// Weights are pre-packed per layer as fp16 [tap][plane][n][8] (same core-matrix order, K-major B).
// Two MMA warpgroups each own 64 of a tile's 128 positions: D accumulates in their registers (fp32), and the same
// threads apply folded BN + leaky + clamp in fp32 and write the next layer's fp16 planes (each thread holds two
// adjacent channels of two positions: 4-byte stores, 128 contiguous bytes per warp and plane).  Warp 0 = bulk-copy
// producer.  Persistent CTAs, grid = #SMs.
#include "oww_internal.h"
#include "tc_common.cuh"
#include <cmath>
#include <cstring>

namespace {

// ---------------------------------------------------------------- layer 0 (CUDA cores) -> fp16 planes
struct Tc0Args {
    WindowSrc src;
    int n_windows; int T_out;         // output rows per window (input rows - 2): 74 for the 76-row window
    const float* w; const float* scale; const float* bias;
    __half* out; int64_t plane;       // units per plane
};

__global__ void __launch_bounds__(256) tc_conv0_kernel(Tc0Args a) {
    __shared__ float s_w[9 * 24];
    __shared__ float s_s[24], s_b[24];
    for (int i = threadIdx.x; i < 9 * 24; i += 256) s_w[i] = a.w[i];
    if (threadIdx.x < 24) { s_s[threadIdx.x] = a.scale[threadIdx.x]; s_b[threadIdx.x] = a.bias[threadIdx.x]; }
    __syncthreads();
    constexpr int Wp = 33;
    const int T = a.T_out;
    const int64_t total = (int64_t)a.n_windows * T * Wp;
    for (int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x; p < total; p += (int64_t)gridDim.x * 256) {
        const int f = (int)(p % Wp);
        const int64_t r = p / Wp;
        const int t = (int)(r % T);
        const int j = (int)(r / T);
        uint4* o = reinterpret_cast<uint4*>(a.out) + kGuard + p;
        if (p == 0) { const uint4 z = make_uint4(0, 0, 0, 0); o[-1] = z; o[a.plane - 1] = z; o[2 * a.plane - 1] = z; }
        if (f == 32) {
            const uint4 z = make_uint4(0, 0, 0, 0);
            o[0] = z; o[a.plane] = z; o[2 * a.plane] = z;
            continue;
        }
        const float* base; int row0, mask;
        if (a.src.count) {
            const int lb = j % a.src.n_streams, i = j / a.src.n_streams;
            const int b = a.src.ids ? a.src.ids[lb] : lb;
            base = a.src.base + (int64_t)b * a.src.stride;
            row0 = a.src.count[b] - 8 * (a.src.n_chunks - 1 - i) - OWW_WINDOW_ROWS;
            mask = a.src.rows_mask;
        } else {
            base = a.src.base + (int64_t)j * a.src.stride; row0 = 0; mask = -1;
        }
        float x[9];
#pragma unroll
        for (int dt = 0; dt < 3; ++dt) {
            int row = row0 + t + dt;
            if (mask >= 0) row &= mask;
            const float* rp = base + (int64_t)row * 32;
#pragma unroll
            for (int df = 0; df < 3; ++df) {
                const int ff = f + df - 1;
                x[dt * 3 + df] = (ff >= 0 && ff < 32) ? __ldg(rp + ff) : 0.f;
            }
        }
#pragma unroll
        for (int g = 0; g < 3; ++g) {
            __half2 h[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                float v2[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int c = g * 8 + u * 2 + e;
                    float acc = 0.f;
#pragma unroll
                    for (int k = 0; k < 9; ++k) acc = fmaf(x[k], s_w[k * 24 + c], acc);
                    acc = fmaxf(acc, 0.f);
                    v2[e] = act(fmaf(acc, s_s[c], s_b[c]));
                }
                h[u] = __floats2half2_rn(v2[0], v2[1]);
            }
            o[g * a.plane] = *reinterpret_cast<uint4*>(h);
        }
    }
}

// ---------------------------------------------------------------- tensor-core conv layer
struct TcConvArgs {
    const __half* in; int64_t in_plane;     // units (16 B) per input plane, guard included
    __half* out; int64_t out_plane;
    float* out_f32;                         // final layer: [n][96] fp32 instead of planes
    const __half* w;                        // packed [3][CGP][NP][8]
    const float* scale; const float* bias;  // [NP]
    int n, T, W, T_out;                     // input extent per window, W excludes the pad column
    int tap_off[3];                         // tile-row offset of each tap
    int lo;                                 // tile starts `lo` positions before its first output
    int rows;                               // tile rows incl. halo (multiple of 8)
    int cg_in;                              // real input planes
    int cg_out;                             // real output planes (Cout/8)
    int apply_act;
    int64_t p_in;                           // n*T*(W+1)
    int n_tiles;
    int out_split;                          // 1: write fp16 hi planes [0, cg_out) and lo planes [cg_out, 2 cg_out) (y = hi + lo)
    int64_t rows_out;                       // final layer: embedding rows per window (T_out valid rows; fully convolutional clips)
    // incremental late layers on plane-major tensors (the reserved[0] bit-4 fallback; the default chain runs
    // tc_conv_blk_kernel below): the output rows land at row offset out_toff inside buffers that hold
    // out_T rows per stream (tails in front), and are mirrored into up to two further buffers where they will serve as
    // tails of later steps.  out_T == 0: plain layout (out_T = T_out, no offset, no mirrors).
    int out_T, out_toff;
    __half* out_b[2]; int out_b_toff[2];    // mirrors (nullptr = unused); same plane pitch as `out`
};

// TERMS = 1: fp16 operands.  TERMS = 3: split operands - the input holds hi planes [0, cg_in) and lo planes
// [cg_in, 2 cg_in), the weights hi and lo blocks of W * 2^s (2^-s folded into `scale`), and every K step issues
// hi*hi + lo*hi + hi*lo into the same fp32 accumulator: the product is fp32-grade (~2^-21), at 3x the MMAs, 2x the
// operand bytes and half the pipeline stages.
// Warp roles: warp 0 lane 0 = bulk-copy producer (warps 1-3 only take part in the set-up); warpgroups 1 and 2 each own
// 64 of the tile's 128 positions: they issue the tile's MMAs (wgmma, accumulators in registers), release the stage and
// run the epilogue from the register fragment.
template <int CGP, int NP, int TERMS>
__global__ void __launch_bounds__(kTcThreads, 1) tc_conv_kernel(TcConvArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    constexpr int kSplit = TERMS == 3 ? 2 : 1;
    constexpr int kStages = TERMS == 3 ? 2 : 4;
    constexpr int W_TERM = 3 * CGP * NP * 16;
    constexpr int W_BYTES = kSplit * W_TERM;
    uint8_t* w_smem = smem;
    const int term_bytes = CGP * a.rows * 16;
    const int stage_bytes = kSplit * term_bytes;
    uint8_t* a_smem = smem + W_BYTES;
    uint64_t* bars = reinterpret_cast<uint64_t*>(a_smem + kStages * stage_bytes);
    // bars: [0..S) full, [S..2S) empty, then w_full
    float* s_sb = reinterpret_cast<float*>(bars + 2 * kStages + 2);          // folded BN scale[NP] | bias[NP]
    for (int i = threadIdx.x; i < NP; i += kTcThreads) { s_sb[i] = a.scale[i]; s_sb[NP + i] = a.bias[i]; }

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t bar0 = smem_u32(bars);
    auto full_bar = [&](int s) { return bar0 + 8u * s; };
    auto empty_bar = [&](int s) { return bar0 + 8u * (kStages + s); };
    const uint32_t wfull_bar = bar0 + 8u * (2 * kStages);

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }   // one arrival per MMA warp
        mbar_init(wfull_bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // zero the pad planes of every A stage once (never overwritten by the bulk copies)
    if (a.cg_in < CGP) {
        for (int s = 0; s < kStages * kSplit; ++s) {
            uint4* pz = reinterpret_cast<uint4*>(a_smem + s * term_bytes + a.cg_in * a.rows * 16);
            for (int i = threadIdx.x; i < (CGP - a.cg_in) * a.rows; i += kTcThreads) pz[i] = make_uint4(0, 0, 0, 0);
        }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    if (warp == 0) {
        // ===================== producer: weights once, then one A tile per stage =====================
        if (lane == 0) {
            mbar_expect_tx(wfull_bar, W_BYTES);
            bulk_g2s(smem_u32(w_smem), a.w, W_BYTES, wfull_bar);
            int stage = 0; uint32_t phase = 0;
            const uint32_t plane_bytes = (uint32_t)a.rows * 16u;
            for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
                mbar_wait(empty_bar(stage), phase ^ 1);
                mbar_expect_tx(full_bar(stage), plane_bytes * a.cg_in * kSplit);
                const int64_t u0 = kGuard + (int64_t)tile * 128 - a.lo;
                for (int t = 0; t < kSplit; ++t)
                    for (int g = 0; g < a.cg_in; ++g)
                        bulk_g2s(smem_u32(a_smem + stage * stage_bytes + t * term_bytes + g * plane_bytes),
                                 reinterpret_cast<const uint4*>(a.in) + (int64_t)(t * a.cg_in + g) * a.in_plane + u0, plane_bytes, full_bar(stage));
                if (++stage == kStages) { stage = 0; phase ^= 1; }
            }
        }
    } else if (warp >= 4) {
        // ===================== MMA + epilogue: warpgroup wg owns accumulator rows [64 wg, 64 wg + 64) =====================
        const int wg = (warp >> 2) - 1, wq = warp & 3, q = lane & 3;
        const uint32_t row_off = (uint32_t)wg * 64u * 16u;                 // 8 core-matrix rows of 128 B per 8 positions
        tc_warp_wait(wfull_bar, 0, lane);
        int stage = 0; uint32_t phase = 0;
        const uint32_t w_addr = smem_u32(w_smem);
        const uint32_t lbo_a = (uint32_t)a.rows * 16u;
        const uint32_t rows16 = (uint32_t)a.rows * 16u;
        const uint32_t tap16[3] = {(uint32_t)a.tap_off[0] * 16u, (uint32_t)a.tap_off[1] * 16u, (uint32_t)a.tap_off[2] * 16u};
        const int Wp = a.W + 1;
        const int per_in = a.T * Wp;
        const int per_out = a.T_out * Wp;
        for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
            tc_warp_wait(full_bar(stage), phase, lane);
            float acc[NP / 2];
            const uint32_t a_addr = smem_u32(a_smem + stage * stage_bytes) + row_off;
            wg_fence();
            {
                uint32_t accumulate = 0;
                if (TERMS == 1 && (a.cg_in & 1)) {
                    // odd plane count, plain operands: the K octets of the three taps are chained exactly as in the fused
                    // step kernel (cnn_tc_inc.cu: the last plane of tap 0 shares an MMA with the first plane of tap 1),
                    // with the weights packed in that order - one MMA per tile less, and the same accumulation order
                    // as the streaming path (bulk == streaming, bit for bit)
                    constexpr int CG = CGP - 1, NPAIR = CG / 2;
                    uint32_t b = w_addr;
                    constexpr uint32_t np2 = 2u * NP * 16u;
                    auto mma = [&](uint32_t a_at, uint32_t lbo) {
                        wg_mma<NP>(acc, make_desc(a_at, lbo, 128u), make_desc(b, NP * 16u, 128u), accumulate);
                        accumulate = 1; b += np2;
                    };
#pragma unroll
                    for (int k = 0; k < NPAIR; ++k) mma(a_addr + tap16[0] + (uint32_t)(2 * k) * rows16, lbo_a);
                    mma(a_addr + tap16[1], (uint32_t)CG * rows16 - rows16 + tap16[0] - tap16[1]);
#pragma unroll
                    for (int k = 0; k < NPAIR; ++k) mma(a_addr + tap16[1] + (uint32_t)(2 * k + 1) * rows16, lbo_a);
#pragma unroll
                    for (int k = 0; k < NPAIR; ++k) mma(a_addr + tap16[2] + (uint32_t)(2 * k) * rows16, lbo_a);
                    mma(a_addr + tap16[2] + (uint32_t)(CG - 1) * rows16, 0u);
                } else {
                    // term order: every K step with the hi activations ((hi,hi), (hi,lo)), then every K step with the lo
                    // activations ((lo,hi)) - the order tc_conv_blk_kernel is bound to (it holds one half at a time), so the
                    // window / clip passes and the incremental late layers accumulate identically (bulk == streaming, bit for bit)
#pragma unroll
                    for (int ph = 0; ph < (TERMS == 3 ? 2 : 1); ++ph) {
#pragma unroll
                        for (int j = 0; j < 3; ++j) {
#pragma unroll
                            for (int qq = 0; qq < CGP / 2; ++qq) {
#pragma unroll
                                for (int wt = 0; wt < (TERMS == 3 && ph == 0 ? 2 : 1); ++wt) {
                                    const uint32_t a_t = a_addr + (ph == 1 ? (uint32_t)term_bytes : 0u);
                                    const uint32_t w_t = w_addr + (wt == 1 ? (uint32_t)W_TERM : 0u);
                                    const uint64_t ad = make_desc(a_t + (uint32_t)(2 * qq) * rows16 + tap16[j], lbo_a, 128u);
                                    const uint64_t bd = make_desc(w_t + (uint32_t)((j * CGP + 2 * qq) * NP) * 16u, NP * 16u, 128u);
                                    wg_mma<NP>(acc, ad, bd, accumulate);
                                    accumulate = 1;
                                }
                            }
                        }
                    }
                }
            }
            wg_commit();
            wg_wait_all();
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(stage));                  // this warp's share of the stage has been read
            if (++stage == kStages) { stage = 0; phase ^= 1; }

#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int row = wg * 64 + wq * 16 + (lane >> 2) + 8 * i;
                const int64_t m = (int64_t)tile * 128 + row;
                if (m >= a.p_in) continue;
                const int n = (int)(m / per_in);
                const int rem = (int)(m - (int64_t)n * per_in);
                const int t = rem / Wp, f = rem - t * Wp;
                if (t >= a.T_out) continue;
                if (a.out_f32) {
                    if (f != 0) continue;
                    float* o = a.out_f32 + ((int64_t)n * a.rows_out + t) * 96;
#pragma unroll
                    for (int j = 0; j < NP / 8; ++j) {
                        const int c = j * 8 + 2 * q;
                        if (c >= 96) continue;
                        float2 r;
                        r.x = fmaf(acc[4 * j + 2 * i], s_sb[c], s_sb[NP + c]);
                        r.y = fmaf(acc[4 * j + 2 * i + 1], s_sb[c + 1], s_sb[NP + c + 1]);
                        *reinterpret_cast<float2*>(o + c) = r;
                    }
                    continue;
                }
                const int64_t po = a.out_T ? (int64_t)n * a.out_T * Wp + (int64_t)(t + a.out_toff) * Wp + f
                                           : (int64_t)n * per_out + (int64_t)t * Wp + f;
                uint4* o = reinterpret_cast<uint4*>(a.out) + kGuard + po;
                const bool pad = f == a.W;
#pragma unroll
                for (int j = 0; j < NP / 8; ++j) {
                    const int g = j;                                       // channel-group plane; this thread holds channels 2q, 2q+1
                    if (g >= a.cg_out) continue;
                    const int c = g * 8 + 2 * q;
                    float y0 = fmaf(acc[4 * j + 2 * i], s_sb[c], s_sb[NP + c]);
                    float y1 = fmaf(acc[4 * j + 2 * i + 1], s_sb[c + 1], s_sb[NP + c + 1]);
                    if (a.apply_act) { y0 = act(y0); y1 = act(y1); }
                    if (pad) { y0 = 0.f; y1 = 0.f; }
                    const __half h0 = __float2half_rn(y0), h1 = __float2half_rn(y1);
                    const __half2 h = __halves2half2(h0, h1);
                    const __half2 l = __floats2half2_rn(y0 - __half2float(h0), y1 - __half2float(h1));
                    const uint32_t hw = *reinterpret_cast<const uint32_t*>(&h), lw = *reinterpret_cast<const uint32_t*>(&l);
                    reinterpret_cast<uint32_t*>(o + (int64_t)g * a.out_plane)[q] = hw;
                    if (po == 0) reinterpret_cast<uint32_t*>(o + (int64_t)g * a.out_plane - 1)[q] = 0u;   // front guard (position -1)
                    if (a.out_split) {
                        reinterpret_cast<uint32_t*>(o + (int64_t)(a.cg_out + g) * a.out_plane)[q] = lw;
                        if (po == 0) reinterpret_cast<uint32_t*>(o + (int64_t)(a.cg_out + g) * a.out_plane - 1)[q] = 0u;
                    }
#pragma unroll
                    for (int kk = 0; kk < 2; ++kk)
                        if (a.out_b[kk]) {
                            uint4* ob = reinterpret_cast<uint4*>(a.out_b[kk]) + kGuard + (int64_t)n * a.out_T * Wp +
                                        (int64_t)(t + a.out_b_toff[kk]) * Wp + f;
                            reinterpret_cast<uint32_t*>(ob + (int64_t)g * a.out_plane)[q] = hw;
                            if (a.out_split) reinterpret_cast<uint32_t*>(ob + (int64_t)(a.cg_out + g) * a.out_plane)[q] = lw;
                        }
                }
            }
        }
    }
}

// ---------------------------------------------------------------- incremental late layers: block-major tensors
// The window-mode kernel above can run a layer of the incremental chain on per-stream "windows" [2 tails | new rows] x
// (W + 1) in plane-major HBM tensors.  Two things make that slow there: of the 128 accumulator rows of a (3,1) tile only
// rows_new / T carry outputs and one column in W + 1 is padding (layer 16: 4 of 12 positions, layer 19: 1 of 6) while an
// MMA costs the same; and a tile's channel-group planes are far apart in HBM, i.e. 24 bulk copies of 2-4 KB per tile.
// Here a late tensor is stored in blocks of S streams, a block being [2*cg planes][units] CONTIGUOUS in HBM (LateLay):
//   input of a (3,1) layer: time-major inside the block, no pad column: unit (row*S + s)*W + f.  Tap k of the conv reads
//     rows k .. k + rows_new - 1 = one contiguous run of rows_new*S*W = 128 units at offset k*S*W: every accumulator row
//     is an output;
//   input of a (1,3) layer: stream-major with the pad column behind a zero guard unit: unit 1 + (s*T + row)*(W+1) + f,
//     taps at unit offsets 0, 1, 2.
// One tile = one block; its hi half and its lo half arrive by ONE bulk copy each.  The two halves of a 96-channel (3,1)
// block (98 KB) do not fit twice beside the 110 KB of split weights, so the two shared-memory slots hold one half each:
// the MMAs of the hi half ((hi,hi), (hi,lo)) run while the lo half lands, the lo MMAs ((lo,hi)) while the next block's
// hi half lands.  The epilogue writes straight into the next layer's block-major tensor(s) (or the plain unpooled temp).
struct TcBlkArgs {
    const __half* in; LateLay lay;          // input tensor
    const __half* w; const float* scale; const float* bias;
    int n, W, rows_new;                     // streams, real width, output rows per stream
    int m_valid, tap;                       // accumulator rows that are positions of the block; unit distance of the taps
    int pool_f;                             // 2: (1,2) max-pool fused into the epilogue (columns f, f^1 sit in adjacent lanes); 0: none
    int cg_in, cg_out, apply_act, n_tiles;
    float* out_f32;                         // final layer: [n][rows_new][96]
    __half* out[3]; int out_toff[3];        // destination buffers (this step / later steps' tails) and their row offsets
    LateLay out_lay;                        // out_lay.S > 0: block-major destination; else the plain temp [n][rows_new][W+1]
    int64_t out_plane;                      //   (plane pitch of the plain temp)
};

template <int CGP, int NP>
__global__ void __launch_bounds__(kTcThreads, 1) tc_conv_blk_kernel(TcBlkArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    constexpr int W_TERM = 3 * CGP * NP * 16;
    constexpr int W_BYTES = 2 * W_TERM;
    uint8_t* w_smem = smem;
    const int units = a.lay.units;
    const int half_bytes = CGP * units * 16;
    uint8_t* a_smem = smem + W_BYTES;                                      // slot 0: hi half, slot 1: lo half
    uint64_t* bars = reinterpret_cast<uint64_t*>(a_smem + 2 * half_bytes);
    // bars: full[2], empty[2], w_full
    float* s_sb = reinterpret_cast<float*>(bars + 6);
    for (int i = threadIdx.x; i < NP; i += kTcThreads) { s_sb[i] = a.scale[i]; s_sb[NP + i] = a.bias[i]; }

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t bar0 = smem_u32(bars);
    auto full_bar = [&](int h) { return bar0 + 8u * h; };
    auto empty_bar = [&](int h) { return bar0 + 8u * (2 + h); };
    const uint32_t wfull_bar = bar0 + 8u * 4;

    if (threadIdx.x == 0) {
        for (int h = 0; h < 2; ++h) { mbar_init(full_bar(h), 1); mbar_init(empty_bar(h), 8); }       // one arrival per MMA warp
        mbar_init(wfull_bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // pad planes (odd cg_in) are never written by the bulk copies: zero them once
    if (a.cg_in < CGP)
        for (int h = 0; h < 2; ++h) {
            uint4* pz = reinterpret_cast<uint4*>(a_smem + h * half_bytes + a.cg_in * units * 16);
            for (int i = threadIdx.x; i < (CGP - a.cg_in) * units; i += kTcThreads) pz[i] = make_uint4(0, 0, 0, 0);
        }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    // Chain of dependent launches: the successor may be scheduled from now on (it waits for this grid's completion itself
    // before it touches a tensor); this CTA's prologue - barriers, the weight copy below - ran beside the predecessor's
    // tail, and only now do we wait for the predecessor's outputs.
    pdl_trigger();

    if (warp == 0) {
        // ===================== producer: weights once, then the hi half and the lo half of one block per tile ==========
        if (lane == 0) {
            mbar_expect_tx(wfull_bar, W_BYTES);
            bulk_g2s(smem_u32(w_smem), a.w, W_BYTES, wfull_bar);
            pdl_wait();
            uint32_t phase = 0;
            const uint32_t bytes = (uint32_t)(a.cg_in * units) * 16u;
            const uint4* in = reinterpret_cast<const uint4*>(a.in);
            for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
                for (int h = 0; h < 2; ++h) {
                    mbar_wait(empty_bar(h), phase ^ 1);
                    mbar_expect_tx(full_bar(h), bytes);
                    bulk_g2s(smem_u32(a_smem + h * half_bytes), in + (int64_t)tile * a.lay.blk_stride + (int64_t)h * a.cg_in * units, bytes, full_bar(h));
                }
                phase ^= 1;
            }
        }
    } else if (warp >= 4) {
        // ===================== MMA + epilogue: warpgroup wg owns accumulator rows [64 wg, 64 wg + 64) =====================
        const int wg = (warp >> 2) - 1, wq = warp & 3, q = lane & 3;
        const uint32_t row_off = (uint32_t)wg * 64u * 16u;
        const uint32_t w_addr = smem_u32(w_smem), a_addr = smem_u32(a_smem) + row_off;
        const uint32_t lbo_a = (uint32_t)units * 16u;
        const uint32_t tap16 = (uint32_t)a.tap * 16u;
        // accumulator rows of this thread -> (stream of the block, output row, column)
        int tr[2], slr[2], fr[2]; bool okr[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int row = wg * 64 + wq * 16 + (lane >> 2) + 8 * i;
            int t, sl, f;
            if (a.lay.kh3) { const int SW = a.lay.S * a.W; t = row / SW; sl = (row - t * SW) / a.W; f = row - t * SW - sl * a.W; }
            else { const int per = a.lay.T * a.lay.Wq; sl = row / per; t = (row - sl * per) / a.lay.Wq; f = row - sl * per - t * a.lay.Wq; }
            tr[i] = t; slr[i] = sl; fr[i] = f;
            okr[i] = row < a.m_valid && f < a.W;                       // (1,3): the pad column computes nothing that is kept
        }
        tc_warp_wait(wfull_bar, 0, lane);
        pdl_wait();                                                     // the stores below must follow the predecessor grid
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
            float acc[NP / 2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                tc_warp_wait(full_bar(h), phase, lane);
                wg_fence();
#pragma unroll
                for (int j = 0; j < 3; ++j) {
#pragma unroll
                    for (int qq = 0; qq < CGP / 2; ++qq) {
#pragma unroll
                        for (int wt = 0; wt < (h == 0 ? 2 : 1); ++wt) {      // hi half: (hi,hi), (hi,lo); lo half: (lo,hi)
                            const uint32_t w_t = w_addr + (wt == 1 ? (uint32_t)W_TERM : 0u);
                            const uint64_t ad = make_desc(a_addr + (uint32_t)h * (uint32_t)half_bytes + (uint32_t)(2 * qq) * lbo_a + (uint32_t)j * tap16,
                                                          lbo_a, 128u);
                            const uint64_t bd = make_desc(w_t + (uint32_t)((j * CGP + 2 * qq) * NP) * 16u, NP * 16u, 128u);
                            wg_mma<NP>(acc, ad, bd, (h | j | qq | wt) != 0);
                        }
                    }
                }
                wg_commit();
                wg_wait_all();
                __syncwarp();
                if (lane == 0) mbar_arrive(empty_bar(h));
            }
            phase ^= 1;

#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int t = tr[i], sl = slr[i], f = fr[i];
                const int n = tile * a.lay.S + sl;
                const bool live = okr[i] && n < a.n;
                if (a.out_f32) {
                    if (!live || f != 0) continue;
                    float* o = a.out_f32 + ((int64_t)n * a.rows_new + t) * 96;
#pragma unroll
                    for (int j = 0; j < NP / 8; ++j) {
                        const int c = j * 8 + 2 * q;
                        if (c >= 96) continue;
                        float2 r;
                        r.x = fmaf(acc[4 * j + 2 * i], s_sb[c], s_sb[NP + c]);
                        r.y = fmaf(acc[4 * j + 2 * i + 1], s_sb[c + 1], s_sb[NP + c + 1]);
                        *reinterpret_cast<float2*>(o + c) = r;
                    }
                    continue;
                }
                // unit of this position in the destination(s), plane 0.  Fused (1,2) pool: columns f and f^1 are adjacent
                // accumulator rows, i.e. lanes 4 apart in the fragment; the even one writes the maximum to column f/2.  The
                // maximum of the fp32 values, split afterwards, is the element the lexicographic (hi, lo) maximum of the
                // separate pool pass picks.
                const bool pooled = a.pool_f == 2;
                const bool writer = live && (!pooled || (f & 1) == 0);
                const int fo = pooled ? f >> 1 : f;
                int64_t dst[3];
#pragma unroll
                for (int kk = 0; kk < 3; ++kk)
                    dst[kk] = a.out_lay.S ? late_unit(a.out_lay, 0, live ? n : 0, t + a.out_toff[kk], fo)
                                          : kGuard + ((int64_t)(live ? n : 0) * a.rows_new + t) * (a.W + 1) + f;
                const int64_t pstride = a.out_lay.S ? (int64_t)a.out_lay.units : a.out_plane;
#pragma unroll
                for (int j = 0; j < NP / 8; ++j) {
                    const int g = j, c = g * 8 + 2 * q;
                    float y0 = fmaf(acc[4 * j + 2 * i], s_sb[c], s_sb[NP + c]);
                    float y1 = fmaf(acc[4 * j + 2 * i + 1], s_sb[c + 1], s_sb[NP + c + 1]);
                    if (a.apply_act) { y0 = act(y0); y1 = act(y1); }
                    if (pooled) {
                        y0 = fmaxf(y0, __shfl_xor_sync(0xffffffffu, y0, 4));
                        y1 = fmaxf(y1, __shfl_xor_sync(0xffffffffu, y1, 4));
                    }
                    if (g >= a.cg_out || !writer) continue;
                    const __half h0 = __float2half_rn(y0), h1 = __float2half_rn(y1);
                    const __half2 hh = __halves2half2(h0, h1);
                    const __half2 ll = __floats2half2_rn(y0 - __half2float(h0), y1 - __half2float(h1));
                    const uint32_t hw = *reinterpret_cast<const uint32_t*>(&hh), lw = *reinterpret_cast<const uint32_t*>(&ll);
#pragma unroll
                    for (int kk = 0; kk < 3; ++kk)
                        if (a.out[kk]) {
                            uint4* o = reinterpret_cast<uint4*>(a.out[kk]) + dst[kk];
                            reinterpret_cast<uint32_t*>(o + (int64_t)g * pstride)[q] = hw;
                            reinterpret_cast<uint32_t*>(o + (int64_t)(a.cg_out + g) * pstride)[q] = lw;
                        }
                }
            }
        }
    }
}

// ---------------------------------------------------------------- max-pool on fp16 planes
// split != 0: planes [0, cg) hold hi parts and [cg, 2cg) lo parts of the same values; the pooled element is the one
// with the largest hi + lo, i.e. the lexicographic maximum of (hi, lo) since |lo| <= ulp(hi)/2.
struct PoolOut { __half* p[3]; int toff[3]; int out_T; LateLay lay = {0, 0, 0, 0, 0, 0}; };   // out_T == 0: plain [n][t_out][wp_out] into p[0]; lay.S > 0: block-major destination
__global__ void __launch_bounds__(256) tc_pool_kernel(const __half* in, int64_t in_plane, PoolOut po, int64_t out_plane,
                                                      int n, int t_in, int w_in, int cg, int pt, int pf, int split) {
    __half* const out = po.p[0];
    pdl_trigger();
    pdl_wait();                 // dependent launch inside the late chain (no-op otherwise)
    const int t_out = t_in / pt, w_out = w_in / pf;
    const int wp_in = w_in + 1, wp_out = w_out + 1;
    const int64_t per_out = (int64_t)t_out * wp_out;
    const int64_t total = (int64_t)n * per_out * cg;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        const int64_t p = i % ((int64_t)n * per_out);
        const int g = (int)(i / ((int64_t)n * per_out));
        const int f = (int)(p % wp_out);
        const int64_t r = p / wp_out;
        const int t = (int)(r % t_out);
        const int64_t s = r / t_out;
        uint4 res = make_uint4(0, 0, 0, 0), res_lo = make_uint4(0, 0, 0, 0);
        if (f < w_out) {
            __half mh[8], ml[8];
            bool first = true;
            for (int da = 0; da < pt; ++da)
                for (int db = 0; db < pf; ++db) {
                    const int64_t pi = s * (int64_t)t_in * wp_in + (int64_t)(t * pt + da) * wp_in + (f * pf + db);
                    const uint4 v = __ldg(reinterpret_cast<const uint4*>(in) + (int64_t)g * in_plane + kGuard + pi);
                    uint4 vl = make_uint4(0, 0, 0, 0);
                    if (split) vl = __ldg(reinterpret_cast<const uint4*>(in) + (int64_t)(cg + g) * in_plane + kGuard + pi);
                    const __half* hv = reinterpret_cast<const __half*>(&v);
                    const __half* lv = reinterpret_cast<const __half*>(&vl);
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        const bool take = first || __hgt(hv[u], mh[u]) || (__heq(hv[u], mh[u]) && __hgt(lv[u], ml[u]));
                        if (take) { mh[u] = hv[u]; ml[u] = lv[u]; }
                    }
                    first = false;
                }
            res = *reinterpret_cast<uint4*>(mh);
            res_lo = *reinterpret_cast<uint4*>(ml);
        }
        if (po.out_T == 0) {
            reinterpret_cast<uint4*>(out)[(int64_t)g * out_plane + kGuard + p] = res;
            if (p == 0) reinterpret_cast<uint4*>(out)[(int64_t)g * out_plane + kGuard - 1] = make_uint4(0, 0, 0, 0);
            if (split) {
                reinterpret_cast<uint4*>(out)[(int64_t)(cg + g) * out_plane + kGuard + p] = res_lo;
                if (p == 0) reinterpret_cast<uint4*>(out)[(int64_t)(cg + g) * out_plane + kGuard - 1] = make_uint4(0, 0, 0, 0);
            }
        } else {
#pragma unroll
            for (int k = 0; k < 3; ++k)
                if (po.p[k]) {
                    if (po.lay.S) {                                     // block-major: pad column untouched (zero since allocation)
                        if (f >= w_out) continue;
                        reinterpret_cast<uint4*>(po.p[k])[late_unit(po.lay, g, (int)s, t + po.toff[k], f)] = res;
                        if (split) reinterpret_cast<uint4*>(po.p[k])[late_unit(po.lay, cg + g, (int)s, t + po.toff[k], f)] = res_lo;
                        continue;
                    }
                    const int64_t q = kGuard + (s * po.out_T + t + po.toff[k]) * wp_out + f;
                    reinterpret_cast<uint4*>(po.p[k])[(int64_t)g * out_plane + q] = res;
                    if (split) reinterpret_cast<uint4*>(po.p[k])[(int64_t)(cg + g) * out_plane + q] = res_lo;
                }
        }
    }
}

// planes -> NHWC fp32 (debug / parity only)
__global__ void tc_unpack_kernel(const __half* in, int64_t plane, float* out, int n, int t, int w, int c, int split) {
    const int wp = w + 1;
    const int64_t total = (int64_t)n * t * w * c;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int ch = (int)(i % c);
        int64_t r = i / c;
        const int f = (int)(r % w); r /= w;
        const int tt = (int)(r % t);
        const int64_t s = r / t;
        const int64_t p = s * (int64_t)t * wp + (int64_t)tt * wp + f;
        float v = __half2float(in[((int64_t)(ch >> 3) * plane + kGuard + p) * 8 + (ch & 7)]);
        if (split) v += __half2float(in[((int64_t)(c / 8 + (ch >> 3)) * plane + kGuard + p) * 8 + (ch & 7)]);
        out[i] = v;
    }
}

struct TcLayerGeom { int T, W, cg, cgp, np, T_out, rows, lo, tap_off[3]; };

inline int round8(int v) { return (v + 7) & ~7; }

template <int CGP, int NP, int TERMS>
int launch_tc(oww_ctx* ctx, const TcConvArgs& a, cudaStream_t s) {
    constexpr int split = TERMS == 3 ? 2 : 1, stages = TERMS == 3 ? 2 : 4;
    const size_t smem = (size_t)split * 3 * CGP * NP * 16 + (size_t)stages * split * CGP * a.rows * 16 +
                        8 * (2 * stages + 2) + 2 * NP * sizeof(float);
    if (smem > 227 * 1024) return oww_fail(ctx, OWW_EUNSUPPORTED, "tensor-core conv tile does not fit shared memory (%zu bytes)", smem);
    // the attribute is per (function, device): tracked per handle (one bit per kernel instance), not per process
    const uint32_t bit = 1u << (((CGP / 2 + NP / 16) + (TERMS == 3 ? 16 : 0)) & 31);     // distinct for the instances in use
    if (!(ctx->tc_attr_mask & bit)) {
        OWW_CUDA(ctx, cudaFuncSetAttribute(tc_conv_kernel<CGP, NP, TERMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        ctx->tc_attr_mask |= bit;
    }
    int grid = ctx->sm_count < a.n_tiles ? ctx->sm_count : a.n_tiles;
    tc_conv_kernel<CGP, NP, TERMS><<<grid, kTcThreads, smem, s>>>(a);
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

template <int CGP, int NP>
int launch_tc_blk(oww_ctx* ctx, const TcBlkArgs& a, cudaStream_t s) {
    const size_t smem = (size_t)2 * 3 * CGP * NP * 16 + (size_t)2 * CGP * a.lay.units * 16 + 8 * 6 + 2 * NP * sizeof(float);
    if (smem > 227 * 1024) return oww_fail(ctx, OWW_EUNSUPPORTED, "blocked late conv tile does not fit shared memory (%zu bytes)", smem);
    const uint32_t bit = 1u << (CGP / 2);
    if (!(ctx->tc_blk_attr_mask & bit)) {
        OWW_CUDA(ctx, cudaFuncSetAttribute(tc_conv_blk_kernel<CGP, NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        ctx->tc_blk_attr_mask |= bit;
    }
    const int grid = ctx->sm_count < a.n_tiles ? ctx->sm_count : a.n_tiles;
    cudaLaunchConfig_t cfg;
    std::memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kTcThreads); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = ctx->late_pdl ? 1 : 0;
    cfg.attrs = at; cfg.numAttrs = 1;
    OWW_CUDA(ctx, cudaLaunchKernelEx(&cfg, tc_conv_blk_kernel<CGP, NP>, a));
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

}  // namespace

// Host-side packing per layer 1..19: fp16 weights [3][CGP][NP][8] + padded scale/bias (TERMS = 1), and for the split
// variant the hi and lo blocks of W * 2^s (s per layer: max |W| * 2^s in [2^13, 2^14), so the lo parts are normal fp16
// numbers) with 2^-s folded exactly into the scale.
int oww_tc_pack_weights(oww_ctx* ctx, const float* h_blob) {
    size_t off = 0, total_h = 0, total_f = 0;
    for (int li = 1; li < OWW_N_CONV; ++li) {
        const ConvLayer& L = ctx->conv[li];
        const int cg = L.cin / 8, cgp = (cg + 1) & ~1, np = (L.cout + 15) & ~15;
        total_h += (size_t)3 * cgp * np * 8;
        total_f += 2 * (size_t)np;
    }
    std::vector<__half> hw(total_h), hw3(2 * total_h);
    std::vector<float> hf(total_f), hf3(total_f);
    size_t oh = 0, of = 0;
    for (int li = 0; li < OWW_N_CONV; ++li) {
        const ConvLayer& L = ctx->conv[li];
        const size_t nw = (size_t)L.kh * L.kw * L.cin * L.cout;
        const float* w = h_blob + off; const float* sc = w + nw; const float* bi = sc + L.cout;
        off += nw + 2 * (size_t)L.cout;
        if (li == 0) continue;
        const int cg = L.cin / 8, cgp = (cg + 1) & ~1, np = (L.cout + 15) & ~15;
        ctx->tc_w_off[li] = oh; ctx->tc_sb_off[li] = of;
        float amax = 0.f;
        for (size_t i = 0; i < nw; ++i) amax = std::fmax(amax, std::fabs(w[i]));
        int sexp = 0;
        if (amax > 0.f && std::isfinite(amax)) { int e; std::frexp(amax, &e); sexp = 14 - e; if (sexp > 24) sexp = 24; if (sexp < -8) sexp = -8; }
        const float up = std::ldexp(1.0f, sexp), down = std::ldexp(1.0f, -sexp);
        const size_t term = (size_t)3 * cgp * np * 8;
        std::fill(hw.begin() + oh, hw.begin() + oh + term, __float2half(0.f));     // pad octets of the chained order stay zero
        for (int j = 0; j < 3; ++j)
            for (int g = 0; g < cgp; ++g)
                for (int n = 0; n < np; ++n)
                    for (int e = 0; e < 8; ++e) {
                        const int c = g * 8 + e;
                        const float v = (c < L.cin && n < L.cout) ? w[((size_t)j * L.cin + c) * L.cout + n] : 0.f;
                        const size_t at = (((size_t)j * cgp + g) * np + n) * 8 + e;
                        // plain weights of a layer with an odd plane count: chained octet order (tc_conv_kernel, TERMS = 1)
                        int oc = j * cgp + g;
                        if ((cg & 1) && g < cg) oc = j == 0 ? (g < cg - 1 ? g : cg) : j == 1 ? (g == 0 ? cg - 1 : cg + g) : 2 * cg + g;
                        if (!(cg & 1) || g < cg) hw[oh + ((size_t)oc * np + n) * 8 + e] = __float2half_rn(v);
                        const __half hi = __float2half_rn(v * up);
                        hw3[2 * oh + at] = hi;
                        hw3[2 * oh + term + at] = __float2half_rn(v * up - __half2float(hi));
                    }
        oh += term;
        for (int n = 0; n < np; ++n) {
            hf[of + n] = n < L.cout ? sc[n] : 0.f; hf[of + np + n] = n < L.cout ? bi[n] : 0.f;
            hf3[of + n] = hf[of + n] * down; hf3[of + np + n] = hf[of + np + n];
        }
        of += 2 * (size_t)np;
    }
    if (!ctx->d_tc_w) OWW_CUDA(ctx, cudaMalloc(&ctx->d_tc_w, total_h * sizeof(__half)));
    if (!ctx->d_tc_sb) OWW_CUDA(ctx, cudaMalloc(&ctx->d_tc_sb, total_f * sizeof(float)));
    if (!ctx->d_tc_w3) OWW_CUDA(ctx, cudaMalloc(&ctx->d_tc_w3, 2 * total_h * sizeof(__half)));
    if (!ctx->d_tc_sb3) OWW_CUDA(ctx, cudaMalloc(&ctx->d_tc_sb3, total_f * sizeof(float)));
    OWW_CUDA(ctx, cudaMemcpy(ctx->d_tc_w, hw.data(), total_h * sizeof(__half), cudaMemcpyHostToDevice));
    OWW_CUDA(ctx, cudaMemcpy(ctx->d_tc_sb, hf.data(), total_f * sizeof(float), cudaMemcpyHostToDevice));
    OWW_CUDA(ctx, cudaMemcpy(ctx->d_tc_w3, hw3.data(), 2 * total_h * sizeof(__half), cudaMemcpyHostToDevice));
    OWW_CUDA(ctx, cudaMemcpy(ctx->d_tc_sb3, hf3.data(), total_f * sizeof(float), cudaMemcpyHostToDevice));
    return OWW_OK;
}

// Largest footprint over all layer outputs of a pass over n inputs of T0 mel rows: planes * plane pitch, in 16-byte
// units (tensors feeding a split layer hold hi and lo planes).
size_t oww_tc_act_units_T(const oww_ctx* ctx, int n, int T0) {
    size_t best = 0;
    int T = T0, W = 32;
    auto upd = [&](int t, int w, int c, int mult) {
        const size_t plane = ((size_t)kGuard + (size_t)n * t * (w + 1) + kGuardBack + 7) & ~(size_t)7;
        const size_t tot = (size_t)(c / 8) * mult * plane;
        if (tot > best) best = tot;
    };
    for (int li = 0; li < OWW_N_CONV; ++li) {
        const ConvLayer& L = ctx->conv[li];
        const int mult = li + 1 >= ctx->split_from ? 2 : 1;
        T -= (L.kh - 1);
        upd(T, W, L.cout, mult);
        if (L.pool_t) { T /= L.pool_t; W /= L.pool_f; upd(T, W, L.cout, mult); }
    }
    return best + 64;
}
size_t oww_tc_act_units(const oww_ctx* ctx, int n_windows) { return oww_tc_act_units_T(ctx, n_windows, OWW_WINDOW_ROWS); }

// Runs the pyramid in tensor-core mode on n inputs of T0 mel rows each (n windows of 76 rows, or n clips: the CNN is
// fully convolutional in time, SURVEY.md F10) -> d_emb [n][(T0 - 76) / 8 + 1][96] fp32.  Layers >= split_from take split
// (hi/lo) operands.  stop_layer >= 0: stop after that layer (and its pool) and unpack it to NHWC fp32 in d_dbg.
int oww_cnn_tc_pyramid_impl(oww_ctx* ctx, const WindowSrc& src, int n, int T0, int split_from, float* d_emb, int stop_layer,
                            float* d_dbg, const TailCapture* cap, cudaStream_t s);
int oww_cnn_tc_pyramid(oww_ctx* ctx, const WindowSrc& src, int n, float* d_emb, int stop_layer, float* d_dbg, cudaStream_t s) {
    return oww_cnn_tc_pyramid_impl(ctx, src, n, OWW_WINDOW_ROWS, ctx->split_from, d_emb, stop_layer, d_dbg, nullptr, s);
}
int oww_cnn_tc_pyramid_cap(oww_ctx* ctx, const WindowSrc& src, int n, float* d_emb, const TailCapture* cap, cudaStream_t s) {
    // tails of the layers inside the fused kernel (all below split_from: plain fp16 there as here) go to the group
    // layout through oww_inc_capture; tails of the incremental late layers (hi/lo) to the late template
    return oww_cnn_tc_pyramid_impl(ctx, src, n, OWW_WINDOW_ROWS, ctx->split_from, d_emb, -1, nullptr, cap, s);
}
int oww_cnn_tc_clip(oww_ctx* ctx, const float* d_mel, int n, int T, float* d_emb, cudaStream_t s) {
    WindowSrc src{d_mel, (int64_t)T * 32, nullptr, -1, 0, 0};
    const int W = (T - OWW_WINDOW_ROWS) / 8 + 1;
    return oww_cnn_tc_pyramid_impl(ctx, src, n, OWW_WINDOW_ROWS + 8 * (W - 1), ctx->split_from, d_emb, -1, nullptr, nullptr, s);
}
// same, the embeddings of input i landing at d_emb + i * out_rows * 96 (rows of a larger per-input array)
int oww_cnn_tc_clip_rows(oww_ctx* ctx, const WindowSrc& src, int n, int T, float* d_emb, int out_rows, cudaStream_t s) {
    ctx->tc_rows_out_override = out_rows;
    int rc = oww_cnn_tc_pyramid_impl(ctx, src, n, T, ctx->split_from, d_emb, -1, nullptr, nullptr, s);
    ctx->tc_rows_out_override = 0;
    return rc;
}

template <int TERMS>
static int dispatch_tc(oww_ctx* ctx, int cgp, int np, const TcConvArgs& a, cudaStream_t s) {
    if (cgp == 4 && np == 32) return launch_tc<4, 32, TERMS>(ctx, a, s);
    if (cgp == 4 && np == 48) return launch_tc<4, 48, TERMS>(ctx, a, s);
    if (cgp == 6 && np == 48) return launch_tc<6, 48, TERMS>(ctx, a, s);
    if (cgp == 6 && np == 80) return launch_tc<6, 80, TERMS>(ctx, a, s);
    if (cgp == 10 && np == 80) return launch_tc<10, 80, TERMS>(ctx, a, s);
    if (cgp == 10 && np == 96) return launch_tc<10, 96, TERMS>(ctx, a, s);
    if (cgp == 12 && np == 96) return launch_tc<12, 96, TERMS>(ctx, a, s);
    return oww_fail(ctx, OWW_EUNSUPPORTED, "no tensor-core conv instance for cgp=%d np=%d", cgp, np);
}

int oww_cnn_tc_pyramid_impl(oww_ctx* ctx, const WindowSrc& src, int n, int T0, int split_from, float* d_emb, int stop_layer,
                            float* d_dbg, const TailCapture* cap, cudaStream_t s) {
    if (oww_tc_act_units_T(ctx, n, T0) > ctx->tc_act_units)
        return oww_fail(ctx, OWW_ENOMEM, "tensor-core activation scratch too small for %d x %d rows", n, T0);
    __half* bufs[2] = {reinterpret_cast<__half*>(ctx->d_tc_act[0]), reinterpret_cast<__half*>(ctx->d_tc_act[1])};
    int cur = 0;
    int T = T0, W = 32;
    auto plane_units = [&](int t, int w) { return (int64_t)((kGuard + (int64_t)n * t * (w + 1) + kGuardBack + 7) & ~7LL); };
    int64_t in_plane = 0;
    for (int li = 0; li < OWW_N_CONV; ++li) {
        const ConvLayer& L = ctx->conv[li];
        const int T_out = T - (L.kh - 1);
        const bool last = li == OWW_N_CONV - 1;
        const bool in_split = li >= split_from;              // this layer takes hi/lo operands
        const bool out_split = li + 1 >= split_from && !last; // the tensor it leaves feeds a split layer
        const int64_t out_plane = plane_units(T_out, W);
        if (li == 0) {
            if (out_split) return oww_fail(ctx, OWW_EUNSUPPORTED, "split_from must be >= 2");
            Tc0Args a{src, n, T_out, L.d_w, L.d_scale, L.d_bias, bufs[cur], out_plane};
            const int64_t total = (int64_t)n * T_out * 33;
            unsigned grid = (unsigned)((total + 255) / 256);
            if (grid > (unsigned)ctx->sm_count * 16) grid = ctx->sm_count * 16;
            tc_conv0_kernel<<<grid, 256, 0, s>>>(a);
            OWW_LAUNCH_CHECK(ctx);
        } else {
            const int cg = L.cin / 8, cgp = (cg + 1) & ~1, np = (L.cout + 15) & ~15;
            const int Wp = W + 1;
            TcConvArgs a;
            std::memset(&a, 0, sizeof(a));
            a.in = bufs[cur ^ 1]; a.in_plane = in_plane;
            a.out = bufs[cur]; a.out_plane = out_plane;
            a.out_f32 = last ? d_emb : nullptr;
            if (in_split) {
                a.w = reinterpret_cast<const __half*>(ctx->d_tc_w3) + 2 * ctx->tc_w_off[li];
                a.scale = ctx->d_tc_sb3 + ctx->tc_sb_off[li];
            } else {
                a.w = reinterpret_cast<const __half*>(ctx->d_tc_w) + ctx->tc_w_off[li];
                a.scale = ctx->d_tc_sb + ctx->tc_sb_off[li];
            }
            a.bias = a.scale + np;
            a.n = n; a.T = T; a.W = W; a.T_out = T_out;
            if (L.kw == 3) { a.lo = 1; a.tap_off[0] = 0; a.tap_off[1] = 1; a.tap_off[2] = 2; a.rows = round8(128 + 2); }
            else { a.lo = 0; a.tap_off[0] = 0; a.tap_off[1] = Wp; a.tap_off[2] = 2 * Wp; a.rows = round8(128 + 2 * Wp); }
            a.cg_in = cg; a.cg_out = L.cout / 8; a.apply_act = last ? 0 : 1;
            a.p_in = (int64_t)n * T * Wp;
            a.n_tiles = (int)((a.p_in + 127) / 128);
            a.out_split = out_split ? 1 : 0;
            a.rows_out = (last && ctx->tc_rows_out_override) ? ctx->tc_rows_out_override : T_out;
            int rc = in_split ? dispatch_tc<3>(ctx, cgp, np, a, s) : dispatch_tc<1>(ctx, cgp, np, a, s);
            if (rc) return rc;
        }
        T = T_out; in_plane = out_plane; cur ^= 1;
        if (L.pool_t && !last) {
            const int T2 = T / L.pool_t, W2 = W / L.pool_f;
            const int64_t op = plane_units(T2, W2);
            const int cgo = L.cout / 8;
            const int64_t total = (int64_t)n * T2 * (W2 + 1) * cgo;
            unsigned grid = (unsigned)((total + 255) / 256);
            if (grid > (unsigned)ctx->sm_count * 16) grid = ctx->sm_count * 16;
            PoolOut pout{{bufs[cur], nullptr, nullptr}, {0, 0, 0}, 0};
            tc_pool_kernel<<<grid, 256, 0, s>>>(bufs[cur ^ 1], in_plane, pout, op, n, T, W, cgo, L.pool_t, L.pool_f, out_split ? 1 : 0);
            OWW_LAUNCH_CHECK(ctx);
            T = T2; W = W2; in_plane = op; cur ^= 1;
        }
        if (cap && cap->n_win > 0 && !last) {
            // the tensor just produced feeds layer li+1; if that is a (3,1) conv its last two rows are the tails
            int rc = oww_inc_capture(ctx, li, bufs[cur ^ 1], in_plane, T, W, cap->win0, cap->n_win, cap->stream0, cap->ids, s);
            if (rc) return rc;
            if (cap->late && (rc = oww_late_capture(ctx, li + 1, bufs[cur ^ 1], in_plane, T, W, s))) return rc;
        }
        if (li == stop_layer && !last) {
            const int64_t total = (int64_t)n * T * W * L.cout;
            tc_unpack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(bufs[cur ^ 1], in_plane, d_dbg, n, T, W, L.cout, out_split ? 1 : 0);
            OWW_LAUNCH_CHECK(ctx);
            return OWW_OK;
        }
    }
    return OWW_OK;
}

// ================================================================================================
// Incremental late layers (cnn_mode 3 with split_from < 20).
//
// The fused step kernel (cnn_tc_inc.cu) runs the frontend and conv layers 0 .. L0-1 of the 8 new mel rows in shared
// memory and leaves the pooled output of layer L0-1 (2 new rows per stream at L0 = 11) in HBM as fp16 hi/lo planes.
// Layers L0 .. 19 - 1.3 of the 5.6 MMAC per frame, but the ones whose fp16 rounding dominates the embedding error -
// then run here as the SAME tensor-core conv / pool kernels as the window mode, with split (hi/lo) operands, on "windows"
// that are the incremental rows of every stream: a (3,1) layer's input holds [2 tail rows | new rows] per stream, and
// every layer mirrors its new rows into the buffer(s) where they are tails of the following step(s) (two buffers for
// tensors that gain two rows per step, three for the one that gains a single row), so no copy or shift pass exists.
// A reset writes the tails of the all-ones window (template) into the slots the stream's next step reads.
// ================================================================================================
namespace {

__global__ void late_capture_kernel(const uint4* planes, int64_t plane_pitch, int T, int Wp, int n_planes, uint4* tmpl) {
    // last two rows of window 0 of every plane -> tmpl[plane][row][f]
    const int total = n_planes * 2 * Wp;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int f = i % Wp, r = (i / Wp) % 2, pl = i / (2 * Wp);
        tmpl[i] = planes[(int64_t)pl * plane_pitch + kGuard + (int64_t)(T - 2 + r) * Wp + f];
    }
}

}  // namespace

int oww_late_alloc(oww_ctx* ctx) {
    // geometry of the incremental tensors X_l (input of conv layer l), l = L0 .. 19
    for (auto& X : ctx->late_x) for (auto& b : X.buf) { cudaFree(b); b = nullptr; }
    for (auto& b : ctx->d_late_tmp) { cudaFree(b); b = nullptr; }
    cudaFree(ctx->d_late_template); ctx->d_late_template = nullptr;
    ctx->late_active = false;
    const int L0 = ctx->split_from;
    if (ctx->cfg.cnn_mode != OWW_CNN_TC_INCREMENTAL || L0 >= OWW_N_CONV) return OWW_OK;
    if (L0 < 2 || ctx->conv[L0].kh != 1 || !ctx->conv[L0 - 1].pool_t)
        return oww_fail(ctx, OWW_EUNSUPPORTED, "split_from=%d: the incremental split must start at a (1,3) layer that follows a pool (3, 7, 11, 15)", L0);
    const int n = ctx->n_streams;
    int rows = 8, W = 32;
    for (int l = 0; l < L0; ++l) if (ctx->conv[l].pool_t) { rows /= ctx->conv[l].pool_t; W /= ctx->conv[l].pool_f; }
    size_t tmpl_units = 0, tmp_units = 0;
    // the block-major kernel is instantiated for 72 / 96 -> 96 channels (every layer from 11 on)
    bool blocked = ctx->late_blocked_ok;
    for (int l = L0; l < OWW_N_CONV; ++l) if ((ctx->conv[l].cin != 96 && ctx->conv[l].cin != 72) || ctx->conv[l].cout != 96) blocked = false;
    for (int l = L0; l < OWW_N_CONV; ++l) {
        const ConvLayer& C = ctx->conv[l];
        oww_ctx::LateTensor& X = ctx->late_x[l];
        const bool kh3 = C.kh == 3;
        X.rows_new = rows; X.W = W; X.cg = C.cin / 8;
        X.T_buf = rows + (kh3 ? 2 : 0);
        X.n_buf = kh3 ? (rows == 1 ? 3 : 2) : 1;
        // block-major layout (tc_conv_blk_kernel): S streams per block so that the block's positions fill the 128
        // accumulator rows ((3,1): rows*S*W outputs, and the whole [T][S][W] block <= 256 units per plane)
        X.lay = LateLay{0, 0, 0, 0, 0, 0};
        size_t buf_units;
        if (blocked) {
            LateLay& Y = X.lay;
            Y.kh3 = kh3 ? 1 : 0; Y.T = X.T_buf; Y.Wq = kh3 ? W : W + 1;
            Y.S = std::max(1, 128 / (rows * Y.Wq));
            if (kh3) while (Y.S > 1 && X.T_buf * Y.S * W > 256) Y.S /= 2;
            const int tap = kh3 ? Y.S * W : 1;
            Y.units = round8(std::max((kh3 ? 0 : 1) + Y.T * Y.S * Y.Wq, 2 * tap + 128));
            Y.blk_stride = (int64_t)2 * X.cg * Y.units;
            buf_units = (size_t)((n + Y.S - 1) / Y.S) * Y.blk_stride;
            X.plane = 0;
        } else {
            X.plane = (int64_t)((kGuard + (int64_t)n * X.T_buf * (W + 1) + kGuardBack + 7) & ~7LL);
            buf_units = (size_t)2 * X.cg * X.plane;
        }
        X.tmpl_off = kh3 ? (int)tmpl_units : -1;
        if (kh3) tmpl_units += (size_t)2 * X.cg * 2 * (W + 1);
        for (int k = 0; k < X.n_buf; ++k) {
            OWW_CUDA(ctx, cudaMalloc(&X.buf[k], buf_units * 16));
            OWW_CUDA(ctx, cudaMemset(X.buf[k], 0, buf_units * 16));
        }
        if (C.pool_t) {
            const size_t u = (size_t)2 * (C.cout / 8) * ((kGuard + (size_t)n * rows * (W + 1) + kGuardBack + 7) & ~(size_t)7);
            if (u > tmp_units) tmp_units = u;
            rows /= C.pool_t; W /= C.pool_f;
        }
    }
    if (tmp_units) {
        OWW_CUDA(ctx, cudaMalloc(&ctx->d_late_tmp[0], tmp_units * 16));
        OWW_CUDA(ctx, cudaMemset(ctx->d_late_tmp[0], 0, tmp_units * 16));
    }
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_late_template, std::max<size_t>(tmpl_units, 1) * 16));
    OWW_CUDA(ctx, cudaMemset(ctx->d_late_template, 0, std::max<size_t>(tmpl_units, 1) * 16));
    ctx->late_step = 0;
    ctx->late_active = true;
    return OWW_OK;
}

// Layers L0 .. 19 for every stream's new rows of this step; d_emb [n_streams][96].
int oww_late_chain(oww_ctx* ctx, float* d_emb, cudaStream_t s) {
    const int L0 = ctx->split_from, n = ctx->n_streams;
    const long k = ctx->late_step;
    for (int l = L0; l < OWW_N_CONV; ++l) {
        const ConvLayer& C = ctx->conv[l];
        const oww_ctx::LateTensor& X = ctx->late_x[l];
        const bool last = l == OWW_N_CONV - 1;
        const int cg = C.cin / 8, cgp = (cg + 1) & ~1, np = (C.cout + 15) & ~15;
        const int W = X.W, Wp = W + 1, T = X.T_buf, T_out = X.rows_new;
        // where the output rows go: the next layer's input buffers (or the unpooled temp)
        auto route = [&](const oww_ctx::LateTensor& Y, __half** p, int* toff, int& n_out) {
            n_out = 0;
            if (Y.n_buf == 1) { p[0] = reinterpret_cast<__half*>(Y.buf[0]); toff[0] = 0; n_out = 1; return; }
            const int r = Y.rows_new;                       // 2 -> two buffers, 1 -> three
            for (int m = 0; m < Y.n_buf; ++m) {
                p[m] = reinterpret_cast<__half*>(Y.buf[(k + m) % Y.n_buf]);
                toff[m] = 2 - m * r;                        // this step: behind the two tails; later steps: as their tails
            }
            n_out = Y.n_buf;
        };
        const int64_t tmp_plane = (int64_t)((kGuard + (int64_t)n * T_out * Wp + kGuardBack + 7) & ~7LL);
        int rc;
        bool pool_fused = false;
        if (X.lay.S) {
            // block-major input: one tile per block of S streams
            TcBlkArgs b;
            std::memset(&b, 0, sizeof(b));
            b.in = reinterpret_cast<const __half*>(X.buf[X.n_buf == 1 ? 0 : (int)(k % X.n_buf)]);
            b.lay = X.lay;
            b.w = reinterpret_cast<const __half*>(ctx->d_tc_w3) + 2 * ctx->tc_w_off[l];
            b.scale = ctx->d_tc_sb3 + ctx->tc_sb_off[l]; b.bias = b.scale + np;
            b.n = n; b.W = W; b.rows_new = T_out;
            b.m_valid = T_out * X.lay.S * X.lay.Wq;
            b.tap = C.kh == 3 ? X.lay.S * W : 1;
            b.cg_in = cg; b.cg_out = C.cout / 8; b.apply_act = last ? 0 : 1;
            b.n_tiles = (n + X.lay.S - 1) / X.lay.S;
            const bool fuse_pool = !last && C.pool_t == 1 && C.pool_f == 2 && X.lay.kh3 && (W & 1) == 0 && ctx->late_x[l + 1].lay.S > 0;
            if (last) {
                b.out_f32 = d_emb;
            } else if (fuse_pool) {
                // (1,2) max-pool in the epilogue: straight into the next layer's tensor, no temp, no pool launch
                const oww_ctx::LateTensor& Y = ctx->late_x[l + 1];
                int n_out = 0;
                route(Y, b.out, b.out_toff, n_out);
                b.out_lay = Y.lay;
                b.pool_f = 2;
                pool_fused = true;
            } else if (C.pool_t) {
                b.out[0] = reinterpret_cast<__half*>(ctx->d_late_tmp[0]);
                b.out_plane = tmp_plane;
            } else {
                const oww_ctx::LateTensor& Y = ctx->late_x[l + 1];
                int n_out = 0;
                route(Y, b.out, b.out_toff, n_out);
                b.out_lay = Y.lay;
            }
            if (cgp == 12 && np == 96) rc = launch_tc_blk<12, 96>(ctx, b, s);
            else if (cgp == 10 && np == 96) rc = launch_tc_blk<10, 96>(ctx, b, s);
            else rc = oww_fail(ctx, OWW_EUNSUPPORTED, "no block-major late conv instance for cgp=%d np=%d", cgp, np);
            if (rc) return rc;
        } else {
        TcConvArgs a;
        std::memset(&a, 0, sizeof(a));
        a.in = reinterpret_cast<const __half*>(X.buf[X.n_buf == 1 ? 0 : (int)(k % X.n_buf)]);
        a.in_plane = X.plane;
        a.w = reinterpret_cast<const __half*>(ctx->d_tc_w3) + 2 * ctx->tc_w_off[l];
        a.scale = ctx->d_tc_sb3 + ctx->tc_sb_off[l]; a.bias = a.scale + np;
        a.n = n; a.T = T; a.W = W; a.T_out = T_out;
        if (C.kw == 3) { a.lo = 1; a.tap_off[0] = 0; a.tap_off[1] = 1; a.tap_off[2] = 2; a.rows = round8(128 + 2); }
        else { a.lo = 0; a.tap_off[0] = 0; a.tap_off[1] = Wp; a.tap_off[2] = 2 * Wp; a.rows = round8(128 + 2 * Wp); }
        a.cg_in = cg; a.cg_out = C.cout / 8; a.apply_act = last ? 0 : 1;
        a.p_in = (int64_t)n * T * Wp;
        a.n_tiles = (int)((a.p_in + 127) / 128);
        a.rows_out = T_out;
        if (last) {
            a.out_f32 = d_emb;
        } else if (C.pool_t) {
            a.out = reinterpret_cast<__half*>(ctx->d_late_tmp[0]);
            a.out_plane = tmp_plane;
            a.out_split = 1;
        } else {
            const oww_ctx::LateTensor& Y = ctx->late_x[l + 1];
            __half* p[3] = {nullptr, nullptr, nullptr}; int toff[3] = {0, 0, 0}; int n_out = 0;
            route(Y, p, toff, n_out);
            a.out = p[0]; a.out_plane = Y.plane; a.out_split = 1;
            a.out_T = Y.T_buf; a.out_toff = toff[0];
            for (int m = 1; m < n_out; ++m) { a.out_b[m - 1] = p[m]; a.out_b_toff[m - 1] = toff[m]; }
        }
        rc = dispatch_tc<3>(ctx, cgp, np, a, s);
        if (rc) return rc;
        }
        if (C.pool_t && !last && !pool_fused) {
            const oww_ctx::LateTensor& Y = ctx->late_x[l + 1];
            PoolOut po{{nullptr, nullptr, nullptr}, {0, 0, 0}, Y.T_buf};
            po.lay = Y.lay;
            int n_out = 0;
            route(Y, po.p, po.toff, n_out);
            const int cgo = C.cout / 8;
            const int64_t total = (int64_t)n * Y.rows_new * (Y.W + 1) * cgo;
            unsigned grid = (unsigned)((total + 255) / 256);
            if (grid > (unsigned)ctx->sm_count * 16) grid = ctx->sm_count * 16;
            cudaLaunchConfig_t cfg;
            std::memset(&cfg, 0, sizeof(cfg));
            cfg.gridDim = dim3(grid); cfg.blockDim = dim3(256); cfg.stream = s;
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
            at[0].val.programmaticStreamSerializationAllowed = ctx->late_pdl ? 1 : 0;
            cfg.attrs = at; cfg.numAttrs = 1;
            OWW_CUDA(ctx, cudaLaunchKernelEx(&cfg, tc_pool_kernel, reinterpret_cast<const __half*>(ctx->d_late_tmp[0]), tmp_plane, po,
                                             Y.plane, n, T_out, W, cgo, C.pool_t, C.pool_f, 1));
            OWW_LAUNCH_CHECK(ctx);
        }
    }
    ctx->late_step = k + 1;
    return OWW_OK;
}

// Called by the full-window pyramid on the all-ones window (template pass): remember the last two rows of every
// tensor that carries tails in the incremental chain.
int oww_late_capture(oww_ctx* ctx, int next_layer, const void* planes, int64_t plane_pitch, int T, int W, cudaStream_t s) {
    if (!ctx->late_active || next_layer < ctx->split_from || next_layer >= OWW_N_CONV) return OWW_OK;
    const oww_ctx::LateTensor& X = ctx->late_x[next_layer];
    if (X.tmpl_off < 0) return OWW_OK;
    if (W != X.W) return oww_fail(ctx, OWW_EINVAL, "late capture: width mismatch at layer %d", next_layer);
    late_capture_kernel<<<4, 256, 0, s>>>(reinterpret_cast<const uint4*>(planes), plane_pitch, T, W + 1, 2 * X.cg,
                                         reinterpret_cast<uint4*>(ctx->d_late_template) + X.tmpl_off);
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}
