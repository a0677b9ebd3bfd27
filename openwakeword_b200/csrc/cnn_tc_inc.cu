// K2 (incremental tensor-core path): ONE persistent kernel runs all 20 layers of the speech-embedding
// CNN for the 8 new mel rows of every stream, with every activation in shared memory.
//
// Why this is exact.  The CNN (reference embedding_model.onnx, openwakeword/utils.py:90-93 of the original project,
// spec notebooks/converting_google_speech_embedding_model.ipynb:871-951) is fully convolutional along
// time with total stride 8, and the reference evaluates it on a 76-row window that slides by exactly
// 8 rows per 80 ms chunk (utils.py:437-443; SURVEY.md F10).  So the newest window's activations are
// the previous window's shifted by 8/4/2/1 rows per level: only the LAST 8/4/2/1 rows of each layer
// are new, and a (3,1) convolution needs just the last two rows of its input from the previous step
// ("tails", 10 small tensors per stream, kept in HBM between steps).  The first step after a reset
// (5 mel rows, SURVEY.md F8) is computed with the full-window kernels (cnn_tc.cu), which also prime
// the tails.
//
// Mapping.  A CTA owns a group of G streams.  Positions are ordered (t, stream, f) with one zero pad
// column, stored as fp16 channel-group planes (16-byte units) in two smem buffers X/Y, exactly the
// no-swizzle K-major core-matrix order of a wgmma operand.  For layer l the A operand is read IN PLACE from the
// previous layer's output planes: a conv tap is a shift of the descriptor start address
// ((1,3): -1/0/+1 units; (3,1): 0/GWp/2GWp units), so there is no im2col and no copy.  Weights
// (+ folded BN scale/bias) of layer l+1 stream into a double buffer by cp.async.bulk while layer l
// computes.  The 16 compute warps form 4 warpgroups; each takes 64-position tiles of the layer in turn, accumulates
// them with wgmma in registers, applies BN + leaky + clamp, writes the next layer's planes to smem and spills the new
// tails to HBM.  Max-pools are an smem->smem pass of the same warps.  Warp 16 = weight producer.
#include "oww_internal.h"
#include "tc_common.cuh"
#include "mel_device.cuh"
#include <cstring>
#include <type_traits>

namespace {

constexpr int kIncEpiWarps = 16;                         // compute warps: four MMA warpgroups
constexpr int kIncThreads = (kIncEpiWarps + 1) * 32;      // 544: + the weight producer
constexpr int kIncMaxG = 7;
constexpr int kMelNF = 2;                                  // frames a warp of the fused frontend processes at once

__device__ __forceinline__ __half2 u32_as_half2(uint32_t v) {
    return __halves2half2(__ushort_as_half((unsigned short)(v & 0xFFFFu)), __ushort_as_half((unsigned short)(v >> 16)));
}

struct IncArgs {
    IncPlan plan;
    const float* mel; const int* mel_count; int64_t mel_stride; int mel_mask; int back;
    const float* w0; const float* s0; const float* b0;       // layer 0 (fp32, CUDA cores)
    const uint8_t* wblob;                                     // packed per layer: fp16 [3][CGP][NP][8] | scale[NP] | bias[NP]
    const uint4* tails_in; uint4* tails_out;                  // [n_groups][tail_units]
    float* emb;                                               // [B][96]
    int B;
    long long* dbg_clock;                                     // optional: 21 clock64 stamps of CTA 0's first group
    // ---- fused step (fused != 0): the same launch also runs the log-mel frontend before layer 0, appends the embedding
    //      to the feature ring and evaluates every head, i.e. PCM in -> scores out ----
    int fused;
    const int16_t* pcm; int64_t pcm_stride;                   // this step's 1280 samples per stream
    int16_t* tail; int* seen; float* mel_rw; int* mel_count_rw;
    const float* mel_window; const float2* mel_twiddle; const int* mel_start; const int* mel_len; const float* mel_w; int mel_kmax;
    float* feat_ring; int64_t feat_stride; int feat_mask; int* feat_count;
    const HeadDev* heads; int n_heads; int max_n_in;
    float* scores; int score_stride;
    int hring_off, hslot_bytes, hns;                          // smem ring the producer streams the heads' first-layer weights through
    const Gate* gates; int n_gates;                           // conditional verifier pairs, applied after the heads phase
    // cut plan (plan.n_layers < 20): the pooled output of the last fused layer leaves the kernel as fp16 hi/lo planes in
    // the block-major layout of the first incremental late layer's input (gx_lay, cnn_tc.cu), or - fallback - the
    // plane-major window layout [plane][stream][row][f + pad]
    uint4* gx; int64_t gx_plane; LateLay gx_lay;     // gx_lay.S > 0: block-major destination (cnn_tc.cu)
};

// Rows of a later head layer (K x D floats) per ring chunk: a multiple of 4 rows (16-byte chunk starts) that fits a slot.
__device__ __forceinline__ int head_rows(int slot_bytes, int K, int D) {
    const int r = (slot_bytes / (D * 4)) & ~3;
    return r < K ? r : K;
}

// kNL: number of conv layers the kernel runs, fixed at compile time (20 = whole CNN, 11 / 15 = cuts before the
// split-operand layers) or 0 = read from the plan (any other cut).  With the count known the full-depth instance
// carries none of the cut layer's code.
template <int kNL>
__global__ void __launch_bounds__(kIncThreads, 1) tc_inc_kernel(const __grid_constant__ IncArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    const IncPlan& P = a.plan;
    const int NL = kNL ? kNL : P.n_layers;
    const int G = P.G;
    // [0, 2048): barriers, per-group stream state, layer-0 weights.  Activations grow from 2048 up; the per-layer weight
    // slots sit at the top of the arena (offsets in the plan, checked against the activation extents).
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem);
    float* s_l0 = reinterpret_cast<float*>(smem + 704);              // 9*24 + 24 + 24 floats: [704, 1760)
    uint4* act0 = reinterpret_cast<uint4*>(smem + 2048);            // activation arena; tensors at plan offsets

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
    const int lane = threadIdx.x & 31;
    const uint32_t bar0 = smem_u32(bars);
    auto wfull = [&](int i) { return bar0 + 8u * i; };
    auto wempty = [&](int i) { return bar0 + 8u * (2 + i); };
    const uint32_t tails_bar = bar0 + 8u * 4;                         // 14 barriers: [0, 112)
    const uint32_t hstart_bar = bar0 + 8u * 5;
    auto hfull = [&](int i) { return bar0 + 8u * (6 + i); };
    auto hempty = [&](int i) { return bar0 + 8u * (10 + i); };

    if (threadIdx.x == 0) {
        for (int i = 0; i < 2; ++i) { mbar_init(wfull(i), 1); mbar_init(wempty(i), 1); }
        mbar_init(tails_bar, 1);
        mbar_init(hstart_bar, 1);
        for (int i = 0; i < 4; ++i) { mbar_init(hfull(i), 1); mbar_init(hempty(i), kIncEpiWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = threadIdx.x; i < 9 * 24; i += kIncThreads) s_l0[i] = a.w0[i];
    if (threadIdx.x < 24) { s_l0[216 + threadIdx.x] = a.s0[threadIdx.x]; s_l0[240 + threadIdx.x] = a.b0[threadIdx.x]; }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    if (warp == kIncEpiWarps) {
        // ===================== weight producer =====================
        if (lane == 0) {
            uint32_t par[2] = {0, 0};
            uint32_t hs_par = 0, he_par = 0; int hchunk = 0;
            for (int grp = blockIdx.x; grp < P.n_groups; grp += gridDim.x) {
                for (int l = 1; l < NL; ++l) {
                    const int i = l & 1;
                    mbar_wait(wempty(i), par[i] ^ 1);
                    mbar_expect_tx(wfull(i), (uint32_t)P.L[l].w_bytes);
                    bulk_g2s(smem_u32(smem + P.L[l].w_smem), a.wblob + P.L[l].w_off, (uint32_t)P.L[l].w_bytes, wfull(i));
                    par[i] ^= 1;
                }
                if (a.fused && a.n_heads > 0) {
                    // heads phase: stream every head's first-layer matrix, one 96-row feature-row chunk at a time
                    mbar_wait(hstart_bar, hs_par); hs_par ^= 1;
                    for (int hh = 0; hh < a.n_heads; ++hh) {
                        const HeadDev& H = a.heads[hh];
                        const uint32_t bytes = (uint32_t)(96 * H.dims[1]) * 4u;
                        const float* W = H.blob + H.w_off[0];
                        for (int c = 0; c < H.n_in; ++c) {
                            const int slot = hchunk % a.hns;
                            mbar_wait(hempty(slot), ((he_par >> slot) & 1u) ^ 1u);
                            mbar_expect_tx(hfull(slot), bytes);
                            bulk_g2s(smem_u32(smem + a.hring_off + slot * a.hslot_bytes), W + (int64_t)c * 96 * H.dims[1], bytes, hfull(slot));
                            he_par ^= 1u << slot;
                            ++hchunk;
                        }
                        // the later (small) layers follow through the same ring, head_rows() weight rows at a time
                        for (int l = 1; l < H.n_layers; ++l) {
                            const int K = H.dims[l], D = H.dims[l + 1];
                            const int rows = head_rows(a.hslot_bytes, K, D);
                            const float* Wl = H.blob + H.w_off[l];
                            for (int k0 = 0; k0 < K; k0 += rows) {
                                const uint32_t cb = ((uint32_t)(min(rows, K - k0) * D) * 4u + 15u) & ~15u;
                                const int slot = hchunk % a.hns;
                                mbar_wait(hempty(slot), ((he_par >> slot) & 1u) ^ 1u);
                                mbar_expect_tx(hfull(slot), cb);
                                bulk_g2s(smem_u32(smem + a.hring_off + slot * a.hslot_bytes), Wl + (int64_t)k0 * D, cb, hfull(slot));
                                he_par ^= 1u << slot;
                                ++hchunk;
                            }
                        }
                    }
                }
            }
        }
    } else {
        // ===================== compute warps (512 threads): frontend, MMAs, epilogues, pools, heads =====================
        const int et = threadIdx.x;                               // 0..511
        uint32_t epar[2] = {0, 0};
        uint32_t epi_tails_par = 0, mma_tails_par = 0;
        uint32_t hf_par = 0; int hchunk_e = 0;
        for (int grp = blockIdx.x; grp < P.n_groups; grp += gridDim.x) {
            const uint4* tin = a.tails_in + (int64_t)grp * P.tail_units;
            uint4* tout = a.tails_out + (int64_t)grp * P.tail_units;
            int* s_cnt = reinterpret_cast<int*>(smem + 512);       // [0..7] mel row count, [8..15] feature count, before this step
            int* s_live = s_cnt + 16;                              // [0..7] stream exists, [8..15] it is fresh (first chunk after a reset)
            float* s_mel = reinterpret_cast<float*>(smem + P.scratch_off + 6144);   // [G][8][32] this step's mel rows
            if (a.dbg_clock && blockIdx.x == 0 && grp == 0 && et == 0) a.dbg_clock[101] = clock64();
            named_bar_sync(2, kIncEpiWarps * 32);                  // every warp is done with the previous group's s_live / s_cnt
            if (et < G) {
                const int b = grp * G + et;
                s_live[et] = b < a.B;
            }
            named_bar_sync(2, kIncEpiWarps * 32);
            if (a.fused) {
                // ===== frontend: log-mel of this step's 8 frames per stream (K1 inside the step kernel) =====
                uint8_t* sc = smem + P.scratch_off;
                float2* s_tw = reinterpret_cast<float2*>(sc);
                float* s_win = reinterpret_cast<float*>(sc + 4096);
                uint8_t* s_work = smem + 2048 + warp * (kMelNF * kMelFrameScratch);   // FFT work buffers: arena base, dead after this phase
                float* s_floor = s_mel + G * 256;
                int seen_v = 1;
                for (int i = et; i < 512; i += kIncEpiWarps * 32) { s_tw[i] = a.mel_twiddle[i]; s_win[i] = a.mel_window[i]; }
                if (et < G) {
                    const int b = grp * G + et;
                    s_cnt[et] = s_live[et] ? a.mel_count_rw[b] : 0;
                    s_cnt[8 + et] = s_live[et] ? a.feat_count[b] : 0;
                    // fresh stream (first chunk after a reset): only 5 mel frames exist (SURVEY.md F8).  Its history is
                    // ones(76,32), which is invariant under a shift in time, so the step is the ordinary 8-row step on
                    // the rows [1, 1, 1, m0..m4] with the tails of the all-ones window (written at reset)
                    seen_v = s_live[et] ? a.seen[b] : 1;
                    s_live[8 + et] = s_live[et] && seen_v == 0;
                }
                named_bar_sync(2, kIncEpiWarps * 32);
                const int my_start = a.mel_start[lane], my_len = a.mel_len[lane];
                const float* my_w = a.mel_w + lane * OWW_MEL_MAXSUPPORT;
                // kMelNF frames per warp at a time (interleaved instruction streams); frames of dead slots in a ragged last
                // group are computed on stream 0's audio and discarded
                for (int fi = warp * kMelNF; fi < G * 8; fi += kIncEpiWarps * kMelNF) {
                    const int16_t* tl[kMelNF]; const int16_t* bd[kMelNF]; int fr[kMelNF]; float db[kMelNF];
#pragma unroll
                    for (int i = 0; i < kMelNF; ++i) {
                        const int fj = fi + i < G * 8 ? fi + i : fi;
                        int b = grp * G + (fj >> 3);
                        if (b >= a.B) b = grp * G;
                        tl[i] = a.tail + (int64_t)b * OWW_TAIL; bd[i] = a.pcm + (int64_t)b * a.pcm_stride; fr[i] = fj & 7;
                    }
                    long long* st = (a.dbg_clock && blockIdx.x == 0 && grp == 0 && warp == 0 && fi == 0) ? a.dbg_clock + 92 : nullptr;
                    mel_frames_db<kMelNF>(tl, OWW_TAIL, bd, fr, s_work, s_tw, s_win, a.mel_kmax, my_start, my_len, my_w, lane, db, st);
#pragma unroll
                    for (int i = 0; i < kMelNF; ++i)
                        if (fi + i < G * 8) s_mel[(fi + i) * 32 + lane] = db[i];
                }
                named_bar_sync(2, kIncEpiWarps * 32);
                if (a.dbg_clock && blockIdx.x == 0 && grp == 0 && et == 0) a.dbg_clock[97] = clock64();
                // the streams' new tails = the last 480 samples of this chunk: 32-bit words, loaded now (every frame has been read)
                // and stored behind the clamp below, so the L2 latency hides under it
                constexpr int kTW = OWW_TAIL / 2;                                  // words per stream
                const bool al = ((size_t)a.pcm & 3) == 0 && (a.pcm_stride & 1) == 0;
                uint32_t tv[4]; int ti[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int i = et + u * kIncEpiWarps * 32;
                    ti[u] = -1; tv[u] = 0;
                    if (i < G * kTW) {
                        const int g = i / kTW, k = i - g * kTW, b = grp * G + g;
                        if (s_live[g]) {
                            const int16_t* src = a.pcm + (int64_t)b * a.pcm_stride + (OWW_SAMPLES_PER_CHUNK - OWW_TAIL) + 2 * k;
                            tv[u] = al ? __ldg(reinterpret_cast<const uint32_t*>(src))
                                       : ((uint32_t)(unsigned short)__ldg(src) | ((uint32_t)(unsigned short)__ldg(src + 1) << 16));
                            ti[u] = b * kTW + k;
                        }
                    }
                }
                if (warp < G) {                                    // per-call (= per stream, this step) maximum -> -80 dB floor
                    float m = -INFINITY;
                    const int j0 = s_live[8 + warp] ? 3 : 0;       // a fresh stream's call holds frames 3..7 only
#pragma unroll
                    for (int j = 0; j < 8; ++j) if (j >= j0) m = fmaxf(m, s_mel[warp * 256 + j * 32 + lane]);
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
                    if (lane == 0) s_floor[warp] = m - 80.0f;
                }
                named_bar_sync(2, kIncEpiWarps * 32);
                for (int i = et; i < G * 256; i += kIncEpiWarps * 32) {
                    const int g = i >> 8, b = grp * G + g;
                    float v = fmaxf(s_mel[i], s_floor[g]);
                    v = v / 10.0f + 2.0f;
                    const int fr = (i >> 5) & 7, skip = s_live[8 + g] ? 3 : 0;
                    if (fr < skip) v = 1.0f;                       // the three rows a fresh stream does not have: ones, like its history
                    s_mel[i] = v;
                    if (s_live[g] && fr >= skip)
                        a.mel_rw[(int64_t)b * a.mel_stride + (int64_t)((s_cnt[g] + fr - skip) & a.mel_mask) * 32 + (i & 31)] = v;
                }
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (ti[u] >= 0) reinterpret_cast<uint32_t*>(a.tail)[ti[u]] = tv[u];
                static_assert(kIncMaxG * (OWW_TAIL / 2) <= 4 * kIncEpiWarps * 32, "tail copy: four words per thread cover a group");
                // the next group's PCM (first touch: HBM) -> L2 while this group's layers run
                if (grp + (int)gridDim.x < P.n_groups && et < G * 20) {
                    const int g = et / 20, ln = et - g * 20, b = (grp + (int)gridDim.x) * G + g;
                    if (b < a.B) asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(a.pcm + (int64_t)b * a.pcm_stride) + ln * 128));
                }
                if (et < G && s_live[et]) {
                    const int b = grp * G + et;
                    a.mel_count_rw[b] = oww_wrap_count(s_cnt[et] + (s_live[8 + et] ? 5 : 8));
                    const int sn = seen_v + 1;                     // read when the group started (same thread)
                    a.seen[b] = sn > (1 << 30) ? (1 << 30) : sn;
                }
                named_bar_sync(2, kIncEpiWarps * 32);
            }
            for (int l = 0; l < NL; ++l) {
                const IncLayer& L = P.L[l];
                const bool to_global = kNL != OWW_N_CONV && l == NL - 1 && NL < OWW_N_CONV;   // cut plan: pooled output -> HBM (hi/lo)
                if (a.dbg_clock && blockIdx.x == 0 && grp == 0 && et == 0) a.dbg_clock[l] = clock64();
                uint4* nx = act0 + L.nx_base;
                // ---- (a) tails of the buffer this phase fills (rows 0..1) and front guards.  In a pool phase that
                //      buffer is still the conv's INPUT, so this is deferred until the tiles are drained. ----
                auto fill_tails_and_guards = [&]() {
                    if (L.nx_tail_off >= 0 && et == 0) {
                        // rows 0..1 of every plane <- the tails the previous step left in HBM: one bulk copy per plane,
                        // asynchronous; the MMA warp waits on tails_bar before it issues layer l+1
                        const uint32_t per_bytes = (uint32_t)(2 * G * L.nx_Wp) * 16u;
                        mbar_expect_tx(tails_bar, per_bytes * L.cg_out);
                        for (int pl = 0; pl < L.cg_out; ++pl)
                            bulk_g2s(smem_u32(nx + pl * L.nx_pitch + 1), tin + L.nx_tail_off + pl * (2 * G * L.nx_Wp), per_bytes, tails_bar);
                    }
                    if (!L.final && et < L.cg_out) nx[et * L.nx_pitch] = make_uint4(0, 0, 0, 0);
                };
                // rows 0..1 of a (3,1) layer's input (the tails copy issued in the previous phase) must have landed
                if (l > 0 && L.kh3) { mbar_wait(tails_bar, mma_tails_par); mma_tails_par ^= 1; }
                if (!L.pool_t) fill_tails_and_guards();
                else if (et < L.cg_out) (act0 + L.tmp_base)[et * L.tmp_pitch] = make_uint4(0, 0, 0, 0);

                if (l == 0) {
                    // ---- layer 0 on CUDA cores: 8 new rows from the last 10 mel rows of each stream ----
                    // A thread computes two adjacent positions (f, f+1): every weight it reads from shared memory (a broadcast
                    // load - the phase is bound by those) feeds two FMAs.  17 pairs per row: 16 real ones and the pad column.
                    const int Wp = 33, NP2 = 17;
                    for (int q = et; q < 8 * G * NP2; q += kIncEpiWarps * 32) {
                        const int j = q % NP2, tg = q / NP2, g = tg % G, t = tg / G;
                        const int f0 = 2 * j;
                        const int b = grp * G + g;
                        uint4* o = nx + 1 + tg * Wp + f0;
                        const uint4 z = make_uint4(0, 0, 0, 0);
                        if (j == 16) { o[0] = z; o[L.nx_pitch] = z; o[2 * L.nx_pitch] = z; continue; }      // pad column f = 32
                        if (!s_live[g]) {
                            o[0] = z; o[L.nx_pitch] = z; o[2 * L.nx_pitch] = z;
                            o[1] = z; o[L.nx_pitch + 1] = z; o[2 * L.nx_pitch + 1] = z;
                            continue;
                        }
                        const float* base = a.mel + (int64_t)b * a.mel_stride;
                        // rows 0..9 of the input = two rows from before this step + the eight new ones
                        const int row0 = (a.fused ? s_cnt[g] - 2 : a.mel_count[b] - a.back - 10) + t;     // fused: the two rows before this step's
                        float x[3][4];                               // mel rows t..t+2, columns f0-1..f0+2
#pragma unroll
                        for (int dt = 0; dt < 3; ++dt) {
                            const float* rp = (a.fused && t + dt >= 2) ? s_mel + (g * 8 + t + dt - 2) * 32
                                                                       : base + (int64_t)((row0 + dt) & a.mel_mask) * 32;
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                const int ff = f0 + i - 1;
                                x[dt][i] = (ff >= 0 && ff < 32) ? rp[ff] : 0.f;
                            }
                        }
#pragma unroll
                        for (int pl = 0; pl < 3; ++pl) {
                            __half2 h0[4], h1[4];
#pragma unroll
                            for (int u = 0; u < 4; ++u) {
                                float v0[2], v1[2];
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    const int c = pl * 8 + u * 2 + e;
                                    float s0 = 0.f, s1 = 0.f;
#pragma unroll
                                    for (int k = 0; k < 9; ++k) {
                                        const float w = s_l0[k * 24 + c];
                                        s0 = fmaf(x[k / 3][k % 3], w, s0);
                                        s1 = fmaf(x[k / 3][k % 3 + 1], w, s1);
                                    }
                                    const float sc = s_l0[216 + c], bi = s_l0[240 + c];
                                    v0[e] = act(fmaf(fmaxf(s0, 0.f), sc, bi));
                                    v1[e] = act(fmaf(fmaxf(s1, 0.f), sc, bi));
                                }
                                h0[u] = __floats2half2_rn(v0[0], v0[1]);
                                h1[u] = __floats2half2_rn(v1[0], v1[1]);
                            }
                            o[pl * L.nx_pitch] = *reinterpret_cast<uint4*>(h0);
                            o[pl * L.nx_pitch + 1] = *reinterpret_cast<uint4*>(h1);
                        }
                    }
                } else {
                    // ---- tensor-core layer: 64-position tiles, warpgroup w takes tiles w, w + 4, ... ----
                    mbar_wait(wfull(l & 1), epar[l & 1]);             // weights (and scale/bias) of layer l have landed
                    epar[l & 1] ^= 1;
                    const float* sb = reinterpret_cast<const float*>(smem + L.w_smem + 3 * L.cgp * L.np * 16);
                    uint4* dst = L.pool_t ? (act0 + L.tmp_base) : nx;
                    const int dpitch = L.pool_t ? L.tmp_pitch : L.nx_pitch;
                    const int t_off_units = L.pool_t ? 0 : L.nx_t_off * G * L.Wp;
                    const int n_t64 = (L.M + 63) / 64;
                    const int tail_start = (L.T_out - 2) * G * L.Wp;
                    const uint32_t wp_magic = 0xFFFFFFFFu / (uint32_t)L.Wp + 1u, g_magic = G > 1 ? 0xFFFFFFFFu / (uint32_t)G + 1u : 0u;
                    const bool edbg = a.dbg_clock && blockIdx.x == 0 && grp == 0 && et == 0;
                    long long e0 = 0;
                    if (edbg) e0 = clock64();
                    const int wg = warp >> 2, wq = warp & 3, q = lane & 3;
                    const uint32_t w_addr = smem_u32(smem + L.w_smem);
                    const uint32_t a_base = smem_u32(act0 + L.in_base);
                    // K = 16 = two channel-group planes per MMA; an odd plane count pairs the last plane with itself
                    // (LBO 0) against zero weights, so no pad plane has to exist in smem.  Only the 14-bit start
                    // address field changes between MMAs.
                    const int nq = L.cgp / 2;
                    const uint32_t a_hi_pair = (uint32_t)make_desc(0, (uint32_t)L.in_pitch * 16u, 128u);   // low word: LBO field
                    const uint32_t a_hi_self = (uint32_t)make_desc(0, 0u, 128u);
                    const uint64_t dhi = make_desc(0, 0u, 128u) & 0xFFFFFFFF00000000ull;                  // high word: SBO field
                    const uint32_t b_lo0 = (uint32_t)make_desc(0, (uint32_t)L.np * 16u, 128u);
                    const uint32_t a_unit0 = (a_base >> 4) + 1u;
                    const uint32_t b_unit0 = w_addr >> 4;
                    const uint32_t tap0 = (uint32_t)L.tap[0], tap1 = (uint32_t)L.tap[1], tap2 = (uint32_t)L.tap[2];
                    const uint32_t pitch2 = 2u * (uint32_t)L.in_pitch, np2 = 2u * (uint32_t)L.np, tap_w = (uint32_t)(L.cgp * L.np);
                    const int n_pair = L.cg_in / 2;                   // K steps whose second plane exists
                    // Odd plane count (24 or 72 channels): instead of padding every tap to an even number of planes (one
                    // half-empty MMA per tap), the K octets of the three taps are chained - the last plane of tap 0 shares an
                    // MMA with the first plane of tap 1 (the LBO field is just the distance of the two octets, whatever tap they
                    // belong to): (3 cg + 1) / 2 MMAs per tile instead of 3 (cg + 1) / 2 (5 instead of 6 at 24 channels).  The
                    // weights of such a layer are packed in the same octet order (oww_inc_setup).
                    const bool chained = (L.cg_in & 1) != 0;
                    const int n_steps = chained ? 3 * n_pair + 2 : 3 * nq;
                    const uint32_t a_cross = (uint32_t)make_desc(0, ((uint32_t)(L.cg_in - 1) * (uint32_t)L.in_pitch + tap0 - tap1) * 16u, 128u);
                    const uint32_t last_plane = (uint32_t)(L.cg_in - 1) * (uint32_t)L.in_pitch;
                    // Work items: (64-position tile, chunk of N: 32 columns, or 16 where N is 48 / 80); warpgroup w takes items
                    // w, w + 4, ... two at a time (both MMA chains in flight, then both epilogues).  The chunks keep the
                    // accumulators at 2 x 16 registers per thread next to the rest of the kernel's state.
                    const int nc = (L.np & 31) ? 16 : 32;
                    const int n_chunks = L.np / nc;
                    const int n_items = n_t64 * n_chunks;
                    // per-layer geometry in registers: inside the item loop every L.field would be an indexed parameter load
                    const int lM = L.M, lWp = L.Wp, lW = L.W, lnp = L.np, lcg_out = L.cg_out, ltail = L.nx_tail_off;
                    const bool lfinal = L.final != 0, lpool = L.pool_t != 0;
                    const uint32_t lin_pitch = (uint32_t)L.in_pitch;
                    const int tail_pitch = 2 * G * lWp;
                    auto mma_item = [&](auto nc_const, auto ns_const, float* acc, int it) {
                        constexpr int NP = decltype(nc_const)::value;          // columns of this chunk
                        constexpr int NS = decltype(ns_const)::value;          // K steps (compile time: unrolled chain)
                        constexpr bool kChained = NS % 3 == 2;
                        constexpr int kPair = kChained ? (NS - 2) / 3 : NS / 3, kNq = NS / 3;
                        const int t64 = it / n_chunks, c0 = (it - t64 * n_chunks) * NP;
                        const uint32_t a_t0 = a_unit0 + (uint32_t)(t64 * 64);
                        const uint32_t b_unit = b_unit0 + (uint32_t)c0;        // weight row n of an octet block: unit n
#pragma unroll
                        for (int s = 0; s < NS; ++s) {
                            uint32_t a_off, a_f, b_off;
                            if (kChained) {
                                const int k1 = s - kPair - 1, k2 = s - 2 * kPair - 1;
                                a_off = s < kPair ? tap0 + (uint32_t)s * pitch2                         // tap 0: planes (0,1) (2,3) ...
                                      : s == kPair ? tap1                                                // (tap 1, plane 0) + (tap 0, last plane)
                                      : k1 < kPair ? tap1 + lin_pitch + (uint32_t)k1 * pitch2            // tap 1: planes (1,2) (3,4) ...
                                      : k2 < kPair ? tap2 + (uint32_t)k2 * pitch2                        // tap 2: planes (0,1) (2,3) ...
                                      : tap2 + last_plane;                                               // tap 2, last plane, with itself
                                a_f = s == kPair ? a_cross : (k2 >= kPair ? a_hi_self : a_hi_pair);
                                b_off = (uint32_t)s * np2;
                            } else {
                                const int j = s / kNq, qq = s - j * kNq;
                                a_off = (j == 0 ? tap0 : j == 1 ? tap1 : tap2) + (uint32_t)qq * pitch2;
                                a_f = a_hi_pair;                                                         // even plane count
                                b_off = (uint32_t)j * tap_w + (uint32_t)qq * np2;
                            }
                            wg_mma<NP>(acc, dhi | a_f | ((a_t0 + a_off) & 0x3FFFu), dhi | b_lo0 | ((b_unit + b_off) & 0x3FFFu), s > 0);
                        }
                    };
                    auto epi_item = [&](auto nc_const, const float* acc, int it) {
                        constexpr int NP = decltype(nc_const)::value;
                        const int t64 = it / n_chunks, c0 = (it - t64 * n_chunks) * NP;
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            const int m = t64 * 64 + wq * 16 + (lane >> 2) + 8 * i;
                            if (m >= lM) continue;
                            // m = (t*G + g)*Wp + f; exact division by multiply-high (m < 2^16, divisors < 2^6)
                            const int tg = (int)__umulhi((uint32_t)m, wp_magic);
                            const int f = m - tg * lWp;
                            const int g = G > 1 ? tg - (int)__umulhi((uint32_t)tg, g_magic) * G : 0;
                            const bool live = s_live[g] != 0;
                            if (lfinal) {
                                if (f != 0 || !live) continue;
                                float* o = a.fused ? a.feat_ring + (int64_t)(grp * G + g) * a.feat_stride + (int64_t)(s_cnt[8 + g] & a.feat_mask) * 96
                                                   : a.emb + (int64_t)(grp * G + g) * 96;
#pragma unroll
                                for (int j = 0; j < NP / 8; ++j) {
                                    const int c = c0 + j * 8 + 2 * q;
                                    float2 r;
                                    r.x = fmaf(acc[4 * j + 2 * i], sb[c], sb[lnp + c]);
                                    r.y = fmaf(acc[4 * j + 2 * i + 1], sb[c + 1], sb[lnp + c + 1]);
                                    *reinterpret_cast<float2*>(o + c) = r;
                                }
                                continue;
                            }
                            const bool pad = f == lW;
                            uint4* d0 = dst + (1 + t_off_units + m);
                            const bool keep_tail = !lpool && ltail >= 0 && m >= tail_start && live;
                            uint4* t0 = tout + (ltail + (m - tail_start));
                            // this thread holds channels 2q, 2q+1 of every plane: one 32-bit word of each 16-byte unit
#pragma unroll
                            for (int j = 0; j < NP / 8; ++j) {
                                const int pl = c0 / 8 + j;
                                if (pl >= lcg_out) break;
                                const int c = pl * 8 + 2 * q;
                                const float y0 = act(fmaf(acc[4 * j + 2 * i], sb[c], sb[lnp + c]));
                                const float y1 = act(fmaf(acc[4 * j + 2 * i + 1], sb[c + 1], sb[lnp + c + 1]));
                                const __half2 h = __floats2half2_rn(y0, y1);
                                const uint32_t hw = pad ? 0u : *reinterpret_cast<const uint32_t*>(&h);
                                reinterpret_cast<uint32_t*>(d0 + pl * dpitch)[q] = hw;
                                if (keep_tail) reinterpret_cast<uint32_t*>(t0 + pl * tail_pitch)[q] = hw;
                                if (to_global) {
                                    // cut layer only (warp-uniform, one layer per step): the unpooled temp also keeps the
                                    // lo parts (y = hi + lo)
                                    const __half2 lo = __floats2half2_rn(y0 - __low2float(h), y1 - __high2float(h));
                                    reinterpret_cast<uint32_t*>(d0 + (lcg_out + pl) * dpitch)[q] = pad ? 0u : *reinterpret_cast<const uint32_t*>(&lo);
                                }
                            }
                        }
                    };
                    auto run_items = [&](auto nc_const, auto ns_const) {
                        constexpr int NP = decltype(nc_const)::value;
                        for (int it = wg; it < n_items; it += 4) {
                            float acc0[NP / 2];
                            wg_fence();
                            mma_item(nc_const, ns_const, acc0, it);
                            wg_commit();
                            wg_wait_all();
                            if (edbg && it == 0) a.dbg_clock[61 + l] = clock64() - e0;     // phase start -> first accumulator ready
                            epi_item(nc_const, acc0, it);
                        }
                    };
                    auto run_steps = [&](auto ns_const) {
                        if (nc == 32) run_items(std::integral_constant<int, 32>{}, ns_const);
                        else run_items(std::integral_constant<int, 16>{}, ns_const);
                    };
                    switch (n_steps) {
                        case 5: run_steps(std::integral_constant<int, 5>{}); break;
                        case 9: run_steps(std::integral_constant<int, 9>{}); break;
                        case 14: run_steps(std::integral_constant<int, 14>{}); break;
                        case 18: run_steps(std::integral_constant<int, 18>{}); break;
                        default: __trap();                                // the plan only holds 24 / 48 / 72 / 96-channel inputs
                    }
                    if (edbg) a.dbg_clock[81 + l] = clock64() - e0;                       // phase start -> last tile stored
                    if (L.pool_t) {
                        // ---- max-pool: tmp (unpooled conv output) -> nx ----
                        named_bar_sync(2, kIncEpiWarps * 32);          // every tile drained: the conv input buffer is free
                        if (!to_global) fill_tails_and_guards();
                        if (L.nx_tail_off >= 0 && L.nx_rows_new == 1) {
                            // single new row: next step's tails are (old tail row 1, new row); copy the old row once it landed
                            mbar_wait(tails_bar, epi_tails_par);
                            const int perrow = G * L.nx_Wp;
                            for (int i = et; i < L.cg_out * perrow; i += kIncEpiWarps * 32) {
                                const int pl = i / perrow, u = i - pl * perrow;
                                if (s_live[u / L.nx_Wp])
                                    tout[L.nx_tail_off + pl * 2 * perrow + u] = nx[pl * L.nx_pitch + 1 + perrow + u];
                            }
                        }
                        const uint4* src = act0 + L.tmp_base;
                        const int T2 = L.T_out / L.pool_t;
                        const int per = T2 * G * L.nx_Wp;
                        // exact division by multiply-high (indices < 2^16): three magics per layer instead of four divisions per unit
                        const uint32_t per_magic = 0xFFFFFFFFu / (uint32_t)per + 1u, nwp_magic = 0xFFFFFFFFu / (uint32_t)L.nx_Wp + 1u;
                        const uint32_t gp_magic = G > 1 ? 0xFFFFFFFFu / (uint32_t)G + 1u : 0u;
                        for (int i = et; i < L.cg_out * per; i += kIncEpiWarps * 32) {
                            const int pl = per > 1 ? (int)__umulhi((uint32_t)i, per_magic) : i, p = i - pl * per;
                            const int tg = (int)__umulhi((uint32_t)p, nwp_magic), f = p - tg * L.nx_Wp;
                            const int t = G > 1 ? (int)__umulhi((uint32_t)tg, gp_magic) : tg, g = tg - t * G;
                            uint4 res = make_uint4(0, 0, 0, 0);
                            if (to_global) {
                                // pool on (hi, lo) pairs: the element with the largest hi + lo = lexicographic maximum
                                uint4 res_lo = make_uint4(0, 0, 0, 0);
                                if (f < L.nx_W) {
                                    // two channels per 32-bit word; mask arithmetic keeps everything in registers
                                    uint32_t bh[4] = {0, 0, 0, 0}, bl[4] = {0, 0, 0, 0};
                                    bool first = true;
                                    for (int da = 0; da < L.pool_t; ++da)
                                        for (int db = 0; db < L.pool_f; ++db) {
                                            const int at = 1 + ((t * L.pool_t + da) * G + g) * L.Wp + f * L.pool_f + db;
                                            const uint4 q = src[pl * L.tmp_pitch + at], ql = src[(L.cg_out + pl) * L.tmp_pitch + at];
                                            const uint32_t qh[4] = {q.x, q.y, q.z, q.w}, qq[4] = {ql.x, ql.y, ql.z, ql.w};
#pragma unroll
                                            for (int u = 0; u < 4; ++u) {
                                                const __half2 h2 = u32_as_half2(qh[u]), l2 = u32_as_half2(qq[u]);
                                                const __half2 b2 = u32_as_half2(bh[u]), c2 = u32_as_half2(bl[u]);
                                                const uint32_t m = first ? 0xFFFFFFFFu
                                                                         : (__hgt2_mask(h2, b2) | (__heq2_mask(h2, b2) & __hgt2_mask(l2, c2)));
                                                bh[u] = (qh[u] & m) | (bh[u] & ~m);
                                                bl[u] = (qq[u] & m) | (bl[u] & ~m);
                                            }
                                            first = false;
                                        }
                                    res = make_uint4(bh[0], bh[1], bh[2], bh[3]);
                                    res_lo = make_uint4(bl[0], bl[1], bl[2], bl[3]);
                                }
                                if (s_live[g]) {
                                    const int64_t q = kGuard + ((int64_t)(grp * G + g) * T2 + t) * L.nx_Wp + f;
                                    if (a.gx_lay.S) {
                                        a.gx[late_unit(a.gx_lay, pl, grp * G + g, t, f)] = res;
                                        a.gx[late_unit(a.gx_lay, L.cg_out + pl, grp * G + g, t, f)] = res_lo;
                                    } else {
                                        a.gx[(int64_t)pl * a.gx_plane + q] = res;
                                        a.gx[(int64_t)(L.cg_out + pl) * a.gx_plane + q] = res_lo;
                                    }
                                }
                                continue;
                            }
                            if (f < L.nx_W) {
                                __half2 mx[4];
                                bool first = true;
                                for (int da = 0; da < L.pool_t; ++da)
                                    for (int db = 0; db < L.pool_f; ++db) {
                                        const uint4 q = src[pl * L.tmp_pitch + 1 + ((t * L.pool_t + da) * G + g) * L.Wp + f * L.pool_f + db];
                                        const __half2* hv = reinterpret_cast<const __half2*>(&q);
#pragma unroll
                                        for (int u = 0; u < 4; ++u) mx[u] = first ? hv[u] : __hmax2(mx[u], hv[u]);
                                        first = false;
                                    }
                                res = *reinterpret_cast<uint4*>(mx);
                            }
                            nx[pl * L.nx_pitch + 1 + L.nx_t_off * G * L.nx_Wp + p] = res;
                            if (L.nx_tail_off >= 0 && s_live[g]) {
                                // the pooled rows are the newest rows of a tails-bearing buffer
                                const int keep = T2 >= 2 ? 2 : 1;
                                if (t >= T2 - keep)
                                    tout[L.nx_tail_off + pl * (2 * G * L.nx_Wp) + ((2 - keep + t - (T2 - keep)) * G + g) * L.nx_Wp + f] = res;
                            }
                        }
                    }
                }
                if (L.nx_tail_off >= 0) epi_tails_par ^= 1;
                // ---- phase done: make generic-proxy smem writes visible to the tensor core; once every warp is past
                //      this barrier, layer l's weight slot (MMA operand, scale / bias) is free for the producer ----
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                named_bar_sync(1, kIncEpiWarps * 32);
                if (l > 0 && et == 0) mbar_arrive(wempty(l & 1));
            }
            if (a.dbg_clock && blockIdx.x == 0 && grp == 0 && et == 0) a.dbg_clock[OWW_N_CONV] = clock64();
            if (a.fused && NL == OWW_N_CONV) {
                // ===== K3 inside the step kernel: every head on this group's streams, straight from the feature ring =====
                named_bar_sync(2, kIncEpiWarps * 32);              // the new embedding rows (written by this CTA) are visible
                if (a.n_heads > 0) {                               // n_heads == 0: the heads run as their own launch after this one
                if (et == 0) mbar_arrive(hstart_bar);              // producer may start streaming head weights
                const int NI = a.max_n_in;
                float* feats = reinterpret_cast<float*>(smem + 2048);            // [G][NI][96]
                float* red = feats + G * NI * 96;                                // [4][G][128]
                float* hA = red + 4 * G * 128;                                   // [G][256]
                float* hB = hA + G * 256;
                // gather the last NI embedding rows of every stream (four independent L2 loads in flight per thread)
                for (int i0 = et; i0 < G * NI * 24; i0 += 4 * kIncEpiWarps * 32) {
                    float4 v[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int i = i0 + u * kIncEpiWarps * 32;
                        v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (i < G * NI * 24) {
                            const int g = i / (NI * 24), r = (i / 24) % NI, c4 = (i % 24) * 4, b = grp * G + g;
                            if (s_live[g]) {
                                const int row = s_cnt[8 + g] + 1 - NI + r;
                                if (row >= 0) v[u] = __ldcg(reinterpret_cast<const float4*>(a.feat_ring + (int64_t)b * a.feat_stride + (int64_t)(row & a.feat_mask) * 96 + c4));
                            }
                        }
                    }
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int i = i0 + u * kIncEpiWarps * 32;
                        if (i < G * NI * 24) *reinterpret_cast<float4*>(feats + i * 4) = v[u];
                    }
                }
                named_bar_sync(2, kIncEpiWarps * 32);
                for (int hh = 0; hh < a.n_heads; ++hh) {
                    const HeadDev& H = a.heads[hh];
                    const int D1 = H.dims[1], off = NI - H.n_in;
                    {   // first layer: 4 K-slices x 128 columns, same summation order as heads_kernel; the weight rows
                        // of feature row c arrive in ring slot (chunk % hns), streamed by the producer warp
                        const int slice = et >> 7, d = et & 127;
                        float acc[kIncMaxG];
#pragma unroll
                        for (int g = 0; g < kIncMaxG; ++g) acc[g] = 0.f;
                        for (int c = 0; c < H.n_in; ++c) {
                            const int slot = hchunk_e % a.hns;
                            mbar_wait(hfull(slot), (hf_par >> slot) & 1u);
                            hf_par ^= 1u << slot;
                            ++hchunk_e;
                            if (d < D1) {
                                const float* wr = reinterpret_cast<const float*>(smem + a.hring_off + slot * a.hslot_bytes) + slice * 24 * D1 + d;
                                const float* xr = feats + (off + c) * 96 + slice * 24;
                                // the features are read four k at a time (one broadcast 16-byte load per stream instead of
                                // four scalar ones: the loop was shared-memory-issue bound); the k order per accumulator is unchanged
#pragma unroll 2
                                for (int k4 = 0; k4 < 24; k4 += 4) {
                                    const float w0 = wr[(k4 + 0) * D1], w1 = wr[(k4 + 1) * D1];
                                    const float w2 = wr[(k4 + 2) * D1], w3 = wr[(k4 + 3) * D1];
#pragma unroll
                                    for (int g = 0; g < kIncMaxG; ++g)
                                        if (g < G) {
                                            const float4 x = *reinterpret_cast<const float4*>(xr + g * NI * 96 + k4);
                                            acc[g] = fmaf(x.x, w0, acc[g]);
                                            acc[g] = fmaf(x.y, w1, acc[g]);
                                            acc[g] = fmaf(x.z, w2, acc[g]);
                                            acc[g] = fmaf(x.w, w3, acc[g]);
                                        }
                                }
                            }
                            __syncwarp();
                            if (lane == 0) mbar_arrive(hempty(slot));
                        }
                        if (d < D1) {
#pragma unroll
                            for (int g = 0; g < kIncMaxG; ++g)
                                if (g < G) red[(slice * G + g) * 128 + d] = acc[g];
                        }
                    }
                    named_bar_sync(2, kIncEpiWarps * 32);
                    for (int i = et; i < G * D1; i += kIncEpiWarps * 32) {
                        const int g = i / D1, d = i - g * D1;
                        float v = __ldg(H.blob + H.b_off[0] + d) + red[(0 * G + g) * 128 + d];
                        v += red[(1 * G + g) * 128 + d];
                        v += red[(2 * G + g) * 128 + d];
                        v += red[(3 * G + g) * 128 + d];
                        hA[g * 256 + d] = v;
                    }
                    named_bar_sync(2, kIncEpiWarps * 32);
                    float* cur = hA; float* nxt = hB;
                    for (int l = 0; l < H.n_layers; ++l) {
                        const int D = H.dims[l + 1], K = H.dims[l];
                        if (l > 0) {
                            // later layers: the producer streams W_l (K x D) through the ring in chunks of head_rows() rows.
                            // A thread owns outputs i = et + 512 j; each accumulates over k in ascending order (as heads_kernel does).
                            const int rows = head_rows(a.hslot_bytes, K, D);
                            const int nown = min(4, max(0, (G * D - et + kIncEpiWarps * 32 - 1) / (kIncEpiWarps * 32)));
                            float accl[4]; int cxo[4], dd[4];
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                const int i = j < nown ? et + j * kIncEpiWarps * 32 : 0;
                                const int g = i / D;
                                dd[j] = i - g * D; cxo[j] = g * 256; accl[j] = 0.f;
                            }
                            for (int k0 = 0; k0 < K; k0 += rows) {
                                const int r = min(rows, K - k0);
                                const int slot = hchunk_e % a.hns;
                                mbar_wait(hfull(slot), (hf_par >> slot) & 1u);
                                hf_par ^= 1u << slot;
                                ++hchunk_e;
                                const float* wr = reinterpret_cast<const float*>(smem + a.hring_off + slot * a.hslot_bytes);
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                    if (j >= nown) break;
                                    const float* cx = cur + cxo[j] + k0;
                                    const float* wc = wr + dd[j];
                                    float sacc = accl[j];
#pragma unroll 8
                                    for (int k = 0; k < r; ++k) sacc = fmaf(cx[k], wc[k * D], sacc);
                                    accl[j] = sacc;
                                }
                                __syncwarp();
                                if (lane == 0) mbar_arrive(hempty(slot));
                            }
#pragma unroll
                            for (int j = 0; j < 4; ++j)
                                if (j < nown) nxt[cxo[j] + dd[j]] = accl[j] + __ldg(H.blob + H.b_off[l] + dd[j]);
                            named_bar_sync(2, kIncEpiWarps * 32);
                            float* t = cur; cur = nxt; nxt = t;
                        }
                        if (l < H.n_layers - 1) {
                            if (warp < G) {
                                float* row = cur + warp * 256;
                                if (H.layernorm) {
                                    float sum = 0.f;
                                    for (int d = lane; d < D; d += 32) sum += row[d];
#pragma unroll
                                    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
                                    const float mu = sum / (float)D;
                                    float sq = 0.f;
                                    for (int d = lane; d < D; d += 32) { const float c = row[d] - mu; sq = fmaf(c, c, sq); }
#pragma unroll
                                    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
                                    const float rstd = 1.0f / sqrtf(sq / (float)D + 1e-5f);
                                    const float* gm = H.blob + H.g_off[l];
                                    const float* hb = H.blob + H.h_off[l];
                                    for (int d = lane; d < D; d += 32)
                                        row[d] = fmaxf((row[d] - mu) * rstd * __ldg(gm + d) + __ldg(hb + d), 0.f);
                                } else {
                                    for (int d = lane; d < D; d += 32) row[d] = fmaxf(row[d], 0.f);
                                }
                            }
                            named_bar_sync(2, kIncEpiWarps * 32);
                        }
                    }
                    if (et < G && s_live[et]) {
                        const int n_out = H.dims[H.n_layers];
                        float* row = cur + et * 256;
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
                        float* o = a.scores + (int64_t)(grp * G + et) * a.score_stride + H.col0;
                        for (int d = 0; d < n_out; ++d) o[d] = row[d];
                    }
                    named_bar_sync(2, kIncEpiWarps * 32);
                }
                }
                if (et < G && s_live[et]) {
                    if (a.n_heads > 0) {
                        // conditional verifier pairs: the thread that wrote this stream's scores rewrites the gated columns
                        float* o = a.scores + (int64_t)(grp * G + et) * a.score_stride;
                        for (int q = 0; q < a.n_gates; ++q)
                            if (o[a.gates[q].main_col] > a.gates[q].thr) o[a.gates[q].main_col] = o[a.gates[q].ver_col];
                    }
                    a.feat_count[grp * G + et] = oww_wrap_count(s_cnt[8 + et] + 1);
                }
                named_bar_sync(2, kIncEpiWarps * 32);
                if (a.dbg_clock && blockIdx.x == 0 && grp == 0 && et == 0) a.dbg_clock[102] = clock64();
            }
        }
    }
}

// ---- capture of tails from the full-window planes (stream-major positions) ----------------------
__global__ void __launch_bounds__(256) tc_capture_kernel(const uint4* planes, int64_t plane_pitch, int T, int Wp, int cg,
                                                         int win0, int n_win, int stream0, const int* ids, int G, int tail_off,
                                                         int tail_units, uint4* tails) {
    const int per = 2 * Wp;
    const int64_t total = (int64_t)n_win * cg * per;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        const int u = (int)(i % per);
        const int pl = (int)((i / per) % cg);
        const int w = (int)(i / ((int64_t)per * cg));
        const int r = u / Wp, f = u - r * Wp;
        const int b = ids ? ids[stream0 + w] : stream0 + w, grp = b / G, g = b - grp * G;
        const uint4 v = planes[(int64_t)pl * plane_pitch + kGuard + (int64_t)(win0 + w) * T * Wp + (int64_t)(T - 2 + r) * Wp + f];
        tails[(int64_t)grp * tail_units + tail_off + pl * (2 * G * Wp) + (r * G + g) * Wp + f] = v;
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// Plan: per-layer geometry of the fused kernel for groups of G streams.
int oww_inc_build_plan(oww_ctx* ctx, int G, int n_streams, int n_layers, IncPlan* out) {
    if (G < 1 || G > kIncMaxG) return oww_fail(ctx, OWW_EINVAL, "group size must be 1..%d", kIncMaxG);
    const int NL = n_layers;            // conv layers inside the kernel: 20, or a cut after a pooled layer (cut plan)
    if (NL < 3 || NL > OWW_N_CONV || (NL < OWW_N_CONV && !ctx->conv[NL - 1].pool_t))
        return oww_fail(ctx, OWW_EINVAL, "fused-CNN plan: cannot cut after layer %d", NL - 1);
    constexpr int kTop = 227 * 1024;     // usable dynamic shared memory per CTA on sm_90
    constexpr int kActBase = 2048;
    IncPlan P;
    std::memset(&P, 0, sizeof(P));
    P.G = G;
    P.n_groups = (n_streams + G - 1) / G;
    P.n_layers = NL;
    for (int l = 0; l < OWW_N_CONV; ++l) P.L[l].nx_tail_off = -1;
    int rows_new = 8, W = 32;            // geometry of the tensor produced by the previous phase
    int tail_units = 0;
    int x_units = 0, y_units = 0;
    size_t w_off = 0;
    auto pitch_of = [&](int rows, int wp) { return (1 + rows * G * wp + 7) & ~7; };
    auto need = [&](int buf, int units) { if (buf) { if (units > y_units) y_units = units; } else { if (units > x_units) x_units = units; } };
    int cur_buf = 0;                      // buffer holding the input of the next layer
    int use_x[OWW_N_CONV] = {0}, use_y[OWW_N_CONV] = {0};   // units of X / Y alive during phase l
    for (int l = 0; l < NL; ++l) {
        const ConvLayer& C = ctx->conv[l];
        IncLayer& L = P.L[l];
        const bool cut = l == NL - 1 && NL < OWW_N_CONV;     // pooled output leaves the kernel (hi/lo planes in HBM)
        L.final = l == OWW_N_CONV - 1;
        L.kh3 = C.kh == 3 && l > 0;
        L.W = W; L.Wp = W + 1;
        L.cg_in = C.cin / 8; L.cgp = (L.cg_in + 1) & ~1; L.np = (C.cout + 15) & ~15; L.cg_out = C.cout / 8;
        L.pool_t = C.pool_t; L.pool_f = C.pool_f;
        auto use = [&](int buf, int units) { need(buf, units); int& u = buf ? use_y[l] : use_x[l]; if (units > u) u = units; };
        if (l == 0) {
            L.T_out = 8; L.M = 0;
        } else {
            L.in_buf = cur_buf;
            L.rows_in = rows_new + (L.kh3 ? 2 : 0);
            L.T_out = rows_new;
            L.M = L.T_out * G * L.Wp;
            L.in_pitch = P.L[l - 1].nx_pitch;
            use(L.in_buf, L.in_pitch * L.cg_in);
            if (L.kh3) { L.tap[0] = 0; L.tap[1] = G * L.Wp; L.tap[2] = 2 * G * L.Wp; }
            else { L.tap[0] = -1; L.tap[1] = 0; L.tap[2] = 1; }
            L.w_off = (int)w_off;
            L.w_bytes = 3 * L.cgp * L.np * 16 + 2 * L.np * 4;
            w_off += (size_t)((L.w_bytes + 127) & ~127);
        }
        // geometry of what this phase leaves for layer l+1
        const bool next_kh3 = !cut && l + 1 < OWW_N_CONV && ctx->conv[l + 1].kh == 3;
        int nrows = L.T_out, nW = W;
        if (L.pool_t) { nrows = L.T_out / L.pool_t; nW = W / L.pool_f; }
        L.nx_W = nW; L.nx_Wp = nW + 1; L.nx_rows_new = nrows;
        L.nx_t_off = (next_kh3 && !L.final) ? 2 : 0;
        L.out_buf = l == 0 ? 0 : (cur_buf ^ 1);
        L.nx_buf = (l == 0) ? 0 : (L.pool_t ? cur_buf : L.out_buf);
        L.nx_pitch = pitch_of(nrows + L.nx_t_off, L.nx_Wp);
        if (L.pool_t) { L.tmp_pitch = pitch_of(L.T_out, L.Wp); use(L.out_buf, L.tmp_pitch * L.cg_out * (cut ? 2 : 1)); }
        if (!L.final && !cut) use(L.nx_buf, L.nx_pitch * L.cg_out);
        L.nx_tail_off = -1;
        if (L.nx_t_off == 2) { L.nx_tail_off = tail_units; tail_units += L.cg_out * 2 * G * L.nx_Wp; }
        cur_buf = L.nx_buf;
        rows_new = nrows; W = nW;
    }
    P.tail_units = tail_units;
    P.x_units = (x_units + 7) & ~7; P.y_units = (y_units + 7) & ~7;
    // ---- placement: class-0 tensors sit at offset 0; a class-1 tensor sits just above the largest class-0 tensor
    //      that is alive at any time during its own lifetime (produced in phase p, consumed in phase p+1) ----
    int size_nx[OWW_N_CONV] = {0}, size_tmp[OWW_N_CONV] = {0}, xlive[OWW_N_CONV + 1];
    for (int l = 0; l < NL; ++l) {
        const IncLayer& L = P.L[l];
        const bool cut = l == NL - 1 && NL < OWW_N_CONV;
        size_nx[l] = (L.final || cut) ? 0 : L.nx_pitch * L.cg_out;
        size_tmp[l] = L.pool_t ? L.tmp_pitch * L.cg_out * (cut ? 2 : 1) : 0;
    }
    for (int l = 0; l <= OWW_N_CONV; ++l) xlive[l] = 0;
    for (int l = 0; l < NL; ++l) {
        const IncLayer& L = P.L[l];
        auto upd = [&](int cls, int sz) { if (cls == 0 && sz > xlive[l]) xlive[l] = sz; };
        if (l > 0) upd(L.in_buf, size_nx[l - 1]);
        if (L.pool_t) upd(L.out_buf, size_tmp[l]);
        upd(L.nx_buf, size_nx[l]);
    }
    auto r8 = [](int v) { return (v + 7) & ~7; };
    int act_high[OWW_N_CONV] = {0};
    for (int l = 0; l < NL; ++l) {
        IncLayer& L = P.L[l];
        L.in_base = l > 0 ? P.L[l - 1].nx_base : 0;
        L.tmp_base = (L.pool_t && L.out_buf == 1) ? r8(xlive[l]) : 0;
        L.nx_base = L.nx_buf == 1 ? r8(xlive[l] > xlive[l + 1] ? xlive[l] : xlive[l + 1]) : 0;
        int hi = 0;
        if (l > 0 && L.in_base + size_nx[l - 1] > hi) hi = L.in_base + size_nx[l - 1];
        if (L.pool_t && L.tmp_base + size_tmp[l] > hi) hi = L.tmp_base + size_tmp[l];
        if (L.nx_base + size_nx[l] > hi) hi = L.nx_base + size_nx[l];
        act_high[l] = kActBase + hi * 16;
    }
    // weight slots, top-down: odd layers end at the top, an even layer sits just below its odd successor's
    // slot (sizes are non-decreasing with depth, so it also clears its odd predecessor).
    auto wsz = [&](int l) { return l >= 1 && l < NL ? (P.L[l].w_bytes + 127) & ~127 : 0; };
    for (int l = 1; l < NL; ++l) {
        // (in a cut plan the last layer can be even: it still sits below its odd predecessor, whose slot is live while
        // this one is prefetched)
        const int above = wsz(l + 1) > wsz(l - 1) ? wsz(l + 1) : wsz(l - 1);
        P.L[l].w_smem = (l & 1) ? kTop - wsz(l) : kTop - above - wsz(l);
    }
    for (int l = 1; l < NL; ++l) {
        // while layer l runs, its own slot and the prefetch of layer l+1 are live next to the activations in use;
        // slot l itself was filled during phase l-1
        int w_low = P.L[l].w_smem;
        if (l + 1 < NL && P.L[l + 1].w_smem < w_low) w_low = P.L[l + 1].w_smem;
        if (act_high[l] > w_low || act_high[l - 1] > P.L[l].w_smem)
            return oww_fail(ctx, OWW_EUNSUPPORTED, "fused-CNN smem plan does not fit at layer %d (G=%d)", l, G);
        if (l >= 2 && wsz(l) < wsz(l - 1)) return oww_fail(ctx, OWW_EUNSUPPORTED, "weight sizes must not shrink with depth");
    }
    // frontend of the fused step: FFT work buffers at the arena base (dead before layer 0 writes its output there);
    // twiddles 4 KB | window 2 KB | G x 8 x 32 mel rows | G floors sit above both, below the weight slots of layers 1-2
    {
        int off = kActBase + r8(size_nx[0]) * 16;
        const int work_end = kActBase + kIncEpiWarps * kMelNF * kMelFrameScratch;
        if (work_end > off) off = (work_end + 127) & ~127;
        const int need_b = 6144 + G * 256 * 4 + 64;
        P.scratch_off = (off + need_b <= P.L[1].w_smem && off + need_b <= P.L[2].w_smem) ? off : 0;
    }
    P.w_total_bytes = (int)w_off;
    P.smem_bytes = kTop;
    *out = P;
    return OWW_OK;
}

int oww_inc_setup(oww_ctx* ctx, const float* h_blob) {
    // packed blob for the fused kernel: per layer fp16 [3][CGP][NP][8] | scale[NP] | bias[NP], 128-byte aligned
    IncPlan P;
    int rc = oww_inc_build_plan(ctx, 1, 1, OWW_N_CONV, &P);
    if (rc) return rc;
    std::vector<uint8_t> blob(P.w_total_bytes, 0);
    size_t off = 0;
    for (int li = 0; li < OWW_N_CONV; ++li) {
        const ConvLayer& C = ctx->conv[li];
        const size_t nw = (size_t)C.kh * C.kw * C.cin * C.cout;
        const float* w = h_blob + off; const float* sc = w + nw; const float* bi = sc + C.cout;
        off += nw + 2 * (size_t)C.cout;
        if (li == 0) continue;
        const IncLayer& L = P.L[li];
        __half* hw = reinterpret_cast<__half*>(blob.data() + L.w_off);
        // octet (tap j, plane g) -> position in the packed block [octet][np][8].  Even plane count: tap-major with the
        // pad plane zero.  Odd plane count: the chained order of the MMA loop in tc_inc_kernel -
        //   t0p0 .. t0p(cg-2) | t1p0, t0p(cg-1) | t1p1 .. t1p(cg-1) | t2p0 .. t2p(cg-2) | t2p(cg-1), zero
        const int cg = L.cg_in;
        auto octet_at = [&](int j, int g) {
            if (!(cg & 1)) return j * L.cgp + g;
            if (j == 0) return g < cg - 1 ? g : cg;
            if (j == 1) return g == 0 ? cg - 1 : cg + g;
            return 2 * cg + g;
        };
        for (int j = 0; j < 3; ++j)
            for (int g = 0; g < cg; ++g)
                for (int n = 0; n < L.np; ++n)
                    for (int e = 0; e < 8; ++e) {
                        const int c = g * 8 + e;
                        const float v = (c < C.cin && n < C.cout) ? w[((size_t)j * C.cin + c) * C.cout + n] : 0.f;
                        hw[(((size_t)octet_at(j, g)) * L.np + n) * 8 + e] = __float2half_rn(v);
                    }
        float* sb = reinterpret_cast<float*>(blob.data() + L.w_off + (size_t)3 * L.cgp * L.np * 16);
        for (int n = 0; n < L.np; ++n) { sb[n] = n < C.cout ? sc[n] : 0.f; sb[L.np + n] = n < C.cout ? bi[n] : 0.f; }
    }
    if (!ctx->d_inc_w) OWW_CUDA(ctx, cudaMalloc(&ctx->d_inc_w, blob.size()));
    OWW_CUDA(ctx, cudaMemcpy(ctx->d_inc_w, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    return OWW_OK;
}

// conv layers inside the fused kernel: all 20, or - with the incremental late layers of cnn_tc.cu - those below split_from
int oww_inc_n_layers(const oww_ctx* ctx) {
    return (ctx->cfg.cnn_mode == OWW_CNN_TC_INCREMENTAL && ctx->split_from < OWW_N_CONV) ? ctx->split_from : OWW_N_CONV;
}

int oww_inc_alloc_streams(oww_ctx* ctx) {
    // Group size: a group's latency is mostly per-layer fixed cost plus a small share per stream (modelled as
    // 50 + 6.5 G), so take the feasible G that minimises rounds(G) * T(G) for this stream count.
    int best_g = 0; double best_cost = 0;
    for (int g = 1; g <= kIncMaxG; ++g) {
        IncPlan P;
        if (oww_inc_build_plan(ctx, g, ctx->n_streams, oww_inc_n_layers(ctx), &P) != OWW_OK) continue;
        const int rounds = (P.n_groups + ctx->sm_count - 1) / ctx->sm_count;
        const double cost = rounds * (50.0 + 6.5 * g);
        if (!best_g || cost < best_cost) { best_g = g; best_cost = cost; }
    }
    if (!best_g) return oww_fail(ctx, OWW_EUNSUPPORTED, "no feasible group size for the fused CNN kernel");
    ctx->err.clear();
    int rc = oww_inc_build_plan(ctx, best_g, ctx->n_streams, oww_inc_n_layers(ctx), &ctx->inc_plan);
    if (rc) return rc;
    const size_t bytes = (size_t)ctx->inc_plan.n_groups * ctx->inc_plan.tail_units * 16;
    for (int i = 0; i < 2; ++i) {
        cudaFree(ctx->d_inc_tails[i]); ctx->d_inc_tails[i] = nullptr;
        OWW_CUDA(ctx, cudaMalloc(&ctx->d_inc_tails[i], bytes));
        OWW_CUDA(ctx, cudaMemset(ctx->d_inc_tails[i], 0, bytes));
    }
    ctx->inc_cur = 0;
    ctx->tails_template_valid = false;                   // the scatter table depends on the group size
    OWW_CUDA(ctx, cudaFuncSetAttribute(tc_inc_kernel<OWW_N_CONV>, cudaFuncAttributeMaxDynamicSharedMemorySize, ctx->inc_plan.smem_bytes));
    OWW_CUDA(ctx, cudaFuncSetAttribute(tc_inc_kernel<11>, cudaFuncAttributeMaxDynamicSharedMemorySize, ctx->inc_plan.smem_bytes));
    OWW_CUDA(ctx, cudaFuncSetAttribute(tc_inc_kernel<15>, cudaFuncAttributeMaxDynamicSharedMemorySize, ctx->inc_plan.smem_bytes));
    OWW_CUDA(ctx, cudaFuncSetAttribute(tc_inc_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, ctx->inc_plan.smem_bytes));
    return OWW_OK;
}

int oww_heads_sync_devs(oww_ctx* ctx) {
    std::vector<HeadDev> v(ctx->heads.size());
    for (size_t i = 0; i < ctx->heads.size(); ++i) {
        const Head& h = ctx->heads[i];
        HeadDev& d = v[i];
        std::memset(&d, 0, sizeof(d));
        d.blob = h.d_blob;
        d.n_in = h.desc.n_in; d.n_layers = h.desc.n_layers; d.layernorm = h.desc.layernorm; d.final_act = h.desc.final_act;
        for (int l = 0; l <= h.desc.n_layers; ++l) d.dims[l] = h.desc.dims[l];
        for (int l = 0; l < h.desc.n_layers; ++l) {
            d.w_off[l] = (int)h.w_off[l]; d.b_off[l] = (int)h.b_off[l];
            d.g_off[l] = (int)h.g_off[l]; d.h_off[l] = (int)h.h_off[l];
        }
        d.col0 = h.col0;
    }
    cudaFree(ctx->d_head_devs); ctx->d_head_devs = nullptr;
    if (v.empty()) return OWW_OK;
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_head_devs, v.size() * sizeof(HeadDev)));
    OWW_CUDA(ctx, cudaMemcpy(ctx->d_head_devs, v.data(), v.size() * sizeof(HeadDev), cudaMemcpyHostToDevice));
    return OWW_OK;
}

// Can the frontend + CNN + ring append of a one-chunk step run as the fused launch?
bool oww_fused_frontend_supported(const oww_ctx* ctx) {
    return ctx->fuse_step && ctx->cfg.cnn_mode == OWW_CNN_TC_INCREMENTAL && ctx->inc_plan.scratch_off != 0;
}

// Can the heads run inside that launch too?  (heads within the in-kernel limits; worthwhile only while re-streaming the
// first-layer matrices once per group of G streams is cheap)
bool oww_fused_heads_supported(const oww_ctx* ctx) {
    if (!oww_fused_frontend_supported(ctx) || ctx->heads.empty() || ctx->heads.size() > 16) return false;
    if (ctx->inc_plan.n_layers < OWW_N_CONV) return false;       // cut plan: the embedding is produced by the late layers' launches
    // In the fused kernel every group of G streams re-streams each head's first-layer matrix from L2; with many
    // groups x many/large heads that traffic (and the 7-row tiles) loses to the stand-alone heads kernel's 32-row tiles.
    {
        size_t w1 = 0;
        for (const Head& h : ctx->heads) w1 += (size_t)h.desc.dims[0] * h.desc.dims[1] * sizeof(float);
        if ((size_t)ctx->inc_plan.n_groups * w1 > ((size_t)256 << 20)) return false;
    }
    for (const Head& h : ctx->heads) {
        if (h.desc.dims[1] > 128) return false;
        for (int l = 1; l <= h.desc.n_layers; ++l) if (h.desc.dims[l] > 256) return false;
    }
    const size_t floats = (size_t)ctx->inc_plan.G * ((size_t)ctx->max_n_in * 96 + 4 * 128 + 2 * 256);
    int d1max = 32;
    for (const Head& h : ctx->heads) d1max = h.desc.dims[1] > d1max ? h.desc.dims[1] : d1max;
    return 2048 + floats * 4 + 128 + (size_t)96 * d1max * 4 <= (size_t)ctx->inc_plan.L[2].w_smem;
}

static void launch_inc(const IncArgs& a, int grid, cudaStream_t s) {
    if (a.plan.n_layers == OWW_N_CONV) tc_inc_kernel<OWW_N_CONV><<<grid, kIncThreads, a.plan.smem_bytes, s>>>(a);
    else if (a.plan.n_layers == 11) tc_inc_kernel<11><<<grid, kIncThreads, a.plan.smem_bytes, s>>>(a);
    else if (a.plan.n_layers == 15) tc_inc_kernel<15><<<grid, kIncThreads, a.plan.smem_bytes, s>>>(a);
    else tc_inc_kernel<0><<<grid, kIncThreads, a.plan.smem_bytes, s>>>(a);
}

static void fill_inc_args(oww_ctx* ctx, IncArgs& a) {
    std::memset(&a, 0, sizeof(a));
    a.plan = ctx->inc_plan;
    a.mel = ctx->d_mel_ring; a.mel_count = ctx->d_mel_count; a.mel_stride = (int64_t)ctx->mel_rows * 32;
    a.mel_mask = ctx->mel_rows - 1;
    a.w0 = ctx->conv[0].d_w; a.s0 = ctx->conv[0].d_scale; a.b0 = ctx->conv[0].d_bias;
    a.wblob = reinterpret_cast<const uint8_t*>(ctx->d_inc_w);
    a.tails_in = reinterpret_cast<const uint4*>(ctx->d_inc_tails[ctx->inc_cur]);
    a.tails_out = reinterpret_cast<uint4*>(ctx->d_inc_tails[ctx->inc_cur ^ 1]);
    a.B = ctx->n_streams;
    a.dbg_clock = reinterpret_cast<long long*>(ctx->d_inc_dbg);
    if (ctx->late_active) {
        a.gx = reinterpret_cast<uint4*>(ctx->late_x[ctx->split_from].buf[0]);
        a.gx_plane = ctx->late_x[ctx->split_from].plane;
        a.gx_lay = ctx->late_x[ctx->split_from].lay;
    }
}

// One launch per step: frontend, 20-layer CNN and ring append for every stream, plus - with_heads - every head and
// the verifier gates, i.e. PCM in -> scores out.
int oww_fused_step(oww_ctx* ctx, const int16_t* d_pcm, int64_t pcm_stride, float* d_scores, int out_stride, bool with_heads,
                   cudaStream_t s) {
    IncArgs a;
    fill_inc_args(ctx, a);
    a.fused = 1;
    a.pcm = d_pcm; a.pcm_stride = pcm_stride;
    a.tail = ctx->d_tail; a.seen = ctx->d_seen; a.mel_rw = ctx->d_mel_ring; a.mel_count_rw = ctx->d_mel_count;
    a.mel_window = ctx->d_window; a.mel_twiddle = ctx->d_twiddle; a.mel_start = ctx->d_mel_start; a.mel_len = ctx->d_mel_len;
    a.mel_w = ctx->d_mel_w; a.mel_kmax = ctx->mel_kmax;
    a.feat_ring = ctx->d_feat_ring; a.feat_stride = (int64_t)ctx->feat_rows * 96; a.feat_mask = ctx->feat_rows - 1;
    a.feat_count = ctx->d_feat_count;
    a.heads = ctx->d_head_devs; a.n_heads = with_heads ? (int)ctx->heads.size() : 0; a.max_n_in = ctx->max_n_in > 0 ? ctx->max_n_in : 1;
    a.scores = d_scores; a.score_stride = out_stride;
    a.gates = ctx->d_gates; a.n_gates = with_heads ? (int)ctx->gates.size() : 0;
    if (with_heads) {   // ring for the heads' first-layer weights: after feats/red/h, below the first weight slot the next group prefetches
        int d1max = 32;
        for (const Head& h : ctx->heads) d1max = h.desc.dims[1] > d1max ? h.desc.dims[1] : d1max;
        const int G = a.plan.G;
        const int used = 2048 + (G * (a.max_n_in * 96 + 4 * 128 + 2 * 256)) * 4;
        a.hring_off = (used + 127) & ~127;
        a.hslot_bytes = 96 * d1max * 4;
        const int avail = a.plan.L[2].w_smem - a.hring_off;
        a.hns = avail / a.hslot_bytes;
        if (a.hns > 4) a.hns = 4;
        if (a.hns < 1 && !ctx->heads.empty()) return oww_fail(ctx, OWW_EUNSUPPORTED, "no room for the fused heads weight ring");
    }
    const int grid = a.plan.n_groups < ctx->sm_count ? a.plan.n_groups : ctx->sm_count;
    launch_inc(a, grid, s);
    OWW_LAUNCH_CHECK(ctx);
    ctx->inc_cur ^= 1;
    return OWW_OK;
}

// One incremental CNN pass for every stream: mel rows ending `back` rows before the newest.
int oww_cnn_inc_step(oww_ctx* ctx, int back, float* d_emb, cudaStream_t s) {
    IncArgs a;
    fill_inc_args(ctx, a);
    a.back = back;
    a.emb = d_emb;
    const int grid = a.plan.n_groups < ctx->sm_count ? a.plan.n_groups : ctx->sm_count;
    launch_inc(a, grid, s);
    OWW_LAUNCH_CHECK(ctx);
    ctx->inc_cur ^= 1;
    if (ctx->late_active) return oww_late_chain(ctx, d_emb, s);
    return OWW_OK;
}

// Tail capture hook for the full-window tensor-core pyramid (cnn_tc.cu): called after the layer
// whose (possibly pooled) output feeds a (3,1) convolution.
int oww_inc_capture(oww_ctx* ctx, int layer, const void* planes, int64_t plane_pitch, int T, int W, int win0, int n_win,
                    int stream0, const int* d_ids, cudaStream_t s) {
    const IncLayer& L = ctx->inc_plan.L[layer];
    if (layer >= ctx->inc_plan.n_layers - (ctx->inc_plan.n_layers < OWW_N_CONV ? 1 : 0) || L.nx_tail_off < 0) return OWW_OK;
    const int Wp = W + 1;
    const int64_t total = (int64_t)n_win * L.cg_out * 2 * Wp;
    unsigned grid = (unsigned)((total + 255) / 256);
    tc_capture_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const uint4*>(planes), plane_pitch, T, Wp, L.cg_out, win0, n_win,
                                          stream0, d_ids, ctx->inc_plan.G, L.nx_tail_off, ctx->inc_plan.tail_units,
                                          reinterpret_cast<uint4*>(ctx->d_inc_tails[ctx->inc_cur]));
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

namespace {
__global__ void fill_ones_kernel(float* p, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = 1.0f;
}
}  // namespace

// Tails of the all-ones window in the compact single-stream (G = 1) layout + the table reset_kernel scatters them with.
// Runs the full-window tensor-core pyramid (cnn_tc.cu) once on ones(76,32) with the tail capture pointed at a G = 1 plan;
// the incremental kernel is bit-identical to that pyramid, so a stream seeded with these tails continues exactly as if
// its (constant) history had been streamed through it.  Synchronous; called lazily by the first reset after a weight load.
int oww_inc_build_template(oww_ctx* ctx) {
    if (!ctx->emb_loaded) return oww_fail(ctx, OWW_EINVAL, "embedding weights not loaded");
    if (!ctx->d_tc_act[0] || !ctx->d_inc_tails[0]) return oww_fail(ctx, OWW_EINVAL, "oww_set_streams has not been called");
    IncPlan P1;
    int rc = oww_inc_build_plan(ctx, 1, 1, ctx->inc_plan.n_layers, &P1);
    if (rc) return rc;
    ctx->n_tail_tab = 0;
    for (int l = 0; l < OWW_N_CONV; ++l)
        if (P1.L[l].nx_tail_off >= 0)
            ctx->tail_tab[ctx->n_tail_tab++] = make_int4(P1.L[l].nx_tail_off, ctx->inc_plan.L[l].nx_tail_off, P1.L[l].cg_out, P1.L[l].nx_Wp);
    cudaFree(ctx->d_tails_template); ctx->d_tails_template = nullptr;
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_tails_template, (size_t)P1.tail_units * 16));
    OWW_CUDA(ctx, cudaMemset(ctx->d_tails_template, 0, (size_t)P1.tail_units * 16));
    float* d_ones = nullptr; float* d_emb = nullptr;
    OWW_CUDA(ctx, cudaMalloc(&d_ones, OWW_WINDOW_ROWS * 32 * sizeof(float)));
    OWW_CUDA(ctx, cudaMalloc(&d_emb, 96 * sizeof(float)));
    fill_ones_kernel<<<(OWW_WINDOW_ROWS * 32 + 255) / 256, 256>>>(d_ones, OWW_WINDOW_ROWS * 32);
    // point the capture hook at the G = 1 layout for this one pass
    const IncPlan saved_plan = ctx->inc_plan;
    void* const saved_tails = ctx->d_inc_tails[ctx->inc_cur];
    ctx->inc_plan = P1;
    ctx->d_inc_tails[ctx->inc_cur] = ctx->d_tails_template;
    WindowSrc src{d_ones, (int64_t)OWW_WINDOW_ROWS * 32, nullptr, -1, 0, 0};
    TailCapture cap{0, 1, 0};
    cap.late = ctx->late_active;
    rc = oww_cnn_tc_pyramid_cap(ctx, src, 1, d_emb, &cap, nullptr);
    cudaError_t e = cudaDeviceSynchronize();
    ctx->inc_plan = saved_plan;
    ctx->d_inc_tails[ctx->inc_cur] = saved_tails;
    cudaFree(d_ones); cudaFree(d_emb);
    if (rc) return rc;
    if (e != cudaSuccess) return oww_fail(ctx, OWW_ECUDA, "tails template: %s", cudaGetErrorString(e));
    ctx->tails_template_valid = true;
    return OWW_OK;
}
