// C ABI of libowwb200.so (include/owwb200.h): handle lifetime, weight upload, stream state and the
// orchestration of one streaming step  PCM -> K1 mel -> K2 embedding CNN -> ring append -> K3 heads.
#include "oww_internal.h"
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <climits>
#include <functional>
#include <numeric>

static thread_local std::string g_create_error;

int oww_fail(oww_ctx* ctx, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (ctx) ctx->err = buf; else g_create_error = buf;
    return code;
}

int oww_order_begin(oww_ctx* ctx, cudaStream_t s) {
    if (s == ctx->own_stream) return OWW_OK;
    OWW_CUDA(ctx, cudaEventRecord(ctx->order_ev[0], ctx->own_stream));
    OWW_CUDA(ctx, cudaStreamWaitEvent(s, ctx->order_ev[0], 0));
    return OWW_OK;
}

int oww_order_end(oww_ctx* ctx, cudaStream_t s) {
    if (s == ctx->own_stream) return OWW_OK;
    OWW_CUDA(ctx, cudaEventRecord(ctx->order_ev[1], s));
    OWW_CUDA(ctx, cudaStreamWaitEvent(ctx->own_stream, ctx->order_ev[1], 0));
    return OWW_OK;
}

namespace {

const int kLayerTable[OWW_N_CONV][6] = {   // kh kw cin cout pool_t pool_f  (SURVEY.md Appendix B)
    {3, 3, 1, 24, 0, 0},
    {1, 3, 24, 24, 0, 0}, {3, 1, 24, 24, 2, 2},
    {1, 3, 24, 48, 0, 0}, {3, 1, 48, 48, 0, 0},
    {1, 3, 48, 48, 0, 0}, {3, 1, 48, 48, 1, 2},
    {1, 3, 48, 72, 0, 0}, {3, 1, 72, 72, 0, 0},
    {1, 3, 72, 72, 0, 0}, {3, 1, 72, 72, 2, 2},
    {1, 3, 72, 96, 0, 0}, {3, 1, 96, 96, 0, 0},
    {1, 3, 96, 96, 0, 0}, {3, 1, 96, 96, 1, 2},
    {1, 3, 96, 96, 0, 0}, {3, 1, 96, 96, 0, 0},
    {1, 3, 96, 96, 0, 0}, {3, 1, 96, 96, 2, 2},
    {3, 1, 96, 96, 0, 0},
};

void fill_layer_table(oww_ctx* ctx) {
    for (int li = 0; li < OWW_N_CONV; ++li) {
        ConvLayer& L = ctx->conv[li];
        L.kh = kLayerTable[li][0]; L.kw = kLayerTable[li][1]; L.cin = kLayerTable[li][2]; L.cout = kLayerTable[li][3];
        L.pool_t = kLayerTable[li][4]; L.pool_f = kLayerTable[li][5];
        L.d_w = L.d_scale = L.d_bias = nullptr;
    }
}

int next_pow2(int v) { int p = 1; while (p < v) p <<= 1; return p; }

// Mode 3: every 16-byte unit of stream b's conv tails state, in the CTA's threads.  early(t, at): unit t of the compact
// G = 1 layout (the template, a stream record) is unit `at` of the G-group tails buffers - layout [(r*G + g)*Wp + f] of
// each tails-bearing tensor.  late(T, i, pl, r, f, at): unit i of late tensor T's [plane][2][Wp] rows is unit `at` of its
// block-major layout (cnn_tc.cu, tc_conv_blk_kernel: no pad column, so cells f >= Wq are not visited).
template <class Early, class Late>
__device__ __forceinline__ void for_each_tail_unit(const ResetTails& rt, int b, Early early, Late late) {
    const int grp = b / rt.G, g = b - grp * rt.G;
    const int64_t base = (int64_t)grp * rt.tail_units;
    for (int k = 0; k < rt.n_tab; ++k) {
        const int off1 = rt.tab[k].x, offG = rt.tab[k].y, cg = rt.tab[k].z, Wp = rt.tab[k].w;
        for (int i = threadIdx.x; i < cg * 2 * Wp; i += blockDim.x) {
            const int pl = i / (2 * Wp), u = i - pl * 2 * Wp, r = u / Wp, f = u - r * Wp;
            early(off1 + i, base + offG + pl * (2 * rt.G * Wp) + (r * rt.G + g) * Wp + f);
        }
    }
    for (int k = 0; k < rt.n_late; ++k) {
        const ResetLate& T = rt.late[k];
        for (int i = threadIdx.x; i < T.n_planes * 2 * T.Wp; i += blockDim.x) {
            const int pl = i / (2 * T.Wp), u = i - pl * 2 * T.Wp, r = u / T.Wp, f = u - r * T.Wp;
            if (f < T.lay.Wq) late(T, i, pl, r, f, late_unit(T.lay, pl, b, r, f));
        }
    }
}

// a late tails row the next step reads: rows 0, 1 of `now`; tensors that gain one row per step also read row 1 as row 0
// of the buffer of the step after
__device__ __forceinline__ void put_late(const ResetLate& T, int b, int pl, int r, int f, int64_t at, uint4 v) {
    T.now[at] = v;
    if (T.next && r == 1) T.next[late_unit(T.lay, pl, b, 0, f)] = v;
}

__global__ void reset_kernel(const int* ids, int n_ids, int n_streams, int16_t* tail, int* seen, int* mel_count,
                             int* feat_count, float* mel_ring, int mel_rows, float* feat_ring, int feat_rows,
                             const float* feat_init, int n_rows, ResetTails rt) {
    const int j = blockIdx.x;
    const int b = ids ? ids[j] : j;
    if (b < 0 || b >= n_streams) return;
    if (rt.tails)       // mode 3: the conv tails of the all-ones window (the stream's history after a reset)
        for_each_tail_unit(rt, b, [&](int t, int64_t at) { rt.tails[at] = rt.tmpl[t]; },
                           [&](const ResetLate& T, int i, int pl, int r, int f, int64_t at) { put_late(T, b, pl, r, f, at, T.tmpl[i]); });
    for (int i = threadIdx.x; i < OWW_TAIL; i += blockDim.x) tail[(int64_t)b * OWW_TAIL + i] = 0;
    float* mr = mel_ring + (int64_t)b * mel_rows * 32;
    for (int i = threadIdx.x; i < mel_rows * 32; i += blockDim.x) mr[i] = 1.0f;     // np.ones((76,32)), utils.py:165
    float* fr = feat_ring + (int64_t)b * feat_rows * 96;
    for (int i = threadIdx.x; i < feat_rows * 96; i += blockDim.x)
        fr[i] = (i < n_rows * 96 && feat_init) ? feat_init[i] : 0.f;
    if (threadIdx.x == 0) {
        seen[b] = 0;
        mel_count[b] = OWW_WINDOW_ROWS;
        feat_count[b] = n_rows;
    }
}

// Ragged step, mode 3: the streams ids[0..n_ids) did not step in the CNN launch that just ran (dead slots: it wrote no
// tails for them).  Their tails state moves unchanged to the buffers the next launch reads - reset_kernel's scatter with
// the stream's own pre-launch rows as the source (ResetTails: tmpl = the G-group tails buffer the launch read, late[].tmpl
// = the late buffer it read; the late chain left rows 0..1 of those untouched).
__global__ void carry_kernel(const int* ids, int n_ids, ResetTails rt) {
    oww_pdl_sync();
    const int b = ids[blockIdx.x];
    for_each_tail_unit(rt, b, [&](int, int64_t at) { rt.tails[at] = rt.tmpl[at]; },
                       [&](const ResetLate& T, int, int pl, int r, int f, int64_t at) { put_late(T, b, pl, r, f, at, T.tmpl[at]); });
}

// ---- stream records (include/owwb200.h, oww_export_streams): one stream's state in a layout that depends only on the
//      cnn_mode, split_from and the weights.  16-byte units:
//        [0, 2)     header: version, record bytes, configuration key | seen, mel count, feature count, 0
//        [2, 62)    the 480-sample PCM tail
//        [62, 670)  the newest 76 mel rows, oldest first
//        [670, 3550) the newest 120 feature rows, oldest first (rows before the stream's first read as zeros)
//        [3550, +u_tails)   mode 3: the conv tails in the compact G = 1 layout of the template (tail_tab)
//        [.., +u_late)      mode 3: rows 0..1 of each tails-bearing late tensor, [plane][2][Wp] at its template offset
constexpr uint32_t kRecVersion = 1;
constexpr int kRecPcm = 2, kRecMel = 62, kRecFeat = 670, kRecTails = 3550;
constexpr int kRecMelRows = OWW_WINDOW_ROWS, kRecFeatRows = 120;      // 120: the reference's feature_buffer cap

struct StreamState {
    int16_t* tail; int* seen; int* mel_count; int* feat_count;
    float* mel_ring; int mel_rows; float* feat_ring; int feat_rows;
    int64_t rec_units;               // units per record
    int u_tails;                     // units of the early conv tails section (the late section follows it)
    uint32_t bytes; uint64_t key;
    int* rejected;
};

// one CTA per record: stream ids[j]'s state -> record j
__global__ void __launch_bounds__(256) stream_export_kernel(const int* ids, StreamState a, ResetTails rt, uint4* rec) {
    const int b = ids[blockIdx.x];
    uint4* r = rec + (int64_t)blockIdx.x * a.rec_units;
    const int mc = a.mel_count[b], fc = a.feat_count[b];
    if (threadIdx.x == 0) {
        r[0] = make_uint4(kRecVersion, a.bytes, (uint32_t)a.key, (uint32_t)(a.key >> 32));
        r[1] = make_uint4((uint32_t)a.seen[b], (uint32_t)mc, (uint32_t)fc, 0u);
    }
    const uint4* tail = reinterpret_cast<const uint4*>(a.tail + (int64_t)b * OWW_TAIL);
    for (int i = threadIdx.x; i < OWW_TAIL / 8; i += blockDim.x) r[kRecPcm + i] = tail[i];
    const uint4* mel = reinterpret_cast<const uint4*>(a.mel_ring + (int64_t)b * a.mel_rows * 32);
    for (int i = threadIdx.x; i < kRecMelRows * 8; i += blockDim.x) {
        const int k = i >> 3;
        r[kRecMel + i] = mel[((mc - kRecMelRows + k) & (a.mel_rows - 1)) * 8 + (i & 7)];
    }
    const uint4* feat = reinterpret_cast<const uint4*>(a.feat_ring + (int64_t)b * a.feat_rows * 96);
    for (int i = threadIdx.x; i < kRecFeatRows * 24; i += blockDim.x) {
        const int k = i / 24, row = fc - kRecFeatRows + k;
        r[kRecFeat + i] = row < 0 ? make_uint4(0, 0, 0, 0) : feat[(row & (a.feat_rows - 1)) * 24 + (i - k * 24)];
    }
    if (!rt.tails) return;
    uint4* tails = r + kRecTails;
    uint4* late = tails + a.u_tails;
    const int64_t n_tails = a.rec_units - kRecTails;                 // pad cells the gather does not visit stay zero
    for (int64_t i = threadIdx.x; i < n_tails; i += blockDim.x) tails[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    for_each_tail_unit(rt, b, [&](int t, int64_t at) { tails[t] = rt.tails[at]; },
                       [&](const ResetLate& T, int i, int, int, int, int64_t at) { late[T.off + i] = T.now[at]; });
}

// one CTA per record: record j -> stream ids[j] (reset_kernel's scatter with the record as the source).  A record whose
// header does not match the handle (or whose counts are impossible) is skipped and counted.  Counts at or past 2^30,
// which no step leaves behind, are rebased as a step would rebase them: a step adds at most 8 * OWW_MAX_CHUNKS rows,
// which then cannot overflow int.
__global__ void __launch_bounds__(256) stream_import_kernel(const int* ids, StreamState a, ResetTails rt, const uint4* rec) {
    const int b = ids[blockIdx.x];
    const uint4* r = rec + (int64_t)blockIdx.x * a.rec_units;
    const uint4 h0 = r[0], h1 = r[1];
    const int seen = (int)h1.x, mc = oww_wrap_count((int)h1.y), fc = oww_wrap_count((int)h1.z);
    if (h0.x != kRecVersion || h0.y != a.bytes || h0.z != (uint32_t)a.key || h0.w != (uint32_t)(a.key >> 32) ||
        seen < 0 || mc < kRecMelRows || fc < 0) {
        if (threadIdx.x == 0) atomicAdd(a.rejected, 1);
        return;
    }
    uint4* tail = reinterpret_cast<uint4*>(a.tail + (int64_t)b * OWW_TAIL);
    for (int i = threadIdx.x; i < OWW_TAIL / 8; i += blockDim.x) tail[i] = r[kRecPcm + i];
    // ring slot s holds row mc - rows + ((s - mc) & mask); the record's row k = that row - (mc - 76).  Older slots get
    // what a reset leaves there (ones / zeros): no step and no read reaches them.
    const float one = 1.0f;
    const uint32_t ones = __float_as_uint(one);
    uint4* mel = reinterpret_cast<uint4*>(a.mel_ring + (int64_t)b * a.mel_rows * 32);
    for (int i = threadIdx.x; i < a.mel_rows * 8; i += blockDim.x) {
        const int k = kRecMelRows - a.mel_rows + (((i >> 3) - mc) & (a.mel_rows - 1));
        mel[i] = k < 0 ? make_uint4(ones, ones, ones, ones) : r[kRecMel + k * 8 + (i & 7)];
    }
    uint4* feat = reinterpret_cast<uint4*>(a.feat_ring + (int64_t)b * a.feat_rows * 96);
    for (int i = threadIdx.x; i < a.feat_rows * 24; i += blockDim.x) {
        const int s = i / 24, k = kRecFeatRows - a.feat_rows + ((s - fc) & (a.feat_rows - 1));
        feat[i] = k < 0 ? make_uint4(0, 0, 0, 0) : r[kRecFeat + k * 24 + (i - s * 24)];
    }
    if (threadIdx.x == 0) { a.seen[b] = seen; a.mel_count[b] = mc; a.feat_count[b] = fc; }
    if (!rt.tails) return;
    const uint4* tails = r + kRecTails;
    const uint4* late = tails + a.u_tails;
    for_each_tail_unit(rt, b, [&](int t, int64_t at) { rt.tails[at] = tails[t]; },
                       [&](const ResetLate& T, int i, int pl, int rr, int f, int64_t at) { put_late(T, b, pl, rr, f, at, late[T.off + i]); });
}

// Ragged step: stream b appends embedding rows n - cnt[b] .. n - 1 of emb [n][B][96] (its own chunks, oldest first) to
// its feature ring and advances its count by cnt[b].  One warp per stream.
__global__ void __launch_bounds__(256) feat_append_ragged_kernel(const float* emb, float* ring, int* count, int B, int n,
                                                                 const int* cnt, int rows_mask, int64_t ring_stride) {
    oww_pdl_sync();
    const int b = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= B) return;
    const int c = cnt[b];
    if (c == 0) return;
    const int c0 = count[b];
    for (int i = lane; i < c * 24; i += 32) {
        const int j = i / 24, c4 = i - j * 24;           // j-th of the stream's chunks = launch n - c + j
        reinterpret_cast<float4*>(ring + (int64_t)b * ring_stride + (int64_t)((c0 + j) & rows_mask) * 96)[c4] =
            __ldg(reinterpret_cast<const float4*>(emb + ((int64_t)(n - c + j) * B + b) * 96) + c4);
    }
    __syncwarp();
    if (lane == 0) count[b] = oww_wrap_count(c0 + c);
}

// Ragged step: score row of stream b = per column the max over its own cnt[b] chunk windows (src [back][B][n_out], back 0
// = newest; verifier gates were applied per window by the heads).  Rows of held streams (cnt 0) are not written.
__global__ void ragged_max_kernel(const float* src, int B, int n_out, const int* cnt, float* dst, int out_stride) {
    oww_pdl_sync();
    const int64_t total = (int64_t)B * n_out;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(i / n_out), col = (int)(i - (int64_t)b * n_out);
        const int k = cnt[b];
        if (k == 0) continue;
        float v = src[i];
        for (int j = 1; j < k; ++j) v = fmaxf(v, src[(int64_t)j * total + i]);
        dst[(int64_t)b * out_stride + col] = v;
    }
}

}  // namespace
// Tails of the all-ones window per tails-bearing tensor, in the compact G = 1 layout, computed once per weight set by
// the full-window tensor-core kernels (cnn_tc.cu) - the state every freshly reset stream starts from (its mel history IS
// ones(76,32), utils.py:165, and a constant history is shift invariant, so no per-stream re-priming pass is needed).
int oww_inc_build_template(oww_ctx* ctx);
namespace {

void free_streams(oww_ctx* c) {
    cudaFree(c->d_tail); cudaFree(c->d_seen); cudaFree(c->d_mel_count); cudaFree(c->d_feat_count);
    cudaFree(c->d_mel_ring); cudaFree(c->d_feat_ring); cudaFree(c->d_act[0]); cudaFree(c->d_act[1]);
    cudaFree(c->d_emb_tmp); cudaFree(c->d_inc_tails[0]); cudaFree(c->d_inc_tails[1]);
    cudaFree(c->d_reset_ids); cudaFree(c->d_reset_init);
    cudaFree(c->d_state_ids); c->d_state_ids = nullptr;
    cudaFree(c->d_scores_tmp);
    cudaFree(c->d_rag_scores); c->d_rag_scores = nullptr; c->rag_scores_floats = 0;
    for (int j = 0; j < oww_ctx::kRagSlots; ++j) {       // set_streams / destroy synchronise the device first
        cudaFreeHost(c->h_rag[j]); cudaFree(c->d_rag[j]); c->h_rag[j] = nullptr; c->d_rag[j] = nullptr;
    }
    c->rag_streams = 0;
    oww_verifiers_free_streams(c);
    oww_detect_free_streams(c);
    oww_audio_free_streams(c);
    oww_ingest_free_streams(c);
    oww_heads_grp_drop_mirror(c);
    for (auto& X : c->late_x) for (auto& b : X.buf) { cudaFree(b); b = nullptr; }
    cudaFree(c->d_late_tmp); c->d_late_tmp = nullptr;
    cudaFree(c->d_late_template); c->d_late_template = nullptr;
    c->late_active = false;
    c->d_tail = nullptr; c->d_seen = c->d_mel_count = c->d_feat_count = nullptr;
    c->d_mel_ring = c->d_feat_ring = c->d_act[0] = c->d_act[1] = c->d_emb_tmp = nullptr;
    c->d_inc_tails[0] = c->d_inc_tails[1] = nullptr;
    c->d_reset_ids = nullptr; c->d_reset_init = nullptr;
    c->d_scores_tmp = nullptr; c->scores_tmp_floats = 0;
    c->act_floats = c->emb_tmp_floats = 0;
    c->n_streams = 0;
}

// grow the fp16 plane scratch of the tensor-core window / clip passes to `units` 16-byte units per buffer
int ensure_tc_units(oww_ctx* ctx, size_t units) {
    if (ctx->tc_act_units >= units) return OWW_OK;
    cudaFree(ctx->d_tc_act[0]); cudaFree(ctx->d_tc_act[1]);
    ctx->d_tc_act[0] = ctx->d_tc_act[1] = nullptr; ctx->tc_act_units = 0;
    for (int i = 0; i < 2; ++i) {
        OWW_CUDA(ctx, cudaMalloc(&ctx->d_tc_act[i], units * 16));
        OWW_CUDA(ctx, cudaMemset(ctx->d_tc_act[i], 0, units * 16));
    }
    ctx->tc_act_units = units;
    return OWW_OK;
}

int ensure_act(oww_ctx* ctx, size_t floats) {
    if (ctx->cfg.cnn_mode == OWW_CNN_TC_WINDOW || ctx->cfg.cnn_mode == OWW_CNN_TC_INCREMENTAL) {
        // `floats` is n_windows * 74*32*24 (layer-1 output of the fp32 path): size the fp16 planes for the same windows
        int n_win = (int)(floats / ((size_t)74 * 32 * 24));
        if (n_win < 1) n_win = 1;
        if (n_win > ctx->window_batch) n_win = ctx->window_batch;
        const int rc = ensure_tc_units(ctx, oww_tc_act_units(ctx, n_win));
        if (rc) return rc;
    }
    if (ctx->act_floats >= floats) return OWW_OK;
    cudaFree(ctx->d_act[0]); cudaFree(ctx->d_act[1]);
    ctx->d_act[0] = ctx->d_act[1] = nullptr; ctx->act_floats = 0;
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_act[0], floats * sizeof(float)));
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_act[1], floats * sizeof(float)));
    ctx->act_floats = floats;
    return OWW_OK;
}

// clips per slab of a clip pass over T mel rows: 1 GiB of fp16 planes per buffer of the tensor-core CNN
int clip_slab(const oww_ctx* ctx, int n, int T) {
    return (int)std::min<size_t>(n, std::max<size_t>(1, ((size_t)1 << 26) / oww_tc_act_units_T(ctx, 1, T)));
}

// Fully convolutional CNN pass over linear mel [n][T][32] (T >= 76, SURVEY.md F10): the (T - 76) / 8 + 1 embedding rows
// of input i land at d_emb + i * out_rows * 96.  Slabs of inputs bounded by the mode's activation scratch.
int oww_cnn_clip(oww_ctx* ctx, const float* d_mel, int n, int T, float* d_emb, int out_rows, cudaStream_t s) {
    if (!ctx->emb_loaded) return oww_fail(ctx, OWW_EINVAL, "embedding weights not loaded");
    if (T < OWW_WINDOW_ROWS) return oww_fail(ctx, OWW_EINVAL, "need at least 76 mel rows");
    const int t_use = OWW_WINDOW_ROWS + 8 * ((T - OWW_WINDOW_ROWS) / 8);
    const bool tc = ctx->cfg.cnn_mode != OWW_CNN_FP32_WINDOW;
    int slab, rc;
    if (tc) {
        slab = clip_slab(ctx, n, t_use);
        rc = ensure_tc_units(ctx, oww_tc_act_units_T(ctx, slab, t_use));
    } else {
        const size_t per = (size_t)(t_use - 2) * 32 * 24;          // layer-1 output of one input, the largest tensor
        rc = ensure_act(ctx, std::max(per, (size_t)ctx->window_batch * 74 * 32 * 24));
        slab = (int)(ctx->act_floats / per);
    }
    if (rc) return rc;
    for (int c0 = 0; c0 < n; c0 += slab) {
        const int m = std::min(slab, n - c0);
        const WindowSrc src{d_mel + (int64_t)c0 * T * 32, (int64_t)T * 32, nullptr, -1, 0, 0};
        float* out = d_emb + (int64_t)c0 * out_rows * 96;
        rc = tc ? oww_cnn_tc_pyramid(ctx, src, m, t_use, out, out_rows, -1, nullptr, s)
                : oww_cnn_fp32_pyramid(ctx, src, m, t_use, out, out_rows, -1, nullptr, s);
        if (rc) return rc;
    }
    return OWW_OK;
}

__global__ void fill_init_rows_kernel(float* feats, int64_t clip_stride, int n_clips, const float* init, int n_rows) {
    const int64_t total = (int64_t)n_clips * n_rows * 24;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % 24);
        const int r = (int)((i / 24) % n_rows);
        const int64_t clip = i / ((int64_t)24 * n_rows);
        reinterpret_cast<float4*>(feats + clip * clip_stride + (int64_t)r * 96)[c4] =
            init ? __ldg(reinterpret_cast<const float4*>(init + (int64_t)r * 96) + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

int ensure_emb_tmp(oww_ctx* ctx, size_t floats) {
    if (ctx->emb_tmp_floats >= floats) return OWW_OK;
    cudaFree(ctx->d_emb_tmp); ctx->d_emb_tmp = nullptr; ctx->emb_tmp_floats = 0;
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_emb_tmp, floats * sizeof(float)));
    ctx->emb_tmp_floats = floats;
    return OWW_OK;
}

// Slabs of the bulk clip path over clips sorted by step count, longest first: neighbours in that order, at most the clips
// whose planes fit the clip pass's scratch at the slab's longest clip (clip_slab), and none more than 1/20 of that
// clip's steps shorter.  Every clip of a slab runs for the longest one's K steps, so the steps computed exceed the steps
// needed by at most 5 %.  Clips of equal length at chunk_size 1280 form the slabs oww_predict_clips always had.
struct ClipSlab { int b, e, K; };
std::vector<ClipSlab> plan_slabs(const oww_ctx* ctx, const std::vector<int>& steps_desc) {
    std::vector<ClipSlab> out;
    const int n = (int)steps_desc.size();
    for (int b = 0; b < n;) {
        const int K = steps_desc[b], seg = std::min(K, 8192);
        const int cap = clip_slab(ctx, n - b, OWW_WINDOW_ROWS + 8 * (seg - 1));
        int e = b + 1;
        while (e < n && e - b < cap && 20 * (int64_t)(K - steps_desc[e]) <= K) ++e;
        out.push_back(ClipSlab{b, e, K});
        b = e;
    }
    return out;
}

// Score row of a call = per column the max over its chunks' rows (verifier gates were applied per chunk by the heads):
// dst[out_row[r]] = max(src[q_last[r] - k[r] + 1 .. q_last[r]]), stepped[out_row[r]] = 1.  q_last / k nullptr: one row, r;
// out_row nullptr: row r (compact).
__global__ void call_max_kernel(const float* src, int n_out, const int* q_last, const int* k, int n, float* dst,
                                const int* out_row, uint8_t* stepped) {
    const int64_t total = (int64_t)n * n_out;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / n_out), col = (int)(i - (int64_t)r * n_out);
        const int q = q_last ? q_last[r] : r, kr = k ? k[r] : 1;
        float v = src[(int64_t)q * n_out + col];
        for (int j = 1; j < kr; ++j) v = fmaxf(v, src[(int64_t)(q - j) * n_out + col]);
        const int64_t o = out_row ? out_row[r] : r;
        dst[o * n_out + col] = v;
        if (stepped && col == 0) stepped[o] = 1;
    }
}

int call_max_launch(oww_ctx* ctx, const float* src, int n_out, const int* q_last, const int* k, int n, float* dst,
                    const int* out_row, uint8_t* stepped, cudaStream_t s) {
    if (n <= 0 || n_out <= 0) return OWW_OK;
    const int64_t total = (int64_t)n * n_out;
    call_max_kernel<<<(int)std::min<int64_t>(4096, (total + 255) / 256), 256, 0, s>>>(src, n_out, q_last, k, n, dst, out_row, stepped);
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

// the embedding rows each clip's own steps appended: feature rows [init_rows, init_rows + steps[p]) of slab clip p ->
// d_emb rows from emb0[p] on
__global__ void emb_rows_kernel(const float* feats, int64_t clip_stride, int init_rows, int K, int m, const int* steps,
                                const int64_t* emb0, float* d_emb) {
    const int64_t total = (int64_t)m * K * 24;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % 24);
        const int r = (int)((i / 24) % K);
        const int p = (int)(i / ((int64_t)24 * K));
        if (r >= steps[p]) continue;
        reinterpret_cast<float4*>(d_emb + (emb0[p] + r) * 96)[c4] =
            reinterpret_cast<const float4*>(feats + p * clip_stride + (int64_t)(init_rows + r) * 96)[c4];
    }
}

// rows of n_chunks * 1280 samples must not overlap: a shorter stride would step one stream on its neighbour's samples
int stride_check(oww_ctx* ctx, int64_t pcm_stride, int n_chunks) {
    if (pcm_stride < (int64_t)n_chunks * OWW_SAMPLES_PER_CHUNK)
        return oww_fail(ctx, OWW_EINVAL, "pcm_stride=%lld < %d samples (%d chunks)", (long long)pcm_stride,
                        n_chunks * OWW_SAMPLES_PER_CHUNK, n_chunks);
    return OWW_OK;
}

// what step_core refuses before it enqueues anything
int step_core_check(oww_ctx* ctx, int64_t pcm_stride, int n_chunks) {
    int rc;
    if (ctx->n_streams <= 0) return oww_fail(ctx, OWW_EINVAL, "oww_set_streams has not been called");
    if (n_chunks < 1 || n_chunks > ctx->cfg.max_chunks)
        return oww_fail(ctx, OWW_EINVAL, "n_chunks=%d outside [1,%d]", n_chunks, ctx->cfg.max_chunks);
    if ((rc = stride_check(ctx, pcm_stride, n_chunks))) return rc;
    if (!ctx->mel_loaded || !ctx->emb_loaded) return oww_fail(ctx, OWW_EINVAL, "weights not loaded");
    return OWW_OK;
}

int step_core(oww_ctx* ctx, const int16_t* d_pcm, int64_t pcm_stride, int n_chunks, float* d_scores, int out_stride,
              cudaStream_t s) {
    const int B = ctx->n_streams;
    int rc;
    if ((rc = step_core_check(ctx, pcm_stride, n_chunks))) return rc;
    const long slot = ctx->timing ? ctx->ev_steps % ctx->ev_slots : 0;
    cudaEvent_t* ev = ctx->timing ? &ctx->ev[4 * slot] : nullptr;
    const bool inc = ctx->cfg.cnn_mode == OWW_CNN_TC_INCREMENTAL;
    const FeatSrc fs0{ctx->d_feat_ring, (int64_t)ctx->feat_rows * 96, ctx->d_feat_count, ctx->feat_rows - 1, 0};

    if (inc && n_chunks == 1 && oww_fused_frontend_supported(ctx)) {
        // ---- one chunk: frontend + CNN + ring append of every stream in ONE launch (fresh streams included: a reset
        //      leaves the tails of the all-ones window behind, see reset_kernel) ----
        const bool heads_inside = oww_fused_heads_supported(ctx);
        if (ev) OWW_CUDA(ctx, cudaEventRecord(ev[1], s));
        if ((rc = oww_fused_step(ctx, d_pcm, pcm_stride, d_scores, out_stride, heads_inside, s))) return rc;
        if (ctx->late_active) {
            // cut plan: conv layers >= split_from run as their own launches (split operands) and the embedding is appended here
            if ((rc = oww_late_chain(ctx, ctx->d_emb_tmp, s))) return rc;
            if ((rc = oww_feat_append(ctx, ctx->d_emb_tmp, 1, s))) return rc;
        }
        if (ev) OWW_CUDA(ctx, cudaEventRecord(ev[2], s));
        if (heads_inside) oww_feat16_invalidate(ctx);
        else if ((rc = oww_feat16_advance(ctx, 1, s))) return rc;
        if (!heads_inside && (rc = oww_heads_all(ctx, fs0, B, d_scores, out_stride, 0, s))) return rc;
        if (heads_inside && (rc = oww_head_banks_launch(ctx, fs0, B, d_scores, out_stride, 0, s))) return rc;
        if ((rc = oww_verifiers_apply(ctx, fs0, B, d_scores, out_stride, false, s))) return rc;
        if (ev) {
            if (heads_inside) ctx->ev_fused[slot] = 1;
            else { OWW_CUDA(ctx, cudaEventRecord(ev[3], s)); ctx->ev_fused[slot] = 2; }
            ctx->ev_steps++;
        }
        return OWW_OK;
    }

    // ---- general path: separate launches (modes 0 / 2, multi-chunk calls, --no-fuse) ----
    if (ev) { OWW_CUDA(ctx, cudaEventRecord(ev[0], s)); ctx->ev_fused[slot] = 0; }
    MelLaunch m{d_pcm, pcm_stride, n_chunks * OWW_SAMPLES_PER_CHUNK, ctx->d_tail, ctx->d_seen, ctx->d_mel_ring,
                (int64_t)ctx->mel_rows * 32, ctx->mel_rows - 1, ctx->d_mel_count, B, 1, n_chunks};
    if ((rc = oww_mel_launch(ctx, m, s))) return rc;
    if (ev) OWW_CUDA(ctx, cudaEventRecord(ev[1], s));
    WindowSrc ws{ctx->d_mel_ring, (int64_t)ctx->mel_rows * 32, ctx->d_mel_count, ctx->mel_rows - 1, B, n_chunks};
    if (inc) {
        // one incremental launch per chunk on the 8 mel rows that chunk added (a fresh stream's first chunk added 5:
        // the three rows before them are ones of its initial ring, which is what the step then reads)
        for (int i = 0; i < n_chunks; ++i)
            if ((rc = oww_cnn_inc_step(ctx, 8 * (n_chunks - 1 - i), ctx->d_emb_tmp + (size_t)i * B * 96, s))) return rc;
    } else {
        if ((rc = oww_cnn_window(ctx, ws, B * n_chunks, ctx->d_emb_tmp, s, false))) return rc;
    }
    if ((rc = oww_feat_append(ctx, ctx->d_emb_tmp, n_chunks, s))) return rc;
    if (ev) OWW_CUDA(ctx, cudaEventRecord(ev[2], s));
    if ((rc = oww_feat16_advance(ctx, n_chunks, s))) return rc;
    for (int i = n_chunks - 1; i >= 0; --i) {
        FeatSrc fs = fs0; fs.back = i;
        if ((rc = oww_heads_all(ctx, fs, B, d_scores, out_stride, i != n_chunks - 1, s))) return rc;
    }
    // custom verifiers: after the max over the chunk windows, on the newest window (model.py:319-328)
    if ((rc = oww_verifiers_apply(ctx, fs0, B, d_scores, out_stride, false, s))) return rc;
    if (ev) { OWW_CUDA(ctx, cudaEventRecord(ev[3], s)); ctx->ev_steps++; }
    return OWW_OK;
}

// Mode 3: where the tails state the next CNN launch reads lives - the G-group tails buffer d_inc_tails[inc_cur] and, per
// tails-bearing late tensor, rows 0..1 of buf[k % n_buf] (+ row 0 of buf[(k + 1) % 3] for tensors that gain one row per
// step) at k = late_step.  The sources (tmpl) are the caller's: reset_kernel's template or carry_kernel's own state.
int next_step_tables(oww_ctx* ctx, ResetTails& rt) {
    std::memset(&rt, 0, sizeof(rt));
    if (!ctx->tails_template_valid) { int rc = oww_inc_build_template(ctx); if (rc) return rc; }   // fills tail_tab
    rt.tails = reinterpret_cast<uint4*>(ctx->d_inc_tails[ctx->inc_cur]);
    rt.G = ctx->inc_plan.G; rt.tail_units = ctx->inc_plan.tail_units; rt.n_tab = ctx->n_tail_tab;
    for (int k = 0; k < ctx->n_tail_tab; ++k) rt.tab[k] = ctx->tail_tab[k];
    if (ctx->late_active) {
        const long k = ctx->late_step;                      // index of the next chunk any stream processes
        for (int l = ctx->split_from; l < OWW_N_CONV; ++l) {
            const oww_ctx::LateTensor& X = ctx->late_x[l];
            if (X.tmpl_off < 0) continue;
            ResetLate& T = rt.late[rt.n_late++];
            T.now = reinterpret_cast<uint4*>(X.buf[k % X.n_buf]);
            T.next = X.n_buf == 3 ? reinterpret_cast<uint4*>(X.buf[(k + 1) % 3]) : nullptr;
            T.Wp = X.W + 1; T.n_planes = 2 * X.cg; T.off = X.tmpl_off; T.lay = X.lay;
        }
    }
    return OWW_OK;
}

// After a CNN launch (and its late chain) of a ragged step: carry the tails state of the n held streams listed at d_ids.
int carry_launch(oww_ctx* ctx, const int* d_ids, int n, cudaStream_t s) {
    if (n <= 0) return OWW_OK;
    ResetTails rt;
    int rc = next_step_tables(ctx, rt);
    if (rc) return rc;
    rt.tmpl = reinterpret_cast<const uint4*>(ctx->d_inc_tails[ctx->inc_cur ^ 1]);   // the buffer the launch read
    for (int i = 0, l = ctx->split_from; i < rt.n_late; ++l) {
        const oww_ctx::LateTensor& X = ctx->late_x[l];
        if (X.tmpl_off >= 0) rt.late[i++].tmpl = reinterpret_cast<const uint4*>(X.buf[(ctx->late_step - 1) % X.n_buf]);
    }
    OWW_CUDA(ctx, oww_launch_pdl(ctx->late_pdl, carry_kernel, dim3(n), dim3(256), 0, s, d_ids, n, rt));
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

// Staging of a ragged step's counts: [B counts | B stream ids by ascending count] in the next slot of the ring, copied on
// `s` -> its device copy; below[c] = number of streams with fewer than c chunks.
int stage_ragged(oww_ctx* ctx, const int32_t* h_chunks, cudaStream_t s, std::vector<int>& below, const int** d_staged) {
    const int B = ctx->n_streams, mc = ctx->cfg.max_chunks;
    if (ctx->rag_streams != B) {
        for (int j = 0; j < oww_ctx::kRagSlots; ++j) {
            if (ctx->rag_ev[j]) OWW_CUDA(ctx, cudaEventSynchronize(ctx->rag_ev[j]));
            cudaFreeHost(ctx->h_rag[j]); cudaFree(ctx->d_rag[j]); ctx->h_rag[j] = nullptr; ctx->d_rag[j] = nullptr;
        }
        ctx->rag_streams = 0;
        for (int j = 0; j < oww_ctx::kRagSlots; ++j) {
            OWW_CUDA(ctx, cudaMallocHost(&ctx->h_rag[j], (size_t)2 * B * sizeof(int32_t)));
            OWW_CUDA(ctx, cudaMalloc(&ctx->d_rag[j], (size_t)2 * B * sizeof(int32_t)));
            if (!ctx->rag_ev[j]) OWW_CUDA(ctx, cudaEventCreateWithFlags(&ctx->rag_ev[j], cudaEventDisableTiming));
        }
        ctx->rag_streams = B;
    }
    const int j = ctx->rag_next;
    ctx->rag_next = (j + 1) % oww_ctx::kRagSlots;
    OWW_CUDA(ctx, cudaEventSynchronize(ctx->rag_ev[j]));          // the copy of the call kRagSlots back has run
    int32_t* h = ctx->h_rag[j];
    below.assign(mc + 2, 0);
    for (int b = 0; b < B; ++b) below[h_chunks[b] + 1]++;
    for (int c = 1; c <= mc + 1; ++c) below[c] += below[c - 1];
    {
        std::vector<int> at(below.begin(), below.end() - 1);
        for (int b = 0; b < B; ++b) { h[b] = h_chunks[b]; h[B + at[h_chunks[b]]++] = b; }
    }
    OWW_CUDA(ctx, cudaMemcpyAsync(ctx->d_rag[j], h, (size_t)2 * B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    OWW_CUDA(ctx, cudaEventRecord(ctx->rag_ev[j], s));
    *d_staged = ctx->d_rag[j];
    return OWW_OK;
}

// Ragged step (oww_step_ragged): stream b steps cnt[b] = h_chunks[b] chunks, the first cnt[b]*1280 samples of its row;
// n = max cnt >= 1 and the counts are not all equal (the caller runs those as oww_step).  Streams that do not step in a
// launch are dead slots there: no state, ring or score write; carry_kernel moves their rotating tails.  Multi-chunk
// calls run right-aligned: CNN launch i steps the streams with cnt >= n - i, so its window offset 8*(n-1-i) is right
// relative to each stream's own mel count.  audio: append the streams' samples to their audio history first (the
// entry point's call; not the calls this one makes on split counts).
int step_ragged_core(oww_ctx* ctx, const int16_t* d_pcm, int64_t pcm_stride, const int32_t* h_chunks, int n, float* d_scores,
                     int out_stride, cudaStream_t s, bool audio) {
    const int B = ctx->n_streams, n_out = ctx->n_out_total, mc = ctx->cfg.max_chunks;
    int rc;
    const bool inc = ctx->cfg.cnn_mode == OWW_CNN_TC_INCREMENTAL;
    std::vector<int> below;
    const int* d_cnt = nullptr;
    if (inc && n > 1 && oww_fused_heads_supported(ctx)) {
        // oww_step(1) runs the heads inside the fused kernel (its own summation order): streams with one chunk take
        // that launch as a ragged step of their own, the others the general path
        std::vector<int32_t> one(B), more(B);
        bool any_one = false;
        for (int b = 0; b < B; ++b) {
            one[b] = h_chunks[b] == 1;
            more[b] = h_chunks[b] >= 2 ? h_chunks[b] : 0;
            any_one = any_one || h_chunks[b] == 1;
        }
        if (any_one) {
            if (audio && ctx->audio) {                     // the whole call's counts, for its one append
                if ((rc = stage_ragged(ctx, h_chunks, s, below, &d_cnt))) return rc;
                if ((rc = oww_audio_append(ctx, d_pcm, pcm_stride, n, d_cnt, s))) return rc;
            }
            if ((rc = step_ragged_core(ctx, d_pcm, pcm_stride, one.data(), 1, d_scores, out_stride, s, false))) return rc;
            return step_ragged_core(ctx, d_pcm, pcm_stride, more.data(), n, d_scores, out_stride, s, false);
        }
    }
    const size_t need = (size_t)mc * B * n_out;
    if (ctx->rag_scores_floats < need) {
        cudaFree(ctx->d_rag_scores); ctx->d_rag_scores = nullptr; ctx->rag_scores_floats = 0;
        OWW_CUDA(ctx, cudaMalloc(&ctx->d_rag_scores, need * sizeof(float)));
        ctx->rag_scores_floats = need;
    }
    if ((rc = stage_ragged(ctx, h_chunks, s, below, &d_cnt))) return rc;
    if (audio && (rc = oww_audio_append(ctx, d_pcm, pcm_stride, n, d_cnt, s))) return rc;
    const int* d_ord = d_cnt + B;
    const FeatSrc fs0{ctx->d_feat_ring, (int64_t)ctx->feat_rows * 96, ctx->d_feat_count, ctx->feat_rows - 1, 0};
    auto append = [&](int n_launch) {
        OWW_CUDA(ctx, oww_launch_pdl(ctx->late_pdl, feat_append_ragged_kernel, dim3((B + 7) / 8), dim3(256), 0, s,
                                     (const float*)ctx->d_emb_tmp, ctx->d_feat_ring, ctx->d_feat_count, B, n_launch, d_cnt,
                                     ctx->feat_rows - 1, (int64_t)ctx->feat_rows * 96));
        OWW_LAUNCH_CHECK(ctx);
        return OWW_OK;
    };
    // heads of every stream on its windows back = 0 .. n-1, then the max over each stream's own cnt windows
    auto heads = [&](int n_launch) {
        if (n_out == 0) return OWW_OK;
        for (int i = 0; i < n_launch; ++i) {
            FeatSrc fs = fs0; fs.back = i;
            int r = oww_heads_all(ctx, fs, B, ctx->d_rag_scores + (size_t)i * B * n_out, n_out, 0, s);
            if (r) return r;
        }
        const int64_t total = (int64_t)B * n_out;
        OWW_CUDA(ctx, oww_launch_pdl(ctx->late_pdl, ragged_max_kernel, dim3((unsigned)std::min<int64_t>(4096, (total + 255) / 256)),
                                     dim3(256), 0, s, (const float*)ctx->d_rag_scores, B, n_out, d_cnt, d_scores, out_stride));
        OWW_LAUNCH_CHECK(ctx);
        return OWW_OK;
    };

    if (inc && n == 1 && oww_fused_frontend_supported(ctx)) {
        // one chunk: the fused launch with the held streams (cnt 0 = ord[0 .. below[1])) as dead slots
        const bool heads_inside = oww_fused_heads_supported(ctx);
        if ((rc = oww_fused_step(ctx, d_pcm, pcm_stride, d_scores, out_stride, heads_inside, s, d_cnt, 1))) return rc;
        if (ctx->late_active) {
            if ((rc = oww_late_chain(ctx, ctx->d_emb_tmp, s))) return rc;
            if ((rc = append(1))) return rc;
        }
        if ((rc = carry_launch(ctx, d_ord, below[1], s))) return rc;
        if (heads_inside) {
            oww_feat16_invalidate(ctx);
            if ((rc = oww_head_banks_launch(ctx, fs0, B, d_scores, out_stride, 0, s, d_cnt))) return rc;
        } else {
            if ((rc = oww_feat16_advance(ctx, 1, s))) return rc;
            if ((rc = oww_feat16_resync(ctx, d_ord, below[1], s))) return rc;     // held: their window did not move
            if ((rc = heads(1))) return rc;
        }
        return oww_verifiers_apply(ctx, fs0, B, d_scores, out_stride, false, s, d_cnt);
    }

    // ---- general path: one mel launch per distinct count on its streams, the CNN launch by launch, masked append ----
    for (int c = 1; c <= n; ++c) {
        const int m = below[c + 1] - below[c];
        if (m == 0) continue;
        MelLaunch ml{d_pcm, pcm_stride, c * OWW_SAMPLES_PER_CHUNK, ctx->d_tail, ctx->d_seen, ctx->d_mel_ring,
                     (int64_t)ctx->mel_rows * 32, ctx->mel_rows - 1, ctx->d_mel_count, m, 1, c};
        ml.ids = d_ord + below[c];
        if ((rc = oww_mel_launch(ctx, ml, s))) return rc;
    }
    if (inc) {
        for (int i = 0; i < n; ++i) {
            if ((rc = oww_cnn_inc_step(ctx, 8 * (n - 1 - i), ctx->d_emb_tmp + (size_t)i * B * 96, s, d_cnt, n - i))) return rc;
            if ((rc = carry_launch(ctx, d_ord, below[n - i], s))) return rc;
        }
    } else {
        // every stream's n newest window positions; those before a stream's own chunks are computed and not appended
        WindowSrc ws{ctx->d_mel_ring, (int64_t)ctx->mel_rows * 32, ctx->d_mel_count, ctx->mel_rows - 1, B, n};
        if ((rc = oww_cnn_window(ctx, ws, B * n, ctx->d_emb_tmp, s, false))) return rc;
    }
    if ((rc = append(n))) return rc;
    if ((rc = oww_feat16_advance(ctx, n, s))) return rc;
    if ((rc = oww_feat16_resync(ctx, d_ord, below[n], s))) return rc;       // streams that appended fewer than n rows
    if ((rc = heads(n))) return rc;
    return oww_verifiers_apply(ctx, fs0, B, d_scores, out_stride, false, s, d_cnt);
}

// validation shared by the ragged entry points: counts in [0, max_chunks], stride for the largest; -> n = max count
int ragged_check(oww_ctx* ctx, const int32_t* h_chunks, int64_t pcm_stride, int* n_max, bool* all_equal) {
    const int B = ctx->n_streams;
    if (B <= 0) return oww_fail(ctx, OWW_EINVAL, "oww_set_streams has not been called");
    if (!ctx->mel_loaded || !ctx->emb_loaded) return oww_fail(ctx, OWW_EINVAL, "weights not loaded");
    int n = 0;
    bool eq = true;
    for (int b = 0; b < B; ++b) {
        if (h_chunks[b] < 0 || h_chunks[b] > ctx->cfg.max_chunks)
            return oww_fail(ctx, OWW_EINVAL, "chunks[%d]=%d outside [0,%d]", b, h_chunks[b], ctx->cfg.max_chunks);
        n = std::max(n, (int)h_chunks[b]);
        eq = eq && h_chunks[b] == h_chunks[0];
    }
    if (n > 0) {
        const int rc = stride_check(ctx, pcm_stride, n);
        if (rc) return rc;
    }
    *n_max = n; *all_equal = eq;
    return OWW_OK;
}

int host_submit(oww_ctx* ctx, const int16_t* h_pcm, int64_t pcm_stride, int n_chunks, const int32_t* h_chunks, int* ticket);

// shared by oww_reset (synchronous) and oww_reset_async: enqueue the state reset of the listed streams on `s`
int reset_enqueue(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const float* h_feature_init, int n_rows, cudaStream_t s) {
    if (ctx->n_streams <= 0) return oww_fail(ctx, OWW_EINVAL, "oww_set_streams has not been called");
    if (n_rows < 0 || n_rows > ctx->feat_rows) return oww_fail(ctx, OWW_EINVAL, "n_rows=%d outside [0,%d]", n_rows, ctx->feat_rows);
    if (!h_stream_ids) n = ctx->n_streams;
    if (n <= 0) return OWW_OK;
    if (n > ctx->n_streams) return oww_fail(ctx, OWW_EINVAL, "more stream ids (%d) than streams (%d)", n, ctx->n_streams);
    if (h_stream_ids) {
        for (int i = 0; i < n; ++i)
            if (h_stream_ids[i] < 0 || h_stream_ids[i] >= ctx->n_streams)
                return oww_fail(ctx, OWW_EINVAL, "stream id %d out of range", h_stream_ids[i]);
        // pageable source: staged by the driver before the call returns; stream-ordered on the device
        OWW_CUDA(ctx, cudaMemcpyAsync(ctx->d_reset_ids, h_stream_ids, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    }
    const bool have_init = h_feature_init && n_rows > 0;
    if (have_init)
        OWW_CUDA(ctx, cudaMemcpyAsync(ctx->d_reset_init, h_feature_init, (size_t)n_rows * 96 * sizeof(float), cudaMemcpyHostToDevice, s));
    // after the host-buffer calls submitted so far, before the later ones (their host counters already see the reset)
    int rc = oww_order_begin(ctx, s);
    if (rc) return rc;
    ResetTails rt;
    std::memset(&rt, 0, sizeof(rt));
    if (ctx->cfg.cnn_mode == OWW_CNN_TC_INCREMENTAL) {
        rc = next_step_tables(ctx, rt);
        if (rc) return rc;
        rt.tmpl = reinterpret_cast<const uint4*>(ctx->d_tails_template);
        for (int i = 0, l = ctx->split_from; i < rt.n_late; ++l)
            if (ctx->late_x[l].tmpl_off >= 0)
                rt.late[i++].tmpl = reinterpret_cast<const uint4*>(ctx->d_late_template) + ctx->late_x[l].tmpl_off;
    }
    reset_kernel<<<n, 256, 0, s>>>(h_stream_ids ? ctx->d_reset_ids : nullptr, n, ctx->n_streams, ctx->d_tail, ctx->d_seen,
                                   ctx->d_mel_count, ctx->d_feat_count, ctx->d_mel_ring, ctx->mel_rows, ctx->d_feat_ring,
                                   ctx->feat_rows, have_init ? ctx->d_reset_init : nullptr, n_rows, rt);
    OWW_LAUNCH_CHECK(ctx);
    rc = oww_detect_reset(ctx, h_stream_ids ? ctx->d_reset_ids : nullptr, n, s);        // the detector's history of those streams
    if (rc) return rc;
    if ((rc = oww_audio_reset(ctx, h_stream_ids ? ctx->d_reset_ids : nullptr, n, s))) return rc;     // ... and their audio
    oww_ingest_reset(ctx, h_stream_ids, n);               // ... and their staged samples (host counters only)
    if ((rc = oww_feat16_resync(ctx, h_stream_ids ? ctx->d_reset_ids : nullptr, n, s))) return rc;  // fp16 mirror (heads_grp.cu)
    return oww_order_end(ctx, s);
}

// Units of a stream record's two conv tails sections (0 outside mode 3).  tail_tab is filled by the reset that
// oww_set_streams ends with.
void record_units(const oww_ctx* ctx, int* u_tails, int* u_late) {
    *u_tails = *u_late = 0;
    if (ctx->cfg.cnn_mode != OWW_CNN_TC_INCREMENTAL) return;
    for (int k = 0; k < ctx->n_tail_tab; ++k)
        *u_tails = std::max(*u_tails, ctx->tail_tab[k].x + ctx->tail_tab[k].z * 2 * ctx->tail_tab[k].w);
    if (!ctx->late_active) return;
    for (int l = ctx->split_from; l < OWW_N_CONV; ++l) {
        const oww_ctx::LateTensor& X = ctx->late_x[l];
        if (X.tmpl_off >= 0) *u_late = std::max(*u_late, X.tmpl_off + 2 * X.cg * 2 * (X.W + 1));
    }
}

int64_t record_bytes(const oww_ctx* ctx) {
    int u_tails, u_late;
    record_units(ctx, &u_tails, &u_late);
    return ((int64_t)kRecTails + u_tails + u_late) * 16;
}

// what a record's state is only valid under: its format, the CNN mode and split point, the mel constants and the
// embedding weights (the conv tails and the rings are their products)
uint64_t record_key(const oww_ctx* ctx) {
    const int32_t cfg[3] = {(int32_t)kRecVersion, ctx->cfg.cnn_mode,
                            ctx->cfg.cnn_mode == OWW_CNN_TC_INCREMENTAL ? ctx->split_from : 0};
    uint64_t h = oww_fnv1a(cfg, sizeof(cfg));
    h = oww_fnv1a(&ctx->mel_key, sizeof(uint64_t), h);
    return oww_fnv1a(&ctx->emb_key, sizeof(uint64_t), h);
}

// shared by oww_export_streams / oww_import_streams: checks on the host, then one launch on `s`, ordered with own_stream
int state_enqueue(oww_ctx* ctx, const int32_t* h_ids, int n, void* d_records, bool import, cudaStream_t s) {
    const int B = ctx->n_streams;
    if (B <= 0) return oww_fail(ctx, OWW_EINVAL, "oww_set_streams has not been called");
    if (n < 0 || n > B) return oww_fail(ctx, OWW_EINVAL, "n=%d outside [0,%d]", n, B);
    if (n == 0) return OWW_OK;
    if (!h_ids || !d_records) return oww_fail(ctx, OWW_EINVAL, "null argument");
    std::vector<uint8_t> hit(import ? B : 0, 0);
    for (int i = 0; i < n; ++i) {
        if (h_ids[i] < 0 || h_ids[i] >= B) return oww_fail(ctx, OWW_EINVAL, "stream id %d out of range", h_ids[i]);
        if (import && hit[h_ids[i]]++) return oww_fail(ctx, OWW_EINVAL, "stream id %d imported twice", h_ids[i]);
    }
    if (!ctx->d_state_ids) OWW_CUDA(ctx, cudaMalloc(&ctx->d_state_ids, (size_t)B * sizeof(int)));
    if (!ctx->d_state_rejected) {
        OWW_CUDA(ctx, cudaMalloc(&ctx->d_state_rejected, sizeof(int)));
        OWW_CUDA(ctx, cudaMemset(ctx->d_state_rejected, 0, sizeof(int)));
    }
    for (auto& e : ctx->state_ev)
        if (!e) OWW_CUDA(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    StreamState a{ctx->d_tail, ctx->d_seen, ctx->d_mel_count, ctx->d_feat_count, ctx->d_mel_ring, ctx->mel_rows,
                  ctx->d_feat_ring, ctx->feat_rows, record_bytes(ctx) / 16, 0, (uint32_t)record_bytes(ctx), record_key(ctx),
                  ctx->d_state_rejected};
    int u_late = 0;
    record_units(ctx, &a.u_tails, &u_late);
    ResetTails rt;
    std::memset(&rt, 0, sizeof(rt));
    if (ctx->cfg.cnn_mode == OWW_CNN_TC_INCREMENTAL) {
        int rc = next_step_tables(ctx, rt);            // where the state between the last step and the next one lives
        if (rc) return rc;
    }
    // the host-buffer steps run on the handle's own stream: after the steps submitted there so far, before later ones
    const bool other = s != ctx->own_stream;
    if (other) {
        OWW_CUDA(ctx, cudaEventRecord(ctx->state_ev[0], ctx->own_stream));
        OWW_CUDA(ctx, cudaStreamWaitEvent(s, ctx->state_ev[0], 0));
    }
    // pageable source: staged by the driver before the call returns; stream-ordered on the device
    OWW_CUDA(ctx, cudaMemcpyAsync(ctx->d_state_ids, h_ids, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    if (import) {
        stream_import_kernel<<<n, 256, 0, s>>>(ctx->d_state_ids, a, rt, static_cast<const uint4*>(d_records));
        OWW_LAUNCH_CHECK(ctx);
        int rc = oww_feat16_resync(ctx, ctx->d_state_ids, n, s);          // fp16 mirror of the rings, as after a reset
        if (rc) return rc;
    } else {
        stream_export_kernel<<<n, 256, 0, s>>>(ctx->d_state_ids, a, rt, static_cast<uint4*>(d_records));
        OWW_LAUNCH_CHECK(ctx);
    }
    if (other) {
        OWW_CUDA(ctx, cudaEventRecord(ctx->state_ev[1], s));
        OWW_CUDA(ctx, cudaStreamWaitEvent(ctx->own_stream, ctx->state_ev[1], 0));
    }
    return OWW_OK;
}

}  // namespace

extern "C" {

const char* oww_version(void) { return "owwb200 0.1 (sm_90a)"; }

const char* oww_last_error(const oww_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int oww_create(const oww_config* cfg, oww_ctx** out) {
    if (!cfg || !out) return oww_fail(nullptr, OWW_EINVAL, "null argument");
    *out = nullptr;
    if (cfg->max_chunks > OWW_MAX_CHUNKS)      // a larger mel ring breaks the count rebase (oww_internal.h)
        return oww_fail(nullptr, OWW_EINVAL, "max_chunks %d above %d", cfg->max_chunks, OWW_MAX_CHUNKS);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return oww_fail(nullptr, OWW_ECUDA, "no CUDA device: %s", e == cudaSuccess ? "count is 0" : cudaGetErrorString(e));
    if (cfg->device < 0 || cfg->device >= ndev) return oww_fail(nullptr, OWW_EINVAL, "device %d out of range", cfg->device);
    if (cfg->cnn_mode != OWW_CNN_FP32_WINDOW && cfg->cnn_mode != OWW_CNN_TC_WINDOW && cfg->cnn_mode != OWW_CNN_TC_INCREMENTAL)
        return oww_fail(nullptr, OWW_EUNSUPPORTED, "cnn_mode %d not built in this version", cfg->cnn_mode);
    oww_ctx* ctx = new (std::nothrow) oww_ctx();
    if (!ctx) return oww_fail(nullptr, OWW_ENOMEM, "out of host memory");
    ctx->cfg = *cfg;
    if (ctx->cfg.max_chunks < 1) ctx->cfg.max_chunks = 1;
    ctx->device = cfg->device;
    ctx->fuse_step = (cfg->reserved[0] & 1) == 0;
    ctx->window_batch = cfg->window_batch > 0 ? cfg->window_batch : (cfg->cnn_mode == OWW_CNN_FP32_WINDOW ? 512 : 1024);
    if ((e = cudaSetDevice(ctx->device)) != cudaSuccess) {
        oww_fail(nullptr, OWW_ECUDA, "cudaSetDevice: %s", cudaGetErrorString(e));
        delete ctx; return OWW_ECUDA;
    }
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, ctx->device);
    ctx->sm_count = prop.multiProcessorCount;
    if (prop.major != 9 || prop.minor != 0) {
        oww_fail(nullptr, OWW_EUNSUPPORTED, "device is sm_%d%d; this library is built for sm_90a only", prop.major, prop.minor);
        delete ctx; return OWW_EUNSUPPORTED;
    }
    ctx->tc_heads = (cfg->reserved[0] & 2) == 0;
    ctx->split_from = (cfg->reserved[1] >= 2 && cfg->reserved[1] <= OWW_N_CONV) ? cfg->reserved[1] : 11;
    ctx->tc_heads_terms = (cfg->reserved[0] & 4) ? 1 : 3;
    ctx->grp_heads = (cfg->reserved[0] & 8) == 0;
    ctx->late_pdl = (cfg->reserved[0] & 32) == 0;
    cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking);
    cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking);
    for (auto& ev : ctx->order_ev) cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    fill_layer_table(ctx);
    *out = ctx;
    return OWW_OK;
}

void oww_destroy(oww_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    free_streams(ctx);
    oww_heads_grp_free(ctx);
    oww_head_banks_free(ctx);
    oww_verifier_fit_free(ctx);
    oww_detect_free(ctx);
    oww_audio_free(ctx);
    oww_ingest_free(ctx);
    oww_mix_free(ctx);
    cudaFree(ctx->d_window); cudaFree(ctx->d_twiddle); cudaFree(ctx->d_mel_start); cudaFree(ctx->d_mel_len);
    cudaFree(ctx->d_mel_w); cudaFree(ctx->d_emb_blob); cudaFree(ctx->d_tc_w); cudaFree(ctx->d_tc_sb);
    cudaFree(ctx->d_tc_w3); cudaFree(ctx->d_tc_sb3);
    cudaFree(ctx->d_tc_act[0]); cudaFree(ctx->d_tc_act[1]); cudaFree(ctx->d_inc_w); cudaFree(ctx->d_head_devs);
    for (auto& h : ctx->heads) { cudaFree(h.d_blob); cudaFree(h.d_w1_tc); }
    cudaFree(ctx->d_gates); cudaFree(ctx->d_tails_template); cudaFree(ctx->d_peer_err); cudaFree(ctx->d_state_rejected);
    for (auto e : ctx->state_ev) if (e) cudaEventDestroy(e);
    for (auto& b : ctx->banks) { cudaFree(b.d_mean); cudaFree(b.d_weight); cudaFree(b.d_bias); }
    for (auto e : ctx->ver_ev) if (e) cudaEventDestroy(e);
    for (auto e : ctx->rag_ev) if (e) cudaEventDestroy(e);
    for (auto& S : ctx->slot) {
        cudaFreeHost(S.h_pcm); cudaFreeHost(S.h_scores); cudaFree(S.d_pcm); cudaFree(S.d_scores);
        if (S.done) cudaEventDestroy(S.done);
        if (S.h2d_done) cudaEventDestroy(S.h2d_done);
    }
    for (auto& S : ctx->det_slot) {
        cudaFreeHost(S.h_pkt); cudaFree(S.d_pkt); cudaFree(S.d_scores); cudaFree(S.d_final); cudaFree(S.d_out);
        cudaFreeHost(S.h_out);
        if (S.done) cudaEventDestroy(S.done);
        if (S.h2d_done) cudaEventDestroy(S.h2d_done);
    }
    for (auto e : ctx->order_ev) if (e) cudaEventDestroy(e);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    for (auto e : ctx->ev) cudaEventDestroy(e);
    cudaStreamDestroy(ctx->own_stream);
    delete ctx;
}

int oww_load_embedding(oww_ctx* ctx, const float* h_blob, size_t n_floats) {
    if (!ctx || !h_blob) return oww_fail(ctx, OWW_EINVAL, "null argument");
    size_t need = 0;
    for (int li = 0; li < OWW_N_CONV; ++li) {
        const ConvLayer& L = ctx->conv[li];
        need += (size_t)L.kh * L.kw * L.cin * L.cout + 2 * (size_t)L.cout;
    }
    if (n_floats != need)
        return oww_fail(ctx, OWW_EINVAL, "embedding blob has %zu floats, the reference CNN needs %zu", n_floats, need);
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->d_emb_blob) OWW_CUDA(ctx, cudaMalloc(&ctx->d_emb_blob, need * sizeof(float)));
    OWW_CUDA(ctx, cudaMemcpy(ctx->d_emb_blob, h_blob, need * sizeof(float), cudaMemcpyHostToDevice));
    size_t off = 0;
    for (int li = 0; li < OWW_N_CONV; ++li) {
        ConvLayer& L = ctx->conv[li];
        L.d_w = ctx->d_emb_blob + off; off += (size_t)L.kh * L.kw * L.cin * L.cout;
        L.d_scale = ctx->d_emb_blob + off; off += L.cout;
        L.d_bias = ctx->d_emb_blob + off; off += L.cout;
    }
    ctx->emb_loaded = true;
    ctx->emb_key = oww_fnv1a(h_blob, need * sizeof(float));
    ctx->tails_template_valid = false;                 // depends on the weights: rebuilt at the next reset
    int rc = oww_tc_pack_weights(ctx, h_blob);
    if (rc) return rc;
    return oww_inc_setup(ctx, h_blob);
}

}  // extern "C"

int oww_check_head_desc(oww_ctx* ctx, const oww_head_desc* desc) {
    if (desc->n_layers < 1 || desc->n_layers > OWW_MAX_HEAD_LAYERS)
        return oww_fail(ctx, OWW_EUNSUPPORTED, "head has %d Linear layers (1..%d supported)", desc->n_layers, OWW_MAX_HEAD_LAYERS);
    if (desc->n_in < 1 || desc->dims[0] != desc->n_in * OWW_EMBEDDING_DIM)
        return oww_fail(ctx, OWW_EINVAL, "dims[0]=%d must equal n_in*96=%d", desc->dims[0], desc->n_in * OWW_EMBEDDING_DIM);
    if (desc->final_act < 0 || desc->final_act > 4) return oww_fail(ctx, OWW_EINVAL, "bad final_act");
    return OWW_OK;
}

int oww_stage_head(oww_ctx* ctx, const oww_head_desc* desc, const float* h_blob, size_t n_floats, Head& h,
                   std::vector<float>& staged) {
    h.desc = *desc;
    // Device layout: the caller's tensors in order, each starting on a 16-byte boundary (the fused step kernel streams
    // weight rows with bulk copies, which need 16-byte aligned sources).  `src` walks the packed host blob.
    size_t off = 0, src = 0;
    auto place = [&](size_t n) {
        off = (off + 3) & ~(size_t)3;
        const size_t at = off;
        if (src + n <= n_floats) {
            staged.resize(at + n + 4, 0.f);
            std::memcpy(staged.data() + at, h_blob + src, n * sizeof(float));
        }
        src += n; off += n;
        return at;
    };
    for (int l = 0; l < desc->n_layers; ++l) {
        const int din = desc->dims[l], dout = desc->dims[l + 1];
        if (dout < 1 || dout > 256) return oww_fail(ctx, OWW_EUNSUPPORTED, "layer width %d outside 1..256", dout);
        h.w_off.push_back(place((size_t)din * dout));
        h.b_off.push_back(place(dout));
        if (desc->layernorm && l < desc->n_layers - 1) {
            h.g_off.push_back(place(dout));
            h.h_off.push_back(place(dout));
        } else { h.g_off.push_back(0); h.h_off.push_back(0); }
    }
    if (src != n_floats) return oww_fail(ctx, OWW_EINVAL, "head blob has %zu floats, descriptor needs %zu", n_floats, src);
    return OWW_OK;
}

extern "C" {

int oww_add_head(oww_ctx* ctx, const oww_head_desc* desc, const float* h_blob, size_t n_floats, int* head_id) {
    if (!ctx || !desc || !h_blob) return oww_fail(ctx, OWW_EINVAL, "null argument");
    int rc = oww_check_head_desc(ctx, desc);
    if (rc) return rc;
    if (ctx->heads.size() >= 16) return oww_fail(ctx, OWW_EUNSUPPORTED, "at most 16 heads per handle");
    Head h;
    std::vector<float> staged;
    if ((rc = oww_stage_head(ctx, desc, h_blob, n_floats, h, staged))) return rc;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaMalloc(&h.d_blob, staged.size() * sizeof(float)));
    OWW_CUDA(ctx, cudaMemcpy(h.d_blob, staged.data(), staged.size() * sizeof(float), cudaMemcpyHostToDevice));
    // tensor-core packing of the first layer (heads_tc.cu); heads it does not cover keep tc_ok == false
    if ((rc = oww_heads_tc_pack(ctx, h, staged.data()))) { cudaFree(h.d_blob); return rc; }
    h.n_out = desc->dims[desc->n_layers];
    h.col0 = ctx->n_out_total;
    ctx->n_out_total += h.n_out;
    ctx->max_n_in = std::max(ctx->max_n_in, desc->n_in);
    ctx->heads.push_back(h);
    if (head_id) *head_id = (int)ctx->heads.size() - 1;
    return oww_heads_sync_devs(ctx);
}

int oww_add_gate(oww_ctx* ctx, int main_head, int verifier_head, float threshold) {
    if (!ctx) return OWW_EINVAL;
    const int nh = (int)ctx->heads.size();
    if (main_head < 0 || main_head >= nh || verifier_head < 0 || verifier_head >= nh || main_head == verifier_head)
        return oww_fail(ctx, OWW_EINVAL, "bad head ids %d / %d", main_head, verifier_head);
    if (ctx->heads[main_head].n_out != 1 || ctx->heads[verifier_head].n_out != 1)
        return oww_fail(ctx, OWW_EUNSUPPORTED, "a verifier gate joins two single-output heads");
    if (ctx->gates.size() >= 16) return oww_fail(ctx, OWW_EUNSUPPORTED, "at most 16 gates per handle");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    ctx->gates.push_back(Gate{ctx->heads[main_head].col0, ctx->heads[verifier_head].col0, threshold});
    cudaFree(ctx->d_gates); ctx->d_gates = nullptr;
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_gates, ctx->gates.size() * sizeof(Gate)));
    OWW_CUDA(ctx, cudaMemcpy(ctx->d_gates, ctx->gates.data(), ctx->gates.size() * sizeof(Gate), cudaMemcpyHostToDevice));
    return OWW_OK;
}

int oww_n_heads(const oww_ctx* ctx) { return ctx ? (int)ctx->heads.size() : 0; }
int oww_n_outputs(const oww_ctx* ctx) { return ctx ? ctx->n_out_total : 0; }
int oww_n_streams(const oww_ctx* ctx) { return ctx ? ctx->n_streams : 0; }
uint64_t oww_launch_count(const oww_ctx* ctx) { return ctx ? ctx->launches : 0; }

int oww_melspectrogram(oww_ctx* ctx, const int16_t* d_pcm, int n_clips, int n_samples, float* d_mel, int affine, void* stream) {
    if (!ctx || !d_pcm || !d_mel) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (n_samples < OWW_FFT_N) return oww_fail(ctx, OWW_EINVAL, "need at least 512 samples, got %d", n_samples);
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    const int T = (n_samples - OWW_FFT_N) / OWW_HOP + 1;
    MelLaunch m{d_pcm, (int64_t)n_samples, n_samples, nullptr, nullptr, d_mel, (int64_t)T * 32, -1, nullptr, n_clips,
                affine, 0};
    return oww_mel_launch(ctx, m, (cudaStream_t)stream);
}

int oww_embed_windows(oww_ctx* ctx, const float* d_windows, int n, float* d_emb, void* stream) {
    if (!ctx || !d_windows || !d_emb) return oww_fail(ctx, OWW_EINVAL, "null argument");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = ensure_act(ctx, (size_t)std::min(n, ctx->window_batch) * 74 * 32 * 24);
    if (rc) return rc;
    WindowSrc src{d_windows, (int64_t)OWW_WINDOW_ROWS * 32, nullptr, -1, 0, 0};
    return oww_cnn_window(ctx, src, n, d_emb, (cudaStream_t)stream);
}

int oww_head_predict(oww_ctx* ctx, int head_id, const float* d_feats, int n, float* d_out, void* stream) {
    if (!ctx || !d_feats || !d_out) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (head_id < 0 || head_id >= (int)ctx->heads.size()) return oww_fail(ctx, OWW_EINVAL, "bad head_id %d", head_id);
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    const Head& h = ctx->heads[head_id];
    FeatSrc fs{d_feats, (int64_t)h.desc.n_in * 96, nullptr, -1, 0};
    if (oww_heads_tc_supported(ctx, head_id))
        return oww_heads_tc_launch(ctx, head_id, fs, n, d_out, h.n_out, 0, 0, (cudaStream_t)stream);
    return oww_heads_launch(ctx, head_id, fs, n, d_out, h.n_out, 0, 0, (cudaStream_t)stream);
}

int oww_set_streams(oww_ctx* ctx, int n_streams) {
    if (!ctx || n_streams < 1) return oww_fail(ctx, OWW_EINVAL, "n_streams must be >= 1");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaDeviceSynchronize());
    free_streams(ctx);
    const int B = n_streams, mc = ctx->cfg.max_chunks;
    ctx->mel_rows = next_pow2(OWW_WINDOW_ROWS + 8 * mc);
    ctx->feat_rows = next_pow2(120 + mc);             // the reference keeps <=120 rows (utils.py:170)
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_tail, (size_t)B * OWW_TAIL * sizeof(int16_t)));
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_seen, (size_t)B * sizeof(int)));
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_mel_count, (size_t)B * sizeof(int)));
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_feat_count, (size_t)B * sizeof(int)));
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_mel_ring, (size_t)B * ctx->mel_rows * 32 * sizeof(float)));
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_feat_ring, (size_t)B * ctx->feat_rows * 96 * sizeof(float)));
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_reset_ids, (size_t)B * sizeof(int)));
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_reset_init, (size_t)ctx->feat_rows * 96 * sizeof(float)));
    ctx->n_streams = B;
    int rc = ensure_act(ctx, (size_t)std::min(B * mc, ctx->window_batch) * 74 * 32 * 24);
    if (rc) return rc;
    if ((rc = ensure_emb_tmp(ctx, (size_t)B * mc * 96))) return rc;
    if (ctx->cfg.cnn_mode == OWW_CNN_TC_INCREMENTAL && (rc = oww_late_alloc(ctx))) return rc;
    if (ctx->cfg.cnn_mode == OWW_CNN_TC_INCREMENTAL && (rc = oww_inc_alloc_streams(ctx))) return rc;
    if ((rc = oww_verifiers_alloc_streams(ctx))) return rc;         // every stream starts without a verifier
    if ((rc = oww_head_banks_alloc_streams(ctx))) return rc;        // ... and without a bank head
    if ((rc = oww_detect_alloc_streams(ctx))) return rc;            // ... and with an empty detector history
    if ((rc = oww_audio_alloc_streams(ctx))) return rc;             // ... and an empty audio history
    if ((rc = oww_ingest_alloc_streams(ctx))) return rc;            // ... and at 16 kHz with nothing staged
    return oww_reset(ctx, nullptr, B, nullptr, OWW_INIT_FEATURE_ROWS);
}

int oww_reset(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const float* h_feature_init, int n_rows) {
    if (!ctx) return OWW_EINVAL;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaDeviceSynchronize());              // steps may be in flight on any stream
    int rc = reset_enqueue(ctx, h_stream_ids, n, h_feature_init, n_rows, nullptr);
    if (rc) return rc;
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return oww_fail(ctx, OWW_ECUDA, "reset failed: %s", cudaGetErrorString(e));
    return OWW_OK;
}

int oww_reset_async(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const float* h_feature_init, int n_rows, void* stream) {
    if (!ctx) return OWW_EINVAL;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    return reset_enqueue(ctx, h_stream_ids, n, h_feature_init, n_rows, (cudaStream_t)stream);
}

int oww_stream_state_info(const oww_ctx* ctx, size_t* record_bytes_out, uint64_t* config_key) {
    if (!ctx) return OWW_EINVAL;
    if (ctx->n_streams <= 0) return oww_fail(const_cast<oww_ctx*>(ctx), OWW_EINVAL, "oww_set_streams has not been called");
    if (record_bytes_out) *record_bytes_out = (size_t)record_bytes(ctx);
    if (config_key) *config_key = record_key(ctx);
    return OWW_OK;
}

int oww_export_streams(oww_ctx* ctx, const int32_t* h_stream_ids, int n, void* d_records, void* stream) {
    if (!ctx) return OWW_EINVAL;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    return state_enqueue(ctx, h_stream_ids, n, d_records, false, (cudaStream_t)stream);
}

int oww_import_streams(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const void* d_records, void* stream) {
    if (!ctx) return OWW_EINVAL;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    return state_enqueue(ctx, h_stream_ids, n, const_cast<void*>(d_records), true, (cudaStream_t)stream);
}

int oww_stream_state_status(oww_ctx* ctx, int* n_rejected) {
    if (!ctx || !n_rejected) return oww_fail(ctx, OWW_EINVAL, "null argument");
    *n_rejected = 0;
    if (!ctx->d_state_rejected) return OWW_OK;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaDeviceSynchronize());              // imports may be in flight on any stream
    OWW_CUDA(ctx, cudaMemcpy(n_rejected, ctx->d_state_rejected, sizeof(int), cudaMemcpyDeviceToHost));
    if (*n_rejected) OWW_CUDA(ctx, cudaMemset(ctx->d_state_rejected, 0, sizeof(int)));
    return OWW_OK;
}

int oww_step(oww_ctx* ctx, const int16_t* d_pcm, int64_t pcm_stride, int n_chunks, float* d_scores, void* stream) {
    if (!ctx || !d_pcm || !d_scores) return oww_fail(ctx, OWW_EINVAL, "null argument");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = step_core_check(ctx, pcm_stride, n_chunks);
    if (rc) return rc;
    if ((rc = oww_audio_append(ctx, d_pcm, pcm_stride, n_chunks, nullptr, (cudaStream_t)stream))) return rc;
    return step_core(ctx, d_pcm, pcm_stride, n_chunks, d_scores, ctx->n_out_total, (cudaStream_t)stream);
}

int oww_step_host_submit(oww_ctx* ctx, const int16_t* h_pcm, int64_t pcm_stride, int n_chunks, int* ticket) {
    if (!ctx || !h_pcm || !ticket) return oww_fail(ctx, OWW_EINVAL, "null argument");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    const int B = ctx->n_streams;
    if (B <= 0) return oww_fail(ctx, OWW_EINVAL, "oww_set_streams has not been called");
    if (n_chunks < 1 || n_chunks > ctx->cfg.max_chunks)
        return oww_fail(ctx, OWW_EINVAL, "n_chunks=%d outside [1,%d]", n_chunks, ctx->cfg.max_chunks);
    const int rc = stride_check(ctx, pcm_stride, n_chunks);
    if (rc) return rc;
    return host_submit(ctx, h_pcm, pcm_stride, n_chunks, nullptr, ticket);
}

int oww_step_ragged(oww_ctx* ctx, const int16_t* d_pcm, int64_t pcm_stride, const int32_t* h_chunks, float* d_scores,
                    void* stream) {
    if (!ctx || !h_chunks || !d_scores) return oww_fail(ctx, OWW_EINVAL, "null argument");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    int n = 0; bool eq = false;
    int rc = ragged_check(ctx, h_chunks, pcm_stride, &n, &eq);
    if (rc) return rc;
    if (n == 0) return OWW_OK;
    if (!d_pcm) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (eq) {
        if ((rc = oww_audio_append(ctx, d_pcm, pcm_stride, n, nullptr, (cudaStream_t)stream))) return rc;
        return step_core(ctx, d_pcm, pcm_stride, n, d_scores, ctx->n_out_total, (cudaStream_t)stream);
    }
    return step_ragged_core(ctx, d_pcm, pcm_stride, h_chunks, n, d_scores, ctx->n_out_total, (cudaStream_t)stream, true);
}

int oww_step_host_ragged_submit(oww_ctx* ctx, const int16_t* h_pcm, int64_t pcm_stride, const int32_t* h_chunks, int* ticket) {
    if (!ctx || !h_chunks || !ticket) return oww_fail(ctx, OWW_EINVAL, "null argument");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    int n = 0; bool eq = false;
    int rc = ragged_check(ctx, h_chunks, pcm_stride, &n, &eq);
    if (rc) return rc;
    if (n > 0 && !h_pcm) return oww_fail(ctx, OWW_EINVAL, "null argument");
    return host_submit(ctx, h_pcm, pcm_stride, n, h_chunks, ticket);
}

int oww_step_host_ragged(oww_ctx* ctx, const int16_t* h_pcm, int64_t pcm_stride, const int32_t* h_chunks, float* h_scores) {
    if (!ctx || !h_scores) return oww_fail(ctx, OWW_EINVAL, "null argument");
    for (int i = 0; i < 2; ++i)
        if (ctx->slot[i].busy) return oww_fail(ctx, OWW_EINVAL, "a submitted step is still in flight: collect it first");
    int ticket = -1;
    int rc = oww_step_host_ragged_submit(ctx, h_pcm, pcm_stride, h_chunks, &ticket);
    if (rc) return rc;
    return oww_step_host_collect(ctx, ticket, h_scores);
}

}  // extern "C"

namespace {

// Host-buffer step on the handle's own stream.  h_chunks == nullptr: every stream steps n_chunks; else the ragged counts
// (validated, n_chunks = their max, which may be 0: nothing is launched and the ticket completes at once).
int host_submit(oww_ctx* ctx, const int16_t* h_pcm, int64_t pcm_stride, int n_chunks, const int32_t* h_chunks, int* ticket) {
    const int B = ctx->n_streams;
    const int si = ctx->next_slot;
    oww_ctx::HostSlot& S = ctx->slot[si];
    if (S.busy) return oww_fail(ctx, OWW_EINVAL, "both host slots are in flight: collect a ticket first");
    const size_t row = (size_t)n_chunks * OWW_SAMPLES_PER_CHUNK;
    const size_t pcm_bytes = (size_t)B * row * sizeof(int16_t);
    const size_t sc_bytes = (size_t)B * std::max(ctx->n_out_total, 1) * sizeof(float);
    if (!S.done) { OWW_CUDA(ctx, cudaEventCreateWithFlags(&S.done, cudaEventDisableTiming)); OWW_CUDA(ctx, cudaEventCreateWithFlags(&S.h2d_done, cudaEventDisableTiming)); }
    if (S.pcm_bytes < pcm_bytes) {
        cudaFreeHost(S.h_pcm); cudaFree(S.d_pcm); S.h_pcm = nullptr; S.d_pcm = nullptr; S.pcm_bytes = 0;
        OWW_CUDA(ctx, cudaMallocHost(&S.h_pcm, pcm_bytes));
        OWW_CUDA(ctx, cudaMalloc(&S.d_pcm, pcm_bytes));
        S.pcm_bytes = pcm_bytes;
    }
    if (S.sc_bytes < sc_bytes) {
        cudaFreeHost(S.h_scores); cudaFree(S.d_scores); S.h_scores = nullptr; S.d_scores = nullptr; S.sc_bytes = 0;
        OWW_CUDA(ctx, cudaMallocHost(&S.h_scores, sc_bytes));
        OWW_CUDA(ctx, cudaMalloc(&S.d_scores, sc_bytes));
        S.sc_bytes = sc_bytes;
    }
    // Source already page-locked (cudaMallocHost / cudaHostRegister / torch pin_memory) and dense: DMA straight from
    // the caller's buffer (it must stay untouched until the ticket is collected).  Otherwise stage through pinned memory.
    const int16_t* src = S.h_pcm;
    cudaPointerAttributes attr;
    const bool pinned = pcm_stride == (int64_t)row && cudaPointerGetAttributes(&attr, h_pcm) == cudaSuccess &&
                        attr.type == cudaMemoryTypeHost;
    cudaGetLastError();                                     // unregistered host memory reports an error on older drivers
    cudaStream_t s = ctx->own_stream;
    // every row written by the step: a lockstep call, or ragged counts all equal to n_chunks >= 1 (all 0: no row)
    bool all_step = h_chunks == nullptr;
    if (h_chunks && n_chunks > 0) {
        all_step = true;
        for (int b = 0; b < B && all_step; ++b) all_step = h_chunks[b] == n_chunks;
    }
    if (all_step) ctx->slot_chunks[si].clear();
    else ctx->slot_chunks[si].assign(h_chunks, h_chunks + B);
    if (n_chunks > 0) {
        if (pinned) {
            src = h_pcm;
        } else if (pcm_stride == (int64_t)row) {
            std::memcpy(S.h_pcm, h_pcm, pcm_bytes);
        } else {
            for (int b = 0; b < B; ++b)
                std::memcpy(S.h_pcm + (size_t)b * row, h_pcm + (size_t)b * pcm_stride, row * sizeof(int16_t));
        }
        OWW_CUDA(ctx, cudaMemcpyAsync(S.d_pcm, src, pcm_bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
        OWW_CUDA(ctx, cudaEventRecord(S.h2d_done, ctx->copy_stream));
        OWW_CUDA(ctx, cudaStreamWaitEvent(s, S.h2d_done, 0));
        int rc = all_step ? step_core_check(ctx, (int64_t)row, n_chunks) : OWW_OK;
        if (!rc && all_step) rc = oww_audio_append(ctx, S.d_pcm, (int64_t)row, n_chunks, nullptr, s);
        if (rc) return rc;
        rc = all_step ? step_core(ctx, S.d_pcm, (int64_t)row, n_chunks, S.d_scores, ctx->n_out_total, s)
                      : step_ragged_core(ctx, S.d_pcm, (int64_t)row, h_chunks, n_chunks, S.d_scores, ctx->n_out_total, s, true);
        if (rc) return rc;
        if (ctx->n_out_total > 0)
            OWW_CUDA(ctx, cudaMemcpyAsync(S.h_scores, S.d_scores, (size_t)B * ctx->n_out_total * sizeof(float),
                                          cudaMemcpyDeviceToHost, s));
    }
    OWW_CUDA(ctx, cudaEventRecord(S.done, s));
    S.busy = true;
    ctx->next_slot = si ^ 1;
    *ticket = si;
    return OWW_OK;
}

}  // namespace

extern "C" {

int oww_step_host_collect(oww_ctx* ctx, int ticket, float* h_scores) {
    if (!ctx || !h_scores) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (ticket < 0 || ticket > 1 || !ctx->slot[ticket].busy) return oww_fail(ctx, OWW_EINVAL, "ticket %d is not in flight", ticket);
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    oww_ctx::HostSlot& S = ctx->slot[ticket];
    OWW_CUDA(ctx, cudaEventSynchronize(S.done));
    const int n_out = ctx->n_out_total;
    const std::vector<int32_t>& cnt = ctx->slot_chunks[ticket];
    if (n_out > 0 && cnt.empty()) {
        std::memcpy(h_scores, S.h_scores, (size_t)ctx->n_streams * n_out * sizeof(float));
    } else if (n_out > 0) {
        // ragged step: the rows of held streams stay as the caller had them (all held: none is copied)
        for (int b = 0; b < ctx->n_streams; ++b)
            if (cnt[b] > 0) std::memcpy(h_scores + (size_t)b * n_out, S.h_scores + (size_t)b * n_out, n_out * sizeof(float));
    }
    S.busy = false;
    return OWW_OK;
}

int oww_step_host(oww_ctx* ctx, const int16_t* h_pcm, int64_t pcm_stride, int n_chunks, float* h_scores) {
    if (!ctx || !h_pcm || !h_scores) return oww_fail(ctx, OWW_EINVAL, "null argument");
    for (int i = 0; i < 2; ++i)
        if (ctx->slot[i].busy) return oww_fail(ctx, OWW_EINVAL, "a submitted step is still in flight: collect it first");
    int ticket = -1;
    int rc = oww_step_host_submit(ctx, h_pcm, pcm_stride, n_chunks, &ticket);
    if (rc) return rc;
    return oww_step_host_collect(ctx, ticket, h_scores);
}

}  // extern "C"

namespace {

// a slot's buffers for a call of B streams, `samples` packet samples, max_events events of `capture` samples, L labels:
// each grows (and only grows) when a call needs more than any before it
int detect_slot_grow(oww_ctx* ctx, oww_ctx::DetectSlot& S, int B, size_t samples, int max_events, int capture, int L) {
    const size_t scores = (size_t)B * std::max(ctx->n_out_total, 1), fin = (size_t)B * L;
    const DetectLayout lay = oww_detect_layout(max_events, capture, B, L);
    if (!S.done) {
        OWW_CUDA(ctx, cudaEventCreateWithFlags(&S.done, cudaEventDisableTiming));
        OWW_CUDA(ctx, cudaEventCreateWithFlags(&S.h2d_done, cudaEventDisableTiming));
    }
    if (S.pkt_samples < samples) {
        cudaFreeHost(S.h_pkt); cudaFree(S.d_pkt); S.h_pkt = nullptr; S.d_pkt = nullptr; S.pkt_samples = 0;
        OWW_CUDA(ctx, cudaMallocHost(&S.h_pkt, samples * sizeof(int16_t)));
        OWW_CUDA(ctx, cudaMalloc(&S.d_pkt, samples * sizeof(int16_t)));
        S.pkt_samples = samples;
    }
    if (S.scores_floats < scores) {
        cudaFree(S.d_scores); S.d_scores = nullptr; S.scores_floats = 0;
        OWW_CUDA(ctx, cudaMalloc(&S.d_scores, scores * sizeof(float)));
        S.scores_floats = scores;
    }
    if (S.final_floats < fin) {
        cudaFree(S.d_final); S.d_final = nullptr; S.final_floats = 0;
        OWW_CUDA(ctx, cudaMalloc(&S.d_final, fin * sizeof(float)));
        S.final_floats = fin;
    }
    if (S.d_out_bytes < lay.final) {
        cudaFree(S.d_out); S.d_out = nullptr; S.d_out_bytes = 0;
        OWW_CUDA(ctx, cudaMalloc(&S.d_out, lay.final));
        S.d_out_bytes = lay.final;
    }
    if (S.h_out_bytes < lay.bytes) {
        cudaFreeHost(S.h_out); S.h_out = nullptr; S.h_out_dev = nullptr; S.h_out_bytes = 0;
        OWW_CUDA(ctx, cudaHostAlloc(&S.h_out, lay.bytes, cudaHostAllocMapped));
        OWW_CUDA(ctx, cudaHostGetDevicePointer(reinterpret_cast<void**>(&S.h_out_dev), S.h_out, 0));
        S.h_out_bytes = lay.bytes;
    }
    return OWW_OK;
}

}  // namespace

extern "C" {

int oww_detect_host_submit(oww_ctx* ctx, const int16_t* h_packets, const int64_t* h_offsets, int max_events,
                           int capture_samples, int want_final, int* ticket) {
    if (!ctx) return OWW_EINVAL;
    if (!h_offsets || !ticket) return oww_fail(ctx, OWW_EINVAL, "null argument");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    const int si = ctx->det_next;
    oww_ctx::DetectSlot& S = ctx->det_slot[si];
    if (S.busy) return oww_fail(ctx, OWW_EINVAL, "two detect tickets are in flight: collect one first");
    // every refusal before anything is enqueued; the capacities count what earlier submits staged (host counters)
    int rc = oww_ingest_check(ctx, h_offsets);
    if (rc) return rc;
    const int L = oww_detect_n_labels(ctx);
    if (L == 0) return oww_fail(ctx, OWW_EINVAL, "no detector configured (oww_set_detector, oww_set_streams)");
    if (max_events < 0) return oww_fail(ctx, OWW_EINVAL, "max_events=%d is negative", max_events);
    const int H = oww_audio_history_samples(ctx);
    if (capture_samples < 0 || (capture_samples > 0 && capture_samples > H))
        return oww_fail(ctx, OWW_EINVAL, H ? "capture_samples=%d outside [0,%d]" : "capture_samples=%d without an audio "
                        "history (oww_set_audio_history)", capture_samples, H);
    const int B = ctx->n_streams;
    const int64_t off0 = h_offsets[0], total = h_offsets[B] - off0;
    if (total > 0 && !h_packets) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if ((rc = detect_slot_grow(ctx, S, B, (size_t)std::max<int64_t>(total, 1), max_events, capture_samples, L))) return rc;
    S.offsets.resize((size_t)B + 1);
    for (int b = 0; b <= B; ++b) S.offsets[b] = h_offsets[b] - off0;
    S.chunks.resize(B);
    S.prepared.resize(B);
    cudaStream_t s = ctx->own_stream;
    if (total > 0) {
        // A dense page-locked span (cudaMallocHost / cudaHostRegister / torch pin_memory) is DMA'd straight from the
        // caller's buffer, which must stay untouched until the ticket is collected; otherwise it is staged
        const int16_t* src = h_packets + off0;
        cudaPointerAttributes a0, a1;
        const bool pinned = cudaPointerGetAttributes(&a0, src) == cudaSuccess && a0.type == cudaMemoryTypeHost &&
                            cudaPointerGetAttributes(&a1, src + total - 1) == cudaSuccess && a1.type == cudaMemoryTypeHost;
        cudaGetLastError();                                 // unregistered host memory reports an error on older drivers
        if (!pinned) {
            std::memcpy(S.h_pkt, src, (size_t)total * sizeof(int16_t));
            src = S.h_pkt;
        }
        OWW_CUDA(ctx, cudaMemcpyAsync(S.d_pkt, src, (size_t)total * sizeof(int16_t), cudaMemcpyHostToDevice, ctx->copy_stream));
        OWW_CUDA(ctx, cudaEventRecord(S.h2d_done, ctx->copy_stream));
        OWW_CUDA(ctx, cudaStreamWaitEvent(s, S.h2d_done, 0));
    }
    uint8_t* d_out = S.d_out;
    const DetectLayout lay = oww_detect_layout(max_events, capture_samples, B, L);
    oww_event* d_events = max_events > 0 ? reinterpret_cast<oww_event*>(d_out + lay.events) : nullptr;
    int32_t* d_n = reinterpret_cast<int32_t*>(d_out);
    if ((rc = oww_ingest(ctx, S.d_pkt, S.offsets.data(), S.chunks.data(), S.prepared.data(), S.d_scores, s))) return rc;
    if ((rc = oww_detect(ctx, S.d_scores, 0, S.prepared.data(), want_final ? S.d_final : nullptr, d_events, max_events, d_n, s)))
        return rc;
    if (capture_samples > 0 &&
        (rc = oww_capture_events(ctx, d_events, d_n, max_events, capture_samples, reinterpret_cast<int16_t*>(d_out + lay.clips),
                                 reinterpret_cast<int64_t*>(d_out + lay.ends), s)))
        return rc;
    if ((rc = oww_detect_deliver(ctx, d_out, S.h_out_dev, max_events, capture_samples, s))) return rc;
    if (want_final)
        OWW_CUDA(ctx, cudaMemcpyAsync(S.h_out + lay.final, S.d_final, (size_t)B * L * sizeof(float), cudaMemcpyDeviceToHost, s));
    OWW_CUDA(ctx, cudaEventRecord(S.done, s));
    S.n_streams = B; S.n_labels = L; S.max_events = max_events; S.capture = capture_samples; S.want_final = want_final != 0;
    S.seq = ++ctx->det_seq;
    S.busy = true;
    ctx->det_next = si ^ 1;
    *ticket = si;
    return OWW_OK;
}

int oww_detect_host_collect(oww_ctx* ctx, int ticket, oww_event* h_events, int32_t* h_n_events, int16_t* h_clips,
                            int64_t* h_ends, int32_t* h_chunks, int32_t* h_prepared, float* h_final) {
    if (!ctx) return OWW_EINVAL;
    if (ticket < 0 || ticket > 1 || !ctx->det_slot[ticket].busy)
        return oww_fail(ctx, OWW_EINVAL, "detect ticket %d is not in flight", ticket);
    oww_ctx::DetectSlot& S = ctx->det_slot[ticket];
    const oww_ctx::DetectSlot& other = ctx->det_slot[ticket ^ 1];
    if (other.busy && other.seq < S.seq)
        return oww_fail(ctx, OWW_EINVAL, "detect ticket %d was submitted before ticket %d: collect it first", ticket ^ 1, ticket);
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaEventSynchronize(S.done));
    const DetectLayout lay = oww_detect_layout(S.max_events, S.capture, S.n_streams, S.n_labels);
    const int n = *reinterpret_cast<const int32_t*>(S.h_out);
    const size_t k = (size_t)std::min(n, S.max_events);
    if (h_n_events) *h_n_events = n;
    if (h_events && k) std::memcpy(h_events, S.h_out + lay.events, k * sizeof(oww_event));
    if (h_ends && S.capture && k) std::memcpy(h_ends, S.h_out + lay.ends, k * sizeof(int64_t));
    if (h_clips && S.capture && k) std::memcpy(h_clips, S.h_out + lay.clips, k * S.capture * sizeof(int16_t));
    if (h_chunks) std::memcpy(h_chunks, S.chunks.data(), (size_t)S.n_streams * sizeof(int32_t));
    if (h_prepared) std::memcpy(h_prepared, S.prepared.data(), (size_t)S.n_streams * sizeof(int32_t));
    if (h_final && S.want_final) std::memcpy(h_final, S.h_out + lay.final, (size_t)S.n_streams * S.n_labels * sizeof(float));
    S.busy = false;
    return OWW_OK;
}

int oww_get_features(oww_ctx* ctx, int stream_id, int n, int back, float* h_out) {
    if (!ctx || !h_out) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (stream_id < 0 || stream_id >= ctx->n_streams) return oww_fail(ctx, OWW_EINVAL, "bad stream id");
    if (n < 0 || back < 0 || n + back > ctx->feat_rows) return oww_fail(ctx, OWW_EINVAL, "n+back exceeds the ring (%d rows)", ctx->feat_rows);
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaDeviceSynchronize());
    int count = 0;
    OWW_CUDA(ctx, cudaMemcpy(&count, ctx->d_feat_count + stream_id, sizeof(int), cudaMemcpyDeviceToHost));
    std::vector<float> ring((size_t)ctx->feat_rows * 96);
    OWW_CUDA(ctx, cudaMemcpy(ring.data(), ctx->d_feat_ring + (size_t)stream_id * ctx->feat_rows * 96,
                             ring.size() * sizeof(float), cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; ++i) {
        const int r = count - back - n + i;
        if (r < 0 || r < count - ctx->feat_rows) std::memset(h_out + (size_t)i * 96, 0, 96 * sizeof(float));
        else std::memcpy(h_out + (size_t)i * 96, ring.data() + (size_t)(r & (ctx->feat_rows - 1)) * 96, 96 * sizeof(float));
    }
    return OWW_OK;
}

int oww_get_counts(oww_ctx* ctx, int stream_id, int* mel_rows, int* feature_rows) {
    if (!ctx) return OWW_EINVAL;
    if (stream_id < 0 || stream_id >= ctx->n_streams) return oww_fail(ctx, OWW_EINVAL, "bad stream id");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaDeviceSynchronize());
    int c[2] = {0, 0};
    OWW_CUDA(ctx, cudaMemcpy(&c[0], ctx->d_mel_count + stream_id, sizeof(int), cudaMemcpyDeviceToHost));
    OWW_CUDA(ctx, cudaMemcpy(&c[1], ctx->d_feat_count + stream_id, sizeof(int), cudaMemcpyDeviceToHost));
    if (mel_rows) *mel_rows = c[0];
    if (feature_rows) *feature_rows = c[1];
    return OWW_OK;
}

int oww_get_mel(oww_ctx* ctx, int stream_id, int n_rows, float* h_out) {
    if (!ctx || !h_out) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (stream_id < 0 || stream_id >= ctx->n_streams) return oww_fail(ctx, OWW_EINVAL, "bad stream id");
    if (n_rows < 0 || n_rows > OWW_WINDOW_ROWS) return oww_fail(ctx, OWW_EINVAL, "n_rows must be <= 76");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaDeviceSynchronize());
    int count = 0;
    OWW_CUDA(ctx, cudaMemcpy(&count, ctx->d_mel_count + stream_id, sizeof(int), cudaMemcpyDeviceToHost));
    std::vector<float> ring((size_t)ctx->mel_rows * 32);
    OWW_CUDA(ctx, cudaMemcpy(ring.data(), ctx->d_mel_ring + (size_t)stream_id * ctx->mel_rows * 32,
                             ring.size() * sizeof(float), cudaMemcpyDeviceToHost));
    for (int i = 0; i < n_rows; ++i) {
        const int r = count - n_rows + i;
        std::memcpy(h_out + (size_t)i * 32, ring.data() + (size_t)(r & (ctx->mel_rows - 1)) * 32, 32 * sizeof(float));
    }
    return OWW_OK;
}

int oww_embed_clips(oww_ctx* ctx, const int16_t* d_pcm, int n_clips, int n_samples, float* d_emb, void* stream) {
    if (!ctx || !d_pcm || !d_emb) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (n_samples < OWW_FFT_N) return oww_fail(ctx, OWW_EINVAL, "need at least 512 samples");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    const int T = (n_samples - OWW_FFT_N) / OWW_HOP + 1;
    if (T < OWW_WINDOW_ROWS)
        return oww_fail(ctx, OWW_EINVAL, "Embedding model requires the input melspectrograms to have at least 76 frames");
    const int W = (T - OWW_WINDOW_ROWS) / 8 + 1;
    cudaStream_t s = (cudaStream_t)stream;
    // per slab of clips: the mel of each clip (one call per clip, as the reference's CPU path runs the graph), then ONE
    // fully convolutional CNN pass over the clips' [T x 32] mel (SURVEY.md F10)
    const int slab = clip_slab(ctx, n_clips, OWW_WINDOW_ROWS + 8 * (W - 1));
    float* d_mel = nullptr;
    OWW_CUDA(ctx, cudaMallocAsync(&d_mel, (size_t)slab * T * 32 * sizeof(float), s));
    int rc = OWW_OK;
    for (int c0 = 0; c0 < n_clips; c0 += slab) {
        const int m = std::min(slab, n_clips - c0);
        MelLaunch ml{d_pcm + (size_t)c0 * n_samples, (int64_t)n_samples, n_samples, nullptr, nullptr, d_mel, (int64_t)T * 32,
                     -1, nullptr, m, 1, 0};
        if ((rc = oww_mel_launch(ctx, ml, s))) break;
        if ((rc = oww_cnn_clip(ctx, d_mel, m, T, d_emb + (size_t)c0 * W * 96, W, s))) break;
    }
    cudaFreeAsync(d_mel, s);
    return rc;
}

int oww_predict_clips(oww_ctx* ctx, const int16_t* d_pcm, int n_clips, int n_samples, int pad_samples,
                      const float* h_feature_init, int n_rows, float* d_scores, void* stream) {
    if (!ctx || !d_pcm || !d_scores) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (n_clips < 1 || n_samples < 1 || pad_samples < 0) return oww_fail(ctx, OWW_EINVAL, "bad clip geometry");
    std::vector<int64_t> off((size_t)n_clips + 1);
    for (int i = 0; i <= n_clips; ++i) off[i] = (int64_t)i * n_samples;
    return oww_predict_clips_ragged(ctx, d_pcm, off.data(), n_clips, pad_samples, OWW_SAMPLES_PER_CHUNK, h_feature_init, n_rows,
                                    d_scores, nullptr, nullptr, stream);
}

int oww_clip_schedule(int chunk_size, int64_t n_padded_samples, int32_t* h_chunks_per_call, int max) {
    if (chunk_size < 1 || n_padded_samples < 0) return oww_fail(nullptr, OWW_EINVAL, "bad chunk_size / length");
    const int64_t n = oww_clip_calls(n_padded_samples, chunk_size);
    if (n > INT32_MAX) return oww_fail(nullptr, OWW_EINVAL, "too many calls");
    for (int64_t j = 0; h_chunks_per_call && j < std::min<int64_t>(n, max); ++j)
        h_chunks_per_call[j] = (int32_t)(oww_call_first_step(j + 1, chunk_size) - oww_call_first_step(j, chunk_size));
    return (int)n;
}

int oww_clip_slab_plan(oww_ctx* ctx, const int32_t* h_steps, int n_clips, int64_t* h_steps_computed, int64_t* h_steps_needed) {
    if (!h_steps || n_clips < 0) return oww_fail(ctx, OWW_EINVAL, "null argument");
    oww_ctx local;                       // ctx may be NULL: the slab bound depends only on the layer table and split_from
    if (!ctx) { fill_layer_table(&local); ctx = &local; }
    std::vector<int> steps;
    for (int i = 0; i < n_clips; ++i)
        if (h_steps[i] > 0) steps.push_back(h_steps[i]);
    std::stable_sort(steps.begin(), steps.end(), std::greater<int>());
    const std::vector<ClipSlab> plan = plan_slabs(ctx, steps);
    int64_t computed = 0, needed = 0;
    for (const ClipSlab& sl : plan) computed += (int64_t)(sl.e - sl.b) * sl.K;
    for (int k : steps) needed += k;
    if (h_steps_computed) *h_steps_computed = computed;
    if (h_steps_needed) *h_steps_needed = needed;
    return (int)plan.size();
}

}  // extern "C"

// oww_predict_clips_ragged (h_clip_streams == nullptr: every clip on the clip slots) and oww_predict_clips_streams
static int predict_clips(oww_ctx* ctx, const int16_t* d_pcm, const int64_t* h_offsets, int n_clips, int pad_samples,
                         int chunk_size, const float* h_feature_init, int n_rows, float* d_scores, uint8_t* d_stepped,
                         float* d_emb, const int32_t* h_clip_streams, void* stream) {
    if (!ctx || !h_offsets) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (n_clips < 0 || pad_samples < 0) return oww_fail(ctx, OWW_EINVAL, "bad clip geometry");
    if (chunk_size < 1 || chunk_size > ctx->cfg.max_chunks * OWW_SAMPLES_PER_CHUNK)
        return oww_fail(ctx, OWW_EINVAL, "chunk_size=%d outside [1, max_chunks*1280 = %d]", chunk_size,
                        ctx->cfg.max_chunks * OWW_SAMPLES_PER_CHUNK);
    if (h_feature_init && n_rows < 0) return oww_fail(ctx, OWW_EINVAL, "n_rows=%d", n_rows);
    if (h_offsets[0] < 0) return oww_fail(ctx, OWW_EINVAL, "offset 0 is negative");
    for (int i = 0; i < n_clips; ++i)
        if (h_offsets[i + 1] < h_offsets[i] || h_offsets[i + 1] - h_offsets[i] > INT32_MAX - 2 * (int64_t)pad_samples)
            return oww_fail(ctx, OWW_EINVAL, "offsets[%d..%d] = %lld, %lld are not monotone (or the clip is too long)", i, i + 1,
                            (long long)h_offsets[i], (long long)h_offsets[i + 1]);
    for (int i = 0; h_clip_streams && i < n_clips; ++i)
        if (h_clip_streams[i] < 0 || h_clip_streams[i] >= ctx->n_streams)
            return oww_fail(ctx, OWW_EINVAL, "clip %d: stream %d outside [0,%d)", i, h_clip_streams[i], ctx->n_streams);
    if (ctx->n_out_total == 0 || n_clips == 0) return OWW_OK;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    const int c = chunk_size, n_out = ctx->n_out_total;
    // per clip: its calls, the chunks they step, its first score row and first embedding row (input order)
    std::vector<int> steps(n_clips);
    std::vector<int64_t> row0(n_clips), emb0(n_clips);
    int64_t rows = 0, emb_rows = 0;
    for (int i = 0; i < n_clips; ++i) {
        const int64_t calls = oww_clip_calls(h_offsets[i + 1] - h_offsets[i] + 2 * (int64_t)pad_samples, c);
        steps[i] = (int)oww_call_first_step(calls, c);
        row0[i] = rows; emb0[i] = emb_rows;
        rows += calls; emb_rows += steps[i];
    }
    if (rows > INT32_MAX) return oww_fail(ctx, OWW_EINVAL, "%lld score rows in one call", (long long)rows);
    // slabs: clips that step, longest first (ties in input order), neighbours in that order (plan_slabs)
    std::vector<int> order;
    for (int i = 0; i < n_clips; ++i)
        if (steps[i] > 0) order.push_back(i);
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return steps[x] > steps[y]; });
    const int n_act = (int)order.size();
    if (n_act == 0) return OWW_OK;
    if (!d_scores || (!d_pcm && h_offsets[n_clips] > h_offsets[0])) return oww_fail(ctx, OWW_EINVAL, "null argument");
    std::vector<int> st_sorted(n_act);
    for (int p = 0; p < n_act; ++p) st_sorted[p] = steps[order[p]];
    const std::vector<ClipSlab> plan = plan_slabs(ctx, st_sorted);

    // One host table, one upload: per sorted clip {sample offset, length, steps, first embedding row}, then per slab the
    // rows of its stepping calls {last chunk row in the slab's step rows, chunks stepped, score row}.  Equal-step slabs of
    // consecutive clips at chunk_size 1280 (every call one step) need no call table: the heads write d_scores directly.
    const bool one_chunk_calls = c == OWW_SAMPLES_PER_CHUNK;
    std::vector<uint8_t> direct(plan.size(), 0);
    std::vector<int64_t> call0(plan.size() + 1, 0);
    size_t max_v = 0, max_f = 0, max_tmp = 0;
    int max_calls = 0;
    const int init_rows = h_feature_init ? n_rows : OWW_INIT_FEATURE_ROWS;
    for (size_t k = 0; k < plan.size(); ++k) {
        const ClipSlab& sl = plan[k];
        const int m = sl.e - sl.b;
        bool d = one_chunk_calls;
        for (int p = sl.b; d && p < sl.e; ++p) d = steps[order[p]] == sl.K && order[p] == order[sl.b] + (p - sl.b);
        direct[k] = d;
        int n_calls = 0;
        if (!d)
            for (int p = sl.b; p < sl.e; ++p) {
                const int64_t calls = oww_clip_calls(h_offsets[order[p] + 1] - h_offsets[order[p]] + 2 * (int64_t)pad_samples, c);
                for (int64_t j = 0; j < calls; ++j) n_calls += oww_call_first_step(j + 1, c) > oww_call_first_step(j, c);
            }
        call0[k + 1] = call0[k] + n_calls;
        max_calls = std::max(max_calls, n_calls);
        const int seg = std::min(sl.K, 8192);
        max_v = std::max(max_v, (size_t)m * (OWW_WINDOW_ROWS + 8 * (seg - 1)) * 32);
        max_f = std::max(max_f, (size_t)m * (init_rows + sl.K) * 96);
        if (!d) max_tmp = std::max(max_tmp, (size_t)m * sl.K * n_out);
    }
    const int64_t n_call_rows = call0.back();
    const size_t sz_off = (size_t)n_act * 8, sz_emb0 = (size_t)n_act * 8, sz_len = (size_t)n_act * 4, sz_st = (size_t)n_act * 4;
    const size_t sz_calls = (size_t)n_call_rows * 4;
    std::vector<uint8_t> tab(sz_off + sz_emb0 + sz_len + sz_st + 3 * sz_calls);
    int64_t* t_off = reinterpret_cast<int64_t*>(tab.data());
    int64_t* t_emb0 = t_off + n_act;
    int* t_len = reinterpret_cast<int*>(t_emb0 + n_act);
    int* t_st = t_len + n_act;
    int* t_qlast = t_st + n_act;
    int* t_k = t_qlast + n_call_rows;
    int* t_row = t_k + n_call_rows;
    for (int p = 0; p < n_act; ++p) {
        const int i = order[p];
        t_off[p] = h_offsets[i]; t_len[p] = (int)(h_offsets[i + 1] - h_offsets[i]); t_st[p] = steps[i]; t_emb0[p] = emb0[i];
    }
    for (size_t k = 0; k < plan.size(); ++k) {
        if (direct[k]) continue;
        const ClipSlab& sl = plan[k];
        int64_t r = call0[k];
        for (int p = sl.b; p < sl.e; ++p) {
            const int i = order[p];
            const int64_t calls = oww_clip_calls(h_offsets[i + 1] - h_offsets[i] + 2 * (int64_t)pad_samples, c);
            for (int64_t j = 0; j < calls; ++j) {
                const int64_t f0 = oww_call_first_step(j, c), f1 = oww_call_first_step(j + 1, c);
                if (f1 == f0) continue;                       // the call only accumulates samples: its row is the host's
                t_qlast[r] = (p - sl.b) * sl.K + (int)f1 - 1; t_k[r] = (int)(f1 - f0); t_row[r] = (int)(row0[i] + j);
                ++r;
            }
        }
    }
    // Per-clip streams: the stream of each sorted clip (the verifiers take its slots), and per slab and head bank an item
    // table over the slab's rows (sample = slab-local clip * K + step): clips grouped by the slot of their stream (host
    // mirror of the assignment), each clip's rows contiguous, items of at most 64 rows of one slot.  They go up with the
    // call's one table upload below: pageable, so the driver stages them before cudaMemcpyAsync returns (a host-side copy
    // of about 4 bytes per row and head bank), so `tab` may be freed when the call returns.
    const int n_hb = h_clip_streams ? (int)ctx->head_banks.size() : 0;
    std::vector<std::vector<int>> hb_items(plan.size() * n_hb), hb_perm(plan.size() * n_hb);
    for (size_t k = 0; k < plan.size() && n_hb; ++k) {
        const ClipSlab& sl = plan[k];
        const int m = sl.e - sl.b, K = sl.K;
        for (int h = 0; h < n_hb; ++h) {
            const std::vector<int>& assign = ctx->head_banks[h].assign;
            std::vector<int> slot(m), lc(m);
            for (int p = 0; p < m; ++p) slot[p] = assign[h_clip_streams[order[sl.b + p]]];
            std::iota(lc.begin(), lc.end(), 0);
            std::stable_sort(lc.begin(), lc.end(), [&](int x, int y) { return slot[x] < slot[y]; });
            std::vector<int>& items = hb_items[k * n_hb + h];
            std::vector<int>& perm = hb_perm[k * n_hb + h];
            for (int i = 0; i < m; ++i)
                for (int st = 0; st < K; ++st) {
                    const int first = (int)perm.size();
                    if (items.empty() || items[items.size() - 4] != slot[lc[i]] || first - items[items.size() - 3] == 64)
                        items.insert(items.end(), {slot[lc[i]], first, 0, 0});
                    items[items.size() - 2]++;
                    perm.push_back(lc[i] * K + st);
                }
            while (perm.size() % 4) perm.push_back(0);               // the next table's items stay 16-byte aligned
        }
    }
    const size_t sz_cs = h_clip_streams ? (size_t)n_act * 4 : 0;
    size_t sz_hb = 0;
    for (size_t i = 0; i < hb_items.size(); ++i) sz_hb += (hb_items[i].size() + hb_perm[i].size()) * 4;
    const size_t hb0 = (tab.size() + sz_cs + 15) & ~(size_t)15;
    if (h_clip_streams) tab.resize(hb0 + sz_hb);
    int* t_cs = reinterpret_cast<int*>(tab.data() + sz_off + sz_emb0 + sz_len + sz_st + 3 * sz_calls);
    for (int p = 0; p < (int)sz_cs / 4; ++p) t_cs[p] = h_clip_streams[order[p]];
    std::vector<size_t> hb_at(hb_items.size());
    for (size_t i = 0, at = hb0; i < hb_items.size(); ++i) {
        hb_at[i] = at;
        std::memcpy(tab.data() + at, hb_items[i].data(), hb_items[i].size() * 4);
        at += hb_items[i].size() * 4;
        std::memcpy(tab.data() + at, hb_perm[i].data(), hb_perm[i].size() * 4);
        at += hb_perm[i].size() * 4;
    }
    const bool verify_calls = oww_verifiers_clip_active(ctx, h_clip_streams != nullptr);
    uint8_t* d_tab = nullptr;
    float *d_v = nullptr, *d_f = nullptr, *d_init = nullptr, *d_tmp = nullptr, *d_call = nullptr;
    OWW_CUDA(ctx, cudaMallocAsync(&d_tab, tab.size(), s));
    OWW_CUDA(ctx, cudaMemcpyAsync(d_tab, tab.data(), tab.size(), cudaMemcpyHostToDevice, s));   // pageable: staged before return
    const int64_t* d_off = reinterpret_cast<const int64_t*>(d_tab);
    const int64_t* d_emb0 = d_off + n_act;
    const int* d_len = reinterpret_cast<const int*>(d_emb0 + n_act);
    const int* d_st = d_len + n_act;
    const int* d_qlast = d_st + n_act;
    const int* d_k = d_qlast + n_call_rows;
    const int* d_row = d_k + n_call_rows;
    const int* d_cs = h_clip_streams ? d_row + n_call_rows : nullptr;
    std::vector<BankRows> bank_rows(hb_items.size());
    for (size_t i = 0; i < hb_items.size(); ++i) {
        const int4* items = reinterpret_cast<const int4*>(d_tab + hb_at[i]);
        bank_rows[i] = BankRows{items, reinterpret_cast<const int*>(items + hb_items[i].size() / 4), (int)hb_items[i].size() / 4};
    }
    OWW_CUDA(ctx, cudaMallocAsync(&d_v, max_v * sizeof(float), s));
    OWW_CUDA(ctx, cudaMallocAsync(&d_f, max_f * sizeof(float), s));
    if (max_tmp) OWW_CUDA(ctx, cudaMallocAsync(&d_tmp, max_tmp * sizeof(float), s));
    if (max_tmp && verify_calls) OWW_CUDA(ctx, cudaMallocAsync(&d_call, (size_t)max_calls * n_out * sizeof(float), s));
    if (h_feature_init && init_rows > 0) {
        OWW_CUDA(ctx, cudaMallocAsync(&d_init, (size_t)init_rows * 96 * sizeof(float), s));
        OWW_CUDA(ctx, cudaMemcpyAsync(d_init, h_feature_init, (size_t)init_rows * 96 * sizeof(float), cudaMemcpyHostToDevice, s));
    }
    // Bulk path (SURVEY.md F10), per slab of clips: for each segment of at most 8192 steps (ending on a call boundary) ONE
    // mel launch over the padded clips (frames grouped and clamped per streaming call, behind the 71 rows of ones a fresh
    // stream's window starts with) and ONE fully convolutional CNN pass over its rows; then the heads over all sliding
    // windows of [feature_init rows | embeddings], the max over each call's chunk rows and the verifiers on each call's
    // newest window.  The same arithmetic as streaming the clips through fresh streams.  A clip shorter than its slab's
    // longest runs on over virtual zeros: a step's rows depend only on samples up to its call's end, so its own calls'
    // rows do not change, and the rows past them are not read.
    int rc = OWW_OK;
    for (size_t k = 0; k < plan.size() && rc == OWW_OK; ++k) {
        const ClipSlab& sl = plan[k];
        const int m = sl.e - sl.b, K = sl.K;
        const int64_t f_stride = (int64_t)(init_rows + K) * 96;
        for (int k0 = 0; k0 < K && rc == OWW_OK;) {
            const int k1 = K - k0 <= 8192 ? K : (int)oww_call_first_step(oww_call_of_step(k0 + 8192, c), c);
            const int T = OWW_WINDOW_ROWS + 8 * (k1 - k0 - 1);
            if ((rc = oww_mel_clips_launch(ctx, d_pcm, d_off + sl.b, d_len + sl.b, m, pad_samples, c, k0, k1, d_v, (int64_t)T * 32, s)))
                break;
            if (k0 == 0 && init_rows > 0) {
                fill_init_rows_kernel<<<std::min(1024, (m * init_rows * 24 + 255) / 256), 256, 0, s>>>(d_f, f_stride, m, d_init, init_rows);
                ctx->launches++;
            }
            // embeddings of step st land at row init_rows + st of the clip's feature array
            rc = oww_cnn_clip(ctx, d_v, m, T, d_f + (int64_t)(init_rows + k0) * 96, init_rows + K, s);
            k0 = k1;
        }
        if (rc) break;
        FeatSrc fs{d_f, f_stride, nullptr, -1, 0};
        fs.steps = K; fs.row0 = init_rows;
        const BankRows* brows = n_hb ? bank_rows.data() + k * n_hb : nullptr;
        const int* cs = d_cs ? d_cs + sl.b : nullptr;
        if (direct[k]) {
            const int64_t r0 = row0[order[sl.b]];
            float* out = d_scores + r0 * n_out;
            if ((rc = oww_heads_all(ctx, fs, m * K, out, n_out, 0, s, brows))) break;
            if ((rc = oww_verifiers_apply(ctx, fs, m * K, out, n_out, true, s, nullptr, cs))) break;   // every step
            if (d_stepped) OWW_CUDA(ctx, cudaMemsetAsync(d_stepped + r0, 1, (size_t)m * K, s));
        } else {
            const int nc = (int)(call0[k + 1] - call0[k]);
            const int* qlast = d_qlast + call0[k];
            const int* kk = d_k + call0[k];
            const int* orow = d_row + call0[k];
            if ((rc = oww_heads_all(ctx, fs, m * K, d_tmp, n_out, 0, s, brows))) break;
            if (!verify_calls) {
                if ((rc = call_max_launch(ctx, d_tmp, n_out, qlast, kk, nc, d_scores, orow, d_stepped, s))) break;
            } else {
                // verifiers after the max, on the call's newest window: on compact call rows, then scattered to their place
                if ((rc = call_max_launch(ctx, d_tmp, n_out, qlast, kk, nc, d_call, nullptr, nullptr, s))) break;
                fs.idx = qlast;
                if ((rc = oww_verifiers_apply(ctx, fs, nc, d_call, n_out, true, s, nullptr, cs))) break;
                if ((rc = call_max_launch(ctx, d_call, n_out, nullptr, nullptr, nc, d_scores, orow, d_stepped, s))) break;
            }
        }
        if (d_emb) {
            const int total = m * K * 24;
            emb_rows_kernel<<<std::min(4096, (total + 255) / 256), 256, 0, s>>>(d_f, f_stride, init_rows, K, m, d_st + sl.b, d_emb0 + sl.b,
                                                                            d_emb);
            OWW_LAUNCH_CHECK(ctx);
        }
    }
    cudaFreeAsync(d_v, s); cudaFreeAsync(d_f, s); cudaFreeAsync(d_tab, s);
    if (d_tmp) cudaFreeAsync(d_tmp, s);
    if (d_call) cudaFreeAsync(d_call, s);
    if (d_init) cudaFreeAsync(d_init, s);
    return rc;
}

extern "C" {

int oww_predict_clips_ragged(oww_ctx* ctx, const int16_t* d_pcm, const int64_t* h_offsets, int n_clips, int pad_samples,
                             int chunk_size, const float* h_feature_init, int n_rows, float* d_scores, uint8_t* d_stepped,
                             float* d_emb, void* stream) {
    return predict_clips(ctx, d_pcm, h_offsets, n_clips, pad_samples, chunk_size, h_feature_init, n_rows, d_scores,
                         d_stepped, d_emb, nullptr, stream);
}

int oww_predict_clips_streams(oww_ctx* ctx, const int16_t* d_pcm, const int64_t* h_offsets, int n_clips, int pad_samples,
                              int chunk_size, const float* h_feature_init, int n_rows, float* d_scores, uint8_t* d_stepped,
                              float* d_emb, const int32_t* h_clip_streams, void* stream) {
    if (!ctx) return OWW_EINVAL;
    if (!h_clip_streams && n_clips > 0) return oww_fail(ctx, OWW_EINVAL, "null argument (h_clip_streams)");
    return predict_clips(ctx, d_pcm, h_offsets, n_clips, pad_samples, chunk_size, h_feature_init, n_rows, d_scores,
                         d_stepped, d_emb, h_clip_streams, stream);
}

int oww_debug_layer(oww_ctx* ctx, const float* d_windows, int n, int layer, float* d_out, void* stream) {
    if (!ctx || !d_windows || !d_out) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (layer < 0 || layer >= OWW_N_CONV - 1) return oww_fail(ctx, OWW_EINVAL, "layer must be in [0,18]");
    if (n < 1 || n > ctx->window_batch) return oww_fail(ctx, OWW_EINVAL, "n must be in [1, window_batch]");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = ensure_act(ctx, (size_t)std::min(n, ctx->window_batch) * 74 * 32 * 24);
    if (rc) return rc;
    WindowSrc src{d_windows, (int64_t)OWW_WINDOW_ROWS * 32, nullptr, -1, 0, 0};
    if (ctx->cfg.cnn_mode == OWW_CNN_TC_WINDOW)
        return oww_cnn_tc_pyramid(ctx, src, n, OWW_WINDOW_ROWS, nullptr, 1, layer, d_out, (cudaStream_t)stream);
    return oww_cnn_fp32_pyramid(ctx, src, n, OWW_WINDOW_ROWS, nullptr, 1, layer, d_out, (cudaStream_t)stream);
}

int oww_debug_inc_plan(oww_ctx* ctx, int group, int n_streams, int32_t* out, int max_ints) {
    return oww_debug_inc_cut_plan(ctx, group, n_streams, 0, out, max_ints);
}

int oww_debug_inc_cut_plan(oww_ctx* ctx, int group, int n_streams, int n_layers, int32_t* out, int max_ints) {
    if (!out) return oww_fail(ctx, OWW_EINVAL, "null argument");
    oww_ctx local;                       // ctx may be NULL: the plan depends only on the fixed layer table
    if (!ctx) { fill_layer_table(&local); ctx = &local; }
    IncPlan P;
    if (group == 0 && ctx != &local) {
        // the plan the handle's fused kernel runs (its group size as oww_inc_alloc_streams chose it)
        if (ctx->inc_plan.G == 0) return oww_fail(ctx, OWW_EINVAL, "the handle has no fused-CNN plan (cnn_mode 3 streams)");
        P = ctx->inc_plan;
    } else {
        int rc = oww_inc_build_plan(ctx, group, n_streams, n_layers ? n_layers : OWW_N_CONV, &P);
        if (rc) return rc;
    }
    const int n = (int)(sizeof(IncPlan) / sizeof(int32_t));
    if (max_ints < n) return oww_fail(ctx, OWW_EINVAL, "need room for %d ints", n);
    std::memcpy(out, &P, sizeof(IncPlan));
    return n;
}

int oww_debug_inc_clocks(oww_ctx* ctx, int64_t* h_out21) {
    if (!ctx || !h_out21) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (ctx->cfg.cnn_mode != OWW_CNN_TC_INCREMENTAL || ctx->n_streams <= 0)
        return oww_fail(ctx, OWW_EINVAL, "needs cnn_mode 3 with streams allocated");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaDeviceSynchronize());
    if (!ctx->d_inc_dbg) OWW_CUDA(ctx, cudaMalloc(&ctx->d_inc_dbg, 104 * sizeof(int64_t)));
    OWW_CUDA(ctx, cudaMemset(ctx->d_inc_dbg, 0, 104 * sizeof(int64_t)));
    // stamps are taken by the NEXT step the caller runs; this call only arms the buffer
    return OWW_OK;
}

int oww_debug_inc_clocks_read(oww_ctx* ctx, int64_t* h_out21) {
    if (!ctx || !h_out21 || !ctx->d_inc_dbg) return oww_fail(ctx, OWW_EINVAL, "clock buffer not armed");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaDeviceSynchronize());
    OWW_CUDA(ctx, cudaMemcpy(h_out21, ctx->d_inc_dbg, 104 * sizeof(int64_t), cudaMemcpyDeviceToHost));
    cudaFree(ctx->d_inc_dbg); ctx->d_inc_dbg = nullptr;
    return OWW_OK;
}

int oww_enable_stage_timing(oww_ctx* ctx, int n_slots) {
    if (!ctx) return OWW_EINVAL;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    ctx->timing = n_slots > 0;
    ctx->ev_steps = 0;
    if (n_slots > 4096) n_slots = 4096;
    while ((int)ctx->ev.size() < 4 * n_slots) {
        cudaEvent_t e;
        OWW_CUDA(ctx, cudaEventCreate(&e));
        ctx->ev.push_back(e);
    }
    if (n_slots > 0) { ctx->ev_slots = n_slots; ctx->ev_fused.assign(n_slots, 0); }
    return OWW_OK;
}

int oww_stage_ms(oww_ctx* ctx, float out_ms[3]) {
    if (!ctx || !out_ms) return OWW_EINVAL;
    if (!ctx->timing || ctx->ev_steps == 0) return oww_fail(ctx, OWW_EINVAL, "no timed step recorded");
    const long n = ctx->ev_steps < ctx->ev_slots ? ctx->ev_steps : ctx->ev_slots;
    double acc[3] = {0, 0, 0};
    for (long k = 0; k < n; ++k) {
        cudaEvent_t* ev = &ctx->ev[4 * k];
        // 0: mel | cnn | heads launches (events 0..3)   1: one fused launch (events 1..2)
        // 2: fused frontend+CNN launch, then a heads launch (events 1..3)
        const int kind = ctx->ev_fused[k];
        const int first = kind == 0 ? 0 : 1, last = kind == 1 ? 2 : 3;
        OWW_CUDA(ctx, cudaEventSynchronize(ev[last]));
        for (int i = first; i < last; ++i) {
            float ms = 0.f;
            OWW_CUDA(ctx, cudaEventElapsedTime(&ms, ev[i], ev[i + 1]));
            acc[i] += ms;
        }
    }
    for (int i = 0; i < 3; ++i) out_ms[i] = (float)(acc[i] / n);
    return OWW_OK;
}

}  // extern "C"
