// Internal declarations shared by the .cu translation units of libowwb200.so.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <string>
#include <utility>
#include <vector>
#include "owwb200.h"

#define OWW_N_CONV 20
#define OWW_FFT_N 512
#define OWW_N_BINS 257
#define OWW_HOP 160
#define OWW_TAIL 480
#define OWW_MEL_MAXSUPPORT 32

struct ConvLayer {
    int kh, kw, cin, cout, pool_t, pool_f;
    int t_in, f_in;      // input extent for the 76-row window
    int t_out, f_out;    // conv output extent (before pool)
    float* d_w;          // [kh*kw*cin][cout]
    float* d_scale;      // [cout]
    float* d_bias;       // [cout]
};

struct Head {
    oww_head_desc desc;
    int n_out;
    int col0;            // first score column
    float* d_blob;       // packed weights (layout of pack_head_blob)
    std::vector<size_t> w_off, b_off, g_off, h_off;   // float offsets per layer
    // tensor-core path (heads_tc.cu): every Linear layer as fp16 hi/lo of W * 2^s in core-matrix order, or tc_ok == false
    struct TcLayer { int K, D, Kp, NP; uint32_t w_off, w_bytes; float unscale; };
    bool tc_ok = false;
    void* d_w1_tc = nullptr;         // packed weights of all layers
    std::vector<TcLayer> tc_layers;
    std::vector<float> tc_w0_host;   // first-layer matrix [n_in*96][D1] (host copy: the grouped kernel packs it per group)
};

// Block-major layout of an incremental late tensor (cnn_tc.cu, tc_conv_blk_kernel): streams in blocks of S, a block is
// [2*cg planes][units] contiguous in HBM (one bulk copy per half), and inside a plane
//   kh3 (input of a (3,1) layer):  unit (row*S + s)*W + f            - time-major, no pad column
//   else (input of a (1,3) layer): unit 1 + (s*T + row)*(W+1) + f    - stream-major, pad column, unit 0 = zero guard
struct LateLay {
    int S, T, Wq, kh3;           // streams per block, rows per stream, row pitch (W or W+1), orientation
    int units;                   // units per plane of a block
    int64_t blk_stride;          // units per block (2*cg*units)
};
#ifdef __CUDACC__
__host__ __device__ __forceinline__ int64_t late_unit(const LateLay& L, int plane, int stream, int row, int f) {
    const int blk = stream / L.S, sl = stream - blk * L.S;
    const int within = L.kh3 ? (row * L.S + sl) * L.Wq + f : 1 + (sl * L.T + row) * L.Wq + f;
    return (int64_t)blk * L.blk_stride + (int64_t)plane * L.units + within;
}
#endif

// what reset_kernel needs to seed a stream's conv tails (mode 3)
struct ResetLate {           // one tails-bearing tensor of the incremental late layers
    uint4* now;              // buffer the stream's next step reads: rows 0, 1 <- template rows 0, 1
    uint4* next;             // tensors that gain ONE row per step: the buffer of the step after, row 0 <- template row 1
    const uint4* tmpl;       // [planes][2][Wp]
    int64_t plane; int T_buf, Wp, n_planes;
    LateLay lay;             // lay.S > 0: block-major destination
};
struct ResetTails { uint4* tails; const uint4* tmpl; int G, tail_units, n_tab; int4 tab[OWW_N_CONV]; int n_late; ResetLate late[6]; };

// conditional verifier pair (hey_jarvis, docs/models/hey_jarvis.md:38): score column `main_col` is replaced by column
// `ver_col` wherever it exceeds `thr`
struct Gate { int main_col, ver_col; float thr; };

// Ring row counters (rows ever written; ring slot = count & (rows-1)) would overflow int32 after ~248 days of
// continuous streaming at 100 mel rows/s.  Past 2^30 they are rebased by a multiple of every ring size (rings are
// powers of two <= 2^20 rows), which keeps the slot and leaves the count >= the ring size, so "row not yet written"
// tests (count - k >= 0) stay true.
#define OWW_COUNT_WRAP (1 << 30)
#define OWW_COUNT_REBASE ((1 << 30) - (1 << 20))
#ifdef __CUDACC__
__device__ __forceinline__ int oww_wrap_count(int c) { return c >= OWW_COUNT_WRAP ? c - OWW_COUNT_REBASE : c; }
#endif

// device-side description of one head (heads.cu launches, and the fused step kernel reads an array of these)
struct HeadDev {
    const float* blob;
    int n_in, n_layers, layernorm, final_act;
    int dims[OWW_MAX_HEAD_LAYERS + 1];
    int w_off[OWW_MAX_HEAD_LAYERS], b_off[OWW_MAX_HEAD_LAYERS], g_off[OWW_MAX_HEAD_LAYERS], h_off[OWW_MAX_HEAD_LAYERS];
    int col0;
};

// ---- fused incremental CNN (cnn_tc_inc.cu): per-layer geometry for a group of G streams --------
struct IncLayer {            // "units" are 16-byte channel-group units (8 fp16 channels of one position)
    int kh3, final;
    int W, Wp;               // input width, Wp = W + 1 (one zero pad column)
    int rows_in, T_out, M;   // input rows (2 tails + new for (3,1)), output rows, positions to compute
    int cg_in, cgp, np, cg_out;
    int in_buf, out_buf;     // buffer class: 0 = low (base 0), 1 = high (base above the live low tensors)
    int in_base, tmp_base, nx_base;   // unit offsets of the input, unpooled temp and produced tensor in the activation arena
    int in_pitch;            // units per plane of the input buffer
    int tap[3];              // unit offset of each conv tap relative to the output position
    int pool_t, pool_f, tmp_pitch;          // max-pool after the conv; pitch of the unpooled temp (in out_buf)
    int nx_buf, nx_pitch, nx_W, nx_Wp, nx_rows_new, nx_t_off, nx_tail_off;   // what this phase leaves for layer l+1
    int w_off, w_bytes, w_smem;             // packed weights: blob offset, size, smem byte offset
};
struct IncPlan {
    int G, n_groups, tail_units, x_units, y_units, w_total_bytes, smem_bytes;
    int scratch_off;         // byte offset of the frontend (mel) scratch used before phase 0; 0 = does not fit
    IncLayer L[OWW_N_CONV];
    int n_layers;            // conv layers inside the kernel (20, or a cut after a pooled layer: the rest run in cnn_tc.cu)
};

struct oww_ctx {
    oww_config cfg;
    int device = 0;
    int sm_count = 132;
    std::string err;
    uint64_t launches = 0;

    // mel constants
    bool mel_loaded = false;
    float* d_window = nullptr;       // [512]
    float2* d_twiddle = nullptr;     // [512] exp(-2 pi i k/512)
    int* d_mel_start = nullptr;      // [32]
    int* d_mel_len = nullptr;        // [32]
    float* d_mel_w = nullptr;        // [32][OWW_MEL_MAXSUPPORT]
    int mel_kmax = 0;                // highest FFT bin any filter touches (+1)

    // embedding CNN
    bool emb_loaded = false;
    ConvLayer conv[OWW_N_CONV];
    float* d_emb_blob = nullptr;

    std::vector<Head> heads;
    int n_out_total = 0;
    int max_n_in = 0;
    std::vector<Gate> gates;         // applied to every chunk's scores before the max over chunks
    Gate* d_gates = nullptr;
    float* d_scores_tmp = nullptr;   // [n_streams][n_out_total]: one chunk's raw scores when gates meet a multi-chunk call
    size_t scores_tmp_floats = 0;

    // streaming state
    int n_streams = 0;
    int mel_rows = 128;              // ring rows (power of two)
    int feat_rows = 128;
    int16_t* d_tail = nullptr;       // [B][480]
    int* d_seen = nullptr;           // [B] chunks seen since reset (saturating)
    int* d_mel_count = nullptr;      // [B] rows ever written (ring slot = count & (mel_rows-1))
    int* d_feat_count = nullptr;     // [B]
    float* d_mel_ring = nullptr;     // [B][mel_rows][32]
    float* d_feat_ring = nullptr;    // [B][feat_rows][96]

    // scratch for the window-mode CNN
    int window_batch = 256;
    float* d_act[2] = {nullptr, nullptr};
    size_t act_floats = 0;           // per buffer
    float* d_emb_tmp = nullptr;      // [max_chunks*B][96]
    size_t emb_tmp_floats = 0;

    // tensor-core path (cnn_tc.cu)
    void* d_tc_w = nullptr;          // packed fp16 weights, all layers
    float* d_tc_sb = nullptr;        // padded scale/bias per layer
    void* d_tc_w3 = nullptr;         // split variant: per layer [hi block | lo block] of W * 2^s (offsets = 2 x tc_w_off)
    float* d_tc_sb3 = nullptr;       // scale * 2^-s | bias
    int tc_rows_out_override = 0;    // clip pass: embedding rows per input in the caller's array (0 = tightly packed)
    int split_from = 11;             // window / clip passes: conv layers >= split_from take fp16 hi/lo split operands
                                     // (fp32-grade products); OWW_N_CONV = plain fp16 everywhere
    size_t tc_w_off[OWW_N_CONV] = {0};
    size_t tc_sb_off[OWW_N_CONV] = {0};
    void* d_tc_act[2] = {nullptr, nullptr};   // fp16 channel-group planes, ping-pong
    size_t tc_act_units = 0;

    // fused incremental path (cnn_tc_inc.cu)
    void* d_inc_w = nullptr;         // packed per-layer {fp16 weights, scale, bias}
    void* d_inc_tails[2] = {nullptr, nullptr};   // [n_groups][tail_units] 16-byte units, double-buffered per step
    int inc_cur = 0;                 // tails buffer the next step reads
    // Incremental late layers (cnn_tc.cu, bottom): tensors X_l = input of conv layer l >= split_from, per stream
    // [tails | new rows], fp16 hi/lo: block-major (LateLay, the default) or plane-major in the window-mode layout
    struct LateTensor { void* buf[3] = {nullptr, nullptr, nullptr}; int n_buf = 0, T_buf = 0, rows_new = 0, W = 0, cg = 0, tmpl_off = -1; int64_t plane = 0;
                        LateLay lay = {0, 0, 0, 0, 0, 0}; };   // lay.S > 0: block-major (tc_conv_blk_kernel); else plane-major [n][T_buf][W + 1]
    LateTensor late_x[OWW_N_CONV];
    void* d_late_tmp[1] = {nullptr};             // unpooled output of a late layer that is followed by a pool
    void* d_late_template = nullptr;             // tails of the all-ones window per tails-bearing late tensor: [plane][2][Wp]
    bool late_active = false;
    bool late_pdl = true;                        // programmatic dependent launches inside the late chain (reserved[0] bit 5 disables)
    bool late_blocked_ok = true;                 // reserved[0] bit 4 keeps the plane-major window layout for every late tensor (A/B)
    long late_step = 0;                          // chunks processed since the buffers were allocated (buffer rotation)

    // Priming.  A reset stream's mel history is ones(76,32) (utils.py:165) and its first chunk yields 5 rows (F8).  A
    // constant history is shift invariant, so that first step equals the ordinary 8-row step on the rows [1,1,1,m0..m4]
    // starting from the tails of the all-ones window: those tails are computed once per weight set (template, compact
    // G = 1 layout) and scattered into the stream's slots by the reset kernel.  No stream is ever "unprimed".
    void* d_tails_template = nullptr;            // [tail units of one stream] x 16 B
    bool tails_template_valid = false;
    int4 tail_tab[OWW_N_CONV];                   // per tails-bearing tensor: {offset in the template, offset in a group, planes, Wp}
    int n_tail_tab = 0;
    int* d_reset_ids = nullptr;      // [n_streams] staging for oww_reset / oww_reset_async
    float* d_reset_init = nullptr;   // [feat_rows][96]
    IncPlan inc_plan;
    void* d_inc_dbg = nullptr;
    HeadDev* d_head_devs = nullptr;  // device copy of the head descriptors (fused step kernel)
    bool fuse_step = true;           // mode 3: run mel + CNN + ring append + heads as ONE launch when the step allows it       // optional per-phase clock stamps (oww_debug_inc_clocks)

    // host staging for oww_step_host / oww_step_host_submit: two slots so the H2D copy of step k+1 (copy_stream)
    // overlaps the kernels of step k (own_stream)
    cudaStream_t own_stream = nullptr;
    cudaStream_t copy_stream = nullptr;
    struct HostSlot {
        int16_t* h_pcm = nullptr; int16_t* d_pcm = nullptr; size_t pcm_bytes = 0;
        float* h_scores = nullptr; float* d_scores = nullptr; size_t sc_bytes = 0;
        cudaEvent_t h2d_done = nullptr, done = nullptr;
        bool busy = false;
    } slot[2];
    int next_slot = 0;

    // stage timing
    bool timing = false;
    std::vector<cudaEvent_t> ev;     // 4 events per slot; step k uses slot k % ev_slots
    std::vector<uint8_t> ev_fused;          // per timing slot: the step was one fused launch (only ev[1], ev[2] recorded)
    int ev_slots = 0;
    long ev_steps = 0;               // timed steps recorded since timing was enabled

    // cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per (function, device): remembered per handle
    bool heads_attr_set = false;
    bool heads_tc_attr_set = false;
    uint32_t tc_blk_attr_mask = 0;
    bool mel_clip_attr_set = false;
    uint32_t tc_attr_mask = 0;
    bool tc_heads = true;            // modes 2/3: first head layer on tensor cores when the head allows it (reserved[0] bit 1 disables)
    int* d_peer_err = nullptr;       // raised by oww_peer_wait's kernel on a timeout (oww_peer_status reads and clears it)
    bool grp_heads = true;           // streaming: heads that share a window run in one CTA per 128 streams (heads_grp.cu; reserved[0] bit 3 disables)
    struct oww_heads_grp* heads_grp = nullptr;
    int tc_heads_terms = 3;          // 3 = hi*hi + lo*hi + hi*lo (fp32-grade), 1 = plain fp16 operands

    // private stream set for oww_predict_clips
    oww_ctx* clip_ctx = nullptr;
};

int oww_fail(oww_ctx* ctx, int code, const char* fmt, ...);
#define OWW_CUDA(ctx, call)                                                                    \
    do {                                                                                       \
        cudaError_t e__ = (call);                                                              \
        if (e__ != cudaSuccess)                                                                \
            return oww_fail((ctx), OWW_ECUDA, "%s failed: %s (%s:%d)", #call,                  \
                            cudaGetErrorString(e__), __FILE__, __LINE__);                      \
    } while (0)
#ifdef __CUDACC__
// Launch with the programmatic-stream-serialization attribute (the kernel calls pdl_wait() before it touches anything
// its predecessor in the stream produced; see tc_common.cuh).  pdl == false: an ordinary launch.
template <typename... KArgs, typename... Args>
inline cudaError_t oww_launch_pdl(bool pdl, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
__device__ __forceinline__ void oww_pdl_sync() {        // trigger the successor, then wait for the predecessor: small kernels
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}
#endif

#define OWW_LAUNCH_CHECK(ctx)                                                                  \
    do {                                                                                       \
        (ctx)->launches++;                                                                     \
        cudaError_t e__ = cudaGetLastError();                                                  \
        if (e__ != cudaSuccess)                                                                \
            return oww_fail((ctx), OWW_ECUDA, "kernel launch failed: %s (%s:%d)",              \
                            cudaGetErrorString(e__), __FILE__, __LINE__);                      \
    } while (0)

// ---- mel.cu ----
// Log-mel of n_clips virtual clips.  Clip c = [prefix (prefix_len samples, may be 0) | body (n_body samples)].
// Streaming: prefix = d_tail row, out rows go to the mel ring at the stream's count; fresh streams
// (seen==0) have no prefix and skip the frames that would touch it.
struct MelLaunch {
    const int16_t* body; int64_t body_stride; int n_body;
    int16_t* tail;                 // [n_clips][480] or nullptr (stateless)
    int* seen;                     // [n_clips] or nullptr
    float* out; int64_t out_stride; int out_rows_mask;   // ring: mask = rows-1 ; linear: mask = -1
    int* out_count;                // ring row counters or nullptr
    int n_clips; int affine; int n_chunks;
    const int* ids = nullptr;      // streaming only: clip j is stream ids[j] (body / tail / seen / ring rows of that stream)
};
int oww_mel_launch(oww_ctx* ctx, const MelLaunch& p, cudaStream_t s);
// bulk path: mel rows of whole padded clips, grouped and clamped per streaming call, behind 71 rows of ones:
// d_out [n_clips][76 + 8 (steps - 1)][32] (the virtual history a fully convolutional CNN pass reproduces predict_clip from)
int oww_mel_clips_launch(oww_ctx* ctx, const int16_t* d_pcm, int64_t clip_stride, int n_clips, int n_samples, int pad, int steps,
                         float* d_out, int64_t out_stride, cudaStream_t s);

// ---- cnn_fp32.cu ----
// Window-mode embedding CNN on n windows.  Source of window j:
//   stateless: src + j*76*32
//   ring     : stream b = j % n_streams, chunk i = j / n_streams (i=0 oldest): rows
//              [count[b] - 8*(n_chunks-1-i) - 76, +76) of the ring.
struct WindowSrc {
    const float* base; int64_t stride;  // per-window (or per-stream) stride in floats
    const int* count; int rows_mask;    // ring addressing (count==nullptr -> linear)
    int n_streams; int n_chunks;
    const int* ids = nullptr;           // ring addressing of a stream subset: local stream b is stream ids[b]
};
// Fully-convolutional pass over linear mel [n][T][32] -> [n][(T-76)/8+1][96] (SURVEY.md F10).
int oww_cnn_clip_fp32(oww_ctx* ctx, const float* d_mel, int n, int T, float* d_emb, cudaStream_t s);
// appends n_chunks embedding rows per stream; ids != nullptr: only the n_ids streams listed (d_emb rows are compact)
int oww_feat_append(oww_ctx* ctx, const float* d_emb, int n_chunks, cudaStream_t s, const int* d_ids = nullptr, int n_ids = 0);
// mode dispatch (fp32 window / tensor-core window) with sub-batching over ctx->window_batch
int oww_cnn_window(oww_ctx* ctx, const WindowSrc& src, int n_windows, float* d_emb, cudaStream_t s, bool capture_tails = false);

// ---- cnn_tc.cu ----
int oww_tc_pack_weights(oww_ctx* ctx, const float* h_blob);
size_t oww_tc_act_units(const oww_ctx* ctx, int n_windows);
size_t oww_tc_act_units_T(const oww_ctx* ctx, int n, int T0);
// fully-convolutional pass over linear mel [n][T][32] -> [n][(T-76)/8+1][96] on the tensor cores
int oww_cnn_tc_clip(oww_ctx* ctx, const float* d_mel, int n, int T, float* d_emb, cudaStream_t s);
int oww_cnn_tc_clip_rows(oww_ctx* ctx, const WindowSrc& src, int n, int T, float* d_emb, int out_rows, cudaStream_t s);
// incremental late layers of mode 3 (split operands)
int oww_late_alloc(oww_ctx* ctx);
int oww_late_chain(oww_ctx* ctx, float* d_emb, cudaStream_t s);
int oww_late_capture(oww_ctx* ctx, int next_layer, const void* planes, int64_t plane_pitch, int T, int W, cudaStream_t s);
int oww_cnn_tc_pyramid(oww_ctx* ctx, const WindowSrc& src, int n, float* d_emb, int stop_layer, float* d_dbg, cudaStream_t s);
// fp32 pyramid with an optional early stop that leaves NHWC fp32 [n][T][W][C] of `stop_layer` in d_dbg
// capture descriptor: which local windows of a full-window pass are the newest window of which streams
struct TailCapture { int win0, n_win, stream0; const int* ids = nullptr; bool late = false; };   // ids: local stream -> stream id;
                                                                  // late: window 0 is the template window of the incremental late layers
int oww_cnn_tc_pyramid_cap(oww_ctx* ctx, const WindowSrc& src, int n, float* d_emb, const TailCapture* cap, cudaStream_t s);

// ---- cnn_tc_inc.cu ----
int oww_inc_build_plan(oww_ctx* ctx, int G, int n_streams, int n_layers, IncPlan* out);
int oww_inc_n_layers(const oww_ctx* ctx);
int oww_inc_setup(oww_ctx* ctx, const float* h_blob);
int oww_inc_alloc_streams(oww_ctx* ctx);
int oww_cnn_inc_step(oww_ctx* ctx, int back, float* d_emb, cudaStream_t s);
// whole step in one launch (n_chunks == 1, primed): PCM -> mel -> CNN -> ring append -> heads -> scores
bool oww_fused_frontend_supported(const oww_ctx* ctx);
bool oww_fused_heads_supported(const oww_ctx* ctx);
int oww_fused_step(oww_ctx* ctx, const int16_t* d_pcm, int64_t pcm_stride, float* d_scores, int out_stride, bool with_heads,
                   cudaStream_t s);
int oww_heads_sync_devs(oww_ctx* ctx);
int oww_inc_capture(oww_ctx* ctx, int layer, const void* planes, int64_t plane_pitch, int T, int W, int win0, int n_win,
                    int stream0, const int* d_ids, cudaStream_t s);
int oww_cnn_fp32_pyramid(oww_ctx* ctx, const WindowSrc& src, int n, float* d_emb, int stop_layer, float* d_dbg, cudaStream_t s);

// ---- heads.cu ----
struct FeatSrc {
    const float* base; int64_t stride;   // per-sample stride in floats
    const int* count; int rows_mask;     // ring addressing (nullptr -> linear [n][n_in][96])
    int back;                            // ring: window ends `back` rows before the newest
    // sliding mode (count == nullptr, steps > 0; bulk clips): sample s = clip * steps + st reads rows
    // [row0 + st + 1 - n_in, row0 + st] of clip's linear rows at base + clip * stride (negative rows read as zeros)
    int steps = 0, row0 = 0;
};
// head_id < 0: every head whose bit is set in head_mask (blockIdx.y walks the selected heads)
int oww_heads_launch(oww_ctx* ctx, int head_id, const FeatSrc& src, int n, float* d_out, int out_stride,
                     int out_col0, int combine_max, cudaStream_t s, uint32_t head_mask = 0xFFFFFFFFu);

// ---- heads_tc.cu: every Linear layer on the tensor cores (wgmma, fp16 hi/lo split operands, fp32 accumulate) ----
int oww_heads_tc_pack(oww_ctx* ctx, Head& h, const float* w1);
bool oww_heads_tc_supported(const oww_ctx* ctx, int head_id);
int oww_heads_tc_launch(oww_ctx* ctx, int head_id, const FeatSrc& src, int n, float* d_out, int out_stride,
                        int out_col0, int combine_max, cudaStream_t s, uint32_t head_mask = 0xFFFFFFFFu);
// ---- heads_grp.cu: streaming / bulk heads, A operand from the fp16 mirror of the feature rings ----
void oww_heads_grp_free(oww_ctx* ctx);
void oww_heads_grp_drop_mirror(oww_ctx* ctx);
void oww_feat16_invalidate(oww_ctx* ctx);        // rows were appended without oww_feat16_advance: rebuild at the next advance
int oww_feat16_advance(oww_ctx* ctx, int n_chunks, cudaStream_t s);
int oww_feat16_resync(oww_ctx* ctx, const int* d_ids, int n, cudaStream_t s);
uint32_t oww_heads_grp_covered(oww_ctx* ctx);
uint32_t oww_heads_grp_bulk(oww_ctx* ctx, const FeatSrc& src, int n, float* d_out, int out_stride, cudaStream_t s, int* rc_out);
int oww_heads_grp_launch(oww_ctx* ctx, int back, int n, float* d_out, int out_stride, int combine_max, cudaStream_t s);
// every head (tensor-core kernel where a head allows it, heads.cu otherwise) + the verifier gates
int oww_heads_all(oww_ctx* ctx, const FeatSrc& src, int n, float* d_out, int out_stride, int combine_max, cudaStream_t s);
