// Internal declarations shared by the .cu translation units of libowwb200.so.
#pragma once
#include <cuda_runtime.h>
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <string>
#include <utility>
#include <vector>
#include "owwb200.h"

// Exponent s of the fp16 weight packings (conv layers, head Linear layers): max |w| * 2^s in [2^13, 2^14), clamped to
// [-8, 24].  W * 2^s is packed and 2^-s folded exactly into the scale that follows, so the fp16 weights (and the lo
// parts of hi/lo splits) stay in the normal range whatever the scale of the weights.
// The rule on the largest magnitude alone, clamped to [lo, hi].  The tensor-core heads apply it per row to their hidden
// activations with [-100, 100], which keeps 2^e and every 2^-(s + e) they fold back normal fp32 numbers.
__host__ __device__ inline int oww_scale_exponent_of_max(float amax, int lo = -8, int hi = 24) {
    if (!(amax > 0.f) || !(amax <= 3.402823466e38f)) return 0;     // zero, inf or NaN
    int e;
    frexpf(amax, &e);                                              // amax = m * 2^e, m in [0.5, 1)
    e = 14 - e;
    return e < lo ? lo : (e > hi ? hi : e);
}
inline int oww_weight_scale_exponent(const float* w, size_t n) {
    float amax = 0.f;
    for (size_t i = 0; i < n; ++i) amax = std::fmax(amax, std::fabs(w[i]));
    return oww_scale_exponent_of_max(amax);
}

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
    int Wp, n_planes;
    int off;                 // unit offset of the tensor's [planes][2][Wp] rows in the late template (and a stream record)
    LateLay lay;             // block-major layout of now / next
};
// late[]: one entry per tails-bearing late tensor X_l, l >= split_from (5 at the default split, 9 at split_from 3)
// The carry of a held stream in a ragged step (api.cu, carry_kernel) fills the same tables with the stream's own state
// as the source: tmpl = the G-group tails buffer the launch read, ResetLate::tmpl = the late buffer it read (same
// layouts as tails / now).
struct ResetTails { uint4* tails; const uint4* tmpl; int G, tail_units, n_tab; int4 tab[OWW_N_CONV]; int n_late; ResetLate late[OWW_N_CONV]; };

// conditional verifier pair (hey_jarvis, docs/models/hey_jarvis.md:38): score column `main_col` is replaced by column
// `ver_col` wherever it exceeds `thr`
struct Gate { int main_col, ver_col; float thr; };

// custom verifier bank (verifier.cu): up to `capacity` speaker verifiers of one head, each the linear form of the
// reference's FunctionTransformer(flatten) -> StandardScaler -> LogisticRegression pipeline over the head's newest n_in
// feature rows (D = n_in*96):  p = 1 / (1 + exp(-(bias + sum_j (x_j - mean_j) * weight_j)))
struct VerifierBank {
    int head_id, col0, n_cols, n_in, capacity;
    int head_bank = -1;              // >= 0: the parent is this head bank (head_id = -1); a row whose bank slot is -1
                                     // (no model) is never verified
    float thr;                       // columns >= thr (fp32) are replaced by p
    float* d_mean = nullptr;         // [capacity][D]
    float* d_weight = nullptr;       // [capacity][D]
    float* d_bias = nullptr;         // [capacity]
    int* d_assign = nullptr;         // [n_streams] slot per stream, -1 = none
    int clip_slot = -1;              // slot oww_predict_clips applies to every clip
};

// wake-word head bank (heads_tc.cu): `capacity` slots that each hold a head of one shape, run by the tensor-core heads
// kernel.  Every stream picks a slot (-1: zeros in the bank's columns).  At assignment time the host sorts the streams by
// slot and cuts each slot's streams into work items of at most 64 (one CTA each).
struct HeadBank {
    Head shape;                      // desc, n_out, col0, the staging offsets of a pack_head_blob blob, tc_layers
    int capacity = 0;
    size_t w_bytes = 0;              // packed fp16 hi/lo weights of one slot (oww_heads_tc_pack's layout)
    size_t p_floats = 0;             // biases | LayerNorm parameters of one slot
    std::vector<int> p_off;          // per layer: offsets of bias, gamma, beta in a slot's parameters (3 per layer)
    uint8_t* d_w = nullptr;          // [capacity][w_bytes]
    float* d_p = nullptr;            // [capacity][p_floats]
    void* d_slots = nullptr;         // [capacity] kernel descriptors of the slots (heads_tc.cu)
    std::vector<uint8_t> h_slots;    // host copy of d_slots
    std::vector<uint8_t> loaded;     // per slot: a head has been loaded
    int clip_slot = -1;              // slot the bulk clip path applies to every clip
    // streams: host mirror of the assignment, and the item table the steps read ([B] int4 {slot, first, rows, 0} |
    // [B] stream ids ordered by slot | [B] slot per stream, read by the bank's verifiers), staged through pinned memory
    std::vector<int> assign;
    int n_items = 0;
    int* d_table = nullptr;
    int* h_stage = nullptr;
    cudaEvent_t stage_ev = nullptr;
};

// Ring row counters (rows ever written; ring slot = count & (rows-1)) would overflow int32 after ~248 days of
// continuous streaming at 100 mel rows/s.  Past 2^30 they are rebased by a multiple of every ring size (rings are
// powers of two <= 2^20 rows: oww_create refuses max_chunks above OWW_MAX_CHUNKS), which keeps the slot and leaves the count >= the ring size, so "row not yet written"
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
    std::vector<HeadBank> head_banks;  // per-stream head banks: their columns are counted in n_out_total
    int n_out_total = 0;
    int max_n_in = 0;
    std::vector<Gate> gates;         // applied to every chunk's scores before the max over chunks
    Gate* d_gates = nullptr;
    float* d_scores_tmp = nullptr;   // [n_streams][n_out_total]: one chunk's raw scores when gates meet a multi-chunk call
    size_t scores_tmp_floats = 0;
    std::vector<VerifierBank> banks; // custom verifiers, applied after the heads (and gates, and the max over chunks)
    int* d_assign_stage = nullptr;   // [2][n_streams] staging of oww_assign_verifier (ids | slots)
    bool verifiers_on = true;        // oww_enable_verifiers: steps and clip calls enqueued while false skip the banks
    cudaEvent_t ver_ev[2] = {nullptr, nullptr};   // orders oww_assign_verifier / oww_load_verifiers with own_stream
    // verifier training (verifier_fit.cu): float64 scratch (per-CTA vectors | per-sample arrays), staged sample offsets,
    // staged slots of oww_load_verifiers; grown on demand
    double* d_fit_scratch = nullptr;
    size_t fit_scratch_doubles = 0;
    int64_t* d_fit_off = nullptr;
    size_t fit_off_cap = 0;
    int* d_load_slots = nullptr;
    size_t load_slots_cap = 0;
    bool fit_attr_set = false;

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
    // [tails | new rows], fp16 hi/lo, in the block-major layout of tc_conv_blk_kernel (LateLay)
    struct LateTensor { void* buf[3] = {nullptr, nullptr, nullptr}; int n_buf = 0, rows_new = 0, W = 0, cg = 0, tmpl_off = -1;
                        LateLay lay = {0, 0, 0, 0, 0, 0}; };
    LateTensor late_x[OWW_N_CONV];
    void* d_late_tmp = nullptr;                  // unpooled output of a late layer that is followed by a separate pool
    void* d_late_template = nullptr;             // tails of the all-ones window per tails-bearing late tensor: [plane][2][Wp]
    bool late_active = false;
    bool late_pdl = true;                        // programmatic dependent launches inside the late chain (reserved[0] bit 5 disables)
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

    // stream records (oww_export_streams / oww_import_streams): configuration key inputs, id staging, rejection count
    uint64_t mel_key = 0, emb_key = 0;           // hashes of the mel constants / embedding blob last loaded
    int* d_state_ids = nullptr;                  // [n_streams]
    int* d_state_rejected = nullptr;             // records an import skipped since oww_stream_state_status last read it
    cudaEvent_t state_ev[2] = {nullptr, nullptr};   // orders the calls with own_stream
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
    std::vector<int32_t> slot_chunks[2];   // per host slot: the ragged counts of its step (empty: every row stepped)
    // orders a call enqueued on the caller's stream with the host-buffer calls on own_stream (oww_order_begin / _end)
    cudaEvent_t order_ev[2] = {nullptr, nullptr};

    // host staging of oww_detect_host_submit / _collect: two slots, like the step's.  Each keeps its ticket's device
    // buffers, the delivery buffer the device writes through a mapped pointer, and what the collect hands out.
    struct DetectSlot {
        int16_t* h_pkt = nullptr; int16_t* d_pkt = nullptr; size_t pkt_samples = 0;   // pinned staging | device packets
        float* d_scores = nullptr; size_t scores_floats = 0;                           // [B][n_out]
        float* d_final = nullptr; size_t final_floats = 0;                             // [B][n_labels]
        uint8_t* d_out = nullptr; size_t d_out_bytes = 0;            // count | events | ends | clips (oww_detect_layout)
        uint8_t* h_out = nullptr; uint8_t* h_out_dev = nullptr; size_t h_out_bytes = 0;   // mapped: the same | final
        std::vector<int64_t> offsets;                                // the call's offsets, rebased to the staged span
        std::vector<int32_t> chunks, prepared;                       // oww_ingest's, filled at submit
        int n_streams = 0, n_labels = 0, max_events = 0, capture = 0, want_final = 0;
        uint64_t seq = 0;                                            // submission order
        cudaEvent_t h2d_done = nullptr, done = nullptr;
        bool busy = false;
    } det_slot[2];
    int det_next = 0;
    uint64_t det_seq = 0;

    // ragged steps (oww_step_ragged): per call [B counts | B stream ids ordered by count], staged through a ring of
    // pinned buffers (a slot is reused once the copy of the call kRagSlots calls back has run)
    static constexpr int kRagSlots = 4;
    int32_t* h_rag[kRagSlots] = {nullptr, nullptr, nullptr, nullptr};
    int32_t* d_rag[kRagSlots] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t rag_ev[kRagSlots] = {nullptr, nullptr, nullptr, nullptr};
    int rag_next = 0, rag_streams = 0;
    float* d_rag_scores = nullptr;   // [max_chunks][n_streams][n_out_total]: per chunk window, before the masked max
    size_t rag_scores_floats = 0;

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
    struct oww_detector* det = nullptr;   // detections on the device (detect.cu); nullptr: no detector configured
    struct oww_audio* audio = nullptr;    // the streams' recent audio (audio.cu); nullptr: no history
    struct oww_ingest_state* ingest = nullptr;  // resampling and staging of packets at any rate (ingest.cu); nullptr: off
    struct oww_clip_resampler* clip_rs = nullptr;  // taps and tile tables of oww_resample_clips (ingest.cu); nullptr: unused
    struct oww_mixer* mixer = nullptr;    // tables and scratch of oww_mix_clips (mix.cu); nullptr: unused
};

int oww_fail(oww_ctx* ctx, int code, const char* fmt, ...);
// api.cu: a call enqueued on `s` that reads or writes state the host-buffer calls use on the handle's own stream runs
// after everything submitted there so far (begin, before its first device work) and before everything submitted later
// (end, after its last).  Both do nothing when s is the own stream.
int oww_order_begin(oww_ctx* ctx, cudaStream_t s);
int oww_order_end(oww_ctx* ctx, cudaStream_t s);
void oww_verifier_fit_free(oww_ctx* ctx);          // verifier_fit.cu: the training scratch
void oww_mix_free(oww_ctx* ctx);                   // mix.cu: the mixer's tables and scratch
// 64-bit FNV-1a of `bytes` bytes, continuing from h (the stream record's configuration key)
inline uint64_t oww_fnv1a(const void* p, size_t bytes, uint64_t h = 14695981039346656037ull) {
    const unsigned char* c = static_cast<const unsigned char*>(p);
    for (size_t i = 0; i < bytes; ++i) h = (h ^ c[i]) * 1099511628211ull;
    return h;
}
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

// ---- call schedule of the bulk clip path ----
// predict_clip(clip, chunk_size = c) makes len(range(0, L - c, c)) calls of c samples on the L padded samples, and
// AudioFeatures._streaming_features steps whole 1280-sample chunks only, keeping the remainder for the next call: after
// calls 0 .. j - 1, floor(j c / 1280) chunks have been stepped.  oww_clip_schedule (api.cu) exports these for the host.
#ifdef __CUDACC__
#define OWW_HD __host__ __device__ __forceinline__
#else
#define OWW_HD inline
#endif
OWW_HD int64_t oww_clip_calls(int64_t L, int c) { return L > c ? (L - 1) / c : 0; }
OWW_HD int64_t oww_call_first_step(int64_t j, int c) { return j * c / OWW_SAMPLES_PER_CHUNK; }
// the call that steps chunk s: the first j with (j + 1) c >= 1280 (s + 1)
OWW_HD int64_t oww_call_of_step(int64_t s, int c) { return ((int64_t)OWW_SAMPLES_PER_CHUNK * (s + 1) + c - 1) / c - 1; }

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
    const int* live = nullptr;     // ragged step: stream b takes part iff live[b] >= live_min (otherwise no write at all)
    int live_min = 0;
    bool pdl = false;              // dependent launch: the kernel waits for its predecessor only before its first store
};
int oww_mel_launch(oww_ctx* ctx, const MelLaunch& p, cudaStream_t s);
// bulk path: mel rows of whole padded clips, grouped and clamped per streaming call of `chunk` samples, behind 71 rows of
// ones - the virtual history a fully convolutional CNN pass reproduces predict_clip from.  Clip i is the d_len[i] samples
// at d_pcm + d_off[i], with `pad` virtual zeros on each side and virtual zeros after that.  Steps [k0, k1) (at most 8192;
// k1 on a call boundary) write its rows [8 k0, 76 + 8 (k1 - 1)) to d_out [n_clips][76 + 8 (k1 - k0 - 1)][32].
int oww_mel_clips_launch(oww_ctx* ctx, const int16_t* d_pcm, const int64_t* d_off, const int* d_len, int n_clips, int pad,
                         int chunk, int k0, int k1, float* d_out, int64_t out_stride, cudaStream_t s);

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
// appends n_chunks embedding rows per stream; ids != nullptr: only the n_ids streams listed (d_emb rows are compact)
int oww_feat_append(oww_ctx* ctx, const float* d_emb, int n_chunks, cudaStream_t s, const int* d_ids = nullptr, int n_ids = 0);
// mode dispatch (fp32 window / tensor-core window) with sub-batching over ctx->window_batch
int oww_cnn_window(oww_ctx* ctx, const WindowSrc& src, int n_windows, float* d_emb, cudaStream_t s, bool capture_tails = false);
// fp32 pyramid, same contract as oww_cnn_tc_pyramid (cnn_tc.cu)
int oww_cnn_fp32_pyramid(oww_ctx* ctx, const WindowSrc& src, int n, int T0, float* d_emb, int out_rows, int stop_layer,
                         float* d_dbg, cudaStream_t s);

// ---- cnn_tc.cu ----
int oww_tc_pack_weights(oww_ctx* ctx, const float* h_blob);
size_t oww_tc_act_units(const oww_ctx* ctx, int n_windows);
size_t oww_tc_act_units_T(const oww_ctx* ctx, int n, int T0);
// incremental late layers of mode 3 (split operands)
int oww_late_alloc(oww_ctx* ctx);
int oww_late_chain(oww_ctx* ctx, float* d_emb, cudaStream_t s);
int oww_late_capture(oww_ctx* ctx, int next_layer, const void* planes, int64_t plane_pitch, int T, int W, cudaStream_t s);
// Pyramid over n inputs of T0 mel rows each (n windows of 76 rows, or clips: the CNN is fully convolutional in time,
// SURVEY.md F10): the embeddings of input i land at d_emb + i * out_rows * 96, rows 0 .. (T0 - 76) / 8.  stop_layer >= 0:
// stop after that layer (and its pool) and leave it as NHWC fp32 [n][T][W][C] in d_dbg.
int oww_cnn_tc_pyramid(oww_ctx* ctx, const WindowSrc& src, int n, int T0, float* d_emb, int out_rows, int stop_layer,
                       float* d_dbg, cudaStream_t s);
// capture descriptor: which local windows of a full-window pass are the newest window of which streams
struct TailCapture { int win0, n_win, stream0; const int* ids = nullptr; bool late = false; };   // ids: local stream -> stream id;
                                                                  // late: window 0 is the template window of the incremental late layers
int oww_cnn_tc_pyramid_cap(oww_ctx* ctx, const WindowSrc& src, int n, float* d_emb, const TailCapture* cap, cudaStream_t s);

// ---- cnn_tc_inc.cu ----
int oww_inc_build_plan(oww_ctx* ctx, int G, int n_streams, int n_layers, IncPlan* out);
int oww_inc_n_layers(const oww_ctx* ctx);
int oww_inc_setup(oww_ctx* ctx, const float* h_blob);
int oww_inc_alloc_streams(oww_ctx* ctx);
// d_chunks != nullptr (ragged step): only the streams with d_chunks[b] >= min_chunks step in this launch; the others are
// dead slots whose tails state the caller carries (api.cu, carry_kernel)
int oww_cnn_inc_step(oww_ctx* ctx, int back, float* d_emb, cudaStream_t s, const int* d_chunks = nullptr, int min_chunks = 0);
// whole step in one launch (n_chunks == 1, primed): PCM -> mel -> CNN -> ring append -> heads -> scores
bool oww_fused_frontend_supported(const oww_ctx* ctx);
bool oww_fused_heads_supported(const oww_ctx* ctx);
int oww_fused_step(oww_ctx* ctx, const int16_t* d_pcm, int64_t pcm_stride, float* d_scores, int out_stride, bool with_heads,
                   cudaStream_t s, const int* d_chunks = nullptr, int min_chunks = 0);
int oww_heads_sync_devs(oww_ctx* ctx);
int oww_inc_capture(oww_ctx* ctx, int layer, const void* planes, int64_t plane_pitch, int T, int W, int win0, int n_win,
                    int stream0, const int* d_ids, cudaStream_t s);

// ---- heads.cu ----
struct FeatSrc {
    const float* base; int64_t stride;   // per-sample stride in floats
    const int* count; int rows_mask;     // ring addressing (nullptr -> linear [n][n_in][96])
    int back;                            // ring: window ends `back` rows before the newest
    // sliding mode (count == nullptr, steps > 0; bulk clips): sample s = clip * steps + st reads rows
    // [row0 + st + 1 - n_in, row0 + st] of clip's linear rows at base + clip * stride (negative rows read as zeros)
    int steps = 0, row0 = 0;
    const int* idx = nullptr;            // sliding mode: sample s reads the window of sliding sample idx[s] (call rows)
};
#ifdef __CUDACC__
// Where sample s's window of n_in rows starts: feature row c of the window is row r0 + c of `base` (ring: slot
// (r0 + c) & mask; linear: mask = -1).  Rows below 0 were never written and read as zeros.
struct FeatRows { const float* base; int r0, mask; };
__device__ __forceinline__ FeatRows feat_rows(const FeatSrc& src, int n_in, int s) {
    if (src.count) return FeatRows{src.base + (int64_t)s * src.stride, src.count[s] - src.back - n_in, src.rows_mask};
    if (src.steps > 0) {
        const int q = src.idx ? src.idx[s] : s;
        const int clip = q / src.steps, st = q - clip * src.steps;
        return FeatRows{src.base + (int64_t)clip * src.stride, src.row0 + st + 1 - n_in, -1};
    }
    return FeatRows{src.base + (int64_t)s * src.stride, 0, -1};
}
// feature row c of the window, or nullptr where it reads as zeros
__device__ __forceinline__ const float* feat_row(const FeatRows& w, int c) {
    const int r = w.r0 + c;
    return r < 0 ? nullptr : w.base + (int64_t)(w.mask >= 0 ? (r & w.mask) : r) * 96;
}
#endif
// head_id < 0: every head whose bit is set in head_mask (blockIdx.y walks the selected heads)
int oww_heads_launch(oww_ctx* ctx, int head_id, const FeatSrc& src, int n, float* d_out, int out_stride,
                     int out_col0, int combine_max, cudaStream_t s, uint32_t head_mask = 0xFFFFFFFFu);

// ---- api.cu: a head blob (weights.py:pack_head_blob) in the device layout: tensors on 16-byte boundaries ----
int oww_check_head_desc(oww_ctx* ctx, const oww_head_desc* desc);
// fills h.desc and h.w_off / b_off / g_off / h_off; staged = the blob at those offsets
int oww_stage_head(oww_ctx* ctx, const oww_head_desc* desc, const float* h_blob, size_t n_floats, Head& h,
                   std::vector<float>& staged);

// ---- heads_tc.cu: every Linear layer on the tensor cores (wgmma, fp16 hi/lo split operands, fp32 accumulate) ----
int oww_heads_tc_pack(oww_ctx* ctx, Head& h, const float* w1);
// per head bank, an item table over rows of the bulk path: CTA i runs items[i] = {slot, first, rows, 0} on the rows
// perm[first .. first + rows) (row = FeatSrc sample = output row)
struct BankRows { const int4* items; const int* perm; int n_items; };
// every head bank on n rows: streams of the handle (src = the feature ring, n = n_streams: each stream's slot) or rows
// of the bulk path (rows[i] != nullptr: head bank i's item table; otherwise the clip slot).  d_step != nullptr (ragged
// step): streams with d_step[b] == 0 are not written.
int oww_head_banks_launch(oww_ctx* ctx, const FeatSrc& src, int n, float* d_out, int out_stride, int combine_max,
                          cudaStream_t s, const int* d_step = nullptr, const BankRows* rows = nullptr);
// head bank `bank`'s slot of every stream on the device ([n_streams], -1 = none), uploaded with its item table
const int* oww_head_bank_stream_slots(const oww_ctx* ctx, int bank);
// (re)allocate every bank's per-stream table for ctx->n_streams streams, every stream on slot -1 (synchronous)
int oww_head_banks_alloc_streams(oww_ctx* ctx);
void oww_head_banks_free(oww_ctx* ctx);
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
// every head (tensor-core kernel where a head allows it, heads.cu otherwise) + the verifier gates; bank_rows: as in
// oww_head_banks_launch
int oww_heads_all(oww_ctx* ctx, const FeatSrc& src, int n, float* d_out, int out_stride, int combine_max, cudaStream_t s,
                  const BankRows* bank_rows = nullptr);

// ---- detect.cu: the detector's per-stream prediction history (nothing happens on a handle without a detector) ----
void oww_detect_free(oww_ctx* ctx);
void oww_detect_free_streams(oww_ctx* ctx);
int oww_detect_alloc_streams(oww_ctx* ctx);      // for ctx->n_streams streams, every history empty; the device is idle
// the listed streams (d_ids == nullptr: streams 0..n-1) start afresh: one launch on `s`
int oww_detect_reset(oww_ctx* ctx, const int* d_ids, int n, cudaStream_t s);
int oww_detect_n_labels(const oww_ctx* ctx);      // labels of the detector; 0 without one (or without streams)
// Byte offsets of one delivery buffer of oww_detect_host_submit for max_events events of `capture` samples: the count
// (int32) at 0, then events, ends and clip rows, each on a 16-byte boundary; `final` is where a host buffer keeps the
// final predictions, `bytes` its size.  A device buffer ends at `final`.
struct DetectLayout { size_t events, ends, clips, final, bytes; };
DetectLayout oww_detect_layout(int max_events, int capture, int n_streams, int n_labels);
// one launch on `s`: the count d_out (layout above) holds, the first min(count, max_events) events and with capture > 0
// their ends and clip rows -> the same places of h_out (a device pointer to mapped host memory)
int oww_detect_deliver(oww_ctx* ctx, const uint8_t* d_out, uint8_t* h_out, int max_events, int capture, cudaStream_t s);

// ---- audio.cu: the streams' recent audio (nothing happens on a handle without history) ----
void oww_audio_free(oww_ctx* ctx);
void oww_audio_free_streams(oww_ctx* ctx);
int oww_audio_alloc_streams(oww_ctx* ctx);       // for ctx->n_streams streams, every history empty; the device is idle
// the listed streams (d_ids == nullptr: streams 0..n-1) start with an empty history: one launch on `s`
int oww_audio_reset(oww_ctx* ctx, const int* d_ids, int n, cudaStream_t s);
int oww_audio_history_samples(const oww_ctx* ctx);   // H; 0 without history (or without streams)
// one launch on `s`: stream b appends the first cnt * 1280 samples of its row, cnt = d_counts[b] (device; nullptr:
// n_chunks for every stream)
int oww_audio_append(oww_ctx* ctx, const int16_t* d_pcm, int64_t pcm_stride, int n_chunks, const int* d_counts,
                     cudaStream_t s);

// ---- ingest.cu: packets at any rate (nothing happens on a handle without ingest state) ----
void oww_ingest_free(oww_ctx* ctx);              // the ingest state and the clip resampler's buffers
void oww_ingest_free_streams(oww_ctx* ctx);
int oww_ingest_alloc_streams(oww_ctx* ctx);      // for ctx->n_streams streams, every one at 16000, nothing staged
// the listed streams (h_ids == nullptr: streams 0..n-1) drop their staged samples and history: host state only
void oww_ingest_reset(oww_ctx* ctx, const int32_t* h_ids, int n);
// what oww_ingest refuses before it enqueues anything (no ingest state, weights, offsets, a packet over its stream's
// capacity), checked without enqueueing
int oww_ingest_check(oww_ctx* ctx, const int64_t* h_offsets);

// ---- verifier.cu: custom verifier banks ----
// every bank of the handle on n rows of final scores (one launch; nothing when the handle has no bank).  The window of
// row r is the newest n_in rows of `src` (FeatSrc sample r).  Its slot is bank.d_assign[r] for streams (rows = streams
// of the handle), or bank.clip_slot for clips (rows = (clip, step) of the bulk path).  d_clip_streams != nullptr
// (clips): row r takes the slots of stream d_clip_streams[q / src.steps], q = its sliding sample (src.idx[r] or r).
// d_chunks != nullptr (ragged step): rows with d_chunks[r] == 0 did not step and are skipped.
int oww_verifiers_apply(oww_ctx* ctx, const FeatSrc& src, int n, float* d_scores, int out_stride, bool clips,
                        cudaStream_t s, const int* d_chunks = nullptr, const int* d_clip_streams = nullptr);
// (re)allocate every bank's per-stream assignment for ctx->n_streams streams, all -1
int oww_verifiers_alloc_streams(oww_ctx* ctx);
// true when oww_verifiers_apply(..., clips = true, d_clip_streams given or not) would launch
bool oww_verifiers_clip_active(const oww_ctx* ctx, bool clip_streams = false);
void oww_verifiers_free_streams(oww_ctx* ctx);
