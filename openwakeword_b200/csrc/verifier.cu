// K3b: custom verifier models (openwakeword/model.py:319-328, openwakeword/custom_verifier_model.py:91-113 of the
// original project).  A verifier is a speaker-specific logistic regression trained on the head's input features; where a
// score of its parent head reaches the threshold, P(positive) of the verifier on the newest window replaces that score.
// The host reduces the reference's pipeline FunctionTransformer(flatten) -> StandardScaler -> LogisticRegression to
//   p = 1 / (1 + exp(-(b + sum_j (x_j - mu_j) * w_j)))     mu = mean_, w = coef_ / scale_, b = intercept_
// and keeps the centred form: with a small scale_ the folded bias b - sum mu_j w_j cancels catastrophically in fp32.
//
// The parent is an ordinary head (oww_add_verifier_bank) or a per-stream head bank (oww_add_bank_verifier_bank).  A row
// whose head-bank slot is -1 has no model: its columns stay 0.0 and it is never verified, whatever the threshold.
//
// One warp per row (a stream, a (clip, step) of the bulk path, or a window of the stateless call) and bank.  The warp
// reads the row's slot and the parent's score columns and leaves when no column reaches the threshold, so a step in
// which nothing fires costs one slot and one score read per stream.  Otherwise it streams the D = n_in*96 features, mu
// and w with 16-byte loads (lane l takes float4 l, l+32, ...), accumulates in fp32 and reduces with a fixed xor-shuffle
// tree: the order depends only on D, so the bulk path, streaming and the stateless entry agree bit for bit.
#include "oww_internal.h"
#include <cmath>

namespace {

constexpr int kVerMaxHeadBanks = 16;    // banks of ordinary heads: one per parent head, at most 16 heads per handle
constexpr int kVerMaxBankBanks = 16;    // banks of head banks: one per head bank
constexpr int kVerMaxBanks = kVerMaxHeadBanks + kVerMaxBankBanks;   // 32 x 64 B (VerBankDev) = 2 KB of kernel parameters
constexpr int kVerWarps = 8;

struct VerBankDev {
    const float* mean; const float* weight; const float* bias;
    const int* assign;                  // per-stream slot, or nullptr: every row uses slot_all
    const int* hslot;                   // parent head bank: its slot per stream (rows on -1 are not verified), or nullptr
    int slot_all, col0, n_cols, n_in;
    float thr;
};
struct VerArgs {
    VerBankDev bank[kVerMaxBanks];
    FeatSrc src;
    int n; float* out; int out_stride;
    int gated;                          // 0: stateless call, write p to column col0 of every row unconditionally
    const int* step;                    // ragged step: rows with step[r] == 0 were held (their score row is not written)
    const int* clip_streams;            // bulk rows: stream of each slab-local clip (its slots apply), or nullptr
};

__global__ void __launch_bounds__(kVerWarps * 32) verifier_kernel(const __grid_constant__ VerArgs a) {
    oww_pdl_sync();
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * kVerWarps + (threadIdx.x >> 5);
    if (r >= a.n || (a.step && a.step[r] == 0)) return;
    const VerBankDev& B = a.bank[blockIdx.y];
    int b = r;                          // the stream whose slots row r takes
    if (a.clip_streams) b = a.clip_streams[(a.src.idx ? a.src.idx[r] : r) / a.src.steps];
    if (B.hslot && B.hslot[b] < 0) return;
    const int slot = B.assign ? B.assign[b] : B.slot_all;
    if (slot < 0) return;
    float* o = a.out + (int64_t)r * a.out_stride + B.col0;
    uint32_t mine = 0;                  // bit k: column 32k + lane reaches the threshold
    if (a.gated) {
        for (int k = 0; 32 * k < B.n_cols; ++k) {
            const int c = 32 * k + lane;
            if (c < B.n_cols && o[c] >= B.thr) mine |= 1u << k;
        }
        if (!__any_sync(0xffffffffu, mine != 0)) return;
    } else {
        mine = lane == 0 ? 1u : 0u;
    }
    const int n_in = B.n_in;
    const FeatRows win = feat_rows(a.src, n_in, r);
    const int64_t D = (int64_t)n_in * 96;
    const float4* mu = reinterpret_cast<const float4*>(B.mean + slot * D);
    const float4* w = reinterpret_cast<const float4*>(B.weight + slot * D);
    float acc = 0.f;
    for (int j = lane; j < n_in * 24; j += 32) {
        const int row = j / 24, c4 = j - row * 24;
        const float* p = feat_row(win, row);
        float4 x = make_float4(0.f, 0.f, 0.f, 0.f);         // rows before the stream's first: zeros, as the heads read them
        if (p) x = reinterpret_cast<const float4*>(p)[c4];
        const float4 m = __ldg(mu + j), v = __ldg(w + j);
        acc = fmaf(x.x - m.x, v.x, acc);
        acc = fmaf(x.y - m.y, v.y, acc);
        acc = fmaf(x.z - m.z, v.z, acc);
        acc = fmaf(x.w - m.w, v.w, acc);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    const float p = 1.0f / (1.0f + expf(-(__ldg(B.bias + slot) + acc)));
    for (int k = 0; mine >> k; ++k)
        if (mine >> k & 1u) o[32 * k + lane] = p;
}

__global__ void assign_kernel(const int* ids, const int* slots, int n, int* assign) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) assign[ids ? ids[i] : i] = slots[i];
}

int launch(oww_ctx* ctx, const VerArgs& a, int n_banks, cudaStream_t s) {
    if (n_banks == 0 || a.n <= 0) return OWW_OK;
    OWW_CUDA(ctx, oww_launch_pdl(ctx->late_pdl, verifier_kernel, dim3((a.n + kVerWarps - 1) / kVerWarps, n_banks),
                                 dim3(kVerWarps * 32), 0, s, a));
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

VerBankDev bank_dev(const VerifierBank& b, int slot_all, const int* assign, const int* hslot) {
    return VerBankDev{b.d_mean, b.d_weight, b.d_bias, assign, hslot, slot_all, b.col0, b.n_cols, b.n_in, b.thr};
}

// the one-clip-slot bulk path: the bank's clip slot verifies, under a model (a head bank's clip slot is not -1)
bool clip_slot_on(const oww_ctx* ctx, const VerifierBank& b) {
    return b.clip_slot >= 0 && (b.head_bank < 0 || ctx->head_banks[b.head_bank].clip_slot >= 0);
}

}  // namespace

int oww_verifiers_apply(oww_ctx* ctx, const FeatSrc& src, int n, float* d_scores, int out_stride, bool clips,
                        cudaStream_t s, const int* d_chunks, const int* d_clip_streams) {
    if (ctx->banks.empty() || !ctx->verifiers_on) return OWW_OK;
    VerArgs a;
    a.step = d_chunks;
    a.clip_streams = clips ? d_clip_streams : nullptr;
    const bool per_stream = !clips || d_clip_streams;
    int nb = 0;
    for (const VerifierBank& b : ctx->banks) {
        if (!per_stream && !clip_slot_on(ctx, b)) continue;   // no clip verifier for this head
        const int* hslot = per_stream && b.head_bank >= 0 ? oww_head_bank_stream_slots(ctx, b.head_bank) : nullptr;
        a.bank[nb++] = bank_dev(b, b.clip_slot, per_stream ? b.d_assign : nullptr, hslot);
    }
    a.src = src; a.n = n; a.out = d_scores; a.out_stride = out_stride; a.gated = 1;
    return launch(ctx, a, nb, s);
}

bool oww_verifiers_clip_active(const oww_ctx* ctx, bool clip_streams) {
    if (!ctx->verifiers_on) return false;
    for (const VerifierBank& b : ctx->banks)
        if (clip_streams || clip_slot_on(ctx, b)) return true;
    return false;
}

int oww_verifiers_alloc_streams(oww_ctx* ctx) {
    oww_verifiers_free_streams(ctx);
    if (ctx->banks.empty() || ctx->n_streams <= 0) return OWW_OK;
    const size_t bytes = (size_t)ctx->n_streams * sizeof(int);
    OWW_CUDA(ctx, cudaMalloc(&ctx->d_assign_stage, 2 * bytes));
    for (VerifierBank& b : ctx->banks) {
        OWW_CUDA(ctx, cudaMalloc(&b.d_assign, bytes));
        OWW_CUDA(ctx, cudaMemset(b.d_assign, 0xFF, bytes));          // -1: no verifier
    }
    return OWW_OK;
}

void oww_verifiers_free_streams(oww_ctx* ctx) {
    for (VerifierBank& b : ctx->banks) { cudaFree(b.d_assign); b.d_assign = nullptr; }
    cudaFree(ctx->d_assign_stage); ctx->d_assign_stage = nullptr;
}

namespace {

// allocate bank b (its parent, columns, n_in, capacity and threshold set) and append it
int add_bank(oww_ctx* ctx, VerifierBank b, int* bank_id) {
    const int capacity = b.capacity;
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t D = (size_t)b.n_in * 96;
    auto fail = [&](cudaError_t e) {
        cudaFree(b.d_mean); cudaFree(b.d_weight); cudaFree(b.d_bias); cudaFree(b.d_assign);
        return oww_fail(ctx, OWW_ENOMEM, "verifier bank of %d slots: %s", capacity, cudaGetErrorString(e));
    };
    cudaError_t e;
    if ((e = cudaMalloc(&b.d_mean, (size_t)capacity * D * sizeof(float))) != cudaSuccess) return fail(e);
    if ((e = cudaMalloc(&b.d_weight, (size_t)capacity * D * sizeof(float))) != cudaSuccess) return fail(e);
    if ((e = cudaMalloc(&b.d_bias, (size_t)capacity * sizeof(float))) != cudaSuccess) return fail(e);
    if (ctx->n_streams > 0) {
        const size_t bytes = (size_t)ctx->n_streams * sizeof(int);
        if ((e = cudaMalloc(&b.d_assign, bytes)) != cudaSuccess) return fail(e);
        if ((e = cudaMemset(b.d_assign, 0xFF, bytes)) != cudaSuccess) return fail(e);
        if (!ctx->d_assign_stage && (e = cudaMalloc(&ctx->d_assign_stage, 2 * bytes)) != cudaSuccess) return fail(e);
    }
    for (auto& ev : ctx->ver_ev)
        if (!ev && (e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)) != cudaSuccess) return fail(e);
    ctx->banks.push_back(b);
    if (bank_id) *bank_id = (int)ctx->banks.size() - 1;
    return OWW_OK;
}

int count_banks(const oww_ctx* ctx, bool of_head_banks) {
    int n = 0;
    for (const VerifierBank& o : ctx->banks) n += (o.head_bank >= 0) == of_head_banks;
    return n;
}

}  // namespace

extern "C" {

int oww_add_verifier_bank(oww_ctx* ctx, int head_id, int capacity, float threshold, int* bank_id) {
    if (!ctx) return OWW_EINVAL;
    if (head_id < 0 || head_id >= (int)ctx->heads.size()) return oww_fail(ctx, OWW_EINVAL, "bad head_id %d", head_id);
    if (capacity < 1 || capacity > (1 << 20)) return oww_fail(ctx, OWW_EINVAL, "capacity %d outside [1, 2^20]", capacity);
    if (count_banks(ctx, false) >= kVerMaxHeadBanks)
        return oww_fail(ctx, OWW_EUNSUPPORTED, "at most %d verifier banks per handle", kVerMaxHeadBanks);
    for (const VerifierBank& o : ctx->banks)     // two banks would write the same score columns in one launch
        if (o.head_id == head_id) return oww_fail(ctx, OWW_EINVAL, "head %d already has a verifier bank", head_id);
    const Head& h = ctx->heads[head_id];
    VerifierBank b;
    b.head_id = head_id; b.col0 = h.col0; b.n_cols = h.n_out; b.n_in = h.desc.n_in; b.capacity = capacity; b.thr = threshold;
    return add_bank(ctx, b, bank_id);
}

int oww_add_bank_verifier_bank(oww_ctx* ctx, int head_bank, int capacity, float threshold, int* bank_id) {
    if (!ctx) return OWW_EINVAL;
    if (head_bank < 0 || head_bank >= (int)ctx->head_banks.size())
        return oww_fail(ctx, OWW_EINVAL, "bad head bank %d", head_bank);
    if (capacity < 1 || capacity > (1 << 20)) return oww_fail(ctx, OWW_EINVAL, "capacity %d outside [1, 2^20]", capacity);
    if (count_banks(ctx, true) >= kVerMaxBankBanks)
        return oww_fail(ctx, OWW_EUNSUPPORTED, "at most %d verifier banks of head banks per handle", kVerMaxBankBanks);
    for (const VerifierBank& o : ctx->banks)
        if (o.head_bank == head_bank) return oww_fail(ctx, OWW_EINVAL, "head bank %d already has a verifier bank", head_bank);
    const HeadBank& h = ctx->head_banks[head_bank];
    VerifierBank b;
    b.head_id = -1; b.head_bank = head_bank;
    b.col0 = h.shape.col0; b.n_cols = h.shape.n_out; b.n_in = h.shape.desc.n_in; b.capacity = capacity; b.thr = threshold;
    return add_bank(ctx, b, bank_id);
}

int oww_load_verifier(oww_ctx* ctx, int bank, int slot, const float* h_mean, const float* h_weight, float bias) {
    if (!ctx || !h_mean || !h_weight) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (bank < 0 || bank >= (int)ctx->banks.size()) return oww_fail(ctx, OWW_EINVAL, "bad verifier bank %d", bank);
    const VerifierBank& b = ctx->banks[bank];
    if (slot < 0 || slot >= b.capacity) return oww_fail(ctx, OWW_EINVAL, "slot %d outside [0,%d)", slot, b.capacity);
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    OWW_CUDA(ctx, cudaDeviceSynchronize());           // steps in flight on any stream finish with the old contents
    const size_t D = (size_t)b.n_in * 96;
    OWW_CUDA(ctx, cudaMemcpy(b.d_mean + slot * D, h_mean, D * sizeof(float), cudaMemcpyHostToDevice));
    OWW_CUDA(ctx, cudaMemcpy(b.d_weight + slot * D, h_weight, D * sizeof(float), cudaMemcpyHostToDevice));
    OWW_CUDA(ctx, cudaMemcpy(b.d_bias + slot, &bias, sizeof(float), cudaMemcpyHostToDevice));
    return OWW_OK;
}

int oww_assign_verifier(oww_ctx* ctx, int bank, const int32_t* h_stream_ids, int n, const int32_t* h_slots, void* stream) {
    if (!ctx || !h_slots) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (bank < 0 || bank >= (int)ctx->banks.size()) return oww_fail(ctx, OWW_EINVAL, "bad verifier bank %d", bank);
    if (ctx->n_streams <= 0) return oww_fail(ctx, OWW_EINVAL, "oww_set_streams has not been called");
    const VerifierBank& b = ctx->banks[bank];
    if (!h_stream_ids) n = ctx->n_streams;
    if (n <= 0) return OWW_OK;
    if (n > ctx->n_streams) return oww_fail(ctx, OWW_EINVAL, "more stream ids (%d) than streams (%d)", n, ctx->n_streams);
    for (int i = 0; i < n; ++i) {
        if (h_stream_ids && (h_stream_ids[i] < 0 || h_stream_ids[i] >= ctx->n_streams))
            return oww_fail(ctx, OWW_EINVAL, "stream id %d out of range", h_stream_ids[i]);
        if (h_slots[i] < -1 || h_slots[i] >= b.capacity)
            return oww_fail(ctx, OWW_EINVAL, "slot %d outside [-1,%d)", h_slots[i], b.capacity);
    }
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    int* d_ids = ctx->d_assign_stage;
    int* d_slots = ctx->d_assign_stage + ctx->n_streams;
    // the host-buffer steps (oww_step_host / _submit) run on the handle's own non-blocking stream: order the assignment
    // after the steps already submitted there and before the ones submitted later, as on `stream` itself
    const bool other = s != ctx->own_stream;
    if (other) {
        OWW_CUDA(ctx, cudaEventRecord(ctx->ver_ev[0], ctx->own_stream));
        OWW_CUDA(ctx, cudaStreamWaitEvent(s, ctx->ver_ev[0], 0));
    }
    // pageable sources: staged by the driver before the call returns; stream-ordered on the device
    if (h_stream_ids) OWW_CUDA(ctx, cudaMemcpyAsync(d_ids, h_stream_ids, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    OWW_CUDA(ctx, cudaMemcpyAsync(d_slots, h_slots, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    assign_kernel<<<(n + 255) / 256, 256, 0, s>>>(h_stream_ids ? d_ids : nullptr, d_slots, n, b.d_assign);
    OWW_LAUNCH_CHECK(ctx);
    if (other) {
        OWW_CUDA(ctx, cudaEventRecord(ctx->ver_ev[1], s));
        OWW_CUDA(ctx, cudaStreamWaitEvent(ctx->own_stream, ctx->ver_ev[1], 0));
    }
    return OWW_OK;
}

int oww_set_verifier_clip_slot(oww_ctx* ctx, int bank, int slot) {
    if (!ctx) return OWW_EINVAL;
    if (bank < 0 || bank >= (int)ctx->banks.size()) return oww_fail(ctx, OWW_EINVAL, "bad verifier bank %d", bank);
    if (slot < -1 || slot >= ctx->banks[bank].capacity)
        return oww_fail(ctx, OWW_EINVAL, "slot %d outside [-1,%d)", slot, ctx->banks[bank].capacity);
    ctx->banks[bank].clip_slot = slot;
    return OWW_OK;
}

int oww_set_verifier_threshold(oww_ctx* ctx, int bank, float threshold) {
    if (!ctx) return OWW_EINVAL;
    if (bank < 0 || bank >= (int)ctx->banks.size()) return oww_fail(ctx, OWW_EINVAL, "bad verifier bank %d", bank);
    ctx->banks[bank].thr = threshold;
    return OWW_OK;
}

int oww_enable_verifiers(oww_ctx* ctx, int enabled) {
    if (!ctx) return OWW_EINVAL;
    ctx->verifiers_on = enabled != 0;
    return OWW_OK;
}

int oww_verifier_predict(oww_ctx* ctx, int bank, int slot, const float* d_feats, int n, float* d_out, void* stream) {
    if (!ctx || !d_feats || !d_out) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (bank < 0 || bank >= (int)ctx->banks.size()) return oww_fail(ctx, OWW_EINVAL, "bad verifier bank %d", bank);
    const VerifierBank& b = ctx->banks[bank];
    if (slot < 0 || slot >= b.capacity) return oww_fail(ctx, OWW_EINVAL, "slot %d outside [0,%d)", slot, b.capacity);
    if (n < 0) return oww_fail(ctx, OWW_EINVAL, "n=%d", n);
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    VerArgs a;
    a.bank[0] = bank_dev(b, slot, nullptr, nullptr);
    a.bank[0].col0 = 0; a.bank[0].n_cols = 1;
    a.src = FeatSrc{d_feats, (int64_t)b.n_in * 96, nullptr, -1, 0};
    a.n = n; a.out = d_out; a.out_stride = 1; a.gated = 0; a.step = nullptr; a.clip_streams = nullptr;
    return launch(ctx, a, 1, (cudaStream_t)stream);
}

}  // extern "C"
