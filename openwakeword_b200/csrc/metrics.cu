// Score metrics on the device (SURVEY.md section 8 f4): false positives per threshold with the reference's grouping rule
// and the ROC counts, over [n_series][n_frames] score tensors that are already in HBM (bulk predict_clips leaves them there).
//
// Replaces openwakeword/metrics.py:24-45 (get_false_positives; the sequential grouping rule is restated
// in oracle/metrics.py and pinned against the reference's own function by tests/golden/metrics.npz), :48-78
// (generate_roc_curve_fprs: the same count at 25 thresholds) and :81-100 (generate_roc_curve_tprs: count of scores >= t).
// The reference walks one Python list per threshold; here one thread owns one (series, threshold) pair and the 32 lanes
// of a warp share a series, so every score load is a broadcast and the whole ROC of a series costs two passes over it.
// HBM bound: 4 B (float32) or 8 B (float64) per score per pass.
//
// Every comparison is (double)score >= threshold.  The host rounds each threshold to the dtype in which NumPy would
// compare it with the scores (openwakeword_b200/metrics.py comparison_dtype) and passes that as a double; widening a
// float32 score, or a threshold already rounded to float16/32/64, to double is exact, so the double comparison is
// exactly NumPy's comparison in that dtype.
#include "oww_internal.h"

namespace {

template <typename T>
__global__ void __launch_bounds__(128) false_positives_kernel(const T* scores, int64_t series_stride, int n_series, int n_frames,
                                                             const double* thr, int n_thr, int window, int* out) {
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int per = (n_thr + 31) & ~31;                       // a warp never straddles two series
    const int sidx = (int)(gid / per), ti = (int)(gid % per);
    if (sidx >= n_series || ti >= n_thr) return;
    const T* s = scores + (int64_t)sidx * series_stride;
    const double t = thr[ti];
    // pass 1: ones and 0->1 transitions of the original sequence
    int ones = 0, n_tr = 0;
    bool prev = false;
    for (int i = 0; i < n_frames; ++i) {
        const bool p = (double)s[i] >= t;
        ones += p;
        n_tr += (i > 0 && !prev && p);
        prev = p;
    }
    // pass 2: the grouping rule only ever touches indices below n_tr (k = min(n_tr - e, window) must be positive)
    int removed = 0, max_end = 0;
    const int lim = n_tr < n_frames ? n_tr : n_frames;
    bool p0 = lim > 0 ? ((double)s[0] >= t) : false;
    for (int i = 0; i + 2 < lim; ++i) {                       // transition at (i, i+1), e = i + 2 < n_tr
        const bool p1 = (double)s[i + 1] >= t;
        if (!p0 && p1) {
            const int e = i + 2;
            const bool alive = e >= max_end && ((double)s[e] >= t);
            if (alive) {
                int k = n_tr - e;
                if (k > window) k = window;
                const int lo = e > max_end ? e : max_end, hi = e + k;
                for (int j = lo; j < hi; ++j) removed += ((double)s[j] >= t);
                if (hi > max_end) max_end = hi;
            }
        }
        p0 = p1;
    }
    out[(int64_t)sidx * n_thr + ti] = ones - removed;
}

template <typename T>
__global__ void __launch_bounds__(256) count_ge_kernel(const T* scores, int64_t n, const double* thr, int n_thr, unsigned long long* out) {
    // grid-stride over the scores; per-thread counters for every threshold (n_thr <= 64), block reduction, one atomic each
    __shared__ unsigned int s_cnt[64];
    if (threadIdx.x < 64) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    for (int ti = 0; ti < n_thr; ++ti) {
        const double t = thr[ti];
        unsigned int c = 0;
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
            c += ((double)scores[i] >= t);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_cnt[ti], c);
    }
    __syncthreads();
    if (threadIdx.x < n_thr && s_cnt[threadIdx.x]) atomicAdd(out + threadIdx.x, (unsigned long long)s_cnt[threadIdx.x]);
}

template <typename T>
int false_positives(oww_ctx* ctx, const T* d_scores, int64_t series_stride, int n_series, int n_frames,
                    const double* h_thresholds, int n_thresholds, int grouping_window, int32_t* h_counts, void* stream) {
    if (!ctx || !d_scores || !h_thresholds || !h_counts) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (n_series < 1 || n_frames < 0 || n_thresholds < 1 || n_thresholds > 4096) return oww_fail(ctx, OWW_EINVAL, "bad sizes");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    double* d_thr = nullptr; int* d_out = nullptr;
    const size_t n_out = (size_t)n_series * n_thresholds;
    OWW_CUDA(ctx, cudaMallocAsync(&d_thr, n_thresholds * sizeof(double), s));
    OWW_CUDA(ctx, cudaMallocAsync(&d_out, n_out * sizeof(int), s));
    OWW_CUDA(ctx, cudaMemcpyAsync(d_thr, h_thresholds, n_thresholds * sizeof(double), cudaMemcpyHostToDevice, s));
    const int per = (n_thresholds + 31) & ~31;
    const int64_t threads = (int64_t)n_series * per;
    false_positives_kernel<<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(d_scores, series_stride, n_series, n_frames, d_thr,
                                                                             n_thresholds, grouping_window, d_out);
    ctx->launches++;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_counts, d_out, n_out * sizeof(int), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    cudaFreeAsync(d_thr, s); cudaFreeAsync(d_out, s);
    if (e != cudaSuccess) return oww_fail(ctx, OWW_ECUDA, "false-positive count failed: %s", cudaGetErrorString(e));
    return OWW_OK;
}

template <typename T>
int count_ge(oww_ctx* ctx, const T* d_scores, int64_t n, const double* h_thresholds, int n_thresholds,
             uint64_t* h_counts, void* stream) {
    if (!ctx || !d_scores || !h_thresholds || !h_counts) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (n < 0 || n_thresholds < 1 || n_thresholds > 64) return oww_fail(ctx, OWW_EINVAL, "1..64 thresholds per call");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    double* d_thr = nullptr; unsigned long long* d_out = nullptr;
    OWW_CUDA(ctx, cudaMallocAsync(&d_thr, n_thresholds * sizeof(double), s));
    OWW_CUDA(ctx, cudaMallocAsync(&d_out, n_thresholds * sizeof(unsigned long long), s));
    OWW_CUDA(ctx, cudaMemsetAsync(d_out, 0, n_thresholds * sizeof(unsigned long long), s));
    OWW_CUDA(ctx, cudaMemcpyAsync(d_thr, h_thresholds, n_thresholds * sizeof(double), cudaMemcpyHostToDevice, s));
    int64_t blocks = (n + 255) / 256;
    if (blocks > (int64_t)ctx->sm_count * 8) blocks = (int64_t)ctx->sm_count * 8;
    if (blocks < 1) blocks = 1;
    count_ge_kernel<<<(unsigned)blocks, 256, 0, s>>>(d_scores, n, d_thr, n_thresholds, d_out);
    ctx->launches++;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_counts, d_out, n_thresholds * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    cudaFreeAsync(d_thr, s); cudaFreeAsync(d_out, s);
    if (e != cudaSuccess) return oww_fail(ctx, OWW_ECUDA, "threshold count failed: %s", cudaGetErrorString(e));
    return OWW_OK;
}

}  // namespace

extern "C" {

int oww_metrics_false_positives(oww_ctx* ctx, const float* d_scores, int64_t series_stride, int n_series, int n_frames,
                                const double* h_thresholds, int n_thresholds, int grouping_window, int32_t* h_counts, void* stream) {
    return false_positives(ctx, d_scores, series_stride, n_series, n_frames, h_thresholds, n_thresholds, grouping_window, h_counts, stream);
}

int oww_metrics_false_positives_f64(oww_ctx* ctx, const double* d_scores, int64_t series_stride, int n_series, int n_frames,
                                    const double* h_thresholds, int n_thresholds, int grouping_window, int32_t* h_counts,
                                    void* stream) {
    return false_positives(ctx, d_scores, series_stride, n_series, n_frames, h_thresholds, n_thresholds, grouping_window, h_counts, stream);
}

int oww_metrics_count_ge(oww_ctx* ctx, const float* d_scores, int64_t n, const double* h_thresholds, int n_thresholds,
                         uint64_t* h_counts, void* stream) {
    return count_ge(ctx, d_scores, n, h_thresholds, n_thresholds, h_counts, stream);
}

int oww_metrics_count_ge_f64(oww_ctx* ctx, const double* d_scores, int64_t n, const double* h_thresholds, int n_thresholds,
                             uint64_t* h_counts, void* stream) {
    return count_ge(ctx, d_scores, n, h_thresholds, n_thresholds, h_counts, stream);
}

}  // extern "C"
