// K3d: training custom verifier models (openwakeword/custom_verifier_model.py:95-113 of the original project) for many
// users in one launch.  For user u with samples i = 0..n-1 (a sample is the window of n_in consecutive feature rows
// starting at row first_row[i], D = n_in*96 contiguous floats) and labels y_i in {0, 1}:
//   StandardScaler   mean_j = sum_i x_ij / n,  var_j = (sum_i (x_ij - mean_j)^2 - (sum_i (x_ij - mean_j))^2 / n) / n
//                    (scikit-learn's formula), scale_j = sqrt(var_j), or 1 where scikit-learn calls the feature constant
//   LogisticRegression on z_ij = (x_ij - mean_j) / scale_j: the minimiser of
//                    f(w, b) = 1/2 |w|^2 + C sum_i [softplus(m_i) - y_i m_i],   m_i = w.z_i + b   (b not penalised)
// Newton's method: each iteration solves H d = -g by conjugate gradients on Hessian-vector products
// (H v = [v_w; 0] + C Z~^T S Z~ v with Z~ = [Z, 1], S = diag(p_i (1 - p_i))), stopped by the forcing term
// min(0.5, sqrt|g|) |g|, then backtracks along d until f decreases by the Armijo condition.
//
// One persistent CTA of kThreads threads per user at a time.  Everything is float64 and every reduction has a fixed
// order that depends only on n and D: a warp per sample for the window dot products (lane l takes float4 l, l+32, ...;
// xor-shuffle tree), a thread per feature for the sums over samples (sequential in sample order), and a fixed shared
// memory tree over the threads of the block.  So a user's outputs do not depend on the other users of the batch, the
// grid size or the order of the users.  No atomics.
#include "oww_internal.h"
#include <cfloat>
#include <cmath>
#include <vector>

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxNin = 120;            // the feature rows a stream keeps (utils.py:449-450): the longest head window
constexpr int kVecs = 6;                // per-CTA float64 vectors of D: scale, g, d, r, p, q
constexpr int kCgMax = 200;             // CG iterations per Newton step
constexpr int kLsMax = 40;              // step halvings per line search

struct FitArgs {
    const float* rows; int64_t n_rows; int n_in, D, n_users;
    const int64_t* first; const int64_t* off; const uint8_t* labels;
    double C, tol; int max_iter;
    double* mean; double* var; double* coef; double* intercept; int* iters; int* status;
    double* vec;                        // [gridDim.x][kVecs][D]
    double* smp;                        // [3][N]: margin, per-sample coefficient, window product
    int64_t N;
};

struct Smem {                           // dynamic shared memory: mu[D] | u[D] | red[kThreads] | ta[kThreads] | tf[kThreads]
    double* mu; double* u; double* red; double* ta; int64_t* tf;
};

__device__ double block_sum(double v, double* red) {
    const int t = threadIdx.x;
    red[t] = v;
    __syncthreads();
#pragma unroll
    for (int s = kThreads / 2; s > 0; s >>= 1) {
        if (t < s) red[t] += red[t + s];
        __syncthreads();
    }
    const double r = red[0];
    __syncthreads();
    return r;
}

__device__ double block_max(double v, double* red) {
    const int t = threadIdx.x;
    red[t] = v;
    __syncthreads();
#pragma unroll
    for (int s = kThreads / 2; s > 0; s >>= 1) {
        if (t < s) red[t] = fmax(red[t], red[t + s]);
        __syncthreads();
    }
    const double r = red[0];
    __syncthreads();
    return r;
}

__device__ __forceinline__ double softplus(double m) { return fmax(m, 0.0) + log1p(exp(-fabs(m))); }
__device__ __forceinline__ double sigmoid(double m) { return 1.0 / (1.0 + exp(-m)); }

// t[i] = sum_j (x_ij - mu_j) u_j + ub for every sample, one warp per sample.  Ends with a barrier.
__device__ void window_dots(const FitArgs& a, const Smem& sm, const int64_t* first, int n, double ub, double* t) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n4 = a.D / 4;
    for (int i = warp; i < n; i += kWarps) {
        const float4* x = reinterpret_cast<const float4*>(a.rows + first[i] * 96);
        double acc = 0.0;
        for (int k = lane; k < n4; k += 32) {
            const float4 v = __ldg(x + k);
            const int j = 4 * k;
            acc = fma((double)v.x - sm.mu[j], sm.u[j], acc);
            acc = fma((double)v.y - sm.mu[j + 1], sm.u[j + 1], acc);
            acc = fma((double)v.z - sm.mu[j + 2], sm.u[j + 2], acc);
            acc = fma((double)v.w - sm.mu[j + 3], sm.u[j + 3], acc);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) t[i] = acc + ub;
    }
    __syncthreads();
}

// For every feature j of this thread (j = tid, tid + kThreads, ...): out(j, sum_i c_i (x_ij - mu_j)) in sample order.
// c == nullptr: c_i = 1.  Samples are staged through shared memory in tiles of kThreads.
template <class Out>
__device__ void feature_sums(const FitArgs& a, const Smem& sm, const int64_t* first, int n, const double* c,
                             const double* mu, Out out) {
    for (int j0 = 0; j0 < a.D; j0 += kThreads) {
        const int j = j0 + threadIdx.x;
        const bool on = j < a.D;
        const double m = (on && mu) ? mu[j] : 0.0;
        double acc = 0.0;
        for (int i0 = 0; i0 < n; i0 += kThreads) {
            __syncthreads();
            if (i0 + threadIdx.x < n) {
                sm.ta[threadIdx.x] = c ? c[i0 + threadIdx.x] : 1.0;
                sm.tf[threadIdx.x] = first[i0 + threadIdx.x] * 96;
            }
            __syncthreads();
            const int cnt = min(kThreads, n - i0);
            if (on) {
#pragma unroll 4
                for (int k = 0; k < cnt; ++k) acc = fma(sm.ta[k], (double)__ldg(a.rows + sm.tf[k] + j) - m, acc);
            }
        }
        if (on) out(j, acc);
    }
    __syncthreads();
}

__device__ void clear_user(const FitArgs& a, int u, int status) {
    const int64_t base = (int64_t)u * a.D;
    for (int j = threadIdx.x; j < a.D; j += kThreads) {
        a.mean[base + j] = 0.0; a.var[base + j] = 0.0; a.coef[base + j] = 0.0;
    }
    if (threadIdx.x == 0) { a.intercept[u] = 0.0; a.iters[u] = 0; a.status[u] = status; }
}

__global__ void __launch_bounds__(kThreads) verifier_fit_kernel(const __grid_constant__ FitArgs a) {
    extern __shared__ double smem[];
    Smem sm;
    sm.mu = smem; sm.u = smem + a.D; sm.red = smem + 2 * a.D; sm.ta = sm.red + kThreads;
    sm.tf = reinterpret_cast<int64_t*>(sm.ta + kThreads);
    const int D = a.D;
    const double C = a.C;
    double* sc = a.vec + (int64_t)blockIdx.x * kVecs * D;
    double* g = sc + D; double* d = g + D; double* r = d + D; double* p = r + D; double* q = p + D;

    for (int u = blockIdx.x; u < a.n_users; u += gridDim.x) {
        const int64_t o0 = a.off[u];
        const int n = (int)(a.off[u + 1] - o0);
        const int64_t* first = a.first + o0;
        const uint8_t* y = a.labels + o0;
        double* m = a.smp + o0;                 // margins w.z_i + b of the current iterate
        double* c = a.smp + a.N + o0;           // per-sample coefficient of the current feature sum
        double* t = a.smp + 2 * a.N + o0;       // window products Z~ v
        double* mean = a.mean + (int64_t)u * D; double* var = a.var + (int64_t)u * D; double* w = a.coef + (int64_t)u * D;

        // windows inside [0, n_rows), and both classes present
        int bad = 0;
        double npos = 0.0;
        for (int i = threadIdx.x; i < n; i += kThreads) {
            const int64_t f = first[i];
            bad |= f < 0 || f > a.n_rows - a.n_in;
            npos += y[i] != 0;
        }
        bad = __syncthreads_or(bad);
        npos = block_sum(npos, sm.red);
        if (bad || n == 0 || npos == 0.0 || npos == (double)n) {
            clear_user(a, u, bad ? 3 : 2);
            __syncthreads();
            continue;
        }

        // scaler statistics (a non-finite value makes the user's status 3)
        feature_sums(a, sm, first, n, nullptr, nullptr, [&](int j, double s) { sm.mu[j] = s / n; });
        int nonfinite = 0;
        for (int j0 = 0; j0 < D; j0 += kThreads) {            // sum of squared and of plain deviations, in one sweep
            const int j = j0 + threadIdx.x;
            const bool on = j < D;
            const double mj = on ? sm.mu[j] : 0.0;
            double s1 = 0.0, s2 = 0.0;
            for (int i0 = 0; i0 < n; i0 += kThreads) {
                __syncthreads();
                if (i0 + threadIdx.x < n) sm.tf[threadIdx.x] = first[i0 + threadIdx.x] * 96;
                __syncthreads();
                const int cnt = min(kThreads, n - i0);
                if (on)
                    for (int k = 0; k < cnt; ++k) {
                        const float x = __ldg(a.rows + sm.tf[k] + j);
                        nonfinite |= !isfinite(x);
                        const double dv = (double)x - mj;
                        s1 += dv; s2 = fma(dv, dv, s2);
                    }
            }
            if (on) {
                const double v = (s2 - s1 * s1 / n) / n;
                mean[j] = mj; var[j] = v;
                constexpr double eps = DBL_EPSILON;
                const double nm = n * mj * eps;
                sc[j] = v <= n * eps * v + nm * nm ? 1.0 : sqrt(v);   // scikit-learn's _is_constant_feature
            }
        }
        if (__syncthreads_or(nonfinite)) {
            clear_user(a, u, 3);
            __syncthreads();
            continue;
        }

        for (int j = threadIdx.x; j < D; j += kThreads) w[j] = 0.0;
        for (int i = threadIdx.x; i < n; i += kThreads) m[i] = 0.0;
        double b = 0.0, ww = 0.0;
        int it = 0, st = 1;
        const double tol_abs = a.tol * C * n;
        for (;;) {
            // value and gradient at (w, b)
            double fl = 0.0, cl = 0.0;
            for (int i = threadIdx.x; i < n; i += kThreads) {
                const double mi = m[i], yi = y[i] != 0 ? 1.0 : 0.0;
                c[i] = sigmoid(mi) - yi;
                fl += softplus(mi) - yi * mi;
                cl += c[i];
            }
            const double fdat = block_sum(fl, sm.red);
            const double g_b = C * block_sum(cl, sm.red);
            double gm = 0.0;
            feature_sums(a, sm, first, n, c, sm.mu, [&](int j, double s) {
                g[j] = w[j] + C * s / sc[j];
                gm = fmax(gm, fabs(g[j]));
            });
            const double f = 0.5 * ww + C * fdat;
            gm = block_max(fmax(gm, fabs(g_b)), sm.red);
            if (gm <= tol_abs) { st = 0; break; }
            if (it == a.max_iter) break;
            ++it;

            // conjugate gradients on H d = -g
            double rl = 0.0;
            for (int j = threadIdx.x; j < D; j += kThreads) { d[j] = 0.0; r[j] = -g[j]; p[j] = r[j]; rl = fma(r[j], r[j], rl); }
            double d_b = 0.0, r_b = -g_b, p_b = r_b;
            double rr = block_sum(rl, sm.red) + r_b * r_b;
            const double target = fmin(0.5, sqrt(sqrt(rr))) * sqrt(rr);
            for (int k = 0; k < kCgMax; ++k) {
                for (int j = threadIdx.x; j < D; j += kThreads) sm.u[j] = p[j] / sc[j];
                __syncthreads();
                window_dots(a, sm, first, n, p_b, t);
                double sl = 0.0;
                for (int i = threadIdx.x; i < n; i += kThreads) {
                    const double pi = sigmoid(m[i]);
                    c[i] = pi * (1.0 - pi) * t[i];
                    sl += c[i];
                }
                const double q_b = C * block_sum(sl, sm.red);      // its barrier publishes c
                double pq = 0.0;
                feature_sums(a, sm, first, n, c, sm.mu, [&](int j, double s) {
                    q[j] = p[j] + C * s / sc[j];
                    pq = fma(p[j], q[j], pq);
                });
                pq = block_sum(pq, sm.red) + p_b * q_b;
                if (!(pq > 0.0)) break;
                const double alpha = rr / pq;
                rl = 0.0;
                for (int j = threadIdx.x; j < D; j += kThreads) {
                    d[j] = fma(alpha, p[j], d[j]); r[j] = fma(-alpha, q[j], r[j]); rl = fma(r[j], r[j], rl);
                }
                d_b = fma(alpha, p_b, d_b); r_b = fma(-alpha, q_b, r_b);
                const double rr_new = block_sum(rl, sm.red) + r_b * r_b;
                if (sqrt(rr_new) <= target) break;
                const double beta = rr_new / rr;
                rr = rr_new;
                for (int j = threadIdx.x; j < D; j += kThreads) p[j] = fma(beta, p[j], r[j]);
                p_b = fma(beta, p_b, r_b);
            }

            // backtracking along d: margins move by step * (Z~ d)_i
            double gl = 0.0, wl = 0.0, dl = 0.0;
            for (int j = threadIdx.x; j < D; j += kThreads) {
                sm.u[j] = d[j] / sc[j];
                gl = fma(g[j], d[j], gl); wl = fma(w[j], d[j], wl); dl = fma(d[j], d[j], dl);
            }
            __syncthreads();
            window_dots(a, sm, first, n, d_b, t);
            const double gd = block_sum(gl, sm.red) + g_b * d_b;
            const double wd = block_sum(wl, sm.red), dd = block_sum(dl, sm.red);
            double step = 1.0;
            bool ok = false;
            for (int ls = 0; ls < kLsMax && !ok; ++ls) {
                double fl2 = 0.0;
                for (int i = threadIdx.x; i < n; i += kThreads) {
                    const double mi = fma(step, t[i], m[i]), yi = y[i] != 0 ? 1.0 : 0.0;
                    fl2 += softplus(mi) - yi * mi;
                }
                const double fn = 0.5 * (ww + step * (2.0 * wd + step * dd)) + C * block_sum(fl2, sm.red);
                // Armijo, with room for the rounding of f itself once the decrease reaches it
                if (fn - f <= 1e-4 * step * gd + 8.0 * DBL_EPSILON * fabs(f)) ok = true;
                else step *= 0.5;
            }
            if (!ok) break;                     // no descent left along d: stop with status 1 at the current iterate
            double wl2 = 0.0;
            for (int j = threadIdx.x; j < D; j += kThreads) { w[j] = fma(step, d[j], w[j]); wl2 = fma(w[j], w[j], wl2); }
            b = fma(step, d_b, b);
            for (int i = threadIdx.x; i < n; i += kThreads) m[i] = fma(step, t[i], m[i]);
            ww = block_sum(wl2, sm.red);        // its barrier publishes m
        }
        if (threadIdx.x == 0) { a.intercept[u] = b; a.iters[u] = it; a.status[u] = st; }
        __syncthreads();
    }
}

__global__ void load_verifiers_kernel(const int* slots, int n, int D, const float* mean, const float* weight,
                                      const float* bias, float* b_mean, float* b_weight, float* b_bias) {
    const int i = blockIdx.x;
    const int64_t dst = (int64_t)slots[i] * D, src = (int64_t)i * D;
    for (int j = threadIdx.x; j < D; j += blockDim.x) {
        b_mean[dst + j] = mean[src + j];
        b_weight[dst + j] = weight[src + j];
    }
    if (threadIdx.x == 0) b_bias[slots[i]] = bias[i];
}

template <class T>
int grow(oww_ctx* ctx, T*& p, size_t& cap, size_t need) {
    if (need <= cap) return OWW_OK;
    cudaFree(p); p = nullptr; cap = 0;
    OWW_CUDA(ctx, cudaMalloc(&p, need * sizeof(T)));
    cap = need;
    return OWW_OK;
}

}  // namespace

void oww_verifier_fit_free(oww_ctx* ctx) {
    cudaFree(ctx->d_fit_scratch); ctx->d_fit_scratch = nullptr; ctx->fit_scratch_doubles = 0;
    cudaFree(ctx->d_fit_off); ctx->d_fit_off = nullptr; ctx->fit_off_cap = 0;
    cudaFree(ctx->d_load_slots); ctx->d_load_slots = nullptr; ctx->load_slots_cap = 0;
}

extern "C" {

int oww_fit_verifiers(oww_ctx* ctx, const float* d_rows, int64_t n_rows, int n_in, const int64_t* d_first_row,
                      const int64_t* h_sample_offsets, const uint8_t* d_labels, int n_users, double C, int max_iter,
                      double tol, double* d_mean, double* d_var, double* d_coef, double* d_intercept, int32_t* d_iters,
                      int32_t* d_status, void* stream) {
    if (!ctx) return OWW_EINVAL;
    if (n_users < 0) return oww_fail(ctx, OWW_EINVAL, "n_users=%d", n_users);
    if (n_users == 0) return OWW_OK;
    if (!h_sample_offsets || !d_mean || !d_var || !d_coef || !d_intercept || !d_iters || !d_status)
        return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (!(C > 0.0) || !std::isfinite(C)) return oww_fail(ctx, OWW_EINVAL, "C=%g must be positive and finite", C);
    if (n_in < 1 || n_in > kMaxNin) return oww_fail(ctx, OWW_EINVAL, "n_in=%d outside [1,%d]", n_in, kMaxNin);
    if (max_iter < 1) return oww_fail(ctx, OWW_EINVAL, "max_iter=%d < 1", max_iter);
    if (!(tol >= 0.0) || !std::isfinite(tol)) return oww_fail(ctx, OWW_EINVAL, "tol=%g must be finite and >= 0", tol);
    if (n_rows < 0) return oww_fail(ctx, OWW_EINVAL, "n_rows=%lld", (long long)n_rows);
    if ((uintptr_t)d_rows % 16) return oww_fail(ctx, OWW_EINVAL, "d_rows must be 16-byte aligned");
    if (h_sample_offsets[0] < 0) return oww_fail(ctx, OWW_EINVAL, "sample offset %lld < 0", (long long)h_sample_offsets[0]);
    for (int u = 0; u < n_users; ++u) {
        const int64_t n = h_sample_offsets[u + 1] - h_sample_offsets[u];
        if (n < 0) return oww_fail(ctx, OWW_EINVAL, "sample offsets decrease at user %d", u);
        if (n > INT32_MAX) return oww_fail(ctx, OWW_EINVAL, "user %d has %lld samples", u, (long long)n);
    }
    const int64_t N = h_sample_offsets[n_users];
    if (N > 0 && (!d_first_row || !d_labels)) return oww_fail(ctx, OWW_EINVAL, "null argument");
    if (N > 0 && n_rows > 0 && !d_rows) return oww_fail(ctx, OWW_EINVAL, "null argument");
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    const int D = n_in * 96;
    const size_t smem = (size_t)(2 * D + 2 * kThreads) * sizeof(double) + kThreads * sizeof(int64_t);
    if (!ctx->fit_attr_set) {
        const size_t most = (size_t)(2 * kMaxNin * 96 + 2 * kThreads) * sizeof(double) + kThreads * sizeof(int64_t);
        OWW_CUDA(ctx, cudaFuncSetAttribute(verifier_fit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)most));
        ctx->fit_attr_set = true;
    }
    int per_sm = 0;
    OWW_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, verifier_fit_kernel, kThreads, smem));
    const int grid = std::max(1, std::min(n_users, ctx->sm_count * std::max(per_sm, 1)));
    int rc;
    if ((rc = grow(ctx, ctx->d_fit_scratch, ctx->fit_scratch_doubles, (size_t)grid * kVecs * D + 3 * (size_t)N))) return rc;
    if ((rc = grow(ctx, ctx->d_fit_off, ctx->fit_off_cap, (size_t)n_users + 1))) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    // pageable source: staged by the driver before the call returns
    OWW_CUDA(ctx, cudaMemcpyAsync(ctx->d_fit_off, h_sample_offsets, (size_t)(n_users + 1) * sizeof(int64_t),
                                  cudaMemcpyHostToDevice, s));
    FitArgs a;
    a.rows = d_rows; a.n_rows = n_rows; a.n_in = n_in; a.D = D; a.n_users = n_users;
    a.first = d_first_row; a.off = ctx->d_fit_off; a.labels = d_labels;
    a.C = C; a.tol = tol; a.max_iter = max_iter;
    a.mean = d_mean; a.var = d_var; a.coef = d_coef; a.intercept = d_intercept; a.iters = d_iters; a.status = d_status;
    a.vec = ctx->d_fit_scratch; a.smp = ctx->d_fit_scratch + (size_t)grid * kVecs * D; a.N = N;
    verifier_fit_kernel<<<grid, kThreads, smem, s>>>(a);
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

int oww_load_verifiers(oww_ctx* ctx, int bank, const int32_t* h_slots, int n, const float* d_mean,
                       const float* d_weight, const float* d_bias, void* stream) {
    if (!ctx) return OWW_EINVAL;
    if (bank < 0 || bank >= (int)ctx->banks.size()) return oww_fail(ctx, OWW_EINVAL, "bad verifier bank %d", bank);
    const VerifierBank& b = ctx->banks[bank];
    if (n < 0 || n > b.capacity) return oww_fail(ctx, OWW_EINVAL, "n=%d outside [0,%d]", n, b.capacity);
    if (n == 0) return OWW_OK;
    if (!h_slots || !d_mean || !d_weight || !d_bias) return oww_fail(ctx, OWW_EINVAL, "null argument");
    std::vector<uint8_t> seen(b.capacity, 0);
    for (int i = 0; i < n; ++i) {
        if (h_slots[i] < 0 || h_slots[i] >= b.capacity)
            return oww_fail(ctx, OWW_EINVAL, "slot %d outside [0,%d)", h_slots[i], b.capacity);
        if (seen[h_slots[i]]++) return oww_fail(ctx, OWW_EINVAL, "slot %d listed twice", h_slots[i]);
    }
    OWW_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc;
    if ((rc = grow(ctx, ctx->d_load_slots, ctx->load_slots_cap, (size_t)b.capacity))) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    // ordered after the host-buffer steps already submitted on the handle's own stream, and before later ones
    const bool other = s != ctx->own_stream;
    if (other) {
        OWW_CUDA(ctx, cudaEventRecord(ctx->ver_ev[0], ctx->own_stream));
        OWW_CUDA(ctx, cudaStreamWaitEvent(s, ctx->ver_ev[0], 0));
    }
    OWW_CUDA(ctx, cudaMemcpyAsync(ctx->d_load_slots, h_slots, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    load_verifiers_kernel<<<n, 256, 0, s>>>(ctx->d_load_slots, n, b.n_in * 96, d_mean, d_weight, d_bias,
                                           b.d_mean, b.d_weight, b.d_bias);
    OWW_LAUNCH_CHECK(ctx);
    if (other) {
        OWW_CUDA(ctx, cudaEventRecord(ctx->ver_ev[1], s));
        OWW_CUDA(ctx, cudaStreamWaitEvent(ctx->own_stream, ctx->ver_ev[1], 0));
    }
    return OWW_OK;
}

}  // extern "C"
