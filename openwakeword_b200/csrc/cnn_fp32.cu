// K2 (fp32 CUDA-core path): the speech-embedding CNN as 20 implicit-GEMM convolutions.
//
// Replaces the embedding_model.onnx session of the reference
// (openwakeword/utils.py:90-93,235,443; graph spec
// notebooks/converting_google_speech_embedding_model.ipynb:871-951, shapes :521-859; SURVEY.md
// Appendix B): 3x3 conv on the 76x32 mel window, then alternating (1,3) "same" / (3,1) "valid"
// dense convs, folded BatchNorm + max(0.2x,x) + max(x,-0.4) after every conv but the last,
// five max-pools.  Activations are NHWC fp32 [window][t][f][c] in two ping-pong buffers.
//
// This file is the bit-faithful fp32 path: every layer is one launch of a register-tiled
// (8x8 per thread) shared-memory implicit GEMM, M = windows*T*F output positions, N = Cout,
// K = taps*Cin, with the tap shift applied while the A tile is gathered (no im2col buffer).
// The window modes differ only in how the first layer addresses the mel rows (ring vs linear);
// clip mode runs the same kernels fully-convolutionally over T > 76 rows (SURVEY.md F10).
#include "oww_internal.h"

namespace {

constexpr float kLeak = 0.20000000298023224f;
constexpr float kFloor = -0.4000000059604645f;

__device__ __forceinline__ float act(float v) {
    v = fmaxf(kLeak * v, v);
    return fmaxf(v, kFloor);
}

// ---------------- layer 0: ZeroPad(0,1) + 3x3 conv (Cin=1) + ReLU + BN + act -----------------
struct L0Args {
    WindowSrc src;
    int n_windows, t_out, t_in;     // t_out = t_in - 2
    const float* w;                 // [9][24]
    const float* scale; const float* bias;
    float* out; int64_t out_stride; // per window
};

__global__ void __launch_bounds__(256) conv0_kernel(L0Args a) {
    __shared__ float s_w[9 * 24];
    __shared__ float s_s[24], s_b[24];
    for (int i = threadIdx.x; i < 9 * 24; i += 256) s_w[i] = a.w[i];
    if (threadIdx.x < 24) { s_s[threadIdx.x] = a.scale[threadIdx.x]; s_b[threadIdx.x] = a.bias[threadIdx.x]; }
    __syncthreads();
    const int64_t total = (int64_t)a.n_windows * a.t_out * 32;
    for (int64_t m = (int64_t)blockIdx.x * 256 + threadIdx.x; m < total; m += (int64_t)gridDim.x * 256) {
        const int f = (int)(m & 31);
        const int64_t r = m >> 5;
        const int t = (int)(r % a.t_out);
        const int j = (int)(r / a.t_out);
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
        float* o = a.out + (int64_t)j * a.out_stride + ((int64_t)t * 32 + f) * 24;
#pragma unroll
        for (int c4 = 0; c4 < 6; ++c4) {
            float v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int c = c4 * 4 + u;
                float acc = 0.f;
#pragma unroll
                for (int k = 0; k < 9; ++k) acc = fmaf(x[k], s_w[k * 24 + c], acc);
                acc = fmaxf(acc, 0.f);                       // activation='relu' before the BN (nb/conv:897)
                v[u] = act(fmaf(acc, s_s[c], s_b[c]));
            }
            reinterpret_cast<float4*>(o)[c4] = make_float4(v[0], v[1], v[2], v[3]);
        }
    }
}

// ---------------- generic (1,3)-same / (3,1)-valid conv as implicit GEMM ----------------------
struct ConvArgs {
    const float* in; int64_t in_stride;    // per sample
    float* out; int64_t out_stride;
    const float* w;                        // [taps*CIN][COUT]
    const float* scale; const float* bias;
    int n, t_out, f;                       // output extent (f_in == f_out)
    int apply_act;
};

template <int CIN, int COUT, int KH, int KW, int BM>
__global__ void __launch_bounds__((BM / 8) * (COUT / 8)) conv_kernel(ConvArgs a) {
    constexpr int TX = COUT / 8, TY = BM / 8, NT = TX * TY;
    constexpr int KC = 8;
    constexpr int NKC = CIN / KC;
    constexpr int NK = KH * KW * NKC;
    constexpr int A_ITEMS = (BM * 2 + NT - 1) / NT;        // float4 gathers per thread per k-step
    constexpr int W_ITEMS = (KC * COUT / 4 + NT - 1) / NT;
    __shared__ __align__(16) float As[2][KC][BM];
    __shared__ __align__(16) float Ws[2][KC][COUT];

    const int tid = threadIdx.x;
    const int tx = tid % TX, ty = tid / TX;
    const int64_t M = (int64_t)a.n * a.t_out * a.f;
    const int64_t m0 = (int64_t)blockIdx.x * BM;

    // per-thread gather descriptors (fixed across the K loop)
    int64_t g_off[A_ITEMS]; int g_f[A_ITEMS]; bool g_ok[A_ITEMS];
#pragma unroll
    for (int it = 0; it < A_ITEMS; ++it) {
        const int q = tid + it * NT;
        const int ml = q >> 1;
        const int64_t m = m0 + ml;
        g_ok[it] = (q < BM * 2) && (m < M);
        const int64_t mm = g_ok[it] ? m : 0;
        const int f = (int)(mm % a.f);
        const int64_t r = mm / a.f;
        const int t = (int)(r % a.t_out);
        const int64_t n = r / a.t_out;
        g_f[it] = f;
        g_off[it] = n * a.in_stride + ((int64_t)t * a.f + f) * CIN + (q & 1) * 4;
    }

    float4 ra[A_ITEMS]; float4 rw[W_ITEMS];
    auto gload = [&](int ks) {
        const int tap = ks / NKC, c0 = (ks % NKC) * KC;
        const int dt = (KH == 3) ? tap : 0;
        const int df = (KW == 3) ? tap - 1 : 0;
#pragma unroll
        for (int it = 0; it < A_ITEMS; ++it) {
            const int ff = g_f[it] + df;
            const bool ok = g_ok[it] && ff >= 0 && ff < a.f;
            ra[it] = ok ? __ldg(reinterpret_cast<const float4*>(
                              a.in + g_off[it] + ((int64_t)dt * a.f + df) * CIN + c0))
                        : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int it = 0; it < W_ITEMS; ++it) {
            const int q = tid + it * NT;
            if (q < KC * COUT / 4)
                rw[it] = __ldg(reinterpret_cast<const float4*>(a.w + (int64_t)(tap * CIN + c0) * COUT) + q);
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int it = 0; it < A_ITEMS; ++it) {
            const int q = tid + it * NT;
            if (q < BM * 2) {
                const int ml = q >> 1, kq = (q & 1) * 4;
                As[buf][kq + 0][ml] = ra[it].x; As[buf][kq + 1][ml] = ra[it].y;
                As[buf][kq + 2][ml] = ra[it].z; As[buf][kq + 3][ml] = ra[it].w;
            }
        }
#pragma unroll
        for (int it = 0; it < W_ITEMS; ++it) {
            const int q = tid + it * NT;
            if (q < KC * COUT / 4) reinterpret_cast<float4*>(&Ws[buf][0][0])[q] = rw[it];
        }
    };

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    gload(0);
    sstore(0);
    __syncthreads();
    for (int ks = 0; ks < NK; ++ks) {
        const int buf = ks & 1;
        if (ks + 1 < NK) gload(ks + 1);
#pragma unroll
        for (int k = 0; k < KC; ++k) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][BM / 2 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Ws[buf][k][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Ws[buf][k][COUT / 2 + tx * 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        if (ks + 1 < NK) sstore(buf ^ 1);
        __syncthreads();
    }

    // epilogue: folded BN + activation, NHWC store
    float sc[8], bi[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = (j < 4 ? tx * 4 + j : COUT / 2 + tx * 4 + (j - 4));
        sc[j] = __ldg(a.scale + c); bi[j] = __ldg(a.bias + c);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int ml = (i < 4 ? ty * 4 + i : BM / 2 + ty * 4 + (i - 4));
        const int64_t m = m0 + ml;
        if (m >= M) continue;
        const int64_t per = (int64_t)a.t_out * a.f;
        const int64_t n = m / per;
        float* o = a.out + n * a.out_stride + (m - n * per) * COUT;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float y = fmaf(acc[i][j], sc[j], bi[j]);
            v[j] = a.apply_act ? act(y) : y;
        }
        *reinterpret_cast<float4*>(o + tx * 4) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4*>(o + COUT / 2 + tx * 4) = make_float4(v[4], v[5], v[6], v[7]);
    }
}

// ---------------- max-pool (pt x pf, stride = size) ---------------------------------------------
__global__ void __launch_bounds__(256) pool_kernel(const float* in, int64_t in_stride, float* out, int64_t out_stride,
                                                   int n, int t_in, int f_in, int c, int pt, int pf) {
    const int t_out = t_in / pt, f_out = f_in / pf, c4 = c / 4;
    const int64_t total = (int64_t)n * t_out * f_out * c4;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        const int cc = (int)(i % c4);
        int64_t r = i / c4;
        const int f = (int)(r % f_out); r /= f_out;
        const int t = (int)(r % t_out);
        const int64_t s = r / t_out;
        float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        for (int a = 0; a < pt; ++a)
            for (int b = 0; b < pf; ++b) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(
                    in + s * in_stride + ((int64_t)(t * pt + a) * f_in + (f * pf + b)) * c) + cc);
                m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
            }
        reinterpret_cast<float4*>(out + s * out_stride + ((int64_t)t * f_out + f) * c)[cc] = m;
    }
}

// ---------------- append embeddings to the per-stream feature rings -----------------------------
__global__ void __launch_bounds__(256) feat_append_kernel(const float* emb, float* ring, int* count, int n_streams,
                                                          int n_chunks, int rows_mask, int64_t ring_stride, const int* ids) {
    const int64_t total = (int64_t)n_streams * n_chunks * 24;   // float4 units
    oww_pdl_sync();
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
        const int c4 = (int)(i % 24);
        const int64_t j = i / 24;                 // window index = chunk * n_streams + stream
        const int lb = (int)(j % n_streams), ch = (int)(j / n_streams);
        const int b = ids ? ids[lb] : lb;
        const int slot = (count[b] + ch) & rows_mask;
        reinterpret_cast<float4*>(ring + (int64_t)b * ring_stride + (int64_t)slot * 96)[c4] =
            __ldg(reinterpret_cast<const float4*>(emb + j * 96) + c4);
    }
}
__global__ void count_add_kernel(int* count, int n, int add, const int* ids) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    oww_pdl_sync();
    if (i < n) { const int b = ids ? ids[i] : i; count[b] = oww_wrap_count(count[b] + add); }
}

template <int CIN, int COUT, int KH, int KW, int BM>
int launch_conv(oww_ctx* ctx, const ConvArgs& a, cudaStream_t s) {
    const int64_t M = (int64_t)a.n * a.t_out * a.f;
    if (M == 0) return OWW_OK;
    const unsigned grid = (unsigned)((M + BM - 1) / BM);
    conv_kernel<CIN, COUT, KH, KW, BM><<<grid, (BM / 8) * (COUT / 8), 0, s>>>(a);
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}

int dispatch_conv(oww_ctx* ctx, const ConvLayer& L, const ConvArgs& a, cudaStream_t s) {
#define OWW_CASE(CI_, CO_, KH_, KW_, BM_) \
    if (L.cin == CI_ && L.cout == CO_ && L.kh == KH_ && L.kw == KW_) return launch_conv<CI_, CO_, KH_, KW_, BM_>(ctx, a, s);
    OWW_CASE(24, 24, 1, 3, 256) OWW_CASE(24, 24, 3, 1, 256)
    OWW_CASE(24, 48, 1, 3, 128) OWW_CASE(48, 48, 3, 1, 128) OWW_CASE(48, 48, 1, 3, 128)
    OWW_CASE(48, 72, 1, 3, 256) OWW_CASE(72, 72, 3, 1, 256) OWW_CASE(72, 72, 1, 3, 256)
    OWW_CASE(72, 96, 1, 3, 128) OWW_CASE(96, 96, 3, 1, 128) OWW_CASE(96, 96, 1, 3, 128)
#undef OWW_CASE
    return oww_fail(ctx, OWW_EUNSUPPORTED, "no conv kernel for %dx%d %d->%d", L.kh, L.kw, L.cin, L.cout);
}

// Runs layers 0..19 on n samples whose mel source has t_mel rows; the W embedding rows of sample i land at
// d_out + i * out_stride.
int run_pyramid(oww_ctx* ctx, const WindowSrc& src, int n, int t_mel, float* d_out, int64_t out_stride, cudaStream_t s,
                int stop_layer = -1, float* d_dbg = nullptr) {
    float* bufs[2] = {ctx->d_act[0], ctx->d_act[1]};
    int cur = 0;
    int t = t_mel, f = 32;
    int64_t stride_in = 0;
    for (int li = 0; li < OWW_N_CONV; ++li) {
        const ConvLayer& L = ctx->conv[li];
        const int t_out = t - (L.kh - 1);
        const bool last = li == OWW_N_CONV - 1;
        float* out = last ? d_out : bufs[cur];
        const int64_t stride_out = last ? out_stride : (int64_t)t_out * f * L.cout;
        if (!last && (size_t)stride_out * n > ctx->act_floats)
            return oww_fail(ctx, OWW_ENOMEM, "activation scratch too small");
        if (li == 0) {
            L0Args a{src, n, t_out, t, L.d_w, L.d_scale, L.d_bias, out, stride_out};
            const int64_t total = (int64_t)n * t_out * 32;
            unsigned grid = (unsigned)((total + 255) / 256);
            if (grid > (unsigned)ctx->sm_count * 16) grid = ctx->sm_count * 16;
            conv0_kernel<<<grid, 256, 0, s>>>(a);
            OWW_LAUNCH_CHECK(ctx);
        } else {
            ConvArgs a{bufs[cur ^ 1], stride_in, out, stride_out, L.d_w, L.d_scale, L.d_bias, n, t_out, f, last ? 0 : 1};
            int rc = dispatch_conv(ctx, L, a, s);
            if (rc) return rc;
        }
        t = t_out;
        stride_in = stride_out;
        cur ^= 1;
        if (L.pool_t) {
            const int t2 = t / L.pool_t, f2 = f / L.pool_f;
            const int64_t so = (int64_t)t2 * f2 * L.cout;
            const int64_t total = (int64_t)n * so / 4;
            unsigned grid = (unsigned)((total + 255) / 256);
            if (grid > (unsigned)ctx->sm_count * 16) grid = ctx->sm_count * 16;
            pool_kernel<<<grid, 256, 0, s>>>(bufs[cur ^ 1], stride_in, bufs[cur], so, n, t, f, L.cout, L.pool_t, L.pool_f);
            OWW_LAUNCH_CHECK(ctx);
            t = t2; f = f2; stride_in = so; cur ^= 1;
        }
        if (li == stop_layer && !last) {
            OWW_CUDA(ctx, cudaMemcpyAsync(d_dbg, bufs[cur ^ 1], (size_t)n * stride_in * sizeof(float), cudaMemcpyDeviceToDevice, s));
            return OWW_OK;
        }
    }
    return OWW_OK;
}

}  // namespace

int oww_cnn_fp32_pyramid(oww_ctx* ctx, const WindowSrc& src, int n, int T0, float* d_emb, int out_rows, int stop_layer,
                         float* d_dbg, cudaStream_t s) {
    return run_pyramid(ctx, src, n, T0, d_emb, (int64_t)out_rows * OWW_EMBEDDING_DIM, s, stop_layer, d_dbg);
}

int oww_cnn_window(oww_ctx* ctx, const WindowSrc& src, int n_windows, float* d_emb, cudaStream_t s, bool capture_tails) {
    if (!ctx->emb_loaded) return oww_fail(ctx, OWW_EINVAL, "embedding weights not loaded");
    const int wb = ctx->window_batch;
    int w0 = 0;
    while (w0 < n_windows) {
        int n = (n_windows - w0 < wb) ? n_windows - w0 : wb;
        WindowSrc sub = src;
        if (src.count) {
            // ring source: window j = chunk * n_streams + stream.  A sub-batch is either whole chunk
            // rows (stream index keeps its meaning) or a run of streams inside one chunk row.
            const int b0 = w0 % src.n_streams, i0 = w0 / src.n_streams;
            sub.n_chunks = src.n_chunks - i0;             // keeps 8*(n_chunks-1-i) for local chunk 0
            if (b0 == 0 && n >= src.n_streams) {
                n -= n % src.n_streams;
            } else {
                if (n > src.n_streams - b0) n = src.n_streams - b0;
                if (src.ids) sub.ids = src.ids + b0;          // the id list carries the offset; base / count stay global
                else { sub.base = src.base + (int64_t)b0 * src.stride; sub.count = src.count + b0; }
                sub.n_streams = n;
            }
        } else {
            sub.base = src.base + (int64_t)w0 * src.stride;
        }
        float* o = d_emb + (int64_t)w0 * OWW_EMBEDDING_DIM;
        int rc;
        if (ctx->cfg.cnn_mode == OWW_CNN_TC_WINDOW || ctx->cfg.cnn_mode == OWW_CNN_TC_INCREMENTAL) {
            TailCapture cap{0, 0, 0};
            if (capture_tails && src.count) {
                // windows of the newest chunk (global chunk index n_chunks-1) inside this sub-batch
                const int b0 = w0 % src.n_streams, i0 = w0 / src.n_streams;
                if (b0 == 0 && n >= src.n_streams) {
                    const int k = n / src.n_streams;
                    if (i0 + k == src.n_chunks) cap = TailCapture{(k - 1) * src.n_streams, src.n_streams, 0, src.ids};
                } else if (i0 == src.n_chunks - 1) {
                    cap = TailCapture{0, n, b0, src.ids};
                }
            }
            rc = oww_cnn_tc_pyramid_cap(ctx, sub, n, o, cap.n_win ? &cap : nullptr, s);
        } else {
            rc = run_pyramid(ctx, sub, n, OWW_WINDOW_ROWS, o, OWW_EMBEDDING_DIM, s);
        }
        if (rc) return rc;
        w0 += n;
    }
    return OWW_OK;
}

int oww_feat_append(oww_ctx* ctx, const float* d_emb, int n_chunks, cudaStream_t s, const int* d_ids, int n_ids) {
    const int B = d_ids ? n_ids : ctx->n_streams;
    if (B <= 0) return OWW_OK;
    const int64_t total = (int64_t)B * n_chunks * 24;
    unsigned grid = (unsigned)((total + 255) / 256);
    OWW_CUDA(ctx, oww_launch_pdl(ctx->late_pdl, feat_append_kernel, dim3(grid), dim3(256), 0, s, d_emb, ctx->d_feat_ring, ctx->d_feat_count, B,
                                 n_chunks, ctx->feat_rows - 1, (int64_t)ctx->feat_rows * 96, d_ids));
    OWW_LAUNCH_CHECK(ctx);
    OWW_CUDA(ctx, oww_launch_pdl(ctx->late_pdl, count_add_kernel, dim3((B + 255) / 256), dim3(256), 0, s, ctx->d_feat_count, B, n_chunks, d_ids));
    OWW_LAUNCH_CHECK(ctx);
    return OWW_OK;
}
