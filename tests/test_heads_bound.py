"""CPU: a per-element round-off bound for whole wake-word heads against float64: LayerNorm, ReLU, the final activations,
the gates of conditional pairs, the max over a call's windows and the custom verifiers.

This extends test_cnn_bound.py's bound of one Linear layer (linear_bound_parts) to whole heads.  The float64 reference
runs on the features the device used, so a head answers only for its own arithmetic.  Bounds are carried through the
layers as (y, A, B) with tau = C A + B: A holds the accumulation terms (sums, FMA chains, K16 steps), B the single
roundings and the propagated operand errors.

LayerNorm of a row h of D values (x^ = (h - mu) / sigma, sigma = sqrt(var + 1e-5), out = x^ g + beta), input bound tau:
  propagated, first order   |g_d| / sigma (tau_d + mean tau + |x^_d| mean(|x^| tau)) (1 + rho),   rho = 2 max tau / sigma
                            (the test asserts rho <= 1/4 on every row it judges: no input leaves the linear regime)
  its own fp32 round-off, for any summation order:
    the mean                e_mu = u D mean|h| (the sum, A) + u |mu| (the division, B); it shifts x^ by e_mu / sigma.
                            This is the term a row with |mu| >> sigma amplifies by up to 1/sqrt(eps) ~ 316.
    the variance            sum of squares u D var (A), the centring's 2 u var, the division by D u var and the + eps
                            u (var + eps) (B); sqrtf and the division 1/sigma u each: a relative error of rstd of
                            u D var / (2 (var + eps)) (A) + 4 u (B), times |x^_d|.
    the element             (v - mu) u |x^|, x rstd u |x^|, x g u |x^ g|, + beta u |out|, the fp32 eps u |x^| / 2:
                            u (|g| (|mu| / sigma + 8 |x^|) + |out|) in all (B, with the mean's and rstd's B parts).
ReLU is 1-Lipschitz and adds no round-off.
sigmoid p = 1 / (1 + exp(-z)): p (1 - p) tau_z (1 + rho), rho = expm1(tau_z) (the log of sigmoid' is 1-Lipschitz), plus
  EXP_K u p: expf's 2 ulp (4 u), the add and the divide.
softmax (relu-softmax: ReLU first) p_i: p_i (tau_i + sum_j p_j tau_j) (1 + rho), rho = expm1(2 max tau), plus
  u p_i (n + EXP_K + |z_i - m| + sum_j p_j |z_j - m|): the n-term sum, expf and the divide, and the rounding of z - m,
  which is an absolute error in the exponent.
Both take an absolute floor of 2^-126: expf(-z) overflows for z < -88.7, where the device returns 0 and p ~ 1e-39, and
the softmax's exp(z - m) underflows likewise.
Tensor-core heads (heads_mma.cuh) split each hidden row v into fp16 hi + lo of v 2^e_r (e_r: max_d v_d 2^e_r in
[2^13, 2^14), clamped to [-100, 100]); linear_bound_parts counts the lo parts' subnormal floor SUB16 per activation, so rows with e_r < 1 add
SUB16 (2^(1 - e_r) - 1) sum|W| (the 1 allows for a device row maximum on the other side of a power of two).

Gates (gate_kernel, the in-kernel gates): the device takes the verifier's score where its own main score is > thr.
Where |main - thr| <= tau_main either branch is accepted and the value must meet the bound of the branch it matches;
elsewhere the reference's branch is required.  A main whose logit is exactly 0 (zero final layer) scores exactly 0.5 on
every implementation, so at thr = 0.5 it must keep its value.
The max over a call's windows: each window gated first, then the max; |max a - max b| <= max |a - b|, so the bound of the
max is the largest bound of its windows (over every accepted branch combination).

Verifier z = b + sum (x - mu) w (verifier_kernel): the fp32 storage of mu, w and b measured against the float64
pipeline's parameters (sum |mu - mu32| |w| + sum |x - mu| |w - w32| + |b - b32|), the subtraction u S, the FMA chains and
the xor tree u (D/32 + 5) S (A), the bias add u |z|, with S = sum |x - mu| |w|; then the sigmoid as above.

Deep LayerNorm heads are outside the bound: the worst-case bound grows by ~3 sqrt(D) through each LayerNorm, so with
three LayerNorms (two at 1 term) it leaves the linear regime (rho > 1/4) on ordinary rows and says nothing there.
outside_bound lists them per path; every other head must have at least MIN_JUDGED of its live rows judged, and the list
is held to the measured fractions both ways.  Those heads stay under test_gpu_tc.py's flat budgets only.

The module checks that float32 emulations of the row-wise implementations (heads.cu and the fused kernel's heads: warp
tree sums; heads_mma.cuh: sequential sums; the tensor-core GEMMs at 3 and 1 terms with the per-row A-tile scale) pass the
bound at C_ROUNDOFF, and that each of a set of defects fails it by at least GUARD_MARGIN.  It reports which of them the
flat budgets of test_gpu_tc.py and test_gpu_verifier.py would accept.  tests/test_gpu_heads_bound.py applies the bound
to the CUDA kernels."""
import itertools

import numpy as np
import pytest
from scipy.special import expit

from helpers import HEAD_SPECS
from openwakeword_b200 import weights as W
from test_cnn_bound import (C_ROUNDOFF, GUARD_MARGIN, SUB16, U, _split16, c_needed, emulate_gemm, head_add_count,
                            head_features, linear_bound_parts, ratio, scale_exponent)

assert head_add_count(96, True, 3) == 18                  # the first layer's K16 steps per 96-wide feature row x terms
LN_EPS = 1e-5
EXP_K = 6
P_FLOOR = 2.0 ** -126
RHO_MAX = 0.25

# The flat budgets the heads and verifiers were held to before this bound, restated (those files stay as they are):
FLAT_TC3 = 2e-4         # test_gpu_tc.test_tc_heads_vs_oracle_and_cuda_core_heads: heads_tc at 3 terms, |err| / max(1, |ref|)
FLAT_CUDA_CORE = 3e-5   # test_gpu_tc.test_tc_heads_vs_oracle_and_cuda_core_heads: heads.cu, |err| / max(1, |ref|)
FLAT_IN_KERNEL = 2e-5   # test_gpu_tc.test_fused_step_heads_with_awkward_shapes: the fused kernel's heads vs a launch
FLAT_GROUPED = 5e-5     # test_gpu_tc.test_grouped_heads_match_per_head_kernels: grouped vs per-head tensor-core heads
FLAT_VERIFIER = 1e-5    # test_gpu_verifier.test_verifier_predict_vs_sklearn: verifier_predict vs scikit-learn


# ---------------------------------------------------------------------------------------------------- the bound
def _row_exponent(v):
    """The A-tile exponent of each row of v (>= 0): max 2^e in [2^13, 2^14), clamped to [-100, 100]; zero rows 0."""
    m = np.asarray(v, np.float64).max(1)
    e = 14 - np.frexp(np.where(m > 0, m, 1.0))[1]
    return np.where(m > 0, np.clip(e, -100, 100), 0)


def ln_parts(h, A, B, g, beta):
    """LayerNorm of rows h with input bound (A, B) -> (out, A, B, rho per row)."""
    D = h.shape[1]
    g64 = np.asarray(g, np.float64)
    ga = np.abs(g64)
    mu = h.mean(1, keepdims=True)
    c = h - mu
    var = (c * c).mean(1, keepdims=True)
    sig = np.sqrt(var + LN_EPS)
    xh = c / sig
    out = xh * g64 + np.asarray(beta, np.float64)
    tau = C_ROUNDOFF * A + B
    rho = 2.0 * tau.max(1, keepdims=True) / sig

    def prop(t):
        return ga / sig * (t + t.mean(1, keepdims=True) + np.abs(xh) * (np.abs(xh) * t).mean(1, keepdims=True)) * (1 + rho)
    A2 = prop(A) + U * ga * (D * np.abs(h).mean(1, keepdims=True) / sig + 0.5 * D * np.abs(xh) * var / (var + LN_EPS))
    B2 = prop(B) + U * (ga * (np.abs(mu) / sig + 8.0 * np.abs(xh)) + np.abs(out))
    return out, A2, B2, rho[:, 0]


def final_parts(final, z, A, B):
    """The final activation of raw outputs z with bound (A, B) -> (y, A, B)."""
    if final == "none":
        return z, A, B
    if final == "relu":
        return np.maximum(z, 0.0), A, B
    tau = C_ROUNDOFF * A + B
    if final == "sigmoid":
        p = expit(z)
        d = p * (1 - p) * (1 + np.expm1(np.minimum(tau, 50.0)))      # tau_z > 50: the bound is vacuous anyway
        return p, d * A, d * B + EXP_K * U * p + P_FLOOR
    assert final in ("softmax", "relu_softmax"), final
    if final == "relu_softmax":
        z = np.maximum(z, 0.0)
    n = z.shape[1]
    m = z.max(1, keepdims=True)
    e = np.exp(z - m)
    p = e / e.sum(1, keepdims=True)
    rho = np.expm1(np.minimum(2 * tau.max(1, keepdims=True), 50.0))

    def prop(t):
        return p * (t + (p * t).sum(1, keepdims=True)) * (1 + rho)
    dz = np.abs(z - m)
    own = U * p * (n + EXP_K + dz + (p * dz).sum(1, keepdims=True))
    return p, prop(A), prop(B) + own + P_FLOOR


def whole_head_parts(h, feats, terms):
    """Float64 outputs of head h on the device's features [n, n_in, 96] and their bound: (y, A, B, LN rho per row).
    terms 3 / 1: the tensor-core heads (hi/lo or fp16 operands), 0: heads.cu and the fused kernel's fp32 heads."""
    L = h["layers"]
    x = np.asarray(feats, np.float64).reshape(len(feats), -1)
    y, A, B = linear_bound_parts(x, L[0]["W"], L[0]["b"], terms, True)
    rho = np.zeros(len(x))
    for l in range(1, len(L)):
        ln = L[l - 1].get("ln")
        if ln is not None:
            y, A, B, r = ln_parts(y, A, B, *ln)
            rho = np.maximum(rho, r)
        y = np.maximum(y, 0.0)
        y2, A2, B2 = linear_bound_parts(y, L[l]["W"], L[l]["b"], terms, False, x_err=(A, B))
        if terms:
            extra = np.maximum(2.0 ** (1 - _row_exponent(y + C_ROUNDOFF * A + B)) - 1.0, 0.0)[:, None]
            B2 = B2 + SUB16 * extra * np.abs(np.asarray(L[l]["W"], np.float64)).sum(0)
        y, A, B = y2, A2, B2
    y, A, B = final_parts(h["final"], y, A, B)
    return y, A, B, rho


def gate_judge(main, ver, thr, dev, main_exact=False):
    """Options [(y, A, B)] per row of a gated column: main = (y, A, B) of the main's score, ver of the verifier's; where
    the reference's branch is not decided within tau_main, both.  main_exact: the device's main equals main's y."""
    (my, mA, mB), (vy, vA, vB) = main, ver
    amb = np.zeros_like(my, bool) if main_exact else np.abs(my - thr) <= C_ROUNDOFF * mA + mB
    take = my > thr
    first = tuple(np.where(take, v, m) for v, m in zip((vy, vA, vB), (my, mA, mB)))
    second = tuple(np.where(amb & ~take, v, np.where(amb & take, m, f)) for v, m, f in zip((vy, vA, vB), (my, mA, mB), first))
    return [first, second]


def max_judge(windows):
    """windows: per window a list of options (y, A, B); -> options of the max over the windows (every combination)."""
    out = []
    for combo in itertools.product(*windows):
        out.append((np.max([o[0] for o in combo], 0), np.max([o[1] for o in combo], 0), np.max([o[2] for o in combo], 0)))
    return out


def options_ratio(dev, options, C=C_ROUNDOFF):
    """(worst ratio, C needed) of device values against the best of several accepted references per element."""
    dev = np.asarray(dev, np.float64)
    r = np.min([np.abs(dev - y) / (C * A + B) for y, A, B in options], 0)
    r = np.where(np.isfinite(dev), r, np.inf)
    cn = np.min([np.maximum(0.0, (np.abs(dev - y) - B) / A) for y, A, B in options], 0)
    cn = np.where(np.isfinite(dev), cn, np.inf)
    return float(r.max()), float(cn.max())


def verifier_parts(feats, mean64, w64, b64, mean32, w32, b32):
    """Float64 P(positive) of a verifier (pipeline parameters mean64, w64 = coef_ / scale_, b64) on the device's
    features, and its bound for the fp32 parameters the device holds: (p, A, B)."""
    x = np.asarray(feats, np.float64).reshape(len(feats), -1)
    D = x.shape[1]
    c = x - mean64
    z = b64 + c @ w64
    S = np.abs(c) @ np.abs(w64)
    A = U * (D // 32 + 5) * S
    B = (np.abs(mean64 - np.asarray(mean32, np.float64)) @ np.abs(w64) + np.abs(c) @ np.abs(w64 - np.asarray(w32, np.float64))
         + abs(b64 - float(b32)) + U * (S + np.abs(z)))
    p, A, B = final_parts("sigmoid", z[:, None], A[:, None], B[:, None])
    return p[:, 0], A[:, 0], B[:, 0]


# ---------------------------------------------------------------------------------------------------- inputs
def rescaled_head(h, k):
    """The same float64 function with every hidden activation x 2^k: without LayerNorm the first layer's W and b and the
    later hidden layers' b x 2^k, with LayerNorm every gamma and beta x 2^k; every later layer's W x 2^-k.  Exact in
    fp32 (powers of two)."""
    f = np.float32(2.0 ** k)
    n = len(h["layers"])
    assert n >= 2
    layernorm = h["layers"][0].get("ln") is not None
    L = []
    for l, lay in enumerate(h["layers"]):
        Wl, bl, ln = lay["W"], lay["b"], lay.get("ln")
        if layernorm:
            Wl = Wl / f if l > 0 else Wl                     # the pre-LN rows stay as they were
            ln = None if ln is None else (ln[0] * f, ln[1] * f)
        else:
            Wl = Wl * f if l == 0 else (Wl / f if l == n - 1 else Wl)
            bl = bl * f if l < n - 1 else bl
        L.append({"W": np.asarray(Wl, np.float32), "b": np.asarray(bl, np.float32), "ln": ln})
    return dict(h, layers=L)


def ill_conditioned_ln_head(n_in, hidden, spread, seed, final="sigmoid", n_out=1):
    """A LayerNorm head whose first layer's columns are nearly equal (differences ~ spread) with a common bias of about
    100: every pre-LN row has |mu| >> sigma whatever the features.  spread ~ 1e-4 puts sigma^2 near eps."""
    h = W.synthetic_head(n_in=n_in, hidden=hidden, n_blocks=0, n_out=n_out, layernorm=True, final=final, seed=seed)
    rng = np.random.default_rng(seed + 1000)
    K = n_in * 96
    common = rng.standard_normal(K) / np.sqrt(K) * 0.05
    lay = h["layers"][0]
    lay["W"] = (common[:, None] + spread * rng.standard_normal((K, hidden)) / np.sqrt(K)).astype(np.float32)
    lay["b"] = (100.0 + spread * rng.standard_normal(hidden)).astype(np.float32)
    return h


def logit_head(n_in, final, offsets, seed):
    """A head whose final logits sit at the given offsets (final layer x 0.01, bias = offsets), one column each."""
    h = W.synthetic_head(n_in=n_in, hidden=30, n_blocks=0, n_out=len(offsets), layernorm=False, final=final, seed=seed)
    last = h["layers"][-1]
    last["W"] = (last["W"] * np.float32(0.01)).astype(np.float32)
    last["b"] = np.asarray(offsets, np.float32)
    return h


def zero_main(n_in, seed):
    """A sigmoid main whose final layer is zero: its score is exactly 0.5 on every implementation."""
    h = W.synthetic_head(n_in=n_in, hidden=30, n_blocks=0, n_out=1, layernorm=False, final="sigmoid", seed=seed)
    h["layers"][-1]["W"] = np.zeros_like(h["layers"][-1]["W"])
    h["layers"][-1]["b"] = np.zeros_like(h["layers"][-1]["b"])
    return h


def head_zoo(tc_only=False):
    """name -> head.  tc_only: only heads every implementation covers (layers at most 128 wide)."""
    hs = {k: W.synthetic_head(**v) for k, v in HEAD_SPECS.items()}
    finals = ("sigmoid", "softmax", "relu_softmax", "relu", "none")
    i = 0
    for ln in (True, False):
        for width in (7, 30, 64, 128, 256):
            for n_blocks, n_in in ((0, 3), (1, 16), (2, 34)):
                fin = finals[i % len(finals)]
                n_out = 1 if fin == "sigmoid" else 3 + i % 5
                i += 1
                if width == 256 and (tc_only or n_blocks == 2):
                    continue
                hs[f"{'ln' if ln else 'relu'}_w{width}_l{n_blocks + 2}_in{n_in}_{fin}"] = W.synthetic_head(
                    n_in=n_in, hidden=width, n_blocks=n_blocks, n_out=n_out, layernorm=ln, final=fin, seed=99 + i)
    hs["ill_ln_mu100"] = ill_conditioned_ln_head(16, 64, 1e-2, 201)
    hs["ill_ln_var_eps"] = ill_conditioned_ln_head(3, 30, 2e-3, 202, final="softmax", n_out=4)
    hs["sigmoid_edges"] = logit_head(3, "sigmoid", (17, -17, 30, -30, 90, -90, 105, -105), 203)
    hs["softmax_above_88.7"] = logit_head(16, "softmax", (95, 89, 100, 60, -30), 204)
    hs["relu_softmax_all_negative"] = logit_head(3, "relu_softmax", (-5, -3, -8), 205)
    return hs


RESCALE_K = (-20, -14, 17)
RESCALE_HEADS = ("timer_v0.1", "alexa_v0.1", "relu_w30_l4_in34_sigmoid", "relu_w7_l3_in16_softmax", "ln_w30_l3_in16_none")


def zoo_features(rng, n, n_in):
    f = head_features(rng, n, n_in)
    f[1::17] = rng.normal(0.0, 30.0, f[1::17].shape)        # large logits: saturated sigmoids, exp shifts
    return f


# ---------------------------------------------------------------------------------------------------- emulation
def _f32(v):
    return np.asarray(v, np.float32)


def _fma(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def _sum_seq(rows):
    s = np.zeros(rows.shape[0], np.float32)
    for d in range(rows.shape[1]):
        s = _f32(s + rows[:, d])
    return s


def _sum_warp(rows, square_of=None):
    """Lane l sums columns l, l + 32, ... (with fmaf(c, c, s) for squares), then the xor tree of 5 levels."""
    n, D = rows.shape
    lanes = np.zeros((n, 32), np.float32)
    for d in range(D):
        if square_of is None:
            lanes[:, d % 32] = _f32(lanes[:, d % 32] + rows[:, d])
        else:
            lanes[:, d % 32] = _fma(rows[:, d], rows[:, d], lanes[:, d % 32])
    for off in (16, 8, 4, 2, 1):
        lanes = _f32(lanes + lanes[:, np.arange(32) ^ off])
    return lanes[:, 0]


def emulate_ln(h, g, beta, order, defects=()):
    """fp32 LayerNorm + ReLU of rows h (float32), sums in the warp-tree or sequential order."""
    h = _f32(h)
    D = h.shape[1]
    if order == "warp":
        mu = _f32(_sum_warp(h) / np.float32(D))[:, None]
        c = _f32(h - mu)
        sq = _sum_warp(c, square_of=True)
    else:
        mu = _f32(_sum_seq(h) / np.float32(D))[:, None]
        c = _f32(h - mu)
        sq = np.zeros(len(h), np.float32)
        for d in range(D):
            sq = _fma(c[:, d], c[:, d], sq)
    if "ln_one_pass_variance" in defects:
        sq = _f32(_sum_seq(_f32(h * h)) - _f32(np.float32(D) * _f32(mu[:, 0] * mu[:, 0])))
    div = np.float32(D - 1 if "ln_unbiased_variance" in defects else D)
    eps = np.float32(1e-3 if "ln_eps_1e-3" in defects else 1e-5)
    rstd = _f32(np.float32(1.0) / np.sqrt(_f32(_f32(sq / div) + eps)))[:, None]
    g = _f32(g).copy()
    if "ln_gamma_off" in defects:
        g[0] = g[0] * np.float32(1 + GAMMA_OFF)
    return np.maximum(_fma(_f32(c * rstd), g, _f32(beta)), np.float32(0))


def emulate_final(final, z, defects=()):
    z = _f32(z)
    if final == "relu":
        return np.maximum(z, np.float32(0))
    if final == "sigmoid":
        with np.errstate(over="ignore"):
            return _f32(np.float32(1) / _f32(np.float32(1) + np.exp(-z)))
    if final in ("softmax", "relu_softmax"):
        if final == "relu_softmax":
            z = np.maximum(z, np.float32(0))
        m = np.zeros((len(z), 1), np.float32) if "softmax_no_max_shift" in defects else z.max(1, keepdims=True)
        with np.errstate(over="ignore", invalid="ignore"):
            e = np.exp(_f32(z - m))
            return _f32(e / _sum_seq(e)[:, None])
    return z


def emulate_tc_linear(x, Wl, b, terms, first, defects=()):
    """One tensor-core Linear layer on rows x (float32): the first layer's features split as they are; a later layer's
    rows x 2^e_r (heads_mma.cuh; 'hidden_split_unscaled': e_r = 0), W 2^s split, K16 steps, fmaf(acc, 2^-s 2^-e_r, b)."""
    s = scale_exponent(Wl)
    e = np.zeros(len(x), int) if first or "hidden_split_unscaled" in defects else _row_exponent(x)
    xs = _f32(x * np.exp2(e.astype(np.float64))[:, None])
    with np.errstate(over="ignore", invalid="ignore"):
        ap = list(_split16(xs))
        wp = list(_split16(np.asarray(Wl, np.float64) * 2.0 ** s))
        acc = emulate_gemm(ap, wp, ((0, 0), (0, 1), (1, 0)) if terms == 3 else ((0, 0),))
        return _fma(acc, _f32(np.exp2(-(s + e)).astype(np.float32))[:, None], _f32(b))


def emulate_head(h, feats, impl, defects=()):
    """impl 'warp': heads.cu / the fused kernel's heads (fp32 GEMMs, warp-tree LayerNorm); 'tc3' / 'tc1': heads_mma.cuh
    (tensor-core GEMMs at 3 / 1 terms, sequential LayerNorm)."""
    L = h["layers"]
    x = _f32(feats).reshape(len(feats), -1)
    for l, lay in enumerate(L):
        if impl == "warp":
            y = _f32(_f32(x @ _f32(lay["W"])) + _f32(lay["b"]))
        else:
            y = emulate_tc_linear(x, lay["W"], lay["b"], 3 if impl == "tc3" else 1, l == 0, defects)
        if l == len(L) - 1:
            return emulate_final(h["final"], y, defects)
        ln = lay.get("ln")
        x = emulate_ln(y, *ln, "warp" if impl == "warp" else "seq", defects) if ln is not None else np.maximum(y, np.float32(0))


def emulate_verifier(feats, mean32, w32, b32, defects=()):
    """verifier_kernel: lane l takes float4 l, l + 32, ... (fmaf(x - mu, w, acc)), the xor tree, the sigmoid.
    'verifier_mean_in_bias': z = (b - sum mu w) + sum x w."""
    x = _f32(feats).reshape(len(feats), -1)
    D = x.shape[1]
    mu, w = _f32(mean32), _f32(w32)
    b = np.float32(b32)
    if "verifier_mean_in_bias" in defects:
        b = np.float32(float(b32) - float(np.asarray(mean32, np.float64) @ np.asarray(w32, np.float64)))
        mu = np.zeros_like(mu)
    lanes = np.zeros((len(x), 32), np.float32)
    for j in range(D // 4):
        for q in range(4):
            d = 4 * j + q
            lanes[:, j % 32] = _fma(_f32(x[:, d] - mu[d]), w[d], lanes[:, j % 32])
    for off in (16, 8, 4, 2, 1):
        lanes = _f32(lanes + lanes[:, np.arange(32) ^ off])
    return emulate_final("sigmoid", _f32(b + lanes[:, :1]))[:, 0]


def verifier_edges(seed=0, n_in=16):
    """Float64 pipeline parameters (mean_, w = coef_ / scale_, intercept_) of D = n_in 96 = 1536 features whose |mean_|
    reaches 1e3 against a spread of 1e-2, and features drawn around them, with logits near 0 and at +-100.  mean_ is
    fp32-representable here, so the fp32 storage of mu costs nothing and a folded bias cannot hide behind it."""
    rng = np.random.default_rng(seed)
    D = n_in * 96
    mean = _f32(np.exp(rng.uniform(np.log(1e-2), np.log(1e3), D)) * rng.choice((-1.0, 1.0), D)).astype(np.float64)
    spread = 1e-2
    w = rng.standard_normal(D) / (spread * np.sqrt(D))
    b = 0.3
    n = 130
    x = mean + spread * rng.standard_normal((n, D))
    x[1::5] = mean + 70.0 * spread * rng.standard_normal((len(x[1::5]), D)) # logits ~ +-100 after the dot product
    x[2::5] = mean + spread * 0.01 * rng.standard_normal((len(x[2::5]), D))  # logits near b
    return mean, w, b, _f32(x).reshape(n, n_in, 96)


def verifier_pipeline(seed=1, n_in=16):
    """A float64 pipeline whose mean_ is not fp32-representable: the storage term counts."""
    mean, w, b, x = verifier_edges(seed, n_in)
    mean = mean * (1 + 1e-9)
    return mean, w, b, x


# ---------------------------------------------------------------------------------------------------- tests
GAMMA_OFF = 2.0 ** -5


def judged_rows(rho):
    """The rows the bound judges: those whose LayerNorms stay in the linear regime (rho <= RHO_MAX)."""
    return rho <= RHO_MAX


MIN_JUDGED = 0.75
# Heads outside the bound, per path (terms 0: heads.cu and the fused kernel's heads, 3 / 1: the tensor-core heads).  The
# worst-case bound grows by ~3 sqrt(D) through each LayerNorm (sum |W| tau, then |g| / sigma), so with three LayerNorms
# (two at 1 term, whose fp16 operand term is 2^-10 S) it leaves the linear regime on ordinary rows: it says nothing
# there, and these heads stay under the flat budgets of test_gpu_tc.py only.  ill_ln_var_eps (sigma^2 ~ eps) is outside
# at 1 term for the same reason.  test_emulated_heads_pass_the_bound holds this list to the measured fractions both ways.
def outside_bound(h, terms, name=""):
    n_ln = sum(l.get("ln") is not None for l in h["layers"])
    return n_ln >= (2 if terms == 1 else 3) or (terms == 1 and name == "ill_ln_var_eps")


def judged_fraction(feats, rho):
    """The fraction of the rows with any non-zero feature that the bound judges (zero rows all give one output)."""
    live = np.abs(np.asarray(feats)).reshape(len(feats), -1).max(1) > 0
    return float((judged_rows(rho) & live).sum() / max(1, live.sum()))


def _judge(h, f, impl, defects=()):
    """-> (worst ratio, C needed, judged fraction of the live rows, device values and references of the judged rows)."""
    terms = {"warp": 0, "tc3": 3, "tc1": 1}[impl]
    y, A, B, rho = whole_head_parts(h, f, terms)
    k = judged_rows(rho)
    dev = emulate_head(h, f, impl, defects)
    if not k.any():
        return 0.0, 0.0, 0.0, dev[k], y[k]
    return (ratio(dev[k], y[k], C_ROUNDOFF * A[k] + B[k]), c_needed(dev[k], y[k], A[k], B[k]), judged_fraction(f, rho),
            dev[k], y[k])


@pytest.fixture(scope="module")
def zoo():
    return head_zoo()


@pytest.mark.parametrize("impl", ["warp", "tc3", "tc1"])
def test_emulated_heads_pass_the_bound(zoo, impl):
    """Every head within the bound on the rows it judges; a head not listed by outside_bound has at least MIN_JUDGED of
    its live rows judged, and a listed one fewer (so the list is exact)."""
    rng = np.random.default_rng(7)
    terms = {"warp": 0, "tc3": 3, "tc1": 1}[impl]
    worst, wrong = 0.0, []
    for name, h in zoo.items():
        if impl != "warp" and any(l["W"].shape[1] > 128 for l in h["layers"]):
            continue
        f = zoo_features(rng, 130, h["n_in"])
        r, cn, frac, _, _ = _judge(h, f, impl)
        out = outside_bound(h, terms, name)
        print(f"{impl} {name}: worst ratio {r:.3g} at C = {C_ROUNDOFF:g} (C needed {cn:.3g}); live rows judged "
              f"{frac:.2f}{' (outside the bound)' if out else ''}")
        assert r <= 1.0, name
        if out != (frac < MIN_JUDGED):
            wrong.append((name, frac))
        worst = max(worst, r)
    print(f"{impl}: worst ratio {worst:.3g}")
    assert not wrong, wrong


@pytest.mark.parametrize("impl", ["warp", "tc3", "tc1"])
@pytest.mark.parametrize("k", RESCALE_K)
def test_rescaled_heads_pass_the_original_bound(zoo, impl, k):
    """x 2^k hidden activations: the same float64 function, judged against the original head's (y, tau)."""
    rng = np.random.default_rng(8)
    for name in RESCALE_HEADS:
        h = zoo[name]
        f = zoo_features(rng, 130, h["n_in"])
        y, A, B, rho = whole_head_parts(h, f, {"warp": 0, "tc3": 3, "tc1": 1}[impl])
        m = judged_rows(rho)
        dev = emulate_head(rescaled_head(h, k), f, impl)
        r = ratio(dev[m], y[m], C_ROUNDOFF * A[m] + B[m])
        print(f"{impl} {name} x2^{k}: worst ratio {r:.3g}")
        assert r <= 1.0, (name, k)


def test_rescaled_heads_are_the_same_function(zoo):
    rng = np.random.default_rng(9)
    for name in RESCALE_HEADS:
        h = zoo[name]
        f = zoo_features(rng, 20, h["n_in"])
        y = whole_head_parts(h, f, 3)[0]
        for k in RESCALE_K:
            assert np.allclose(whole_head_parts(rescaled_head(h, k), f, 3)[0], y, rtol=1e-12, atol=1e-300), (name, k)


def test_ill_conditioned_rows_are_what_they_claim(zoo):
    rng = np.random.default_rng(10)
    for name in ("ill_ln_mu100", "ill_ln_var_eps"):
        h = zoo[name]
        f = zoo_features(rng, 130, h["n_in"])
        pre = np.asarray(f, np.float64).reshape(130, -1) @ np.asarray(h["layers"][0]["W"], np.float64) + h["layers"][0]["b"]
        mu, var = np.abs(pre.mean(1)), pre.var(1)
        print(f"{name}: min |mu| / sigma {np.min(mu / np.sqrt(var)):.3g}, median sigma^2 {np.median(var):.3g}")
        assert np.min(mu / np.sqrt(var)) > 50, name
        if name == "ill_ln_var_eps":
            assert 0.1 * LN_EPS < np.median(var) < 10 * LN_EPS


def small_head(seed):
    """A sigmoid head of 3 feature rows and one hidden layer of 7, whose scores straddle 0.5."""
    return W.synthetic_head(n_in=3, hidden=7, n_blocks=0, n_out=1, layernorm=False, final="sigmoid", seed=seed)


def test_gated_pair_and_call_max_emulation():
    rng = np.random.default_rng(11)
    ver = small_head(41)
    for main, exact in ((zero_main(3, 42), True), (small_head(43), False)):
        wins = []
        devs = {"gt": [], "ge": []}
        for w in range(3):
            f = zoo_features(rng, 130, 3)
            my, mA, mB, _ = whole_head_parts(main, f, 0)
            vy, vA, vB, _ = whole_head_parts(ver, f, 0)
            m_dev, v_dev = emulate_head(main, f, "warp"), emulate_head(ver, f, "warp")
            if exact:
                assert np.all(m_dev == 0.5) and np.all(my == 0.5)
            opts = gate_judge((my, mA, mB), (vy, vA, vB), 0.5, None, main_exact=exact)
            wins.append(opts)
            devs["gt"].append(np.where(m_dev > 0.5, v_dev, m_dev))
            devs["ge"].append(np.where(m_dev >= 0.5, v_dev, m_dev))
            r, _ = options_ratio(devs["gt"][-1], opts)
            assert r <= 1.0
        r, cn = options_ratio(np.max(devs["gt"], 0), max_judge(wins))
        print(f"gated pair (exact main {exact}): 3-window call max worst ratio {r:.3g} (C needed {cn:.3g})")
        assert r <= 1.0


def test_verifier_emulation_passes_the_bound():
    for mean, w, b, x in (verifier_edges(), verifier_pipeline()):
        m32, w32, b32 = _f32(mean), _f32(w), np.float32(b)
        p, A, B = verifier_parts(x, mean, w, b, m32, w32, b32)
        dev = emulate_verifier(x, m32, w32, b32)
        z = b + (np.asarray(x, np.float64).reshape(len(x), -1) - mean) @ w
        assert np.abs(z).max() > 90 and np.abs(z).min() < 1
        r, cn = ratio(dev, p, C_ROUNDOFF * A + B), c_needed(dev, p, A, B)
        print(f"verifier: worst ratio {r:.3g} (C needed {cn:.3g})")
        assert r <= 1.0


# name -> (what it runs, flat budget it is reported against)
GUARDS = {
    "ln_one_pass_variance": ("warp", "ill_ln_mu100", FLAT_CUDA_CORE),
    "ln_eps_1e-3": ("warp", "ill_ln_var_eps", FLAT_CUDA_CORE),
    "ln_unbiased_variance": ("warp", "ln_w7_l2_in3_sigmoid", FLAT_CUDA_CORE),
    "ln_gamma_off": ("tc3", "ln_w7_l2_in3_sigmoid", FLAT_TC3),
    "softmax_no_max_shift": ("warp", "softmax_above_88.7", FLAT_CUDA_CORE),
    "gate_ge": ("warp", None, FLAT_IN_KERNEL),
    "call_max_newest": ("warp", None, FLAT_IN_KERNEL),
    "verifier_mean_in_bias": ("verifier", None, FLAT_VERIFIER),
    "hidden_split_unscaled": ("tc3", None, FLAT_TC3),
}


def _flat_pass(dev, ref, budget):
    dev = np.asarray(dev, np.float64)
    return bool(np.isfinite(dev).all() and (np.abs(dev - ref) / np.maximum(1.0, np.abs(ref))).max() < budget)


def _guard(name, zoo):
    """-> (worst ratio, whether the flat budget accepts the defective output)."""
    impl, hname, budget = GUARDS[name]
    rng = np.random.default_rng(12)
    if hname is not None:
        h = zoo[hname]
        f = zoo_features(rng, 130, h["n_in"])
        r, _, _, dev, y = _judge(h, f, impl, (name,))
        flat = _flat_pass(dev, y, budget)
        if name.startswith("ln_"):                       # and on every other LayerNorm head inside the bound
            caught, inside = [], []
            terms = {"warp": 0, "tc3": 3}[impl]
            for other, g in zoo.items():
                if g["layers"][0].get("ln") is None or outside_bound(g, terms, other) or other == hname \
                        or (impl != "warp" and any(l["W"].shape[1] > 128 for l in g["layers"])):
                    continue
                f2 = zoo_features(rng, 130, g["n_in"])
                r2 = _judge(g, f2, impl, (name,))[0]
                inside.append(other)
                if r2 >= GUARD_MARGIN:
                    caught.append(other)
            print(f"  {name} also fails the bound by >= {GUARD_MARGIN:g}x on {len(caught)} of the {len(inside)} other "
                  f"LayerNorm heads inside it: {', '.join(caught)}")
        return r, flat
    if name == "verifier_mean_in_bias":
        mean, w, b, x = verifier_edges()
        m32, w32 = _f32(mean), _f32(w)
        p, A, B = verifier_parts(x, mean, w, b, m32, w32, np.float32(b))
        dev = emulate_verifier(x, m32, w32, np.float32(b), (name,))
        return ratio(dev, p, C_ROUNDOFF * A + B), _flat_pass(dev, p, budget)
    if name == "hidden_split_unscaled":
        worst, flat = 0.0, True
        for hname in RESCALE_HEADS:
            h = zoo[hname]
            f = zoo_features(rng, 130, h["n_in"])
            y, A, B, rho = whole_head_parts(h, f, 3)
            m = judged_rows(rho)
            for k in RESCALE_K:
                dev = emulate_head(rescaled_head(h, k), f, "tc3", (name,))[m]
                r = ratio(dev, y[m], C_ROUNDOFF * A[m] + B[m])
                print(f"  {hname} x2^{k}: worst ratio {r:.3g}")
                worst, flat = max(worst, r), flat and _flat_pass(dev, y[m], budget)
        return worst, flat
    main, ver = zero_main(3, 42), small_head(41)
    wins, devs, refs = [], [], []
    for _ in range(3 if name == "call_max_newest" else 1):
        f = zoo_features(rng, 130, 3)
        if name == "call_max_newest":
            main = small_head(43)
        m, v = whole_head_parts(main, f, 0)[:3], whole_head_parts(ver, f, 0)[:3]
        m_dev, v_dev = emulate_head(main, f, "warp"), emulate_head(ver, f, "warp")
        wins.append(gate_judge(m, v, 0.5, None, main_exact=name == "gate_ge"))
        devs.append(np.where(m_dev >= 0.5, v_dev, m_dev) if name == "gate_ge" else np.where(m_dev > 0.5, v_dev, m_dev))
        refs.append(np.where(m[0] > 0.5, v[0], m[0]))
    if name == "call_max_newest":
        r, _ = options_ratio(devs[-1], max_judge(wins))
        return r, _flat_pass(devs[-1], np.max(refs, 0), budget)
    r, _ = options_ratio(devs[0], wins[0])
    return r, _flat_pass(devs[0], refs[0], budget)


@pytest.mark.parametrize("name", list(GUARDS))
def test_defects_fail_the_bound(zoo, name):
    r, flat = _guard(name, zoo)
    print(f"\n{name}: worst ratio {r:.3g} at C = {C_ROUNDOFF:g}; flat budget {GUARDS[name][2]:g}: "
          f"{'PASS (the flat budget cannot see it)' if flat else 'fail'}")
    assert r >= GUARD_MARGIN, (name, r)


def test_report_which_guards_the_flat_budgets_accept(zoo):
    accepted = [name for name in GUARDS if _guard(name, zoo)[1]]
    print("\nguards the flat budgets accept:", ", ".join(accepted) or "none")
    # On these inputs the flat budgets catch every guard too: the bound's gain is that it holds each element to its own
    # round-off (a flat budget relative to max(1, |ref|) cannot tell a saturated sigmoid's 1e-30 from 0), not that these
    # particular defects escape the flat budgets.  A guard they accept would show up here.
    assert accepted == [], accepted
