"""CPU: a per-element round-off bound for the embedding CNN's layers and the heads' Linear layers against float64.

The CNN is judged one layer at a time.  The reference computes layer l in float64 from the tensor the device handed to
it (the device's output of layer l-1, or the mel windows for layer 0): conv, folded BN, leaky, clamp and pool, through
oracle.embedding's _conv and _pool.  Errors do not compound, so each kernel answers for its own arithmetic only.

With S = sum |a_k| |w_k| over an output element's products (_conv on absolute values), the conv's bound is

    C u n S                                   u = 2^-24, n = the accumulator's add count: K16 steps x MMA terms on the
                                              tensor cores, K for an FMA chain (the CUDA cores)
  + 2^-11 S                                   fp16 operands (the activations arrive as fp16, the weights are rounded)
    or 3 2^-22 S                              hi/lo operands (hi.hi + lo.hi + hi.lo; lo.lo and the lo parts' own
                                              rounding are left out)
  + 2^-25 sum|w| + 2^-25 2^-s sum|a|          fp16 subnormals: the activation's lo part and the weight's part of
                                              W 2^s, where s is the packing's per-layer exponent (scale_exponent)

It is carried through the epilogue (x |scale|, + the fmaf and leaky roundings, 2 u |v|; leaky, clamp and max-pool are
1-Lipschitz, so a pooled element takes the largest bound of its window) and the store: 2^-11 |y| + 2^-25 for fp16
planes, (2^-22 + 2^-24) |y| + 2^-25 for hi/lo planes read back as hi + lo in fp32, u |y| for fp32.  The device output is
compared with the unrounded float64 value, so rounding ties need no special case.

This module checks that a float32 emulation of the kernels (operands exactly as packed, one fp32 rounding per K16
block and MMA term, in the kernels' term order) passes the bound at the constant C the GPU tests hold the kernels to,
and that each of a set of small defects fails it by at least 2x.  tests/test_gpu_cnn_bound.py applies the same bounds
to the CUDA kernels."""
import numpy as np
import pytest

from helpers import emb_weights
from oracle import embedding as E
from openwakeword_b200 import weights as Wt

U = 2.0 ** -24
# Round-off constant of the bound: the smallest power of two at least 4x the worst C the CUDA kernels need (the largest
# (|dev - y| - B) / A over all elements, which tests/test_gpu_cnn_bound.py prints per layer, mode, split point and
# weight set).  Measured on an H100 80GB HBM3 (700 W limit): 0.144 on the CNN (cnn_fp32.cu; 0.109 on the tensor-core
# layers) and 0.025 on the heads (heads_tc at 3 terms; 0.003 in the fused kernel's heads), so C = 1.  The worst ratio at C = 1 is 0.994: fp16 stores, whose rounding (2^-11 |y|)
# the bound states exactly.  Above 2 the BN-scale guard would lose its 2x margin (3.7x at C = 1, 2.04x at C = 2).
C_ROUNDOFF = 1.0
GUARD_MARGIN = 2.0
N_CONV = len(E.LAYERS)
SPLIT_OP = 3.0 * 2.0 ** -22
FP16_OP = 2.0 ** -11
SUB16 = 2.0 ** -25                      # half the fp16 subnormal spacing


def scale_exponent(w):
    """The packing's exponent s of one weight tensor: max |w| 2^s in [2^13, 2^14), clamped to [-8, 24]."""
    amax = float(np.max(np.abs(w)))
    if not amax > 0 or not np.isfinite(amax):
        return 0
    return int(min(24, max(-8, 14 - int(np.frexp(amax)[1]))))


def layer_params(weights):
    """[(w HWIO, folded scale, bias)] per conv layer, float32, exactly as oww_load_embedding receives them."""
    blob = Wt.pack_embedding_blob(weights)
    out, off = [], 0
    for kh, kw, cin, cout, _ in E.LAYERS:
        nw = kh * kw * cin * cout
        w = blob[off:off + nw].reshape(kh, kw, cin, cout)
        out.append((w, blob[off + nw:off + nw + cout], blob[off + nw + cout:off + nw + 2 * cout]))
        off += nw + 2 * cout
    return out


def scaled_weights(weights, k):
    """The same network with conv layers 0..18 x 2^k and their BatchNorms compensating (gamma 2^-k, moving mean 2^k):
    every folded scale is 2^-k times the original and every bias is unchanged, bit for bit.  Layer 19 is unscaled."""
    f = np.float32(2.0 ** k)
    conv = [c * f if li < N_CONV - 1 else c for li, c in enumerate(weights["conv"])]
    bn = [(g / f, beta, m * f, v) for g, beta, m, v in weights["bn"]]
    return {"conv": conv, "bn": bn}


def layer_modes(li, cnn_mode, split_from):
    """(operands, store) of conv layer li: operands 'f32' (CUDA-core FMA chains), 'fp16' or 'split'; store 'f16',
    'split' (hi and lo planes) or 'f32'."""
    if cnn_mode == 0:
        return "f32", "f32"
    ops = "f32" if li == 0 else ("split" if li >= split_from else "fp16")
    if li == N_CONV - 1:
        return ops, "f32"
    return ops, ("split" if li + 1 >= split_from else "f16")


def add_count(li, operands):
    kh, kw, cin, _, _ = E.LAYERS[li]
    if operands == "f32":
        return kh * kw * cin
    return kh * kw * -(-cin // 16) * (3 if operands == "split" else 1)


def store_bound(y, store):
    a = np.abs(y)
    if store == "f16":
        return FP16_OP * a + SUB16
    if store == "split":
        return (2.0 ** -22 + U) * a + SUB16
    return U * a


def layer_bound_parts(li, x, w, scale, bias, operands, store):
    """Float64 reference of conv layer li computed from the device's input x [N, T, F, cin] (layer 0: the mel windows
    [N, 76, 32]), after the layer's pool, and its bound split as tau = C * A + B: (y, A, B).  A and B are pooled apart,
    which can only widen the bound."""
    kh, kw, cin, cout, pool = E.LAYERS[li]
    x = np.asarray(x, np.float64)
    if li == 0:
        x = x[..., None]
    w64 = np.asarray(w, np.float64)
    z = E._conv(x, w64, np.float64)
    S = E._conv(np.abs(x), np.abs(w64), np.float64)
    A = U * add_count(li, operands) * S
    B = np.zeros_like(S)
    if operands != "f32":
        sum_a = E._conv(np.abs(x), np.ones((kh, kw, cin, 1)), np.float64)
        B = (FP16_OP if operands == "fp16" else SPLIT_OP) * S + SUB16 * np.abs(w64).sum((0, 1, 2)) \
            + SUB16 * 2.0 ** -scale_exponent(w) * sum_a
    if li == 0:
        z = np.maximum(z, 0.0)
    sc, b = np.asarray(scale, np.float64), np.asarray(bias, np.float64)
    v = z * sc + b
    A, B = A * np.abs(sc), B * np.abs(sc)
    if li < N_CONV - 1:
        y, B = np.maximum(np.maximum(float(E.LEAK) * v, v), float(E.FLOOR)), B + 2 * U * np.abs(v)
    else:
        y, B = v, B + U * np.abs(v)
    if pool is not None:
        y, A, B = E._pool(y, *pool), E._pool(A, *pool), E._pool(B, *pool)
    return y, A, B + store_bound(y, store)


def layer_bound(li, x, w, scale, bias, operands, store, C=C_ROUNDOFF):
    """(y, tau) of conv layer li (layer_bound_parts)."""
    y, A, B = layer_bound_parts(li, x, w, scale, bias, operands, store)
    return y, C * A + B


def ratio(dev, y, tau):
    """Worst |dev - y| / tau; inf where the device value is not finite."""
    dev = np.asarray(dev, np.float64)
    r = np.abs(dev - y) / tau
    return float(np.where(np.isfinite(dev), r, np.inf).max())


def c_needed(dev, y, A, B):
    """The smallest C at which every element passes (0 when the C-free part B alone covers every error)."""
    dev = np.asarray(dev, np.float64)
    if not np.isfinite(dev).all():
        return np.inf
    return float(max(0.0, ((np.abs(dev - y) - B) / A).max()))


# ---------------------------------------------------------------------------------------------------- inputs
def bound_windows(n_noise, seed=0):
    """(groups, mel windows [n, 76, 32] float32): the frontend zoo's signals, silence, the all-ones reset window, windows
    half at the -80 dB floor (many equal values, so many hi ties in the pools) and noise at three levels."""
    from oracle import mel
    from test_frontend_bound import zoo
    L = 12400 + 512
    groups, wins = [], []
    for g, x in zoo(L, seed=7):
        groups.append("zoo_" + g)
        wins.append(mel.melspectrogram(x)[:76])
    groups.append("silence")
    wins.append(mel.melspectrogram(np.zeros(L, np.int16))[:76])
    groups.append("ones")
    wins.append(np.ones((76, 32), np.float32))
    rng = np.random.default_rng(seed)
    for k in range(2):
        m = mel.melspectrogram(np.clip(rng.normal(0, 8000, L), -32768, 32767).astype(np.int16))[:76].copy()
        if k == 0:
            m[38:] = m.max() - 8.0                      # x/10 + 2 scale: 80 dB below the window's maximum
        else:
            m[:, 16:] = m.max() - 8.0
        groups.append("half_floor")
        wins.append(m)
    for i in range(n_noise):
        amp = (300, 3000, 12000)[i % 3]
        groups.append(f"noise_{amp}")
        wins.append(mel.melspectrogram(np.clip(rng.normal(0, amp, L), -32768, 32767).astype(np.int16))[:76])
    return groups, np.stack(wins).astype(np.float32)


# ---------------------------------------------------------------------------------------------------- emulation
def _f16(v):
    return np.asarray(v, np.float32).astype(np.float16).astype(np.float64)


def _split16(v):
    v = np.asarray(v, np.float32)
    hi = v.astype(np.float16)
    return hi.astype(np.float64), (v - hi.astype(np.float32)).astype(np.float16).astype(np.float64)


def _im2col(x, kh, kw, pad_column=True):
    """[N, T, F, C] -> [N * To * F, kh * kw * C16], each tap's channels zero-padded to a multiple of 16 (the K16 steps).
    pad_column=False: a (1,3) tap reads the neighbouring position in (window, t, f) order, across the row's end."""
    N, T, F, Cn = x.shape
    c16 = -(-Cn // 16) * 16
    x = np.pad(np.asarray(x, np.float64), ((0, 0), (0, 0), (0, 0), (0, c16 - Cn)))
    if kw == 3:
        xp = np.pad(x, ((0, 0), (0, 0), (1, 1), (0, 0)))
        if not pad_column:
            flat = x.reshape(-1, c16)
            prev = np.concatenate([np.zeros((1, c16)), flat[:-1]]).reshape(x.shape)
            nxt = np.concatenate([flat[1:], np.zeros((1, c16))]).reshape(x.shape)
            xp[:, :, 0], xp[:, :, F + 1] = prev[:, :, 0], nxt[:, :, F - 1]
        x = xp
    To = T - kh + 1
    cols = [x[:, dt:dt + To, df:df + F, :] for dt in range(kh) for df in range(kw)]
    return np.concatenate(cols, axis=-1).reshape(-1, kh * kw * c16)


def _pad_weights(w):
    kh, kw, cin, cout = w.shape
    c16 = -(-cin // 16) * 16
    return np.pad(np.asarray(w, np.float64), ((0, 0), (0, 0), (0, c16 - cin), (0, 0))).reshape(kh * kw * c16, cout)


def emulate_gemm(a_parts, b_parts, terms):
    """fp32 accumulation in K16 steps: each step's products summed exactly and rounded once to fp32, then added to the fp32
    accumulator; the (a part, b part) terms in the kernels' order: every step with the hi activations first ((0, 0),
    (0, 1)), then every step with the lo activations ((1, 0))."""
    K = a_parts[0].shape[1]
    acc = np.zeros((a_parts[0].shape[0], b_parts[0].shape[1]), np.float32)
    for ph in (0, 1):
        for k in range(0, K, 16):
            for ta, tb in terms:
                if ta == ph:
                    acc = acc + (a_parts[ta][:, k:k + 16] @ b_parts[tb][k:k + 16]).astype(np.float32)
    return acc


SPLIT_TERMS = ((0, 0), (0, 1), (1, 0))
BN_GUARD = (12, 7)                      # (layer, channel) of the BN-scale defect


def emulate_layer(li, x, w, scale, bias, operands, store, defects=()):
    """conv layer li as the kernels compute it, in float32 on the CPU; x is the (emulated) device input.  defects name
    the perturbations the bound must catch (GUARDS)."""
    kh, kw, cin, cout, pool = E.LAYERS[li]
    if li == 0:                                          # tc_conv0_kernel / cnn_fp32.cu: fp32 FMA chain of 9 taps
        xp =np.pad(np.asarray(x, np.float64), ((0, 0), (0, 0), (1, 1)))
        N, T = x.shape[0], x.shape[1] - 2
        acc = np.zeros((N, T, 32, cout), np.float32)
        for dt in range(3):
            for df in range(3):
                acc = (acc + xp[:, dt:dt + T, df:df + 32, None] * np.asarray(w[dt, df, 0], np.float64)).astype(np.float32)
        acc = np.maximum(acc, np.float32(0)).reshape(-1, cout)
        s = 0
    else:
        A = _im2col(x, kh, kw, "no_pad_column" not in defects)
        if operands == "f32":
            acc = (A @ _pad_weights(w)).astype(np.float32)
            s = 0
        elif operands == "fp16":
            s = 0 if "plain_unscaled" in defects else scale_exponent(w)
            acc = emulate_gemm([A], [_f16(_pad_weights(w) * 2.0 ** s)], [(0, 0)])
        else:
            s = scale_exponent(w)
            terms = [(0, 0)] if "one_term" in defects else \
                [t for t in SPLIT_TERMS if not ("no_hi_lo" in defects and t == (0, 1)) and not ("no_lo_hi" in defects and t == (1, 0))]
            acc = emulate_gemm(list(_split16(A)), list(_split16(_pad_weights(w) * 2.0 ** s)), terms)
    sc = np.asarray(scale, np.float32) * np.float32(2.0 ** -s)
    if "bn_scale" in defects and li == BN_GUARD[0]:
        sc = sc.copy()
        sc[BN_GUARD[1]] *= np.float32(1 + 2.0 ** -12)
    v = (acc.astype(np.float64) * sc + np.asarray(bias, np.float64)).astype(np.float32)
    if li < N_CONV - 1:
        v = np.maximum(np.maximum(E.LEAK * v, v), E.FLOOR)
    To = x.shape[1] - kh + 1
    y = v.reshape(x.shape[0], To, 32 if li == 0 else x.shape[2], cout)
    if store == "f16" or (li == N_CONV - 1 and "layer19_fp16" in defects):
        y = y.astype(np.float16).astype(np.float32)
    elif store == "split":
        hi, lo = _split16(y)
        if pool is not None and "hi_only_pool" in defects:
            N, T, F, Cc = y.shape
            pt, pf = pool
            T2, F2 = T // pt, F // pf

            def win(a):
                a = a[:, :T2 * pt, :F2 * pf].reshape(N, T2, pt, F2, pf, Cc)
                return a.transpose(0, 1, 3, 5, 2, 4).reshape(N, T2, F2, Cc, pt * pf)
            h, l_ = win(hi), win(lo)
            k = np.argmax(h, axis=-1)[..., None]
            return (np.take_along_axis(h, k, -1) + np.take_along_axis(l_, k, -1))[..., 0].astype(np.float32)
        y = (hi + lo).astype(np.float32)
    if pool is not None:
        y = E._pool(y, *pool)
    return y


def run_layers(params, wins, cnn_mode, split_from, defects=(), C=C_ROUNDOFF):
    """Emulated device, each layer fed the previous emulated output: ([device output per layer], [ratio per layer])."""
    outs, ratios, x = [], [], wins
    for li, (w, s, b) in enumerate(params):
        ops, store = layer_modes(li, cnn_mode, split_from)
        y_dev = emulate_layer(li, x, w, s, b, ops, store, defects)
        y, tau = layer_bound(li, x, w, s, b, ops, store, C)
        outs.append(y_dev)
        ratios.append(ratio(y_dev, y, tau))
        x = y_dev
    return outs, ratios


def reference_chain(params, wins, split_from):
    """The float64 chain the flat budgets compare against: at split_from 2 layer 1 on fp16 operands with its input stored
    as fp16 (test_gpu_tc's fp16-below oracle), otherwise the exact oracle."""
    x, out = np.asarray(wins, np.float64)[..., None], []
    for li, ((kh, kw, cin, cout, pool), (w, s, b)) in enumerate(zip(E.LAYERS, params)):
        a, wt = x, np.asarray(w, np.float64)
        if split_from == 2 and li == 1:
            up = 2.0 ** scale_exponent(w)
            a, wt = _f16(a), _f16(wt * up) / up
        z = E._conv(a, wt, np.float64)
        if li == 0:
            z = np.maximum(z, 0)
        v = z * np.asarray(s, np.float64) + np.asarray(b, np.float64)
        x = np.maximum(np.maximum(float(E.LEAK) * v, v), float(E.FLOOR)) if li < N_CONV - 1 else v
        if pool is not None:
            x = E._pool(x, *pool)
        out.append(x)
    return out


def flat_budgets_pass(outs, ref, split_from):
    """Would test_gpu_tc.test_tc_layers_vs_oracle accept these layer outputs?  Its own budgets (LAYER_BUDGET,
    layer_max_budget), against reference_chain."""
    from test_gpu_tc import LAYER_BUDGET, layer_max_budget
    _, _, mean_b, emb_b = LAYER_BUDGET[split_from]
    for li in range(N_CONV - 1):
        r = ref[li] if not (split_from == 2 and li == 0) else _f16(ref[li])
        e = np.abs(outs[li] - r)
        if not np.isfinite(outs[li]).all() or e.max() / max(np.abs(r).max(), 1.0) >= layer_max_budget(split_from, li) \
                or e.mean() >= mean_b:
            return False
    return bool(np.abs(outs[-1] - ref[-1]).max() < emb_b)


# name -> (split point, weight scale exponent, defects)
GUARDS = {"split_layers_one_term": (2, 0, ("one_term",)),
          "hi_lo_missing": (2, 0, ("no_hi_lo",)),
          "lo_hi_missing": (2, 0, ("no_lo_hi",)),
          "hi_only_pool": (2, 0, ("hi_only_pool",)),
          "no_pad_column": (2, 0, ("no_pad_column",)),
          "bn_scale_off_2^-12": (2, 0, ("bn_scale",)),
          "layer19_stored_fp16": (2, 0, ("layer19_fp16",)),
          "unscaled_plain_packing_x2^-14": (20, -14, ("plain_unscaled",))}
# configurations the emulation must pass: (cnn_mode, split point, weight scale exponent)
CONFIGS = [(2, 2, 0), (2, 11, 0), (2, 20, 0), (2, 20, -14), (2, 11, -14), (2, 20, 17), (0, 20, 0)]


@pytest.fixture(scope="module")
def windows():
    return bound_windows(6)[1]


def _params(k):
    w = emb_weights(0)
    return layer_params(w if k == 0 else scaled_weights(w, k))


def test_scaled_weight_sets_fold_to_the_same_network():
    """x 2^k weights with compensating BN: folded scales exactly 2^-k times the original, biases bit for bit equal."""
    base = _params(0)
    for k in (-14, 17):
        for li, ((w0, s0, b0), (w1, s1, b1)) in enumerate(zip(base, _params(k))):
            f = 2.0 ** k if li < N_CONV - 1 else 1.0
            assert np.array_equal(w1, w0 * np.float32(f)) and np.array_equal(s1, s0 / np.float32(f)) and np.array_equal(b1, b0)


def test_scale_exponent_matches_the_packing_rule():
    assert scale_exponent(np.array([0.75])) == 14 and scale_exponent(np.array([1.0])) == 13
    assert scale_exponent(np.array([2.0 ** -40])) == 24 and scale_exponent(np.array([1e8])) == -8
    assert scale_exponent(np.zeros(3)) == 0
    for w in (np.array([0.3, -5.5]), np.array([2.0 ** -9]), np.array([3000.0])):
        s = scale_exponent(w)
        assert 2.0 ** 13 <= np.abs(w).max() * 2.0 ** s < 2.0 ** 14


@pytest.mark.parametrize("cnn_mode,split_from,k", CONFIGS)
def test_emulated_kernels_pass_the_bound(windows, cnn_mode, split_from, k):
    _, ratios = run_layers(_params(k), windows, cnn_mode, split_from)
    print(f"\ncnn_mode {cnn_mode} split {split_from} weights x2^{k}: worst ratio per layer at C = {C_ROUNDOFF:g}:",
          " ".join(f"{r:.3f}" for r in ratios))
    assert max(ratios) <= 1.0, ratios


@pytest.mark.parametrize("name", sorted(GUARDS))
def test_defects_fail_the_bound(windows, name):
    split_from, k, defects = GUARDS[name]
    params = _params(k)
    outs, ratios = run_layers(params, windows, 2, split_from, defects)
    flat = flat_budgets_pass(outs, reference_chain(params, windows, split_from), split_from)
    worst = int(np.argmax(ratios))
    print(f"\n{name}: worst ratio {ratios[worst]:.3g} (layer {worst}) at C = {C_ROUNDOFF:g}; "
          f"test_gpu_tc's flat budgets at split {split_from}: {'PASS' if flat else 'fail'}")
    assert ratios[worst] >= GUARD_MARGIN, (name, ratios)


def test_flat_budgets_pass_the_defect_free_emulation(windows):
    """The flat budgets are met by the emulation itself, so a guard they pass is a defect they cannot see."""
    for split_from in (2, 20):
        params = _params(0)
        outs, _ = run_layers(params, windows, 2, split_from)
        assert flat_budgets_pass(outs, reference_chain(params, windows, split_from), split_from), split_from


# ---------------------------------------------------------------------------------------------------- heads
def head_add_count(K, first, terms):
    """K16 steps x terms of a head's Linear layer on the tensor cores (layer 0 in blocks of one 96-wide feature row);
    terms = 0: heads.cu's fp32 FMA chains (K, + the bias)."""
    if terms == 0:
        return K + 1
    return (K // 96 * 6 if first else -(-K // 16)) * terms


def linear_bound_parts(x, W, b, terms, first, x_err=None):
    """Float64 y = x W + b of one Linear layer and its per-element bound tau = C * A + B (terms 3: hi/lo operands, 1:
    fp16, 0: fp32): (y, A, B).  x_err = (A, B) of the input's own bound, carried through |W|."""
    x, W64, b64 = np.asarray(x, np.float64), np.asarray(W, np.float64), np.asarray(b, np.float64)
    ax = np.abs(x) if x_err is None else np.abs(x) + C_ROUNDOFF * x_err[0] + x_err[1]
    S = ax @ np.abs(W64)
    y = x @ W64 + b64
    A = U * head_add_count(W64.shape[0], first, terms) * S
    B = U * (2 * np.abs(y) + np.abs(b64))
    if terms:
        floor = SUB16 * (np.abs(W64).sum(0) + 2.0 ** -scale_exponent(W) * ax.sum(1, keepdims=True))
        B = B + (SPLIT_OP if terms == 3 else 2 * FP16_OP) * S + floor
    if x_err is not None:
        A, B = A + x_err[0] @ np.abs(W64), B + x_err[1] @ np.abs(W64)
    return y, A, B


def head_bound_parts(h, feats, terms):
    """Raw outputs of a head of one Linear layer, or of two without LayerNorm (ReLU between), final 'none', and their
    bound: (y, A, B), tau = C * A + B.  ReLU is 1-Lipschitz, so layer 2 takes |W2|^T tau1 on top of its own round-off."""
    L = h["layers"]
    assert h["final"] == "none" and len(L) in (1, 2) and all(l.get("ln") is None for l in L[:-1])
    x = np.asarray(feats, np.float64).reshape(len(feats), -1)
    y, A, B = linear_bound_parts(x, L[0]["W"], L[0]["b"], terms, True)
    if len(L) == 2:
        y, A, B = linear_bound_parts(np.maximum(y, 0.0), L[1]["W"], L[1]["b"], terms, False, x_err=(A, B))
    return y, A, B


def head_bound(h, feats, terms, C=C_ROUNDOFF):
    y, A, B = head_bound_parts(h, feats, terms)
    return y, C * A + B


def emulate_linear(x, W, b, defects=()):
    """heads_tc's first GEMM at 3 terms in float32 on the CPU: features split to hi/lo, W 2^s split, K16 steps per
    96-wide row, fmaf(acc, 2^-s, b)."""
    s = scale_exponent(W)
    W64 = np.asarray(W, np.float64)
    if "w_fp16_unscaled" in defects:
        s = 0
        acc = emulate_gemm(list(_split16(x)), [_f16(W64)], [(0, 0), (1, 0)])
    else:
        terms = [t for t in SPLIT_TERMS if not ("two_terms" in defects and t == (0, 1))]
        acc = emulate_gemm(list(_split16(x)), list(_split16(W64 * 2.0 ** s)), terms)
    bias = 0.0 if "no_bias" in defects else np.asarray(b, np.float64)
    return (acc.astype(np.float64) * 2.0 ** -s + bias).astype(np.float32)


HEAD_GUARDS = ("two_terms", "w_fp16_unscaled", "no_bias")


def bound_head(n_in, width, seed):
    rng = np.random.default_rng(seed)
    K = n_in * 96
    return {"n_in": n_in, "final": "none",
            "layers": [{"W": (rng.standard_normal((K, width)) / np.sqrt(K)).astype(np.float32),
                        "b": rng.normal(0, 0.1, width).astype(np.float32), "ln": None}]}


def head_features(rng, n, n_in):
    """Features from N(0.3, 1.5), every 7th row x 4, every 11th row of mean 100 and std 1, every 13th row zero."""
    f = rng.normal(0.3, 1.5, (n, n_in, 96)).astype(np.float32)
    f[::7] *= 4.0
    f[5::11] = rng.normal(100.0, 1.0, f[5::11].shape)
    f[3::13] = 0.0
    return f


@pytest.mark.parametrize("defect", (None,) + HEAD_GUARDS)
def test_heads_emulation_and_guards(defect):
    rng = np.random.default_rng(2)
    worst = 0.0
    for n_in, width in ((3, 1), (16, 64), (34, 128)):
        h = bound_head(n_in, width, seed=n_in)
        f = head_features(rng, 130, n_in)
        y, tau = head_bound(h, f, 3)
        lay = h["layers"][0]
        dev = emulate_linear(f.reshape(130, -1), lay["W"], lay["b"], () if defect is None else (defect,))
        worst = max(worst, ratio(dev, y, tau))
    print(f"\nheads_tc 3-term emulation, {defect or 'no defect'}: worst ratio {worst:.3g} at C = {C_ROUNDOFF:g}")
    if defect is None:
        assert worst <= 1.0
    else:
        assert worst >= GUARD_MARGIN
