"""Speech-embedding CNN restatement (the graph inside ``embedding_model.onnx``).

Follows notebooks/converting_google_speech_embedding_model.ipynb
lines 871-951 (layer code) and 521-859 (shapes): 20 bias-free dense convs
(3x3 then alternating (1,3) 'same' / (3,1) 'valid'), each but the last followed
by BatchNorm(eps=1e-3) -> max(0.2x, x) -> max(x, -0.4); the first conv also has
ReLU before its BN (nb/conv:897-899); five max-pools.  NHWC [N,76,32,1] ->
[N,96].  Weights are plain arrays supplied by the caller.
"""
import numpy as np

# (kh, kw, cin, cout, pool_after) ; pool = (pt, pf) or None       SURVEY.md App. B
LAYERS = [
    (3, 3, 1, 24, None),
    (1, 3, 24, 24, None), (3, 1, 24, 24, (2, 2)),
    (1, 3, 24, 48, None), (3, 1, 48, 48, None),
    (1, 3, 48, 48, None), (3, 1, 48, 48, (1, 2)),
    (1, 3, 48, 72, None), (3, 1, 72, 72, None),
    (1, 3, 72, 72, None), (3, 1, 72, 72, (2, 2)),
    (1, 3, 72, 96, None), (3, 1, 96, 96, None),
    (1, 3, 96, 96, None), (3, 1, 96, 96, (1, 2)),
    (1, 3, 96, 96, None), (3, 1, 96, 96, None),
    (1, 3, 96, 96, None), (3, 1, 96, 96, (2, 2)),
    (3, 1, 96, 96, None),
]
BN_EPS = 1e-3
LEAK = np.float32(0.20000000298023224)
FLOOR = np.float32(-0.4000000059604645)
MACS_PER_WINDOW = 41955840


def fold_bn(gamma, beta, mean, var, eps=BN_EPS):
    scale = gamma / np.sqrt(var + eps)
    return scale.astype(np.float32), (beta - mean * scale).astype(np.float32)


def _conv(x, w, dtype):
    """x [N,T,F,Cin], w [kh,kw,Cin,Cout]; time 'valid'; freq: 'same' for kw=3 of a
    (1,3) layer, and the 3x3 first layer sees ZeroPadding2D((0,1)) (nb/conv:896)."""
    kh, kw, cin, cout = w.shape
    N, T, F, _ = x.shape
    if kw == 3:
        x = np.pad(x, ((0, 0), (0, 0), (1, 1), (0, 0)))
    To = T - kh + 1
    cols = []
    for dt in range(kh):
        for df in range(kw):
            cols.append(x[:, dt:dt + To, df:df + F, :])
    a = np.concatenate(cols, axis=-1).reshape(-1, kh * kw * cin).astype(dtype)
    y = a @ w.reshape(kh * kw * cin, cout).astype(dtype)
    return y.reshape(N, To, F, cout)


def _pool(x, pt, pf):
    N, T, F, C = x.shape
    T2, F2 = T // pt, F // pf
    x = x[:, :T2 * pt, :F2 * pf, :].reshape(N, T2, pt, F2, pf, C)
    return x.max(axis=(2, 4))


def forward(weights, mel, dtype=np.float32, quant=None, return_all=False):
    """mel [N,T,32] float32 (T>=76; T=76 is the reference window) -> [N,(T-76)//8+1,96].
    ``weights`` = {"conv": [20 arrays HWIO], "bn": [19 x (gamma,beta,mean,var)]}.
    ``quant``: optional callable applied to every conv's activations and weights
    (used to study fp16/bf16 operand rounding); accumulation stays in ``dtype``."""
    x = np.asarray(mel, dtype=np.float32)[..., None].astype(dtype)
    outs = []
    for li, (kh, kw, cin, cout, pool) in enumerate(LAYERS):
        w = weights["conv"][li].astype(dtype)
        a = x
        if quant is not None and li > 0:
            a = quant(a).astype(dtype)
            w = quant(w).astype(dtype)
        x = _conv(a, w, dtype)
        if li == 0:
            x = np.maximum(x, 0)
        if li < len(LAYERS) - 1:
            s, b = fold_bn(*[np.asarray(p, dtype=np.float64) for p in weights["bn"][li]])
            x = x * s.astype(dtype) + b.astype(dtype)
            x = np.maximum(dtype(LEAK) * x, x)
            x = np.maximum(x, dtype(FLOOR))
        if pool is not None:
            x = _pool(x, *pool)
        if return_all:
            outs.append(x.astype(np.float32))
    y = x[:, :, 0, :].astype(np.float32)          # [N, n_windows, 96]
    return (y, outs) if return_all else y


def embed_windows(weights, windows, dtype=np.float32, quant=None):
    """``embedding_model_predict`` on [N,76,32] windows -> [N,96] (utils.py:93)."""
    return forward(weights, windows, dtype, quant)[:, 0, :]
