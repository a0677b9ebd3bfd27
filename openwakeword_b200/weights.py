"""Weight containers for the CUDA backend.

The released model files of the reference (``melspectrogram.onnx``,
``embedding_model.onnx``, ``<head>_v0.1.onnx``; registry at
openwakeword/__init__.py:8-51) are download-only and absent from
this image, so every test and benchmark runs on *synthetic, seeded weights of
the exact reference architecture* (SURVEY.md F3).  This module builds those,
packs weights into the flat float32 blobs the C ABI takes
(include/owwb200.h: ``oww_load_embedding`` / ``oww_add_head``) and stores /
loads them as ``.npz``.  No inference arithmetic happens here.
"""
import math
import numpy as np

_erf = math.erf

# (kh, kw, cin, cout, pool_t, pool_f): the speech-embedding CNN, SURVEY.md App. B
# (nb/conv:871-951).  pool = 0 -> none.
EMBEDDING_LAYERS = [
    (3, 3, 1, 24, 0, 0),
    (1, 3, 24, 24, 0, 0), (3, 1, 24, 24, 2, 2),
    (1, 3, 24, 48, 0, 0), (3, 1, 48, 48, 0, 0),
    (1, 3, 48, 48, 0, 0), (3, 1, 48, 48, 1, 2),
    (1, 3, 48, 72, 0, 0), (3, 1, 72, 72, 0, 0),
    (1, 3, 72, 72, 0, 0), (3, 1, 72, 72, 2, 2),
    (1, 3, 72, 96, 0, 0), (3, 1, 96, 96, 0, 0),
    (1, 3, 96, 96, 0, 0), (3, 1, 96, 96, 1, 2),
    (1, 3, 96, 96, 0, 0), (3, 1, 96, 96, 0, 0),
    (1, 3, 96, 96, 0, 0), (3, 1, 96, 96, 2, 2),
    (3, 1, 96, 96, 0, 0),
]
BN_EPS = 1e-3
LN_EPS = 1e-5
EMBEDDING_DIM = 96
N_EMBEDDING_PARAMS = 332088          # nb/conv:859

# Per-layer variance of the pre-BatchNorm activations under synthetic_embedding()
# init, measured once with the oracle on seeded noise (recorded in DESIGN.md).
# Baked in so that the generator is closed-form and activations stay O(1).
_PRE_BN_VAR = [0.6914, 0.9152, 0.6638, 1.4282, 0.9623, 1.0618, 0.888, 1.3352, 1.0612, 1.2764,
               1.2048, 1.361, 1.0875, 1.5599, 1.1395, 0.6771, 1.2109, 0.7107, 1.3346]
_PRE_BN_MEAN = [0.2156, -0.0759, 0.0574, 0.0159, -0.0224, 0.0469, 0.1931, 0.017, -0.1188, -0.2009,
                0.0322, -0.1334, 0.0649, -0.049, 0.1022, 0.0404, 0.0874, 0.0161, -0.1357]


def synthetic_embedding(seed=0):
    """Seeded weights with the reference CNN's exact shapes: HWIO conv kernels
    (bias-free), 19 BatchNorms as (gamma, beta, moving_mean, moving_var)."""
    rng = np.random.default_rng(seed)
    conv, bn = [], []
    for li, (kh, kw, cin, cout, _, _) in enumerate(EMBEDDING_LAYERS):
        fan_in = kh * kw * cin
        w = rng.standard_normal((kh, kw, cin, cout)) * np.sqrt(1.6 / fan_in)
        if li == 0:   # kernel_constraint=CenterAround(0.0), nb/conv:897,975
            w = w - w.mean(axis=(0, 1), keepdims=True)
        conv.append(w.astype(np.float32))
        if li < len(EMBEDDING_LAYERS) - 1:
            gamma = rng.uniform(0.6, 1.4, cout)
            beta = rng.normal(0.15, 0.25, cout)
            mean = _PRE_BN_MEAN[li] + rng.normal(0.0, 0.2, cout) * np.sqrt(_PRE_BN_VAR[li])
            var = _PRE_BN_VAR[li] * rng.uniform(0.6, 1.6, cout)
            bn.append(tuple(a.astype(np.float32) for a in (gamma, beta, mean, var)))
    return {"conv": conv, "bn": bn}


def synthetic_head(n_in=16, hidden=64, n_blocks=1, n_out=1, layernorm=True,
                   final="sigmoid", seed=1):
    """Seeded head of the reference's DNN family (train.py:56-83):
    Linear(n_in*96,hidden) [LN] ReLU, n_blocks x (Linear [LN] ReLU), Linear(hidden,n_out)."""
    rng = np.random.default_rng(seed)
    dims = [n_in * EMBEDDING_DIM] + [hidden] * (1 + n_blocks) + [n_out]
    layers = []
    for i in range(len(dims) - 1):
        last = i == len(dims) - 2
        gain = 3.0 if last else 1.0
        W = rng.standard_normal((dims[i], dims[i + 1])) * gain / np.sqrt(dims[i])
        b = rng.normal(0.0, 0.1, dims[i + 1])
        ln = None
        if layernorm and not last:
            ln = (rng.uniform(0.7, 1.3, dims[i + 1]).astype(np.float32),
                  rng.normal(0.1, 0.2, dims[i + 1]).astype(np.float32))
        if last and layernorm and n_out == 1:
            # centre the logit so synthetic scores straddle 0.5 (maximum sigmoid slope
            # -> the most sensitive parity test): hidden unit i is relu(N(beta_i, gamma_i^2))
            # after LayerNorm, whose mean is beta*Phi(beta/gamma) + gamma*phi(beta/gamma).
            g, h = (a.astype(np.float64) for a in layers[-1]["ln"])
            z = h / g
            phi = np.exp(-0.5 * z * z) / np.sqrt(2 * np.pi)
            Phi = 0.5 * (1.0 + np.array([_erf(v / np.sqrt(2.0)) for v in z]))
            b = b - (W[:, 0] @ (h * Phi + g * phi))
        layers.append({"W": W.astype(np.float32), "b": b.astype(np.float32), "ln": ln})
    return {"n_in": int(n_in), "layers": layers, "final": final}


def fold_bn(gamma, beta, mean, var, eps=BN_EPS):
    """BatchNorm(inference) -> per-channel (scale, bias), computed in float64."""
    g, b, m, v = (np.asarray(a, dtype=np.float64) for a in (gamma, beta, mean, var))
    s = g / np.sqrt(v + eps)
    return s.astype(np.float32), (b - m * s).astype(np.float32)


def pack_embedding_blob(weights):
    """Flat float32 blob for ``oww_load_embedding``: per layer the HWIO kernel
    (kh*kw*cin*cout), then folded BN scale[cout], bias[cout] (identity for the
    last, BN-less layer)."""
    parts = []
    for li, (kh, kw, cin, cout, _, _) in enumerate(EMBEDDING_LAYERS):
        w = np.asarray(weights["conv"][li], dtype=np.float32)
        assert w.shape == (kh, kw, cin, cout), (li, w.shape)
        parts.append(w.ravel())
        if li < len(EMBEDDING_LAYERS) - 1:
            s, b = fold_bn(*weights["bn"][li])
        else:
            s, b = np.ones(cout, np.float32), np.zeros(cout, np.float32)
        parts += [s, b]
    return np.ascontiguousarray(np.concatenate(parts), dtype=np.float32)


FINAL_CODES = {"none": 0, "sigmoid": 1, "softmax": 2, "relu_softmax": 3, "relu": 4}


def is_gated(head):
    """A conditional verifier pair (the released ``hey_jarvis`` graph, docs/models/hey_jarvis.md:9,38):
    ``{"main": head, "verifier": head, "threshold": 0.5}`` - the verifier's score replaces the main network's wherever
    the latter exceeds the threshold."""
    return isinstance(head, dict) and "verifier" in head


def synthetic_gated_head(seed_main=31, seed_verifier=32, threshold=0.5, **kw):
    return {"main": synthetic_head(seed=seed_main, **kw), "verifier": synthetic_head(seed=seed_verifier, **kw),
            "threshold": float(threshold), "n_in": int(kw.get("n_in", 16))}


def head_desc(head):
    """(n_in, dims list, layernorm flag, final code) of a head dict."""
    L = head["layers"]
    dims = [L[0]["W"].shape[0]] + [l["W"].shape[1] for l in L]
    ln = any(l.get("ln") is not None for l in L[:-1])
    if ln and not all(l.get("ln") is not None for l in L[:-1]):
        raise ValueError("heads with LayerNorm on only some hidden layers are not supported")
    return head["n_in"], dims, ln, FINAL_CODES[head["final"]]


def pack_head_blob(head):
    """Flat float32 blob for ``oww_add_head``: per layer W[in,out] row-major,
    b[out], and (hidden layers of LayerNorm heads) ln_gamma[out], ln_beta[out]."""
    parts = []
    L = head["layers"]
    for i, lay in enumerate(L):
        parts += [np.asarray(lay["W"], np.float32).ravel(), np.asarray(lay["b"], np.float32).ravel()]
        if lay.get("ln") is not None and i < len(L) - 1:
            parts += [np.asarray(lay["ln"][0], np.float32), np.asarray(lay["ln"][1], np.float32)]
    return np.ascontiguousarray(np.concatenate(parts), dtype=np.float32)


def save_head(path, head, class_mapping=None):
    d = {}
    parts = [("", head)] if not is_gated(head) else [("", head["main"]), ("v_", head["verifier"])]
    if is_gated(head):
        d["gate_threshold"] = np.float64(head["threshold"])
    for pre, hd in parts:
        d[pre + "n_in"] = np.int64(hd["n_in"]); d[pre + "final"] = np.str_(hd["final"])
        d[pre + "n_layers"] = np.int64(len(hd["layers"]))
        for i, lay in enumerate(hd["layers"]):
            d[f"{pre}W{i}"], d[f"{pre}b{i}"] = lay["W"], lay["b"]
            if lay.get("ln") is not None:
                d[f"{pre}g{i}"], d[f"{pre}h{i}"] = lay["ln"]
    if class_mapping:
        d["class_keys"] = np.array(list(class_mapping.keys()))
        d["class_vals"] = np.array(list(class_mapping.values()))
    np.savez(path, **d)


def load_head(path):
    z = np.load(path, allow_pickle=False)

    def one(pre):
        layers = []
        for i in range(int(z[pre + "n_layers"])):
            ln = (z[f"{pre}g{i}"], z[f"{pre}h{i}"]) if f"{pre}g{i}" in z.files else None
            layers.append({"W": z[f"{pre}W{i}"], "b": z[f"{pre}b{i}"], "ln": ln})
        return {"n_in": int(z[pre + "n_in"]), "layers": layers, "final": str(z[pre + "final"])}
    head = one("")
    if "gate_threshold" in z.files:
        head = {"main": head, "verifier": one("v_"), "threshold": float(z["gate_threshold"]), "n_in": head["n_in"]}
    cm = None
    if "class_keys" in z.files:
        cm = {str(k): str(v) for k, v in zip(z["class_keys"], z["class_vals"])}
    return head, cm


def save_embedding(path, weights):
    d = {}
    for i, w in enumerate(weights["conv"]):
        d[f"conv{i}"] = w
    for i, p in enumerate(weights["bn"]):
        d[f"bn{i}"] = np.stack(p)
    np.savez(path, **d)


def load_embedding(path):
    z = np.load(path, allow_pickle=False)
    conv = [z[f"conv{i}"] for i in range(len(EMBEDDING_LAYERS))]
    bn = [tuple(z[f"bn{i}"]) for i in range(len(EMBEDDING_LAYERS) - 1)]
    return {"conv": conv, "bn": bn}
