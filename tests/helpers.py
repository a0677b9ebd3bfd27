"""Shared test helpers: golden-case loading, the synthetic weight set the goldens were made with, the Models the host
tests build, and the verifier arithmetic of verifier.cu in NumPy."""
import glob
import os

import numpy as np

import openwakeword_b200 as owb
from openwakeword_b200 import weights as W
from openwakeword_b200.custom_verifier_model import load_verifier

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = ["alexa_v0.1", "timer_v0.1", "hey_jarvis_v0.1"]
VERIFIER_CASES = ["verifier_alexa_c1280", "verifier_alexa_c2560", "verifier_timer_c1280", "verifier_timer_c2560"]

HEAD_SPECS = {   # must match tests/golden/make_golden.py
    "alexa_v0.1": dict(n_in=16, hidden=64, n_blocks=1, n_out=1, layernorm=True, final="sigmoid", seed=1),
    "hey_mycroft_v0.1": dict(n_in=16, hidden=64, n_blocks=1, n_out=1, layernorm=True, final="sigmoid", seed=2),
    "timer_v0.1": dict(n_in=34, hidden=128, n_blocks=1, n_out=7, layernorm=False, final="relu_softmax", seed=9),
    "big_v0.1": dict(n_in=16, hidden=128, n_blocks=2, n_out=1, layernorm=True, final="sigmoid", seed=4),
}
GATED_SPECS = {"hey_jarvis_v0.1": dict(seed_main=31, seed_verifier=32, threshold=0.5)}
TIMER_MAP = {"1": "1_minute_timer", "2": "5_minute_timer", "3": "10_minute_timer",
             "4": "20_minute_timer", "5": "30_minute_timer", "6": "1_hour_timer"}

_cache = {}


def emb_weights(seed=0):
    if ("emb", seed) not in _cache:
        _cache[("emb", seed)] = W.synthetic_embedding(seed)
    return _cache[("emb", seed)]


def head(name):
    if name not in _cache:
        _cache[name] = W.synthetic_gated_head(**GATED_SPECS[name]) if name in GATED_SPECS else W.synthetic_head(**HEAD_SPECS[name])
    return _cache[name]


def class_mapping(names):
    return {"timer_v0.1": dict(TIMER_MAP)} if "timer_v0.1" in names else {}


def golden_cases(kind=None):
    out = []
    for p in sorted(glob.glob(os.path.join(GOLDEN, "*.npz"))):
        z = np.load(p, allow_pickle=False)
        if "kind" not in z.files:          # not a hot-path case file (e.g. metrics.npz)
            continue
        if kind is None or str(z["kind"]) == kind:
            out.append(os.path.splitext(os.path.basename(p))[0])
    return out


def load_case(tag):
    z = np.load(os.path.join(GOLDEN, tag + ".npz"), allow_pickle=False)
    c = {k: z[k] for k in z.files}
    kw = {}
    for k in list(c):
        if k.startswith("kw_") and k.endswith("_keys"):
            base = k[3:-5]
            kw[base] = {str(a): float(b) for a, b in zip(c[k], c["kw_" + base + "_vals"])}
        elif k.startswith("kw_") and not k.endswith("_vals"):
            kw[k[3:]] = float(c[k])
    if "patience" in kw:
        kw["patience"] = {a: int(b) for a, b in kw["patience"].items()}
    c["kw"] = kw
    for k in ("names", "labels"):
        if k in c:
            c[k] = [str(s) for s in c[k]]
    return c


def case_model(c, **kw):
    """the Model of golden case c: its models, embedding seed and feature_init, max_chunks 8"""
    specs = [{"name": n, "head": head(n), "class_mapping": class_mapping([n]).get(n)} for n in c["names"]]
    return owb.Model(wakeword_models=specs, embedding_model_path=emb_weights(int(c["emb_seed"])),
                     feature_init=c["feature_init"], max_chunks=8, **kw)


def streams_model(B, fi, names=NAMES, max_chunks=2, **kw):
    """a Model of B streams on the models `names`"""
    specs = [{"name": n, "head": head(n), "class_mapping": class_mapping([n]).get(n)} for n in names]
    return owb.Model(wakeword_models=specs, embedding_model_path=emb_weights(), feature_init=fi, n_streams=B,
                     max_chunks=max_chunks, **kw)


def verifier_pipeline(tag):
    return load_verifier(os.path.join(GOLDEN, f"verifier_{tag}.pkl"))


def kernel_order_proba(mean, weight, bias, feats):
    """verifier.cu in NumPy fp32: lane l accumulates float4 l, l+32, ... with fmaf (x - mu) * w in x, y, z, w order,
    then the xor-shuffle tree; p = 1 / (1 + exp(-(bias + acc))).  feats [n, n_in, 96] -> float32 [n]."""
    x = np.asarray(feats, np.float32).reshape(len(feats), -1)
    d = (x - mean[None]).astype(np.float32)
    n, D = x.shape
    lanes = np.zeros((n, 32), np.float32)
    for j in range(D // 4):
        for e in range(4):
            k = 4 * j + e
            # fmaf: the fp32 product is exact in float64, one rounding of the sum
            lanes[:, j % 32] = (d[:, k].astype(np.float64) * np.float64(weight[k]) + lanes[:, j % 32]).astype(np.float32)
    off = 16
    while off:
        lanes = (lanes + lanes[:, np.arange(32) ^ off]).astype(np.float32)
        off >>= 1
    z = (np.float32(bias) + lanes[:, 0]).astype(np.float32)
    return (np.float32(1) / (np.float32(1) + np.exp(-z))).astype(np.float32)
