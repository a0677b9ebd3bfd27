"""Shared test helpers: golden-case loading, the synthetic weight set the goldens were made with, the Models the host
tests build, the verifier arithmetic of verifier.cu in NumPy, the seven bench networks and the test audio of the stream
tests, and the judge of resampled samples against the float64 oracle."""
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


def seven_heads():
    """the bench's seven networks: five 16-row sigmoid heads (the third a gated pair) and a 34-row 7-class head"""
    hs = []
    for i in range(5):
        hs.append(W.synthetic_gated_head(seed_main=10 + i, seed_verifier=40 + i, threshold=0.5) if i == 2
                  else W.synthetic_head(seed=10 + i))
    hs.append(W.synthetic_head(n_in=34, hidden=128, n_out=7, layernorm=False, final="relu_softmax", seed=20))
    return hs


def bank_heads():
    """three heads of one shape for a head bank"""
    return [W.synthetic_head(seed=300 + i, n_in=16, hidden=64, n_out=1) for i in range(3)]


def mixes(rng, n, length):
    """+-1000 noise, full scale, gated bursts, silence, tone"""
    out = np.empty((n, length), np.int16)
    t = np.arange(length)
    for i in range(n):
        k = (i + int(rng.integers(0, 5))) % 5
        if k == 0:
            x = rng.integers(-1000, 1000, length)
        elif k == 1:
            x = rng.uniform(-1, 1, length) * 32767
        elif k == 2:
            x = rng.normal(0, 8000, length) * ((t // 4000) % 2)
        elif k == 3:
            x = np.zeros(length)
        else:
            x = 12000 * np.sin(2 * np.pi * (300 + 40 * i) * t / 16000) + rng.normal(0, 20, length)
        out[i] = np.clip(x, -32768, 32767).astype(np.int16)
    return out


def judge_resampled(got, y64, s, up, down, n_taps):
    """int16 samples `got` against the float64 outputs y64 of the same input, s = sum |h32 * x| of each, under the
    round-off bound |y - y64| <= gamma_K * s (K = taps per phase): outside the bound's band around a rounding boundary
    got equals clip(rint(y64)) exactly, inside it differs by at most one -> the fraction judged"""
    from oracle import resample as ores
    assert got.size == y64.size
    K = -(-n_taps // up)
    u = 2.0 ** -24
    band = K * u / (1 - K * u) * s
    ref = ores.to_int16(y64)
    frac = y64 - np.floor(y64)
    near = np.abs(frac - 0.5) <= band
    sat = (y64 > 32767 + band) | (y64 < -32768 - band)
    judged = ~near | sat
    assert np.array_equal(got[judged], ref[judged]), (up, down, np.nonzero(got[judged] != ref[judged])[0][:5])
    assert (np.abs(got.astype(np.int32) - ref) <= 1).all()
    return judged.mean()


# ---- long-running streams: the counter rules of oww_internal.h and detect.cu restated, and the twin comparators ----
COUNT_WRAP = 1 << 30                    # OWW_COUNT_WRAP
COUNT_REBASE = (1 << 30) - (1 << 20)    # OWW_COUNT_REBASE: a multiple of every ring size (<= 2^20 rows)
DET_REBASE = 35791392 * 30              # DET_COUNT_REBASE = 2^30 - 64, a multiple of 30
REC_COUNT_WORDS = (5, 6)                # int32 words of a stream record's header: mel count, feature count


def ring_count(c, added):
    """a ring row count after `added` rows: c' = c + added - REBASE * [c + added >= 2^30]"""
    c = int(c) + int(added)
    return c - COUNT_REBASE if c >= COUNT_WRAP else c


def imported_count(c):
    """the count a stream takes from a record holding c (< 2^31): rebased once, as a step would"""
    return int(c) - COUNT_REBASE if int(c) >= COUNT_WRAP else int(c)


def det_count(c):
    """the detector's count after one prediction is appended to a stream at count c"""
    c = int(c) + 1
    return c - DET_REBASE if c >= COUNT_WRAP else c


def det_imported(c):
    c = max(int(c), 0)
    return c - DET_REBASE if c >= COUNT_WRAP else c


def event_index(c):
    """`index` of an event of a stream at count c before the call: the count before the append, in the count's frame
    after this call's rebase (the count after the call, minus one)"""
    return det_count(c) - 1


def record_words(rec):
    return np.ascontiguousarray(np.asarray(rec, np.uint8)).view(np.int32)


def record_diff(ctrl, twin, counts):
    """Stream record `twin` against `ctrl` (uint8 [record bytes] each): byte for byte outside the header's count words,
    which must hold counts = (mel, feature).  -> a list of what differs (empty: the twin holds)."""
    a, b = record_words(ctrl).copy(), record_words(twin).copy()
    out = []
    got = (int(b[REC_COUNT_WORDS[0]]), int(b[REC_COUNT_WORDS[1]]))
    if got != tuple(int(v) for v in counts):
        out.append(f"counts {got}, want {tuple(counts)}")
    a[list(REC_COUNT_WORDS)] = 0
    b[list(REC_COUNT_WORDS)] = 0
    bad = np.nonzero(a != b)[0]
    if bad.size:
        out.append(f"{bad.size} words differ, first at word {bad[0]}")
    return out


def events_diff(ev_ctrl, ev_twin, twin_of, index_of):
    """Events of the controls against their twins': the same (label, score) per pair, and each twin event's index =
    index_of[twin stream].  twin_of: {control stream: twin stream}.  -> a list of what differs."""
    out = []
    twins = set(twin_of.values())
    c = {(int(e["stream"]), int(e["label"])): e for e in ev_ctrl if int(e["stream"]) in twin_of}
    t = {(int(e["stream"]), int(e["label"])): e for e in ev_twin if int(e["stream"]) in twins}
    want = {(twin_of[s], j) for s, j in c}
    if set(t) != want:
        out.append(f"twin events {sorted(set(t) ^ want)[:4]} differ from the controls'")
    for (s, j), e in c.items():
        f = t.get((twin_of[s], j))
        if f is None:
            continue
        if np.float32(f["score"]).view(np.int32) != np.float32(e["score"]).view(np.int32):
            out.append(f"stream {s} label {j}: score {f['score']} != {e['score']}")
        if int(f["index"]) != index_of[twin_of[s]]:
            out.append(f"stream {twin_of[s]} label {j}: index {int(f['index'])}, want {index_of[twin_of[s]]}")
    return out
