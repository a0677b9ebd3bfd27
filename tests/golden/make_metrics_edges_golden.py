"""Generate tests/golden/metrics_edges.npz from the UNMODIFIED reference functions
(openwakeword/metrics.py of the original openWakeWord project, OWW_REFERENCE = its root directory):
    OWW_REFERENCE=/path/to/openWakeWord python tests/golden/make_metrics_edges_golden.py

The edges of get_false_positives / generate_roc_curve_* that tests/golden/metrics.npz does not reach: the precision of
the comparison ``np.array(scores) >= threshold`` (NumPy >= 2 promotion: a Python float threshold takes the scores'
dtype, a NumPy scalar promotes), and the grouping rule at the very start of a series.
* Series in float16, float32 and float64, built around base thresholds t with float32(t) < t, > t and == t: the
  float32 / float16 value nearest t and its neighbours, and float64 values within half a float32 ulp of t.
* Every base threshold as a Python float, np.float64 and np.float32; grouping windows 0, 1, 5 and 50.
* Shapes: first rise at index 0 or 1, alternating 0101... starts (the densest grouping), all ones, all zeros, short
  series of 1-4 frames and random mixes of near-threshold values.
* ROC fprs and tprs of float32 and float64 series that hold the linspace thresholds and their neighbours.
A series whose last element is a fresh 0->1 rise makes the reference raise IndexError at some threshold; such series
are not written (the oracle defines that case as a no-op and the tests check it there)."""
import importlib.util
import os

import numpy as np

spec = importlib.util.spec_from_file_location("ref_metrics", os.path.join(os.environ["OWW_REFERENCE"], "openwakeword", "metrics.py"))
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)

BASE = np.array([0.7, 0.1, 0.5, 0.3, 0.01, 0.99, 0.25, 1.0 / 3.0])   # f32(0.7) < 0.7, f32(0.1) > 0.1, f32(0.5) == 0.5
WINDOWS = [0, 1, 5, 50]
KINDS = ("float", "float64", "float32")                               # how a threshold is passed


def threshold(value, kind):
    return {"float": float, "float64": np.float64, "float32": np.float32}[kind](value)


def neighbours(x, dtype):
    x = dtype(x)
    return [np.nextafter(x, dtype(-np.inf)), x, np.nextafter(x, dtype(np.inf))]


def pool(t, dtype):
    """Values right at t in the series dtype."""
    if dtype is np.float64:
        u = float(np.spacing(np.float32(t)))
        return [t, np.nextafter(t, -1.0), np.nextafter(t, 2.0), t - 0.25 * u, t + 0.25 * u, t - 0.49 * u, t + 0.49 * u,
                float(np.float32(t))] + [float(v) for v in neighbours(t, np.float32)]
    return neighbours(t, dtype)


def shapes(rng, vals, dtype):
    """Series over near-threshold values `vals` (low = 0, high = 1 as fillers)."""
    v = list(vals)
    out = [
        [0, v[0], 0] + v + [0],                                           # first rise at index 0
        [0, 0, v[-1], 1, 0] + v[::-1] + [0],                              # first rise at index 1
        [v[0], 0, v[1 % len(v)], 0],                                      # starts high
        sum(([0, x] for x in v * 3), []) + [0],                           # alternating 0101... start
        [0, 1] * 20 + [0],
        [0, 1] * 20 + [1, 1, 0],
        [1] * 37,
        [0] * 37,
        [v[0]], [0, v[0], v[0]], [v[0], 0], [0, 1, 1], [1, 0, 1, 1],
    ]
    for n in (8, 30, 120):
        for _ in range(3):
            s = rng.choice(np.array(v + [0.0, 1.0], np.float64), n)
            s[-1] = 0.0
            out.append(list(s))
    return [np.array(s, dtype) for s in out]


def trailing_rise(s, thresholds):
    return any(len(s) > 1 and not (s[-2] >= t) and s[-1] >= t for t in thresholds)


def main():
    rng = np.random.default_rng(2026)
    all_thr = [threshold(t, k) for t in BASE for k in KINDS]
    sers = []
    for t in BASE:
        for dtype in (np.float16, np.float32, np.float64):
            for s in shapes(rng, pool(t, dtype), dtype):
                if not trailing_rise(s, all_thr):
                    sers.append(s)
    # the two cases where float32 rounding of scores or thresholds decides the count
    sers.append(np.array([0, np.float32(0.7), 0, 0], np.float32))
    sers.append(np.array([0, 0.5 - 1e-10, 0, 0], np.float64))
    fp = np.zeros((len(sers), len(BASE), len(KINDS), len(WINDOWS)), np.int64)
    for i, s in enumerate(sers):
        for a, t in enumerate(BASE):
            for b, k in enumerate(KINDS):
                for c, w in enumerate(WINDOWS):
                    fp[i, a, b, c] = int(ref.get_false_positives(s, threshold=threshold(t, k), grouping_window=w))
    out = {"n_series": np.int64(len(sers)), "base": BASE, "kinds": np.array(KINDS), "windows": np.array(WINDOWS),
           "fp": fp}                                                      # [series][base threshold][kind][window]
    for i, s in enumerate(sers):
        out[f"s{i}"] = s
    # ROC: float32 and float64 series holding the linspace thresholds and their neighbours
    lin = np.linspace(0.01, 0.99, 25)
    roc = []
    for dtype in (np.float32, np.float64):
        vals = np.concatenate([np.array(pool(t, dtype), np.float64) for t in lin])
        s = np.zeros(3 * vals.size + 1)
        s[1::3] = rng.permutation(vals)
        s[2::3] = rng.permutation(vals)
        s[:40] = np.tile([0.0, 1.0], 20)
        roc.append(s.astype(dtype))
    for j, (s, w) in enumerate(zip(roc, (50, 5))):
        out[f"roc_s{j}"] = s
        out[f"roc_window{j}"] = np.int64(w)
        out[f"roc_fprs{j}"] = np.array(ref.generate_roc_curve_fprs(s, n_points=25, time_per_prediction=0.08, grouping_window=w))
        out[f"roc_tprs{j}"] = np.array(ref.generate_roc_curve_tprs(s, n_points=25), np.float64)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "metrics_edges.npz")
    np.savez_compressed(path, **out)
    kinds_differ = int((fp[:, :, 0] != fp[:, :, 1]).any(axis=(1, 2)).sum())
    print("wrote", path, "series", len(sers), "fp", fp.shape, "series whose count depends on the threshold's type:",
          kinds_differ, "grouping effect:", int((fp[..., 1] != fp[..., 3]).sum()))


if __name__ == "__main__":
    main()
