"""Score metrics (SURVEY.md section 8 f4): the oracle restatement against golden values produced by the reference's own
functions (not-gpu), and the device kernels against both (gpu).  tests/golden/metrics_edges.npz holds the reference's
counts at the precision edges of its comparison and at the start-of-series edges of its grouping rule; the comparison
dtype rule (openwakeword_b200.metrics.comparison_dtype) is checked here against NumPy itself.  The device kernels'
layout edges and the edge goldens on the device are in tests/test_gpu_metrics.py."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import metrics as om


def _golden():
    return np.load(os.path.join(GOLDEN, "metrics.npz"))


def edge_golden():
    return np.load(os.path.join(GOLDEN, "metrics_edges.npz"))


def edge_threshold(value, kind):
    """A base threshold of metrics_edges.npz as the reference was given it: Python float, np.float64 or np.float32."""
    return {"float": float, "float64": np.float64, "float32": np.float32}[str(kind)](value)


def test_oracle_metrics_match_reference_goldens():
    z = _golden()
    for i in range(int(z["n_series"])):
        s = z[f"s{i}"]
        for wi, w in enumerate(z["windows"]):
            got = [om.get_false_positives(s, t, int(w)) for t in z["thresholds"]]
            assert got == list(z["fp"][i, wi]), (i, int(w))
    s = z[f"s{int(z['roc_series'])}"]
    np.testing.assert_allclose(om.generate_roc_curve_fprs(s, 25, 0.08, grouping_window=50), z["roc_fprs"], rtol=0, atol=0)
    np.testing.assert_allclose(om.generate_roc_curve_tprs(s, 25), z["roc_tprs"], rtol=0, atol=0)


def test_oracle_metrics_edge_cases():
    assert om.get_false_positives([], 0.5) == 0
    assert om.get_false_positives([0.9], 0.5) == 1
    assert om.get_false_positives([0.1, 0.9], 0.5) == 1          # the reference raises IndexError here; defined as a no-op
    assert om.get_false_positives(np.ones(10), 0.5) == 10        # no 0->1 transition at all


def test_oracle_metrics_match_reference_edge_goldens():
    z = edge_golden()
    for i in range(int(z["n_series"])):
        s = z[f"s{i}"]
        got = [[[om.get_false_positives(s, edge_threshold(t, k), int(w)) for w in z["windows"]] for k in z["kinds"]]
               for t in z["base"]]
        assert np.array_equal(got, z["fp"][i]), (i, s.dtype, s)
    for j in range(2):
        s, w = z[f"roc_s{j}"], int(z[f"roc_window{j}"])
        assert om.generate_roc_curve_fprs(s, 25, 0.08, grouping_window=w) == list(z[f"roc_fprs{j}"])
        assert om.generate_roc_curve_tprs(s, 25) == list(z[f"roc_tprs{j}"])


def test_oracle_metrics_precision_of_the_comparison():
    """The two cases where the comparison's dtype decides the count: float32 scores against a Python float threshold
    compare in float32; a list of Python floats is a float64 array."""
    assert om.get_false_positives(np.array([0, np.float32(0.7), 0, 0], np.float32), 0.7) == 1
    assert om.get_false_positives(np.array([0, np.float32(0.7), 0, 0], np.float32), np.float64(0.7)) == 0
    assert om.get_false_positives([0, 0.5 - 1e-10, 0, 0], 0.5) == 0
    assert om.get_false_positives(np.float32([0, 0.5 - 1e-10, 0, 0]), 0.5) == 1


SCORE_FORMS = {"float16": lambda v: np.asarray(v, np.float16), "float32": lambda v: np.asarray(v, np.float32),
               "float64": lambda v: np.asarray(v, np.float64), "list": lambda v: [float(x) for x in v]}
THRESHOLD_FORMS = {"float": float, "int": int, "np.float32": np.float32, "np.float64": np.float64}


@pytest.mark.parametrize("score_form", list(SCORE_FORMS))
@pytest.mark.parametrize("thr_form", list(THRESHOLD_FORMS))
def test_comparison_dtype_is_numpys(score_form, thr_form):
    """comparison_dtype is the dtype NumPy compares ``np.array(scores) >= threshold`` in, and a score widened to float64
    against the threshold rounded to that dtype (what the device compares) is NumPy's comparison, element by element,
    on values at and next to the threshold in every precision."""
    from openwakeword_b200 import metrics as M
    for base in (0.7, 0.1, 0.5, 1.0 / 3.0, 1e-5, 0.0, 1.0, 3.0, 70000.0, 1e300):
        with np.errstate(over="ignore", invalid="ignore"):          # 70000 and 1e300 overflow float16 / float32
            t = THRESHOLD_FORMS[thr_form](base)
            vals = [0.0, 1.0, -1.0, np.inf, -np.inf, np.nan, float(t)]
            for d in (np.float16, np.float32, np.float64):
                x = d(float(t))
                vals += [float(v) for v in (np.nextafter(x, d(-np.inf)), x, np.nextafter(x, d(np.inf)))]
            a = np.array(SCORE_FORMS[score_form](vals))
            want = a >= t
            d = M.comparison_dtype(a.dtype, t)
            got = a.astype(np.float64) >= M._rounded_thresholds(a.dtype, [t])[0]
        assert d == np.result_type(a, t) == np.result_type(a.dtype, t), (score_form, thr_form, base)
        assert np.array_equal(got, want), (score_form, thr_form, base, a[got != want])
    assert M.comparison_dtype(np.dtype(np.float32), 0.7) == np.float32
    assert M.comparison_dtype(np.dtype(np.float32), np.float64(0.7)) == np.float64
    assert M.comparison_dtype(np.dtype(np.float16), 1) == np.float16


def test_rounded_thresholds_keep_each_elements_type():
    """A list of thresholds keeps each element's type (Python floats stay weak); an array's elements are NumPy
    scalars of its dtype."""
    from openwakeword_b200 import metrics as M
    f32 = np.dtype(np.float32)
    got = M._rounded_thresholds(f32, [0.7, np.float64(0.7), np.float32(0.7), 1])
    assert list(got) == [float(np.float32(0.7)), 0.7, float(np.float32(0.7)), 1.0]
    assert list(M._rounded_thresholds(f32, np.array([0.7, 0.1]))) == [0.7, 0.1]
    assert list(M._rounded_thresholds(f32, 0.1)) == [float(np.float32(0.1))]
    assert list(M._rounded_thresholds(np.dtype(np.float16), [0.7, 1e6])) == [float(np.float16(0.7)), np.inf]


def test_roc_fprs_pass_keywords_on_as_the_reference():
    """generate_roc_curve_fprs hands its keyword arguments to the false-positive count, as the reference hands them to
    get_false_positives: an unknown one is a TypeError (raised before anything reaches the device)."""
    from openwakeword_b200 import metrics as M
    for fn in (M.generate_roc_curve_fprs, om.generate_roc_curve_fprs):
        with pytest.raises(TypeError):
            fn([0.1, 0.9, 0.0], 5, grouping_windw=3)


@pytest.mark.gpu
def test_device_metrics_match_reference_goldens_and_oracle(built_library):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from openwakeword_b200 import metrics as M
    z = _golden()
    thr = z["thresholds"]
    for i in range(int(z["n_series"])):
        s = z[f"s{i}"]
        for wi, w in enumerate(z["windows"]):
            got = M.false_positives_batch(s, thr, int(w))[0]
            assert list(got) == list(z["fp"][i, wi]), (i, int(w))
    s = z[f"s{int(z['roc_series'])}"]
    np.testing.assert_allclose(M.generate_roc_curve_fprs(list(s), 25, 0.08, grouping_window=50), z["roc_fprs"], rtol=1e-12)
    np.testing.assert_allclose(M.generate_roc_curve_tprs(s, 25), z["roc_tprs"], rtol=1e-12)
    assert M.get_false_positives(list(s), 0.5) == int(z["fp"][int(z["roc_series"]), 2, 12])
    # batched: [64 series, 5000 frames] CUDA tensor against the oracle, series by series
    rng = np.random.default_rng(3)
    big = rng.uniform(0, 1, (64, 5000)).astype(np.float32) ** 3
    big[:, :40] = rng.uniform(0, 1, (64, 40))                       # dense start: the grouping rule has something to do
    t = torch.from_numpy(big).cuda()
    got = M.false_positives_batch(t, [0.2, 0.5, 0.8], grouping_window=7)
    for b in range(64):
        assert list(got[b]) == [om.get_false_positives(big[b], x, 7) for x in (0.2, 0.5, 0.8)]
    assert M.generate_roc_curve_tprs(t, 9) == om.generate_roc_curve_tprs(big.reshape(-1), 9)
