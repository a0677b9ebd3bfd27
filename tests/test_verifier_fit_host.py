"""not-gpu: the float64 verifier fit against scikit-learn, the host arithmetic of train_custom_verifier (offsets, RNG
order, the framing of the enrollment clip) against the reference's predict loop, and the pickle it writes."""
import pickletools

import numpy as np
import pytest

from verifier_fit_ref import fit_verifier_f64, linear_proba

sklearn = pytest.importorskip("sklearn")


def _data(rng, n_pos, n_neg, n_in=16, offset=0.0):
    sc = rng.uniform(0.2, 3, 96)
    x = (rng.normal(0, 1, (n_pos + n_neg, n_in, 96)) * sc + rng.normal(0, 2, 96) + offset).astype(np.float32)
    x[:n_pos] += rng.normal(0, 0.4, 96).astype(np.float32)
    return x, np.array([1] * n_pos + [0] * n_neg)


def _sk_fit(x, y, C=0.001):
    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import FunctionTransformer, StandardScaler
    from openwakeword_b200.custom_verifier_model import flatten_features
    return make_pipeline(FunctionTransformer(flatten_features), StandardScaler(),
                         LogisticRegression(random_state=0, max_iter=2000, C=C)).fit(x, y)


@pytest.mark.parametrize("n_pos,n_neg,offset,const", [(60, 140, 0.0, False), (30, 470, 1e3, True)])
def test_fit_f64_against_sklearn(n_pos, n_neg, offset, const):
    rng = np.random.default_rng(n_pos)
    x, y = _data(rng, n_pos, n_neg, offset=offset)
    if const:
        x[:, 3, 7] = 2.5
        x[:, 0, :5] = 0.0
    f = fit_verifier_f64(x, y)
    p = _sk_fit(x, y)
    sc = p.steps[1][1]
    np.testing.assert_allclose(f["mean"], sc.mean_, rtol=1e-12, atol=0)
    np.testing.assert_allclose(f["var"], sc.var_, rtol=1e-12, atol=1e-300)
    np.testing.assert_array_equal(f["scale"] == 1.0, sc.scale_ == 1.0)
    probe, _ = _data(np.random.default_rng(7), 100, 100, offset=offset)
    for z in (x, probe):
        d = np.abs(linear_proba(f["mean"], f["scale"], f["coef"], f["intercept"], z) - p.predict_proba(z)[:, 1]).max()
        print(f"n = {len(x)}: max |p_f64 - p_sklearn| = {d:.2e}")
        assert d <= 1e-3            # scikit-learn's lbfgs stops short of the optimum by up to ~6e-4 in p
    assert f["iters"] <= 10


def test_fit_f64_is_the_minimiser():
    """the gradient of the objective at the f64 solution is at round-off (its definition, checked independently)."""
    rng = np.random.default_rng(3)
    x, y = _data(rng, 20, 80, n_in=2)
    for C in (1e-3, 1.0, 100.0):
        f = fit_verifier_f64(x, y, C=C)
        z = (x.reshape(len(x), -1).astype(np.float64) - f["mean"]) / f["scale"]
        p = linear_proba(f["mean"], f["scale"], f["coef"], f["intercept"], x)
        g = np.concatenate([f["coef"] + C * z.T @ (p - y), [C * (p - y).sum()]])
        assert np.abs(g).max() <= 1e-11 * max(1.0, C * len(x)), C


class _Recorder:
    """A stand-in of Model for get_reference_clip_features: records the PCM of each predict call; score by a table."""

    def __init__(self, scores):
        self.calls, self.scores = [], scores
        self.model_inputs = {"m": 2}
        self.preprocessor = self

    def predict(self, x):
        self.calls.append(np.array(x))
        return {"m": self.scores[len(self.calls) - 1]}

    def get_features(self, n):
        return np.full((1, n, 96), len(self.calls), np.float32)


def test_enrollment_clip_frames_the_reference_loop():
    """The passes of train_custom_verifier, concatenated into one clip plus a chunk, step exactly the chunks the
    reference's get_reference_clip_features loop feeds predict, in order, and draw the same offsets from the seeded
    NumPy RNG."""
    from openwakeword_b200.custom_verifier_model import (enrollment_clip, enrollment_passes,
                                                         get_reference_clip_features)
    rng = np.random.default_rng(0)
    pos = [rng.integers(-3000, 3000, L).astype(np.int16) for L in (1280 * 7 + 5, 20000, 1281, 1280 * 2)]
    neg = [rng.integers(-3000, 3000, L).astype(np.int16) for L in (30001, 1280, 5000)]
    scores = rng.uniform(0, 1, 10000)
    rec = _Recorder(scores)
    np.random.seed(1234)
    for c in pos:
        get_reference_clip_features(c, rec, "m", N=5)
    for c in neg:
        get_reference_clip_features(c, rec, "m", threshold=0.0, N=1)
    after_ref = np.random.randint(0, 1 << 30)
    np.random.seed(1234)
    passes = enrollment_passes([len(c) for c in pos], [len(c) for c in neg])
    assert np.random.randint(0, 1 << 30) == after_ref          # same number of draws
    pcm, lab = enrollment_clip(pos, neg, passes)
    steps = len(range(0, pcm.size - 1280, 1280))               # the bulk path's framing at padding 0
    assert steps == len(rec.calls) == lab.size
    ref = np.concatenate(rec.calls) if rec.calls else np.zeros(0, np.int16)
    np.testing.assert_array_equal(pcm[:steps * 1280], ref)
    assert lab.sum() == sum(k for p, _, _, k in passes if p)


def _fake_fit(rng, D):
    var = rng.uniform(0.5, 2, D)
    var[3] = 0.0
    return {"mean": rng.normal(0, 1, (1, D)), "var": var[None], "coef": rng.normal(0, 0.1, (1, D)),
            "intercept": np.array([0.3]), "iters": np.array([5], np.int32)}


def test_pickle_names_the_reference_function_and_round_trips(tmp_path):
    from openwakeword_b200.custom_verifier_model import (_pipeline, dumps_verifier, linear_verifier_params,
                                                         load_verifier)
    rng = np.random.default_rng(5)
    x, y = _data(rng, 10, 30, n_in=3)
    fit = _fake_fit(rng, 3 * 96)
    pipe = _pipeline(len(x), 3, np.array([0, 1]), fit)
    blob = dumps_verifier(pipe)
    strings, globals_ = [], []
    for op, arg, _ in pickletools.genops(blob):
        if op.name in ("SHORT_BINUNICODE", "BINUNICODE", "UNICODE"):
            strings.append(arg)
        if op.name == "STACK_GLOBAL":
            globals_.append(tuple(strings[-2:]))
        if op.name == "GLOBAL":
            globals_.append(tuple(arg.split(" ")))
    assert ("openwakeword.custom_verifier_model", "flatten_features") in globals_
    assert not any(m.startswith("openwakeword_b200") for m, _ in globals_)
    path = tmp_path / "v.pkl"
    path.write_bytes(blob)
    v = load_verifier(str(path))
    mean, w, b = linear_verifier_params(v)
    assert v.steps[1][1].scale_[3] == 1.0
    np.testing.assert_array_equal(mean, fit["mean"][0].astype(np.float32))
    z = x.reshape(len(x), -1).astype(np.float64)
    p_lin = 1.0 / (1.0 + np.exp(-(b + (z - mean) @ w.astype(np.float64))))
    np.testing.assert_allclose(v.predict_proba(x)[:, 1], p_lin, atol=1e-5)
    np.testing.assert_allclose(v.predict_proba(x), pipe.predict_proba(x), rtol=0, atol=0)
