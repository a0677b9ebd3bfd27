"""not-gpu tests of custom verifier models: loading the reference's pickles without the reference package, the
reduction of the pipeline to the device's linear form, and the Model's verifier logic driven through a fake context
that applies verifier banks the way verifier.cu does, against the verifier goldens of the reference plumbing."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import openwakeword_b200 as owb
from openwakeword_b200 import _native
from openwakeword_b200.custom_verifier_model import linear_verifier_params, flatten_features
from helpers import (GOLDEN, VERIFIER_CASES, case_model as _model, emb_weights, head, class_mapping, kernel_order_proba,
                     load_case, verifier_pipeline as _pipeline)
import fake_backend

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def fake_vctx(monkeypatch):
    monkeypatch.setattr(_native, "Context", fake_backend.FakeContext)


def test_golden_pickle_loads_without_the_reference_package():
    code = ("import sys; sys.modules['openwakeword'] = None\n"
            "try:\n    import openwakeword\nexcept ImportError:\n    pass\nelse:\n    raise SystemExit('importable')\n"
            "import numpy as np\n"
            "from openwakeword_b200.custom_verifier_model import load_verifier, linear_verifier_params\n"
            f"v = load_verifier({os.path.join(GOLDEN, 'verifier_alexa.pkl')!r})\n"
            "assert linear_verifier_params(v) is not None\n"
            "print(v.predict_proba(np.zeros((1, 16, 96), np.float32))[0][-1])\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    with pytest.raises(Exception):       # the plain unpickler needs the reference package
        subprocess.run([sys.executable, "-c", "import sys, pickle; sys.modules['openwakeword'] = None; "
                        f"pickle.load(open({os.path.join(GOLDEN, 'verifier_alexa.pkl')!r}, 'rb'))"],
                       cwd=ROOT, check=True, capture_output=True)


@pytest.mark.parametrize("tag", ["alexa", "timer"])
def test_linear_params_reproduce_predict_proba(tag):
    v = _pipeline(tag)
    mean, w, b = linear_verifier_params(v)
    n_in = mean.size // 96
    assert mean.dtype == np.float32 and w.dtype == np.float32 and mean.size == n_in * 96
    rng = np.random.default_rng(3)
    x = (rng.normal(0, 1, (2000, n_in, 96)) * rng.uniform(0.5, 3, 96) + rng.normal(0, 2, 96)).astype(np.float32)
    ref = v.predict_proba(x)[:, -1]
    got = kernel_order_proba(mean, w, b, x)
    print(f"{tag}: max |kernel order fp32 - predict_proba| = {np.abs(got - ref).max():.2e}")
    assert np.abs(got - ref).max() <= 1e-6
    from oracle.verifier import verifier_proba
    np.testing.assert_allclose(verifier_proba(v, x), ref, rtol=0, atol=1e-12)


def test_only_the_reference_pipeline_is_recognised():
    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import FunctionTransformer, StandardScaler, MinMaxScaler
    rng = np.random.default_rng(0)
    x = rng.normal(0, 1, (30, 2, 96)).astype(np.float32)
    y2 = np.arange(30) % 2
    good = make_pipeline(FunctionTransformer(flatten_features), StandardScaler(), LogisticRegression(max_iter=200)).fit(x, y2)
    assert linear_verifier_params(good) is not None
    multi = make_pipeline(FunctionTransformer(flatten_features), StandardScaler(), LogisticRegression(max_iter=200))
    assert linear_verifier_params(multi.fit(x, np.arange(30) % 3)) is None
    extra = make_pipeline(FunctionTransformer(flatten_features), MinMaxScaler(), StandardScaler(), LogisticRegression(max_iter=200))
    assert linear_verifier_params(extra.fit(x, y2)) is None
    from test_abi_and_host import _ConstVerifier
    assert linear_verifier_params(_ConstVerifier(0.5)) is None


@pytest.mark.parametrize("tag", VERIFIER_CASES)
def test_fake_backend_model_reproduces_verifier_golden(fake_vctx, tag):
    c = load_case(tag)
    parent = str(c["parent"])
    path = os.path.join(GOLDEN, str(c["verifier"]))
    m = _model(c, custom_verifier_models={parent: path}, custom_verifier_threshold=float(c["threshold"]))
    assert parent in m._vbanks and not m._host_verifiers
    res = m.predict_clip(c["pcm"], padding=int(c["padding"]), chunk_size=int(c["chunk"]))
    got = np.array([[r[lab] for lab in c["labels"]] for r in res], np.float32)
    print(f"{tag}: max |fake Model - reference| = {np.abs(got - c['scores']).max():.2e}")
    assert np.abs(got - c["scores"]).max() <= 1e-5
    assert not np.allclose(c["scores"], c["unverified"])          # the verifier changed some scores


def test_multi_stream_model_equals_single_stream_models(fake_vctx):
    """3 streams: stream 0 with the golden verifier, stream 1 with a second one, stream 2 without; a chunk of 640 samples
    (no step: the previous prediction is re-verified on the stateless entry), 1- and 2-chunk calls, then a mid-run
    reassignment."""
    c = load_case("verifier_alexa_c1280")
    name = c["names"][0]
    v0 = _pipeline("alexa")
    rng = np.random.default_rng(5)
    x = rng.normal(0, 1, (60, 16, 96)).astype(np.float32)
    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import FunctionTransformer, StandardScaler
    v1 = make_pipeline(FunctionTransformer(flatten_features), StandardScaler(),
                       LogisticRegression(C=0.001, max_iter=2000)).fit(x, np.arange(60) % 2)
    thr = 0.0
    pcm = np.clip(rng.normal(0, 3000, (3, 40 * 1280)), -32768, 32767).astype(np.int16)
    plan = [1280] * 7 + [640, 640, 2560, 1280, 2560] + [1280] * 3
    swap_at = 12

    m = owb.Model(wakeword_models=[{"name": name, "head": head(name)}], embedding_model_path=emb_weights(),
                  feature_init=c["feature_init"], max_chunks=8, n_streams=3,
                  custom_verifier_models={name: {0: v0, 1: v1}}, custom_verifier_threshold=thr)
    multi, pos = [], 0
    for k, n in enumerate(plan):
        if k == swap_at:
            m.set_custom_verifier(name, v0, [1])
            m.set_custom_verifier(name, v1, [2])
            m.set_custom_verifier(name, None, [0])
        multi.append(m.predict(pcm[:, pos:pos + n])[name])
        pos += n
    multi = np.stack(multi, axis=1)
    singles = []
    for b, (v_before, v_after) in enumerate([(v0, None), (v1, v0), (None, v1)]):
        m = owb.Model(wakeword_models=[{"name": name, "head": head(name)}], embedding_model_path=emb_weights(),
                      feature_init=c["feature_init"], max_chunks=8, custom_verifier_threshold=thr)
        if v_before is not None:
            m.set_custom_verifier(name, v_before)
        row, pos = [], 0
        for k, n in enumerate(plan):
            if k == swap_at:
                m.set_custom_verifier(name, v_after)
            row.append(m.predict(pcm[b, pos:pos + n])[name])
            pos += n
        singles.append(row)
    np.testing.assert_array_equal(multi, np.array(singles, np.float32))
    assert (multi[:, 5:] != 0).all()


def test_set_custom_verifier_rejects_what_the_device_cannot_run(fake_vctx, tmp_path):
    from test_abi_and_host import _ConstVerifier
    c = load_case("verifier_alexa_c1280")
    name = c["names"][0]
    m = _model(c)
    with pytest.raises(ValueError):
        m.set_custom_verifier(name, _ConstVerifier(0.5))
    with pytest.raises(ValueError):
        m.set_custom_verifier(name, _pipeline("timer"))          # trained on another head's 34-row window
    with pytest.raises(ValueError):
        m.set_custom_verifier("not_loaded", _pipeline("alexa"))
    with pytest.raises(ValueError):
        m.set_custom_verifier(name, _pipeline("alexa"), streams=[1])
    p = str(tmp_path / "const.pkl")
    with open(p, "wb") as f:
        pickle.dump(_ConstVerifier(0.5), f)
    with pytest.raises(ValueError):
        _model(c, custom_verifier_models={name: {0: p}})


@pytest.mark.parametrize("tag", VERIFIER_CASES)
def test_verified_oracle_model_reproduces_verifier_golden(tag):
    """oracle/verifier.py: the float64 restatement inside the oracle's streaming state machine against the reference."""
    from oracle import streaming
    from oracle.verifier import VerifiedOracleModel
    c = load_case(tag)
    parent = str(c["parent"])
    om = VerifiedOracleModel(emb_weights(int(c["emb_seed"])), {n: head(n) for n in c["names"]},
                             verifiers={parent: _pipeline(parent.split("_")[0])}, threshold=float(c["threshold"]),
                             class_mapping=class_mapping(c["names"]), feature_init=c["feature_init"])
    res = om.predict_clip(c["pcm"], padding=int(c["padding"]), chunk_size=int(c["chunk"]))
    got = np.array([[r[lab] for lab in c["labels"]] for r in res], np.float32)
    print(f"{tag}: max |VerifiedOracleModel - reference| = {np.abs(got - c['scores']).max():.2e}")
    assert np.abs(got - c["scores"]).max() <= 1e-5


def test_calls_longer_than_max_chunks_verify_the_max_once(fake_vctx):
    """A call of more than max_chunks*1280 samples runs as several device steps; the verifier must see the max over all
    its chunk windows and the newest window (model.py:287-328), as VerifiedOracleModel does for the whole call."""
    from oracle.verifier import VerifiedOracleModel
    c = load_case("verifier_alexa_c1280")
    name = c["names"][0]
    v = _pipeline("alexa")
    rng = np.random.default_rng(12)
    plan = [1280] * 6 + [5 * 1280, 1280, 7 * 1280, 640, 640, 3 * 1280]
    pcm = np.clip(rng.normal(0, 3000, sum(plan)), -32768, 32767).astype(np.int16)
    specs = [{"name": name, "head": head(name)}]
    thr = 0.06
    m = owb.Model(wakeword_models=specs, embedding_model_path=emb_weights(), feature_init=c["feature_init"],
                  max_chunks=2, custom_verifier_models={name: os.path.join(GOLDEN, "verifier_alexa.pkl")},
                  custom_verifier_threshold=thr)
    om = VerifiedOracleModel(emb_weights(), {name: head(name)}, verifiers={name: v}, threshold=thr,
                             feature_init=c["feature_init"])
    plain = owb.Model(wakeword_models=specs, embedding_model_path=emb_weights(), feature_init=c["feature_init"],
                      max_chunks=2)
    got, ref, raw, pos = [], [], [], 0
    for n in plan:
        got.append(m.predict(pcm[pos:pos + n])[name])
        ref.append(om.predict(pcm[pos:pos + n])[name])
        raw.append(plain.predict(pcm[pos:pos + n])[name])
        pos += n
    got, ref, raw = np.array(got, np.float32), np.array(ref, np.float32), np.array(raw, np.float32)
    print("device path", got, "oracle", ref, "unverified", raw, sep="\n")
    long = [k for k, n in enumerate(plan) if n > 2 * 1280]
    assert (raw[long] >= np.float32(thr)).any() and (got[long] != raw[long]).any()       # verified long calls
    assert np.abs(got - ref).max() <= 1e-5


def test_threshold_removal_and_attribute_follow_set_custom_verifier(fake_vctx, tmp_path):
    from test_abi_and_host import _ConstVerifier
    c = load_case("verifier_alexa_c1280")
    name = c["names"][0]
    p = str(tmp_path / "const.pkl")
    with open(p, "wb") as f:
        pickle.dump(_ConstVerifier(0.7), f)
    m = _model(c, custom_verifier_models={name: p}, custom_verifier_threshold=0.0)
    assert name in m._host_verifiers and name in m.custom_verifier_models
    m.set_custom_verifier(name, None)                       # removes the host-side verifier too
    assert not m._host_verifiers and name not in m.custom_verifier_models
    v = _pipeline("alexa")
    m.set_custom_verifier(name, v)
    assert m.custom_verifier_models[name] is v
    ctx = m.preprocessor.ctx
    bank = ctx.banks[m._vbanks[name]["bank"]]
    m.custom_verifier_threshold = 0.25                      # follows on the device banks
    assert bank["thr"] == np.float32(0.25)
    rng = np.random.default_rng(2)
    for _ in range(7):
        m.predict(rng.integers(-1000, 1000, 1280).astype(np.int16))
    m.set_custom_verifier(name, None)
    assert name not in m.custom_verifier_models and (bank["assign"] == -1).all()
