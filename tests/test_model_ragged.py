"""Model.predict_ragged and Model.reset_streams on the CPU (no GPU): every stream of a multi-stream Model fed its own
arrays must give, label for label, what an independent reference-semantics OracleModel gives when fed the same arrays -
per-stream chunk accumulation, the n_prepared < 1280 rules, first-5 zeroing (again after reset_streams), patience,
debounce, and lockstep predict calls interleaved."""
import numpy as np
import pytest

import fake_backend
import openwakeword_b200 as owb
from helpers import NAMES, class_mapping, emb_weights, head
from openwakeword_b200 import _native
from oracle import streaming

MAX_CHUNKS = 2


@pytest.fixture
def fake_ctx(monkeypatch):
    monkeypatch.setattr(_native, "Context", fake_backend.FakeContext)


def _models(B, fi):
    specs = [{"name": n, "head": head(n), "class_mapping": class_mapping([n]).get(n)} for n in NAMES]
    m = owb.Model(wakeword_models=specs, embedding_model_path=emb_weights(), feature_init=fi, n_streams=B,
                  max_chunks=MAX_CHUNKS)
    oracles = [streaming.OracleModel(emb_weights(), {n: head(n) for n in NAMES}, class_mapping=class_mapping(NAMES),
                                     feature_init=fi) for _ in range(B)]
    return m, oracles


def _length(rng, allow_zero):
    k = rng.integers(0 if allow_zero else 1, 5)
    return [0, int(rng.integers(1, 401)), 1280, int(rng.integers(1281, 4000)),
            int(rng.integers(MAX_CHUNKS * 1280 + 1, 6 * 1280))][k]


@pytest.mark.parametrize("B,post", [(6, "none"), (7, "patience"), (9, "debounce")])
def test_predict_ragged_equals_independent_models(fake_ctx, B, post):
    rng = np.random.default_rng(B)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    m, oracles = _models(B, fi)
    thr = {n: 0.3 for n in NAMES}
    kw = {"none": {}, "patience": dict(patience={"alexa_v0.1": 2, "hey_jarvis_v0.1": 3}, threshold=thr),
          "debounce": dict(debounce_time=0.5, threshold=thr)}[post]
    # the reference's debounce divides by the samples prepared: with debounce no call is empty (tested separately)
    allow_zero = post != "debounce"
    n_calls, reset_at, reset_ids = 60, 31, [1, B - 2]
    lockstep = 0
    for t in range(n_calls):
        if t == reset_at:
            m.reset_streams(reset_ids)
            for b in reset_ids:
                oracles[b].reset(feature_init=fi)
        if t < 4 or t % 9 == 0:                            # lockstep predict, equal lengths
            n = _length(rng, allow_zero=False)
            xs = [rng.integers(-3000, 3000, n).astype(np.int16) for _ in range(B)]
            got = m.predict(np.stack(xs), **kw)
            lockstep += 1
        else:
            xs = [rng.integers(-3000, 3000, _length(rng, allow_zero)).astype(np.int16) for _ in range(B)]
            got = m.predict_ragged(xs, **kw)
        for b in range(B):
            ref = oracles[b].predict(xs[b], **kw)
            assert list(got) == list(ref)
            for lab, v in ref.items():
                assert abs(float(got[lab][b]) - float(v)) <= 1e-5, (t, b, lab, float(got[lab][b]), float(v))
    assert lockstep >= 8
    for b in range(B):
        np.testing.assert_allclose(m.preprocessor.get_features(16, stream=b)[0], oracles[b].preprocessor.get_features(16)[0],
                                   atol=1e-4)


def test_debounce_with_nothing_prepared_takes_the_whole_history(fake_ctx):
    """n_prepared == 0: the reference's debounce window divides by zero; here it is the whole 30-entry history."""
    rng = np.random.default_rng(5)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    m, oracles = _models(2, fi)
    thr = {n: 0.0 for n in NAMES}                          # every score is a hit: a non-zero prediction is debounced
    for t in range(8):
        x = rng.integers(-3000, 3000, 1280).astype(np.int16)
        m.predict_ragged([x, x], debounce_time=0.5, threshold=thr)
    got = m.predict_ragged([rng.integers(-3000, 3000, 1280).astype(np.int16), np.zeros(0, np.int16)],
                           debounce_time=0.5, threshold=thr)
    for lab in got:
        assert got[lab][1] == 0.0


def test_predict_ragged_errors(fake_ctx):
    fi = np.zeros((41, 96), np.float32)
    m, _ = _models(3, fi)
    with pytest.raises(ValueError):
        m.predict_ragged([np.zeros(1280, np.int16)] * 2)           # one array per stream
    with pytest.raises(ValueError):
        m.predict_ragged([np.zeros(1280, np.int16), [0] * 1280, np.zeros(1280, np.int16)])   # not an ndarray
    with pytest.raises(ValueError):
        m.predict_ragged(5)
    with pytest.raises(ValueError):
        m.reset_streams([3])
