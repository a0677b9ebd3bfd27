"""Model(stream_models=...) and set_stream_model on a CPU stand-in of the head-bank ABI (oracle arithmetic): every stream
against an independent single-model Model, slot sharing and freeing, and the refusals."""
import numpy as np
import pytest

import fake_backend
from helpers import emb_weights, head
from openwakeword_b200 import _native, weights as W
import openwakeword_b200 as owb


@pytest.fixture
def fake_bctx(monkeypatch):
    monkeypatch.setattr(_native, "Context", fake_backend.FakeContext)


FI = np.random.default_rng(0).normal(0, 1, (41, 96)).astype(np.float32)


def _cands():
    return [W.synthetic_head(seed=200 + i) for i in range(3)]


def _model(**kw):
    return owb.Model(wakeword_models=[{"name": "alexa_v0.1", "head": head("alexa_v0.1")}],
                     embedding_model_path=emb_weights(), feature_init=FI, max_chunks=4, **kw)


def _solo(h):
    return owb.Model(wakeword_models=[{"name": "mine", "head": h}], embedding_model_path=emb_weights(), feature_init=FI,
                     max_chunks=4)


def test_per_stream_models_equal_independent_models(fake_bctx):
    cands = _cands()
    B = 3
    m = _model(n_streams=B, stream_models={"mine": {None: cands[0], 1: cands[1]}})
    assert m.model_inputs["mine"] == 16 and m.model_outputs["mine"] == 1
    st = m._sbanks["mine"]
    assert st["slots"].tolist() == [0, 1, 0]               # one slot for the object shared by streams 0 and 2
    rng = np.random.default_rng(1)
    sizes = [1280, 1280, 2560, 640, 1280, 3840, 1280, 1280, 1280, 2560, 1280]
    pcm = np.clip(rng.normal(0, 4000, (B, sum(sizes))), -32768, 32767).astype(np.int16)
    solos = {(b, k): _solo(cands[k]) for b in range(B) for k in range(3)}
    plan = {b: 0 for b in range(B)}
    plan[1] = 1
    pos = 0
    for t, n in enumerate(sizes):
        if t == 6:
            m.set_stream_model("mine", None, [2])                # stream 2 loses its model
            m.set_stream_model("mine", cands[2], [1])            # stream 1 switches; slot 1 is free again
            plan[2], plan[1] = None, 2
            assert st["slots"].tolist() == [0, 1, -1]
        x = pcm[:, pos:pos + n]
        pos += n
        got = m.predict(x)
        for b in range(B):
            want = {}
            for k in range(3):
                r = solos[(b, k)].predict(x[b])
                if plan[b] == k:
                    want = r
            assert got["alexa_v0.1"][b] is not None
            if plan[b] is None:
                assert got["mine"][b] == 0.0
            else:
                assert np.float32(got["mine"][b]) == np.float32(want["mine"]), (t, b)


@pytest.mark.parametrize("kw", [dict(patience={"mine": 2}, threshold={"mine": 0.3}),
                                dict(debounce_time=0.3, threshold={"mine": 0.3})])
def test_patience_debounce_and_reset_streams(fake_bctx, kw):
    cands = _cands()
    B = 2
    m = _model(n_streams=B, stream_models={"mine": {0: cands[0], 1: cands[1]}})
    solos = [_solo(cands[0]), _solo(cands[1])]
    rng = np.random.default_rng(2)
    pcm = np.clip(rng.normal(0, 6000, (B, 12 * 1280)), -32768, 32767).astype(np.int16)
    for t in range(12):
        if t == 8:
            m.reset_streams([1], feature_init=FI)
            solos[1].reset(feature_init=FI)
        x = pcm[:, t * 1280:(t + 1) * 1280]
        got = m.predict(x, **kw)
        for b in range(B):
            assert np.float32(got["mine"][b]) == np.float32(solos[b].predict(x[b], **kw)["mine"]), (t, b)


def test_slots_capacity_and_refusals(fake_bctx, tmp_path):
    cands = _cands()
    m = _model(n_streams=4, stream_models={"mine": {0: cands[0]}}, stream_model_capacity=2)
    st = m._sbanks["mine"]
    m.set_stream_model("mine", cands[1], [1, 2])
    assert st["slots"].tolist() == [0, 1, 1, -1]
    with pytest.raises(ValueError, match="distinct models"):
        m.set_stream_model("mine", cands[2], [3])
    m.set_stream_model("mine", cands[2], [0])               # slot 0 is freed by the same call
    assert st["slots"].tolist() == [0, 1, 1, -1]
    path = str(tmp_path / "h.npz")
    W.save_head(path, cands[0])
    m.set_stream_model("mine", path, [0])
    m.set_stream_model("mine", path, [1, 2, 3])
    assert st["slots"].tolist() == [0, 0, 0, 0]               # one path, one slot
    with pytest.raises(ValueError, match="shape"):
        m.set_stream_model("mine", W.synthetic_head(hidden=32, seed=3), [0])
    with pytest.raises(ValueError, match="stream ids"):
        m.set_stream_model("mine", cands[0], [4])
    with pytest.raises(ValueError, match="no stream models"):
        m.set_stream_model("alexa_v0.1", cands[0])
    with pytest.raises(ValueError, match="wakeword_models"):
        _model(stream_models={"alexa_v0.1": {0: cands[0]}})
    with pytest.raises(ValueError):
        _model(stream_models={"mine": {0: cands[0]}}, custom_verifier_models={"mine": path})
    with pytest.raises(ValueError, match="stream models"):
        m.set_custom_verifier("mine", None)
    assert m.labels() == ["alexa_v0.1", "mine"]
