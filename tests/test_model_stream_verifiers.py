"""not-gpu tests of verifiers on stream models (Model(stream_verifiers=), set_stream_verifier): a fake context applies
head banks and verifier banks of both kinds the way verifier.cu does (oracle arithmetic), and every stream of a Model
with stream models and stream verifiers must equal an independent single-stream Model whose ordinary head and custom
verifier are that stream's; bookkeeping, threshold propagation and refusals."""
import numpy as np
import pytest

import openwakeword_b200 as owb
from openwakeword_b200 import _native
from openwakeword_b200 import weights as W
from helpers import emb_weights, verifier_pipeline as _pipeline
import fake_backend


@pytest.fixture
def fake_svctx(monkeypatch):
    monkeypatch.setattr(_native, "Context", fake_backend.FakeContext)


FI = np.random.default_rng(0).normal(0, 1, (41, 96)).astype(np.float32)


def _cands():
    return [W.synthetic_head(seed=200 + i) for i in range(3)]


def _solo(h, v, thr):
    kw = dict(custom_verifier_models={"mine": {0: v}}) if v is not None else {}
    return owb.Model(wakeword_models=[{"name": "mine", "head": h}], embedding_model_path=emb_weights(), feature_init=FI,
                     max_chunks=4, custom_verifier_threshold=thr, **kw)


@pytest.mark.parametrize("kw", [{}, {"patience": {"mine": 2}, "threshold": {"mine": 0.5}},
                                {"debounce_time": 0.2, "threshold": {"mine": 0.5}}])
def test_stream_verifiers_equal_independent_models(fake_svctx, kw):
    cands = _cands()
    v = _pipeline("alexa")
    B, thr = 4, 0.0
    sm = {0: cands[0], 1: cands[1], 2: cands[0]}                # stream 3 has no model
    sv = {0: v, 2: v, 3: v}                                     # stream 1 has no verifier; stream 3's never runs
    m = owb.Model(wakeword_models=[{"name": "x", "head": cands[2]}], embedding_model_path=emb_weights(), feature_init=FI,
                  max_chunks=4, n_streams=B, stream_models={"mine": sm}, stream_verifiers={"mine": sv},
                  custom_verifier_threshold=thr)
    solos = {b: _solo(sm[b], sv.get(b), thr) for b in sm}
    rng = np.random.default_rng(1)
    sizes = [1280, 1280, 2560, 640, 1280, 6400, 1280, 640, 1280, 2560, 1280, 1280]
    pcm = np.clip(rng.normal(0, 4000, (B, sum(sizes))), -32768, 32767).astype(np.int16)
    pos, n_ver = 0, 0
    for n in sizes:
        got = m.predict(pcm[:, pos:pos + n], **kw)["mine"]
        for b in range(B):
            if b in solos:
                want = solos[b].predict(pcm[b, pos:pos + n], **kw)["mine"]
                assert got[b] == np.float32(want), (pos, b)
            else:
                assert got[b] == 0.0
        n_ver += int(got[0] != 0.0)
        pos += n
    assert n_ver > 0 or kw                                      # patience / debounce may zero every score here


def test_bookkeeping_threshold_and_refusals(fake_svctx):
    cands = _cands()
    v = _pipeline("alexa")
    B = 4
    m = owb.Model(wakeword_models=[{"name": "x", "head": cands[2]}], embedding_model_path=emb_weights(), feature_init=FI,
                  max_chunks=4, n_streams=B, stream_models={"mine": {None: cands[0]}})
    ctx = m.preprocessor.ctx
    assert m.stream_verifiers == {}
    m.set_stream_verifier("mine", v, [1, 2])
    st = m._svbanks["mine"]
    assert st["slots"].tolist()[1] >= 0 and st["slots"].tolist()[0] == -1
    assert m.stream_verifiers["mine"] == {1: v, 2: v}
    m.set_stream_verifier("mine", v)
    assert m.stream_verifiers["mine"] is v
    assert len(set(st["slots"].tolist())) == 1                  # one slot for every stream
    m.set_stream_verifier("mine", None, [0])
    assert set(m.stream_verifiers["mine"]) == {1, 2, 3}
    m.set_stream_verifier("mine", None)
    assert "mine" not in m.stream_verifiers and (st["slots"] == -1).all()
    m.custom_verifier_threshold = 0.25
    assert ctx.banks[st["bank"]]["thr"] == np.float32(0.25)
    assert "mine" not in m.custom_verifier_models
    # a stream whose model is removed stays 0.0 even at threshold 0
    m.set_stream_verifier("mine", v)
    m.custom_verifier_threshold = 0.0
    m.set_stream_model("mine", None, [2])
    x = np.clip(np.random.default_rng(2).normal(0, 4000, (B, 1280 * 8)), -32768, 32767).astype(np.int16)
    for s in range(8):
        assert m.predict(x[:, s * 1280:(s + 1) * 1280])["mine"][2] == 0.0
    # refusals
    with pytest.raises(ValueError):
        m.set_stream_verifier("nope", v)
    with pytest.raises(ValueError):
        m.set_stream_verifier("x", v)                            # an ordinary model: set_custom_verifier
    with pytest.raises(ValueError):
        m.set_stream_verifier("mine", _pipeline("timer"))        # another input window
    with pytest.raises(ValueError):
        m.set_stream_verifier("mine", object())
    with pytest.raises(ValueError):
        m.set_custom_verifier("mine", v)
    with pytest.raises(ValueError):
        owb.Model(wakeword_models=[{"name": "x", "head": cands[2]}], embedding_model_path=emb_weights(),
                  feature_init=FI, stream_verifiers={"x": {0: v}})
    with pytest.raises(ValueError):
        m.train_stream_verifiers("x", {0: ([], [])})
