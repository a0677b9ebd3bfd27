"""Model.export_streams / Model.import_streams on the CPU (no GPU), on the CPU stand-in of the C ABI: a stream
moved to another Model of the same configuration returns, call for call, what the unmoved stream returns - through
lockstep ``predict`` and ``predict_ragged``, remainders below 1280 samples, the first-5 zeroing, patience and debounce
history - also after a pickle round trip of the CPU StreamState.  The refusals raise ValueError."""
import pickle

import numpy as np
import pytest

import fake_backend
import openwakeword_b200 as owb
from helpers import NAMES, class_mapping, emb_weights, head
from openwakeword_b200 import _native

MAX_CHUNKS = 2


@pytest.fixture
def fake_ctx(monkeypatch):
    monkeypatch.setattr(_native, "Context", fake_backend.FakeContext)


def _model(B, fi, names=NAMES, **kw):
    specs = [{"name": n, "head": head(n), "class_mapping": class_mapping([n]).get(n)} for n in names]
    return owb.Model(wakeword_models=specs, embedding_model_path=emb_weights(), feature_init=fi, n_streams=B,
                     max_chunks=MAX_CHUNKS, **kw)


def _length(rng):
    return [0, int(rng.integers(1, 1280)), 1280, int(rng.integers(1281, 4000)),
            int(rng.integers(MAX_CHUNKS * 1280 + 1, 5 * 1280))][int(rng.integers(0, 5))]


def _call(m, xs, kw, lockstep):
    return m.predict(np.stack(xs), **kw) if lockstep else m.predict_ragged(xs, **kw)


@pytest.mark.parametrize("post", ["none", "patience", "debounce"])
def test_moved_stream_continues_as_the_unmoved_one(fake_ctx, post):
    """Model A runs 5 streams; after call 2 (within the first-5 zeroing, holding remainders) streams 0, 3, 4 are exported
    and imported into slots 5, 1, 3 of Model B, which had run calls of its own.  From then on every moved slot gets its
    source stream's samples and must return its source stream's predictions, while A keeps running the originals."""
    rng = np.random.default_rng({"none": 1, "patience": 2, "debounce": 3}[post])
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    thr = {n: 0.3 for n in NAMES}
    kw = {"none": {}, "patience": dict(patience={"alexa_v0.1": 2, "hey_jarvis_v0.1": 3}, threshold=thr),
          "debounce": dict(debounce_time=0.5, threshold=thr)}[post]
    a, b = _model(5, fi), _model(6, fi)
    src, dst = [0, 3, 4], [5, 1, 3]

    def pcm(lengths):
        return [rng.integers(-3000, 3000, n).astype(np.int16) for n in lengths]

    for t in range(6):                                   # B's own history first (its counts pass the first-5 zeroing)
        b.predict_ragged(pcm([_length(rng) for _ in range(6)]), **kw)
    for t in range(2):
        a.predict(np.stack(pcm([700] * 5)), **kw)
    a.predict_ragged(pcm([300, 1500, 0, 1279, 2600]), **kw)
    state = a.export_streams(src)
    assert len(state) == 3 and [p.size for p in state.pending] == [420, 119, 160]
    assert all((c == 3).all() for c in state.counts.values())
    state = pickle.loads(pickle.dumps(state.to("cpu")))
    b.import_streams(dst, state)
    assert b.preprocessor.pending_ragged
    for t in range(40):
        lock = t % 7 == 0                                # lockstep predict: one length for every stream
        if lock:
            n = max(_length(rng), 1)
            xa, xb = pcm([n] * 5), pcm([n] * 6)
        else:
            xa, xb = pcm([_length(rng) for _ in range(5)]), pcm([_length(rng) for _ in range(6)])
        for s, d in zip(src, dst):
            xb[d] = xa[s]
        ga, gb = _call(a, xa, kw, lock), _call(b, xb, kw, lock)
        assert list(ga) == list(gb)
        for lab in ga:
            for s, d in zip(src, dst):
                assert ga[lab][s] == gb[lab][d], (t, lab, s, d, ga[lab][s], gb[lab][d])


def test_untouched_streams(fake_ctx):
    """Streams that are not import targets keep their remainders and history."""
    rng = np.random.default_rng(9)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    a, b = _model(3, fi), _model(4, fi)
    for m, B in ((a, 3), (b, 4)):
        m.predict_ragged([rng.integers(-3000, 3000, 2000 + 300 * i).astype(np.int16) for i in range(B)])
    b_before = {lab: b._h(lab)[0].copy() for lab in b.labels()}
    b.import_streams([2], a.export_streams([1]))
    for lab in b.labels():
        np.testing.assert_array_equal(np.delete(b._h(lab)[0], 2, axis=1), np.delete(b_before[lab], 2, axis=1))
        np.testing.assert_array_equal(b._h(lab)[0][:, 2], a._h(lab)[0][:, 1])
    buf, lens = b.preprocessor._ragged_pending()
    abuf, alens = a.preprocessor._ragged_pending()
    assert lens[2] == alens[1] and np.array_equal(buf[2, :lens[2]], abuf[1, :alens[1]])
    assert [int(v) for v in lens[[0, 1, 3]]] == [2000 % 1280, 2300 % 1280, 2900 % 1280]


def test_import_refusals(fake_ctx):
    fi = np.zeros((41, 96), np.float32)
    a = _model(3, fi)
    a.predict(np.zeros((3, 1280), np.int16))
    st = a.export_streams([0, 1])
    with pytest.raises(ValueError):
        _model(3, fi, split_from=7).import_streams([0, 1], st)           # another configuration
    with pytest.raises(ValueError):
        _model(3, fi, names=NAMES[:2]).import_streams([0, 1], st)       # another label set
    other = _model(3, fi)
    with pytest.raises(ValueError):
        other.import_streams([0], st)                                    # one id per exported stream
    with pytest.raises(ValueError):
        other.import_streams([1, 1], st)                                 # distinct ids
    with pytest.raises(ValueError):
        other.import_streams([0, 3], st)                                 # out of range
    with pytest.raises(ValueError):
        other.export_streams([-1])
    other.speex_ns = object()                                            # Speex state cannot be exported
    with pytest.raises(ValueError):
        other.import_streams([0, 1], st)
