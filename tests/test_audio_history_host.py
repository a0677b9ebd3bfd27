"""Stream audio without a GPU: ``AudioFeatures.raw_data_buffer`` against the reference's own deque (the fixture
tests/golden/raw_buffer.npz, recorded by make_raw_buffer_golden.py from the unmodified reference), on the lockstep and
the ragged accumulation paths, and the host-side rules of the audio calls (ValueError / AttributeError), on a stand-in
of the C ABI whose audio history is a NumPy ring with the semantics of include/owwb200.h (oww_set_audio_history)."""
import os

import numpy as np
import pytest

import fake_backend
from openwakeword_b200 import _native
from openwakeword_b200.utils import AudioFeatures, audio_history_samples
from helpers import emb_weights, streams_model as _model

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "raw_buffer.npz")


@pytest.fixture
def audio_only(monkeypatch):
    """steps record the audio and nothing else (no features, no scores)"""
    monkeypatch.setattr(_native, "Context", fake_backend.FakeContext)
    monkeypatch.setattr(fake_backend.FakeContext, "features", False)


@pytest.fixture
def audio_detect(monkeypatch):
    monkeypatch.setattr(_native, "Context", fake_backend.FakeContext)


def _features(n_streams=1, seconds=10.0):
    return AudioFeatures(embedding_model_path=emb_weights(), n_streams=n_streams,
                         feature_init=np.zeros((41, 96), np.float32), audio_history=seconds)


def _expected(z, k):
    return z["signal"][z["raw_lo"][k]:z["raw_hi"][k]]


def test_raw_data_buffer_matches_the_reference_lockstep(audio_only):
    z = np.load(GOLDEN)
    af = _features()
    off = 0
    for k, c in enumerate(z["calls"]):
        if c < 0:
            af.reset()
        else:
            assert af(z["signal"][off:off + c]) == z["ret"][k], k
            off += c
        buf = af.raw_data_buffer
        assert buf.maxlen == 160000
        assert np.array_equal(np.array(buf, np.int16), _expected(z, k)), k
        assert all(type(v) is int for v in list(buf)[:3])


def test_raw_data_buffer_matches_the_reference_ragged(audio_only):
    """Stream 0 gets the fixture's calls while stream 1 gets other lengths, so the streams hold different remainders
    and the per-stream accumulation (with its per-stream flag) runs throughout."""
    z = np.load(GOLDEN)
    af = _features(n_streams=2)
    rng = np.random.default_rng(3)
    scores = np.zeros((2, 1), np.float32)
    off = 0
    for k, c in enumerate(z["calls"]):
        if c < 0:
            af.reset(stream_ids=[0])
        else:
            other = rng.integers(-2000, 2000, int(rng.integers(0, 3000))).astype(np.int16)
            n_prep = af._streaming_features_ragged([z["signal"][off:off + c], other], scores)[0]
            assert n_prep[0] == z["ret"][k], k
            off += c
        assert np.array_equal(np.array(af.raw_data_buffer, np.int16), _expected(z, k)), k


def test_raw_data_buffer_shorter_history_keeps_the_last_samples(audio_only):
    af = _features(seconds=0.16)
    x = np.arange(5000, dtype=np.int16)
    af(x)                                       # steps 3840, holds 1160 (a remainder: not in the buffer)
    assert np.array_equal(np.array(af.raw_data_buffer, np.int16), x[3840 - 2560:3840])
    af(x[:100])                                 # steps nothing: 1260 held, all in the reference's buffer
    assert np.array_equal(np.array(af.raw_data_buffer, np.int16), np.concatenate((x, x[:100]))[-2560:])


def test_audio_history_rules(audio_only):
    af = _features(seconds=0.0)
    with pytest.raises(AttributeError, match="audio_history"):
        af.raw_data_buffer
    assert not hasattr(af, "raw_data_buffer")
    for bad in (0.05, -0.08, 60.08, 1.0001):
        with pytest.raises(ValueError, match="audio_history"):
            _features(seconds=bad)
    assert audio_history_samples(10) == 160000 and audio_history_samples(0.08) == 1280
    assert audio_history_samples(60) == 960000


def _mk(B, seconds, **kw):
    m = _model(B, np.zeros((41, 96), np.float32), audio_history=seconds, **kw)
    m.preprocessor._ensure_streams()
    return m


def _feed(m, host, xs, call):
    """call(xs) on Model m; host[b] += the samples stream b stepped in it"""
    held, lens0 = m.preprocessor._ragged_pending()
    out = call(xs)
    lens = m.preprocessor._ragged_pending()[1]
    for b in range(len(host)):
        allx = np.concatenate((held[b, :lens0[b]], xs[b]))
        host[b] = np.concatenate((host[b], allx[:allx.size - lens[b]]))
    return out


def test_model_get_audio_and_capture_on_the_stand_in(audio_detect):
    B = 3
    m = _mk(B, 0.32)
    rng = np.random.default_rng(5)
    host = [np.zeros(0, np.int16) for _ in range(B)]
    for _ in range(4):
        xs = [rng.integers(-3000, 3000, int(rng.integers(0, 4000))).astype(np.int16) for _ in range(B)]
        _feed(m, host, xs, m.predict_ragged)
    clips, ends = m.get_audio([2, 0, 2], 0.08)
    for i, b in enumerate([2, 0, 2]):
        assert ends[i] == host[b].size
        want = host[b][-1280:]
        assert np.array_equal(clips[i, 1280 - want.size:], want)
    clips, ends = m.get_audio([1], 0.16, end=host[1].size + 1280)        # post-roll not stepped yet: zeros
    assert ends[0] == host[1].size + 1280 and not clips[0, 1280:].any()
    assert np.array_equal(clips[0, :1280], host[1][-1280:])
    xs = [rng.integers(-3000, 3000, 1280).astype(np.int16) for _ in range(B)]
    ev = _feed(m, host, xs, lambda x: m.detect_ragged(x, threshold=0.0, capture=0.08))
    assert ev and all(len(e) == 5 for e in ev)
    for s, lab, sc, clip, end in ev:
        assert end == host[s].size and clip.dtype == np.int16 and np.array_equal(clip, host[s][-1280:])
    assert all(len(e) == 3 for e in m.detect(np.zeros((B, 1280), np.int16), threshold=0.0))


def test_model_audio_refusals(audio_detect):
    on, off, other = _mk(2, 0.16), _mk(2, 0.0), _mk(2, 0.32)
    with pytest.raises(ValueError, match="audio_history"):
        off.get_audio([0], 0.08)
    with pytest.raises(ValueError, match="audio_history"):
        off.detect(np.zeros((2, 1280), np.int16), threshold=0.5, capture=0.08)
    with pytest.raises(ValueError, match="outside"):
        on.get_audio([0], 0.32)                     # longer than the history
    with pytest.raises(ValueError):
        on.get_audio([2], 0.08)                     # no such stream
    st_on, st_off = on.export_streams([0]), off.export_streams([0])
    assert st_off.audio is None and st_on.audio[0].shape == (1, 2560)
    for dst, st in ((off, st_on), (on, st_off), (other, st_on)):
        with pytest.raises(ValueError, match="audio history"):
            dst.import_streams([1], st)
    on.predict(np.arange(2 * 2000, dtype=np.int16).reshape(2, 2000) % 700)
    on2 = _mk(2, 0.16)
    on2.import_streams([1], on.export_streams([0]))
    assert np.array_equal(on2.get_audio([1], 0.16)[0], on.get_audio([0], 0.16)[0])
    assert on2.get_audio([1], 0.16)[1][0] == 1280
    on.reset_streams([0])
    assert on.get_audio([0], 0.08)[1][0] == 0 and not on.get_audio([0], 0.08)[0].any()
