"""Detections on the bulk clip path without a GPU: the clip restatement (tests/clip_detect_ref.py, the oracle
StreamDetector per clip) against ``Model.predict_clip(clip, **kw)`` after ``reset`` on the host stand-in of the C ABI,
over chunk sizes below, at and above 1280 samples, patience 1..30, debounce, a multi-class label mapped past its
head's outputs and a gated pair; the debounce and patience goldens; the verifier rule of a repeated call; and the
refusals of the bulk entry points, which come before any device work."""
import numpy as np
import pytest

import fake_backend
import openwakeword_b200 as owb
from clip_detect_ref import ClipDetector, chunks_of_call, detect_clips, prepared_of_call
from helpers import NAMES, TIMER_MAP, emb_weights, head, load_case
from openwakeword_b200 import _native
from oracle import detect as odet

f32 = np.float32
# class 7 lies past the timer head's 7 outputs: a label whose column is -1
TIMER_PAST = dict(TIMER_MAP, **{"7": "2_hour_timer"})


@pytest.fixture
def fake_ctx(monkeypatch):
    monkeypatch.setattr(_native, "Context", fake_backend.FakeContext)


def _model(fi, names=NAMES, max_chunks=3):
    specs = [{"name": n, "head": head(n), "class_mapping": TIMER_PAST if n == "timer_v0.1" else None} for n in names]
    return owb.Model(wakeword_models=specs, embedding_model_path=emb_weights(), feature_init=fi, max_chunks=max_chunks)


def _raw_rows(m, clip, padding, chunk):
    """the raw score row of each predict call of predict_clip (the stand-in's step output; stale on calls that step
    nothing, which the rules never read)"""
    m.reset()
    z = np.zeros(16000 * padding, np.int16)
    data = np.concatenate((z, clip, z))
    rows = []
    for i in range(0, data.shape[0] - chunk, chunk):
        m.predict(data[i:i + chunk])
        rows.append(m._scores[0].copy())
    return np.array(rows, np.float32).reshape(len(rows), m._scores.shape[1])


def _predicted(m, clip, padding, chunk, kw):
    m.reset()
    labels = m.labels()
    return np.array([[r[lab] for lab in labels] for r in m.predict_clip(clip, padding, chunk, **kw)],
                    np.float32).reshape(-1, len(labels))


def _restated(m, raw, chunk, kw):
    table = m._clip_table(kw.get("patience", {}), kw.get("threshold", {}), kw.get("debounce_time", 0.0))
    labels = [odet.Label(*row) for row in table]
    return detect_clips(labels, kw.get("debounce_time", 0.0), raw, np.array([0, raw.shape[0]]), chunk)


def test_prepared_follows_the_call_schedule():
    for c in (1, 400, 1024, 1280, 2000, 2560, 3840):
        done = 0
        for j in range(200):
            k = chunks_of_call(j, c)
            assert done + k == (j + 1) * c // 1280
            p = prepared_of_call(j, c)
            assert (p == 1280 * k) if k else (p == (j + 1) * c % 1280 and p != 0)
            done += k


# per chunk size: (clip samples, padding) so that every size sees calls that step and, below 1280, calls that do not
CASES = {1: (2700, 0), 400: (12000, 0), 1024: (16000, 1), 1280: (24000, 1), 2000: (24000, 1), 2560: (20000, 1),
         3840: (30000, 1)}


@pytest.mark.parametrize("chunk", sorted(CASES))
def test_restatement_equals_predict_clip(fake_ctx, chunk):
    rng = np.random.default_rng(chunk)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    m = _model(fi)
    n, padding = CASES[chunk]
    clip = rng.integers(-4000, 4000, n).astype(np.int16)
    raw = _raw_rows(m, clip, padding, chunk)
    labels = m.labels()
    assert -1 in [row[0] for row in m._clip_table({}, {}, 0.0)]
    # thresholds at each model's median score, so that rules fire and are suppressed
    thr = {}
    for mdl in NAMES:
        js = [j for j, lab in enumerate(labels) if m.get_parent_model_from_label(lab) == mdl]
        cols = [row[0] for row in (m._clip_table({}, {}, 0.0)[j] for j in js) if row[0] >= 0]
        thr[mdl] = float(np.median(raw[5:, cols])) if raw.shape[0] > 5 else 0.5
    patiences = range(1, 31) if chunk == 1280 else (1, 2, 5, 30)
    settings = [{}, dict(threshold=thr)] + [dict(threshold=thr, debounce_time=d) for d in (0.25, 1.25, 3.0)] + \
        [dict(threshold=thr, patience={"alexa_v0.1": p, "hey_jarvis_v0.1": max(1, p // 2)}) for p in patiences]
    n_events = 0
    for kw in settings:
        want = _predicted(m, clip, padding, chunk, kw)
        got, events = _restated(m, raw, chunk, kw)
        np.testing.assert_array_equal(got, want, err_msg=str(kw))
        n_events += len(events)
    assert n_events > 0


@pytest.mark.parametrize("n_calls", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("chunk", [400, 1280, 2560])
def test_short_clips(fake_ctx, n_calls, chunk):
    """clips of 0 to 4 calls (padding 0): every call lies in the zeroed first five"""
    rng = np.random.default_rng(100 + n_calls)
    m = _model(rng.normal(0, 1, (41, 96)).astype(np.float32))
    clip = rng.integers(-4000, 4000, n_calls * chunk + 1).astype(np.int16)
    raw = _raw_rows(m, clip, 0, chunk)
    assert raw.shape[0] == n_calls
    kw = dict(threshold={n: 0.0 for n in NAMES}, debounce_time=1.25)
    got, events = _restated(m, raw, chunk, kw)
    np.testing.assert_array_equal(got, _predicted(m, clip, 0, chunk, kw))
    assert not got.any() and len(events) == n_calls * len(m.labels())


@pytest.mark.parametrize("tag", ["jane_debounce", "jane_patience"])
def test_restatement_reproduces_the_goldens(fake_ctx, tag):
    c = load_case(tag)
    name = c["names"][0]
    m = owb.Model(wakeword_models=[{"name": name, "head": head(name)}], embedding_model_path=emb_weights(int(c["emb_seed"])),
                  feature_init=c["feature_init"], max_chunks=8)
    chunk, padding = int(c["chunk"]), int(c["padding"])
    raw = _raw_rows(m, c["pcm"], padding, chunk)
    got, events = _restated(m, raw, chunk, c["kw"])
    np.testing.assert_allclose(got, c["scores"], atol=1e-5)
    thr = f32(c["kw"]["threshold"][name])
    assert [e[3] for e in events] == np.nonzero(c["scores"][:, 0] >= thr)[0].tolist()


def test_verifier_rule_of_a_repeated_call():
    """below 1280 samples a prediction >= the verifier threshold becomes p, whatever the threshold (at 0 even a 0.0
    does); a label without p, and a call that steps, keep the rules of StreamDetector"""
    nan = float("nan")
    labels = [odet.Label(0, True), odet.Label(1, False), odet.Label(-1, False)]
    p = np.array([0.9, 0.8, 0.7], np.float32)
    for vthr, want in ((f32(0.5), [0.9, 0.0, 0.0]), (f32(0.0), [0.9, 0.8, 0.7])):
        d = ClipDetector(labels)
        for _ in range(5):
            d.detect_call(np.array([0.6, 0.6], f32), 1280, p, vthr)
        assert d.detect_call(np.array([0.6, 0.6], f32), 1280, p, vthr)[0].tolist() == [f32(0.6), f32(0.6), 0.0]
        assert d.detect_call(None, 400, p, vthr)[0].tolist() == [f32(v) for v in want]
    d = ClipDetector(labels)
    for _ in range(6):
        d.detect_call(np.array([0.3, 0.6], f32), 1280)
    assert d.detect_call(None, 400, np.array([nan, 0.8, nan], f32), f32(0.5))[0].tolist() == [f32(0.3), 0.0, 0.0]
    assert d.detect_call(None, 400, np.array([0.95, 0.8, nan], f32), f32(0.5))[0].tolist() == [f32(0.3), 0.0, 0.0]


def test_debounce_window_of_a_repeated_call():
    """a call that steps nothing at 400 samples per call prepares 400, 800, 1200 samples: windows of 50, 25, 17 calls
    at 1.25 s, capped at the 30 entries of the history"""
    assert [prepared_of_call(j, 400) for j in range(4)] == [400, 800, 1200, 1280]
    d = ClipDetector([odet.Label(0, True, 0.5)], debounce_time=1.25)
    hist = np.zeros((1, 30), f32)
    hist[0, 29] = 0.8
    d.load(hist, 40)
    assert d.detect_call(None, 1200)[0][0] == 0.0          # the repeat of 0.8 is inside its own window


def test_bulk_refusals(fake_ctx):
    fi = np.zeros((41, 96), np.float32)
    m = _model(fi)
    clips = [np.zeros(16000, np.int16)]
    for call in (m.predict_clips, lambda c, **kw: m.predict_clips_ragged(np.zeros(16000, np.int16), [0, 16000], **kw)):
        with pytest.raises(ValueError, match="threshold"):
            call(clips, patience={"alexa_v0.1": 2})                                    # patience without thresholds
        with pytest.raises(ValueError, match="threshold"):
            call(clips, debounce_time=1.0)
        with pytest.raises(ValueError, match="together"):
            call(clips, patience={"alexa_v0.1": 2}, threshold={"alexa_v0.1": 0.5}, debounce_time=1.0)
        with pytest.raises(ValueError):
            call(clips, patience={"alexa_v0.1": 2}, threshold={"timer_v0.1": 0.5})      # patience of a model without one
    with pytest.raises(ValueError, match="together"):
        m.predict_clips_array(np.zeros((2, 16000), np.int16), patience={"alexa_v0.1": 2}, threshold=0.5,
                              debounce_time=1.0)
    with pytest.raises(ValueError, match="together"):
        m.detect_clips(clips, 0.5, patience={"alexa_v0.1": 2}, debounce_time=1.0)
    with pytest.raises(ValueError, match="patience"):
        m.detect_clips(clips, 0.5, patience={"alexa_v0.1": 31})
