"""Detections without a GPU: oracle/detect.py against hand-written values for each branch of the rules, and the host
side of ``Model.detect`` / ``detect_ragged`` on a stand-in of the C ABI (the detector calls restated with the oracle):
the goldens that pin debounce and patience through the whole pipeline, equality with ``predict`` / ``predict_ragged``
on a twin Model, the hand-over of the history between the two, and the refusals."""
import numpy as np
import pytest

import fake_backend
import openwakeword_b200 as owb
from helpers import NAMES, emb_weights, head, load_case, streams_model as _model
from openwakeword_b200 import _native
from oracle import detect as odet

f32 = np.float32


@pytest.fixture
def fake_ctx(monkeypatch):
    monkeypatch.setattr(_native, "Context", fake_backend.FakeContext)


# ---- the oracle, branch by branch ----
def _run(det, rows, prepared=1280):
    return [det.detect(np.array(r, f32), prepared) for r in rows]


def test_oracle_first_five_are_zero_and_counted():
    d = odet.StreamDetector([odet.Label(0, True, 0.5)])
    out = _run(d, [[0.9]] * 7)
    assert [float(f[0]) for f, _ in out] == [0, 0, 0, 0, 0, float(f32(0.9)), float(f32(0.9))]
    assert [e for _, e in out][:5] == [[]] * 5
    assert out[5][1] == [(0, f32(0.9), 5)] and out[6][1] == [(0, f32(0.9), 6)]
    assert d.count == 7


def test_oracle_repeat_rules():
    d = odet.StreamDetector([odet.Label(0, True), odet.Label(1, False)])
    assert d.detect(None, 400)[0].tolist() == [0.0, 0.0]            # empty history: 0.0, the scores are not read
    _run(d, [[0.7, 0.6]] * 5)
    assert d.detect(np.array([0.7, 0.6], f32), 1280)[0].tolist() == [f32(0.7), f32(0.6)]
    assert d.detect(None, 1279)[0].tolist() == [f32(0.7), 0.0]      # the single-output label repeats, the class reads 0.0
    assert d.detect(None, 0)[0].tolist() == [f32(0.7), 0.0]
    assert d.detect(None, -1) is None and d.count == 9             # skipped: nothing appended


def test_oracle_patience():
    d = odet.StreamDetector([odet.Label(0, True, 0.5, 3)])
    _run(d, [[0.0]] * 5)
    got = [float(f[0]) for f, _ in _run(d, [[0.9], [0.9], [0.9], [0.9], [0.4], [0.9]])]
    # the history holds final values: a zeroed prediction does not count towards the next one's patience
    assert got == [0, 0, 0, 0, 0, 0]
    d = odet.StreamDetector([odet.Label(0, True, 0.5, 2)])
    d.load(np.array([[0.0] * 28 + [0.6, 0.7]], f32), 30)
    f, e = d.detect(np.array([0.9], f32), 1280)
    assert f[0] == f32(0.9) and e == [(0, f32(0.9), 30)]            # satisfied: two of the last two are >= 0.5
    d.load(np.array([[0.0] * 28 + [0.7, 0.4]], f32), 30)
    assert d.detect(np.array([0.9], f32), 1280)[0][0] == 0.0        # not satisfied
    d.load(np.array([[0.0] * 28 + [0.7, 0.7]], f32), 30)
    assert d.detect(np.array([0.3], f32), 1280)[0][0] == f32(0.3)   # satisfied; below the threshold it is no event
    d = odet.StreamDetector([odet.Label(0, True, 0.5, 8)])
    d.load(np.array([[0.0] * 24 + [0.9] * 6], f32), 6)              # fewer entries than the patience: never satisfied
    assert d.detect(np.array([0.9], f32), 1280)[0][0] == 0.0


@pytest.mark.parametrize("prepared,window", [(1280, 7), (2560, 4)])
def test_oracle_debounce_window(prepared, window):
    """n_frames = ceil(0.5 / (prepared / 16000)): a hit at the edge of the window suppresses, one entry older does not"""
    for age, suppressed in ((window, True), (window + 1, False)):
        d = odet.StreamDetector([odet.Label(0, True, 0.5)], debounce_time=0.5)
        hist = np.zeros((1, 30), f32)
        hist[0, 30 - age] = 0.8
        d.load(hist, 40)
        assert d.detect(np.array([0.9], f32), prepared)[0][0] == (0.0 if suppressed else f32(0.9)), age
    d.load(np.zeros((1, 30), f32), 3)                   # fewer entries than the window: capped by the entries present
    _run(d, [[0.9]] * 2)
    assert d.detect(np.array([0.9], f32), prepared)[0][0] == f32(0.9)
    assert d.detect(np.array([0.4], f32), prepared)[0][0] == f32(0.4)          # below the threshold: untouched


@pytest.mark.parametrize("prepared", [400, 0])
def test_oracle_debounce_on_a_repeated_prediction(prepared):
    """below 1280 samples the prediction is the newest entry, which lies inside its own window (20 entries at 400
    samples, the whole history at 0): at or above the threshold it is suppressed, below it is repeated"""
    for prev, want in ((0.6, 0.0), (0.45, f32(0.45))):
        d = odet.StreamDetector([odet.Label(0, True, 0.5)], debounce_time=0.5)
        hist = np.zeros((1, 30), f32)
        hist[0, 29] = prev
        d.load(hist, 40)
        assert d.detect(None, prepared)[0][0] == want


def test_oracle_nan_threshold_column_minus_one_and_errors():
    d = odet.StreamDetector([odet.Label(0, True, float("nan")), odet.Label(-1, False, 0.0)], debounce_time=1.0)
    d.load(np.full((2, 30), 0.9, f32), 30)
    f, e = d.detect(np.array([0.95], f32), 1280)
    assert f.tolist() == [f32(0.95), 0.0]                           # no threshold: no debounce, no event
    assert e == [(1, f32(0.0), 30)]                                 # 0.0 >= 0.0 fires; its value is not "nonzero"
    with pytest.raises(ValueError):
        odet.Label(0, True, None, 2)
    with pytest.raises(ValueError):
        odet.Label(0, True, 0.5, 31)
    with pytest.raises(ValueError):
        odet.StreamDetector([odet.Label(0, True, 0.5, 2)], debounce_time=0.5)


def test_oracle_export_load_round_trip():
    rng = np.random.default_rng(0)
    d = odet.StreamDetector([odet.Label(0, True, 0.5), odet.Label(1, False, 0.5)], debounce_time=0.3)
    for n in (3, 47):
        d.reset()
        _run(d, rng.uniform(0, 1, (n, 2)))
        h, c = d.export()
        assert c == n and (h[:, :30 - min(n, 30)] == 0).all()
        e = odet.StreamDetector(d.labels, 0.3)
        e.load(h, c)
        row = rng.uniform(0, 1, 2)
        a, b = d.detect(row.astype(f32), 1280), e.detect(row.astype(f32), 1280)
        assert a[0].tolist() == b[0].tolist() and a[1] == b[1]


# ---- Model.detect on the stand-in ----
@pytest.mark.parametrize("tag", ["jane_debounce", "jane_patience"])
def test_detect_fires_where_the_golden_scores_reach_the_threshold(fake_ctx, tag):
    c = load_case(tag)
    name = c["names"][0]
    m = owb.Model(wakeword_models=[{"name": name, "head": head(name)}], embedding_model_path=emb_weights(int(c["emb_seed"])),
                  feature_init=c["feature_init"], max_chunks=8)
    thr = c["kw"]["threshold"][name]
    z = np.zeros(16000 * int(c["padding"]), np.int16)
    data = np.concatenate((z, c["pcm"], z))
    chunk = int(c["chunk"])
    fired = [bool(m.detect(data[i:i + chunk], **c["kw"])) for i in range(0, data.shape[0] - chunk, chunk)]
    want = (c["scores"][:, 0] >= f32(thr)).tolist()
    assert fired == want and any(want) == (tag == "jane_debounce")      # the patience case never reaches its threshold
    hist, cnt = m.preprocessor.ctx.detector_history([0])
    n = len(want)
    assert cnt[0] == n
    np.testing.assert_allclose(hist[0, 0], c["scores"][n - 30:, 0], atol=1e-5)
    np.testing.assert_allclose(list(m.prediction_buffer[name]), c["scores"][n - 30:, 0], atol=1e-5)


def _thresholded(res, labels, thr, model):
    """predict's {label: float32 [B]} -> detect's event list"""
    out = []
    B = len(next(iter(res.values())))
    for b in range(B):
        for lab in labels:
            t = thr if not isinstance(thr, dict) else thr.get(model.get_parent_model_from_label(lab))
            if t is not None and res[lab][b] >= f32(t):
                out.append((b, lab, float(res[lab][b])))
    return out


@pytest.mark.parametrize("post", ["none", "patience", "debounce"])
def test_detect_equals_thresholded_predict_on_a_twin(fake_ctx, post):
    rng = np.random.default_rng({"none": 4, "patience": 5, "debounce": 6}[post])
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    B = 4
    thr = {"alexa_v0.1": 0.3, "timer_v0.1": 0.12} if post != "none" else 0.2      # hey_jarvis: no threshold in the dict
    kw = {"none": {}, "patience": dict(patience={"alexa_v0.1": 2}), "debounce": dict(debounce_time=0.4)}[post]
    thr_dict = thr if isinstance(thr, dict) else {n: thr for n in NAMES}
    p, d = _model(B, fi), _model(B, fi)
    labels = p.labels()
    n_events = 0
    for t in range(36):
        if t == 14:
            p.reset_streams([1, 3])
            d.reset_streams([1, 3])
        if t == 22:                     # a predict-only Model's streams continue on the detect Model, and the reverse
            sp, sd = p.export_streams([0, 2]), d.export_streams([0, 2])
            for lab in labels:
                np.testing.assert_array_equal(sp.history[lab], sd.history[lab])
                np.testing.assert_array_equal(sp.counts[lab], sd.counts[lab])
            p.import_streams([2, 0], sd)
            d.import_streams([2, 0], sp)
        lock = t % 3 == 0
        if lock:
            n = [1280, 2560, 1024, 0][(t // 3) % 4]
            xs = [rng.integers(-3000, 3000, n).astype(np.int16) for _ in range(B)]
            if t >= 22:
                xs[0], xs[2] = xs[2], xs[0]
            want = _thresholded(p.predict(np.stack(xs), threshold=thr_dict, **kw), labels, thr, p)
            got = d.detect(np.stack(xs), thr, **kw)
        else:
            xs = [rng.integers(-3000, 3000, [0, 700, 1280, 1024, 2560, 3000][int(rng.integers(0, 6))]).astype(np.int16)
                  for _ in range(B)]
            want = _thresholded(p.predict_ragged(xs, threshold=thr_dict, **kw), labels, thr, p)
            got = d.detect_ragged(xs, thr, **kw)
        assert got == want, (t, got, want)
        n_events += len(got)
        if t % 5 == 0:
            for lab in labels:
                assert list(d.prediction_buffer[lab]) == list(p.prediction_buffer[lab])
    assert n_events > 10


def test_predict_and_detect_mix_on_one_model(fake_ctx):
    """the history moves to the device at the first detect and back at the next predict"""
    rng = np.random.default_rng(12)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    thr = {n: 0.2 for n in NAMES}
    kw = dict(debounce_time=0.3, threshold=thr)
    p, m = _model(2, fi), _model(2, fi)
    labels = p.labels()
    for t in range(30):
        x = rng.integers(-3000, 3000, (2, [1280, 640, 2560][t % 3])).astype(np.int16)
        want = p.predict(x, **kw)
        if (t // 4) % 2:
            assert m.detect(x, thr, debounce_time=0.3) == _thresholded(want, labels, thr, p)
        else:
            got = m.predict(x, **kw)
            assert all((got[lab] == want[lab]).all() for lab in labels)
    m.reset()
    assert not m.prediction_buffer and m.detect(x, thr) == []


def test_detect_refusals(fake_ctx):
    fi = np.zeros((41, 96), np.float32)
    m = _model(2, fi)
    x = np.zeros((2, 1280), np.int16)
    with pytest.raises(ValueError):
        m.detect([0] * 1280, 0.5)                                               # not an array
    with pytest.raises(ValueError):
        m.detect(x, {"alexa_v0.1": 0.5}, patience={"timer_v0.1": 2})            # patience without a threshold
    with pytest.raises(ValueError):
        m.detect(x, 0.5, patience={"alexa_v0.1": 2}, debounce_time=1.0)         # patience with debounce
    with pytest.raises(ValueError):
        m.detect(x, 0.5, patience={"alexa_v0.1": 31})
    with pytest.raises(ValueError):
        m.detect_ragged([x[0]], 0.5)                                            # one array per stream
    m._host_verifiers["alexa_v0.1"] = object()
    with pytest.raises(ValueError, match="host"):
        m.detect(x, 0.5)
    m._host_verifiers.clear()
    m.speex_ns = object()
    with pytest.raises(ValueError, match="Speex"):
        m.detect(x, 0.5)
    m.speex_ns = None
    m._vbanks["alexa_v0.1"] = object()                                          # device verifier banks loaded
    with pytest.raises(ValueError, match="max_chunks"):
        m.detect(np.zeros((2, 3 * 1280), np.int16), 0.5)
    m._vbanks.clear()
    assert m.detect(np.zeros((2, 3 * 1280), np.int16), 0.5) == []               # without banks a long call is split
    assert m.preprocessor.ctx.detector_history([0])[1][0] == 1                  # the refused calls appended nothing
