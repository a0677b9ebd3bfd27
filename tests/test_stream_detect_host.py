"""Per-stream detection settings without a GPU: the float64 restatement of the rules (stream_detect_ref.py) against the
per-handle oracle, the record layout against include/owwb200.h, and the host side of ``Model.set_stream_detection`` on
the CPU stand-in of the C ABI, extended here with the settings calls: how names resolve, what is refused, and that each
stream detects what ``predict`` on a one-stream Model returns under that stream's settings."""
import os
import re

import numpy as np
import pytest

import fake_backend
import openwakeword_b200 as owb
from helpers import NAMES, streams_model
from openwakeword_b200 import _native, weights as W
from oracle import detect as odet
from stream_detect_ref import StreamRules, events

f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class SettingsContext(fake_backend.FakeContext):
    """the stand-in plus oww_set_stream_detection / oww_get_stream_detection: a stream with settings of its own runs its
    oracle detector on its resolved labels; oww_set_detector clears every stream's settings"""

    def set_detector(self, labels, debounce_time=0.0):
        super().set_detector(labels, debounce_time)
        self._sd = (np.zeros((self._n, len(labels)), _native.STREAM_DETECT_DTYPE), np.full(self._n, np.nan))
        self._sd[0]["threshold"], self._sd[0]["patience"] = np.nan, -1

    def set_stream_detection(self, stream_ids, records, debounce=None, stream=None):
        ids = self._ids(stream_ids)
        rec, deb = self._sd
        if records is None:
            rec[ids] = (np.nan, -1, 0)
            deb[ids] = np.nan
        else:
            rec[ids] = records
            deb[ids] = np.nan if debounce is None else debounce
        for b in ids:
            labels = []
            for j, (lab, r) in enumerate(zip(self._labels, rec[b])):
                thr = lab.threshold if np.isnan(r["threshold"]) else r["threshold"]
                thr = None if r["flags"] & _native.DETECT_NO_THRESHOLD or thr is None else float(thr)
                labels.append(odet.Label(lab.column, lab.repeats, thr, lab.patience if r["patience"] < 0 else r["patience"]))
            self.det[b].configure(labels, self._debounce if np.isnan(deb[b]) else float(deb[b]))

    def stream_detection(self, stream_ids=None):
        ids = self._ids(stream_ids)
        return self._sd[0][ids].copy(), self._sd[1][ids].copy()


@pytest.fixture
def fake_ctx(monkeypatch):
    monkeypatch.setattr(_native, "Context", SettingsContext)


# ---- the restatement ----
def _oracle_run(rng, B, table, debounce, calls):
    """random scores and `prepared` through one oracle StreamDetector per stream -> per call (final, events)"""
    ods = [odet.StreamDetector([odet.Label(*r) for r in table], debounce) for _ in range(B)]
    out = []
    for t in range(calls):
        scores = rng.choice(np.array([0.0, 0.25, 0.5, np.nextafter(f32(0.5), f32(0)), 0.7, 0.9], f32), (B, 4))
        prep = rng.choice(np.array([-1, 0, 400, 1280, 2560], np.int64), B)
        fin = np.full((B, len(table)), np.nan)
        ev = []
        for b in range(B):
            r = ods[b].detect(scores[b], int(prep[b]))
            if r is not None:
                fin[b] = r[0]
                ev += [(b, j, s, i) for j, s, i in r[1]]
        out.append((scores, prep, fin, ev))
    return out


@pytest.mark.parametrize("mode", ["none", "patience", "debounce"])
def test_restatement_at_the_handle_values_equals_the_oracle(mode):
    rng = np.random.default_rng({"none": 1, "patience": 2, "debounce": 3}[mode])
    B = 9
    table = [(0, True, 0.5, 2 if mode == "patience" else 0), (1, False, 0.25, 0), (-1, False, None, 0),
             (3, True, 0.7, 3 if mode == "patience" else 0)]
    debounce = 0.5 if mode == "debounce" else 0.0
    rules = StreamRules(B, [r[0] for r in table], [r[1] for r in table])
    thr = np.tile([np.nan if r[2] is None else r[2] for r in table], (B, 1))
    pat = np.tile([r[3] for r in table], (B, 1))
    n_ev = 0
    for scores, prep, fin, ev in _oracle_run(rng, B, table, debounce, 120):
        before = rules.count.copy()
        got, fired = rules.step(scores, prep, thr, pat, debounce)
        np.testing.assert_array_equal(got, fin)
        assert events(got, fired, before) == ev
        n_ev += len(ev)
    assert n_ev > 20


def test_restatement_per_stream_equals_one_oracle_per_stream():
    """every stream its own thresholds, patience and debounce (as the device resolves a stream's records)"""
    rng = np.random.default_rng(7)
    B, L = 12, 3
    columns, repeats = [0, 2, -1], [True, False, True]
    thr = rng.choice(np.array([0.25, 0.5, 0.7, np.nan]), (B, L))
    pat = np.where(rng.random((B, L)) < 0.4, rng.integers(1, 5, (B, L)), 0) * ~np.isnan(thr)
    deb = np.where(pat.any(1), 0.0, rng.choice([0.0, 0.2, 0.5, 1.3], B))
    ods = [odet.StreamDetector([odet.Label(columns[j], repeats[j], None if np.isnan(thr[b, j]) else thr[b, j], pat[b, j])
                                for j in range(L)], deb[b]) for b in range(B)]
    rules = StreamRules(B, columns, repeats)
    n_ev = 0
    for t in range(150):
        scores = rng.choice(np.array([0.0, 0.25, 0.5, 0.7, 0.9], f32), (B, 3))
        prep = rng.choice(np.array([-1, 0, 300, 1280, 2560]), B)
        before = rules.count.copy()
        got, fired = rules.step(scores, prep, thr, pat, deb)
        want = []
        for b in range(B):
            r = ods[b].detect(scores[b], int(prep[b]))
            if r is None:
                assert np.isnan(got[b]).all()
                continue
            assert got[b].tolist() == r[0].tolist(), (t, b)
            want += [(b, j, s, i) for j, s, i in r[1]]
        assert events(got, fired, before) == want
        n_ev += len(want)
    assert n_ev > 20


# ---- the record against the header ----
def test_record_layout_matches_the_header():
    with open(os.path.join(ROOT, "include", "owwb200.h")) as fh:
        h = fh.read()
    body = re.search(r"typedef struct oww_stream_detect \{([^}]*)\} oww_stream_detect;", h).group(1)
    fields = [tuple(f.split()) for f in body.split(";") if f.strip()]
    assert fields == [("float", "threshold"), ("int32_t", "patience"), ("int32_t", "flags")]
    assert "sizeof(oww_stream_detect) == 12" in h
    assert int(re.search(r"#define OWW_DETECT_NO_THRESHOLD (\d+)", h).group(1)) == _native.DETECT_NO_THRESHOLD
    dt = _native.STREAM_DETECT_DTYPE
    assert dt.itemsize == 12 and [dt.fields[k][1] for k in ("threshold", "patience", "flags")] == [0, 4, 8]
    assert [dt.fields[k][0] for k in ("threshold", "patience", "flags")] == [np.dtype("<f4"), np.dtype("<i4"), np.dtype("<i4")]
    assert "oww_set_stream_detection" in _native.EXPORTED_SYMBOLS and "oww_get_stream_detection" in _native.EXPORTED_SYMBOLS


# ---- Model.set_stream_detection on the stand-in ----
def _fi():
    return np.random.default_rng(0).normal(0, 1, (41, 96)).astype(np.float32)


def test_names_resolve_as_the_call_arguments_do(fake_ctx):
    """a multi-class model's labels take its value, stream models their name, the rest the call's; NaN-free records"""
    m = streams_model(3, _fi(), stream_models={"user": {None: W.synthetic_head(seed=70)}})
    labels = m.labels()
    m.set_stream_detection([1], threshold={"timer_v0.1": 0.3, "user": None}, patience={"alexa_v0.1": 2})
    m.set_stream_detection([2], threshold=0.6, debounce_time=1.5)
    rec, deb = m._stream_detection_table({"alexa_v0.1": 0.5, "user": 0.4}, {}, 0.0)
    assert rec.shape == (3, len(labels))
    assert np.isnan(rec["threshold"][0]).all() and (rec["patience"][0] == -1).all() and np.isnan(deb[0])
    timer = [j for j, lab in enumerate(labels) if m.get_parent_model_from_label(lab) == "timer_v0.1"]
    assert len(timer) == 6
    for j, lab in enumerate(labels):
        parent = m.get_parent_model_from_label(lab)
        t, flags, p = rec["threshold"][1, j], rec["flags"][1, j], rec["patience"][1, j]
        want = {"timer_v0.1": 0.3, "alexa_v0.1": 0.5}.get(parent)
        if want is None:                                   # hey_jarvis: none in the call; user: opted out
            assert flags == _native.DETECT_NO_THRESHOLD and np.isnan(t), lab
        else:
            assert flags == 0 and t == f32(want), lab
        assert p == (2 if parent == "alexa_v0.1" else 0)
        assert rec["threshold"][2, j] == f32(0.6) and rec["flags"][2, j] == 0 and rec["patience"][2, j] == 0
    assert deb[1] == 0.0 and deb[2] == 1.5
    assert m.stream_detection(1) == dict(threshold={"timer_v0.1": 0.3, "user": None}, patience={"alexa_v0.1": 2},
                                         debounce_time=None)
    assert m.stream_detection(0) is None
    m.clear_stream_detection([1, 2])
    assert m._stream_detection_table(0.5, {}, 0.0) is None


def test_refusals(fake_ctx):
    m = streams_model(3, _fi())
    x = np.zeros((3, 1280), np.int16)
    with pytest.raises(ValueError, match="0..30"):
        m.set_stream_detection([0], threshold=0.5, patience={"alexa_v0.1": 31})
    with pytest.raises(ValueError, match="cannot be used together"):
        m.set_stream_detection([0], threshold=0.5, patience={"alexa_v0.1": 2}, debounce_time=0.5)
    with pytest.raises(ValueError, match="no model named"):
        m.set_stream_detection([0], threshold={"alexa": 0.5})
    with pytest.raises(ValueError, match="no model named"):
        m.set_stream_detection([0], patience={"1_minute_timer": 2})           # a label, not its model
    with pytest.raises(ValueError, match="stream ids"):
        m.set_stream_detection([3], threshold=0.5)
    with pytest.raises(ValueError, match="debounce_time"):
        m.set_stream_detection([0], debounce_time=-1.0)
    assert m.stream_detection(0) is None
    # refused at the call, by the checks of predict, before anything runs: patience where the stream has no threshold,
    # and a stream's patience against the call's debounce
    m.detect(x, 0.5)
    m.set_stream_detection([1], threshold={"alexa_v0.1": None})
    with pytest.raises(ValueError, match="threshold values must be provided"):
        m.detect(x, 0.5, patience={"alexa_v0.1": 2})
    m.set_stream_detection([1], patience={"alexa_v0.1": 2})
    with pytest.raises(ValueError, match="cannot be used together"):
        m.detect(x, 0.5, debounce_time=0.5)
    assert m.preprocessor.ctx.detector_history([1])[1][0] == 1
    m.detect(x, 0.5)                                                         # a valid call goes through
    assert m.preprocessor.ctx.detector_history([1])[1][0] == 2


def _predict_events(model, res, thr, b):
    out = []
    for lab in model.labels():
        t = thr if not isinstance(thr, dict) else thr.get(model.get_parent_model_from_label(lab))
        if t is not None and res[lab] >= f32(t):
            out.append((b, lab, float(res[lab])))
    return out


SETTINGS = [                     # per stream: (set_stream_detection kwargs or None, the predict kwargs they amount to)
    (None, None),
    (dict(threshold={"alexa_v0.1": 0.1, "hey_jarvis_v0.1": None}, debounce_time=0.3),
     dict(threshold={"alexa_v0.1": 0.1, "timer_v0.1": 0.12}, debounce_time=0.3)),
    (dict(threshold=0.15, patience={"alexa_v0.1": 2, "timer_v0.1": 1}),
     dict(threshold={n: 0.15 for n in NAMES}, patience={"alexa_v0.1": 2, "timer_v0.1": 1})),
    (dict(threshold={"alexa_v0.1": 0.2, "timer_v0.1": 0.12, "hey_jarvis_v0.1": 0.2}),      # the call's own values
     dict(threshold={"alexa_v0.1": 0.2, "timer_v0.1": 0.12, "hey_jarvis_v0.1": 0.2})),
]
CALL = dict(threshold={"alexa_v0.1": 0.2, "timer_v0.1": 0.12, "hey_jarvis_v0.1": 0.2})


@pytest.mark.parametrize("ragged", [False, True])
def test_each_stream_detects_what_predict_gives_under_its_settings(fake_ctx, ragged):
    rng = np.random.default_rng(40 + ragged)
    fi = _fi()
    B = len(SETTINGS)
    d = streams_model(B, fi)
    singles = [streams_model(1, fi) for _ in range(B)]
    for b, (own, _) in enumerate(SETTINGS):
        if own is not None:
            d.set_stream_detection([b], **own)
    n_events = 0
    for t in range(24):
        if ragged:
            xs = [rng.integers(-4000, 4000, [0, 700, 1280, 2560][int(rng.integers(0, 4))]).astype(np.int16) for _ in range(B)]
            got = d.detect_ragged(xs, **CALL)
        else:
            x = rng.integers(-4000, 4000, (B, [1280, 2560, 640][t % 3])).astype(np.int16)
            xs = list(x)
            got = d.detect(x, **CALL)
        want = []
        for b, (_, kw) in enumerate(SETTINGS):
            kw = kw or CALL
            res = singles[b].predict_ragged([xs[b]], **kw) if ragged else singles[b].predict(xs[b], **kw)
            want += _predict_events(singles[b], res, kw["threshold"], b)
        assert got == want, (t, got, want)
        n_events += len(got)
    assert n_events > 10
    # the settings and the history follow a stream to another slot
    st = d.export_streams([1, 2])
    assert st.detection[0] == (SETTINGS[1][0]["threshold"], {}, 0.3)
    d.import_streams([2, 1], st)
    assert d.stream_detection(2)["debounce_time"] == 0.3 and d.stream_detection(1)["patience"] == {"alexa_v0.1": 2,
                                                                                                 "timer_v0.1": 1}
    d.reset_streams([0])                                                   # a reset keeps them
    assert d.stream_detection(2) is not None
