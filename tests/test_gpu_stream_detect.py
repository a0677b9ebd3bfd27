"""-m gpu: per-stream detection settings (oww_set_stream_detection, csrc/detect.cu).

* A mixed handle - streams with their own thresholds, patience, debounce, opt-outs, the handle's own values, and none -
  over 240 calls with ragged `prepared`, against the float64 restatement (stream_detect_ref.py): d_final, every event
  field and the count, bit for bit; the streams without settings also against a twin handle that never had any.
* Lifecycle: reset keeps the settings, set_detector clears them, set_streams keeps those below the new count, and a
  stream's settings and history moved to another slot and into a second handle continue bit for bit.
* Refused arguments.
* Model.set_stream_detection + detect / detect_ragged (with capture) against predict on one-stream Models under each
  stream's settings."""
import numpy as np
import pytest

from helpers import NAMES, emb_weights, head, streams_model
from stream_detect_ref import StreamRules, events

pytestmark = pytest.mark.gpu
NAN = float("nan")
PREPARED = np.array([-1, 0, 400, 1280, 2560], np.int32)
TABLE = [(0, True, 0.5, 0), (3, False, 0.25, 0), (-1, False, None, 0), (1, False, 0.5, 0), (5, True, 0.3, 0)]


@pytest.fixture(scope="module")
def torch_cuda(built_library):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _engine(B):
    """alexa (1 column) + timer (7 columns): 8 score columns"""
    from openwakeword_b200.engine import StreamEngine
    return StreamEngine([head("alexa_v0.1"), head("timer_v0.1")], B, embedding=emb_weights(), max_chunks=2)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _scores(rng, shape):
    pool = np.array([0.5, np.nextafter(np.float32(0.5), np.float32(0)), 0.25, 0.3, 0.0, 0.9, 0.7], np.float32)
    pick = rng.integers(0, pool.size + 2, shape)
    return np.where(pick < pool.size, pool[np.minimum(pick, pool.size - 1)], rng.uniform(0, 1, shape).astype(np.float32))


def _mixed(B, L, debounce):
    """per stream kind k = b % 6: 0 none; 1 own thresholds; 2 own patience; 3 own debounce; 4 opt-outs; 5 the handle's
    values given explicitly -> (ids with settings, their records and debounce, the resolved thr / pat / deb [B, ...])"""
    from openwakeword_b200 import _native
    thr = np.tile([NAN if t[2] is None else t[2] for t in TABLE], (B, 1)).astype(np.float64)
    pat = np.zeros((B, L), np.int64)
    deb = np.full(B, debounce)
    ids, recs, debs = [], [], []
    for b in range(B):
        k = b % 6
        if k == 0:
            continue
        r = np.zeros(L, _native.STREAM_DETECT_DTYPE)
        r["threshold"], r["patience"] = NAN, -1
        d = NAN
        if k == 1:
            r["threshold"][[0, 1, 2]] = [0.3 + 0.01 * (b % 7), 0.7, 0.25]           # label 2 gains a threshold
            thr[b, [0, 1, 2]] = r["threshold"][[0, 1, 2]]
        elif k == 2:
            r["patience"][[0, 3]] = [1 + b % 3, 30 if b % 2 else 2]
            pat[b, [0, 3]] = r["patience"][[0, 3]]
            d = 0.0
            deb[b] = 0.0
        elif k == 3:
            d = [0.2, 1.1, 2.5][b % 3]
            deb[b] = d
        elif k == 4:
            r["flags"][[0, 4]] = _native.DETECT_NO_THRESHOLD
            thr[b, [0, 4]] = NAN
        else:
            r["threshold"] = thr[b]
            r["patience"] = 0
            d = debounce
        ids.append(b)
        recs.append(r)
        debs.append(d)
    return np.array(ids, np.int32), np.stack(recs), np.array(debs), thr, pat, deb


@pytest.mark.parametrize("B", [36, 2053])
def test_mixed_handle_equals_the_restatement_and_the_twin(torch_cuda, B):
    torch = torch_cuda
    rng = np.random.default_rng(B)
    L, debounce = len(TABLE), 0.4
    eng, twin = _engine(B), _engine(B)
    for e in (eng, twin):
        e.ctx.set_detector(TABLE, debounce)
    ids, recs, debs, thr, pat, deb = _mixed(B, L, debounce)
    eng.set_stream_detection_records(ids, recs, debs)
    got_rec, got_deb = eng.stream_detection(ids)
    assert (got_rec.view(np.uint8) == recs.view(np.uint8)).all() and np.array_equal(got_deb, debs, equal_nan=True)
    rules = StreamRules(B, [t[0] for t in TABLE], [t[1] for t in TABLE])
    none = np.arange(B) % 6 == 0
    d_final = torch.empty((B, L), dtype=torch.float32, device="cuda")
    t_final = torch.empty((B, L), dtype=torch.float32, device="cuda")
    n_total = 0
    for t in range(240):
        sc = torch.from_numpy(_scores(rng, (B, eng.n_cols))).cuda()
        prep = PREPARED[rng.integers(0, PREPARED.size, B)] if t % 7 else np.full(B, 1280, np.int32)
        d_final.fill_(-7.0)
        ev, n = eng.detect(sc, prep, final=d_final)
        tev, _ = twin.detect(sc, prep, final=t_final)
        before = rules.count.copy()
        want_final, fired = rules.step(sc.cpu().numpy(), prep, thr, pat, deb)
        final = d_final.cpu().numpy()
        live = prep >= 0
        assert (final[~live] == -7.0).all()
        assert (_bits(final[live]) == _bits(want_final[live])).all(), t
        want = events(want_final, fired, before)
        assert n == len(want) == ev.size
        assert ev.tolist() == [(s, j, float(v), i) for s, j, v, i in want], t
        # the streams without settings: what a handle that never had any gives them
        assert (_bits(final[none & live]) == _bits(t_final.cpu().numpy()[none & live])).all()
        mine, theirs = ev[none[ev["stream"]]], tev[none[tev["stream"]]]
        assert mine.tobytes() == theirs.tobytes()
        n_total += n
    assert n_total > 1000
    # the handle's own values given explicitly (kind 5) decide exactly as no settings (kind 0): same history bits
    hist, cnt = eng.detector_history(np.arange(B))
    assert rules.count.tolist() == cnt.tolist()
    assert (_bits(hist) == _bits(rules.hist.astype(np.float32))).all()


def test_lifecycle_reset_set_detector_set_streams_and_moves(torch_cuda):
    torch = torch_cuda
    from openwakeword_b200._native import NativeError
    rng = np.random.default_rng(11)
    B, L, debounce = 30, len(TABLE), 0.0
    a, b, ref = _engine(B), _engine(B), _engine(B)
    for e in (a, b, ref):
        e.ctx.set_detector(TABLE, debounce)
    ids, recs, debs, thr, pat, deb = _mixed(B, L, debounce)
    a.set_stream_detection_records(ids, recs, debs)
    ref.set_stream_detection_records(ids, recs, debs)
    a.reset(stream_ids=np.array([1, 2], np.int32))                               # oww_reset keeps them
    a.reset_async(stream_ids=np.array([3], np.int32))
    torch.cuda.synchronize()
    r1, d1 = a.stream_detection()
    assert (r1[ids].view(np.uint8) == recs.view(np.uint8)).all()
    # stream 7 (own thresholds) moves to slot 12 of `a` and to slot 5 of `b`; `ref` keeps it in place
    src, dst_a, dst_b = 7, 12, 5
    n_ev = 0
    for t in range(60):
        if t == 20:
            rec_s, deb_s = a.stream_detection([src])
            h_s = a.detector_history([src])
            a.set_stream_detection_records([dst_a], rec_s, deb_s)
            a.set_detector_history([dst_a], *h_s)
            b.set_stream_detection_records([dst_b], rec_s, deb_s)
            b.set_detector_history([dst_b], *h_s)
        sc = _scores(rng, (B, a.n_cols))
        prep = PREPARED[rng.integers(1, PREPARED.size, B)]
        evr, _ = ref.detect(torch.from_numpy(sc).cuda(), prep)
        mine = evr[evr["stream"] == src]
        n_ev += mine.size
        if t < 20:
            a.detect(torch.from_numpy(sc).cuda(), prep)
            continue
        for e, dst in ((a, dst_a), (b, dst_b)):
            s2, p2 = sc.copy(), prep.copy()
            s2[dst], p2[dst] = sc[src], prep[src]
            ev, _ = e.detect(torch.from_numpy(s2).cuda(), p2)
            moved = ev[ev["stream"] == dst]
            assert moved["label"].tolist() == mine["label"].tolist() and moved["index"].tolist() == mine["index"].tolist()
            assert (_bits(moved["score"]) == _bits(mine["score"])).all(), t
    assert n_ev > 5
    # set_streams: the first streams keep theirs, new streams have none
    a.set_streams(40)
    r2, d2 = a.stream_detection()
    assert (r2[:B].view(np.uint8) == a_rec_after_move(r1, dst_a, src).view(np.uint8)).all()
    assert np.isnan(r2["threshold"][B:]).all() and (r2["patience"][B:] == -1).all() and (r2["flags"][B:] == 0).all()
    assert np.isnan(d2[B:]).all()
    a.set_streams(10)
    assert (a.stream_detection()[0].view(np.uint8) == r2[:10].view(np.uint8)).all()
    # set_detector clears every stream's settings, even under the same labels
    a.ctx.set_detector(TABLE, 0.0)
    r3, d3 = a.stream_detection()
    assert np.isnan(r3["threshold"]).all() and (r3["patience"] == -1).all() and np.isnan(d3).all()
    # refused before anything changes
    good = a.stream_detection([0])[0]
    bad = good.copy()
    bad["patience"][0, 0] = 31
    nothr = good.copy()
    nothr["patience"][0, 0], nothr["flags"][0, 0] = 2, 1
    flags = good.copy()
    flags["flags"][0, 1] = 2
    for args in (([0], bad, NAN), ([0], nothr, NAN), ([0], flags, NAN), ([10], good, NAN), ([0, 0], np.concatenate([good] * 2), NAN),
                 ([0], good, -1.0), ([0], good, float("inf"))):
        with pytest.raises(NativeError):
            a.set_stream_detection_records(*args)
    patience = good.copy()
    patience["patience"][0, 0] = 2
    a.set_stream_detection_records([0], patience, NAN)
    with pytest.raises(NativeError):
        a.set_stream_detection_records([1], patience, 0.5)                       # patience with a debounce
    a.ctx.set_detector(TABLE, 0.5)
    with pytest.raises(NativeError):
        a.set_stream_detection_records([1], patience, NAN)                       # ... the handle's debounce
    assert np.isnan(a.stream_detection()[0]["threshold"]).all() and (a.stream_detection()[0]["patience"] == -1).all()


def a_rec_after_move(r1, dst, src):
    r = r1.copy()
    r[dst] = r1[src]
    return r


def _predict_events(model, res, thr, b):
    out = []
    for lab in model.labels():
        t = thr.get(model.get_parent_model_from_label(lab))
        if t is not None and res[lab] >= np.float32(t):
            out.append((b, lab, float(res[lab])))
    return out


CALL = dict(threshold={"alexa_v0.1": 0.05, "timer_v0.1": 0.12, "hey_jarvis_v0.1": 0.05})
SETTINGS = [
    (None, CALL),
    (dict(threshold={"alexa_v0.1": 0.02, "hey_jarvis_v0.1": None}, debounce_time=0.3),
     dict(threshold={"alexa_v0.1": 0.02, "timer_v0.1": 0.12}, debounce_time=0.3)),
    (dict(threshold=0.04, patience={"alexa_v0.1": 2, "timer_v0.1": 1}),
     dict(threshold={n: 0.04 for n in NAMES}, patience={"alexa_v0.1": 2, "timer_v0.1": 1})),
    (dict(debounce_time=1.0), dict(CALL, debounce_time=1.0)),
    (dict(CALL), CALL),
]


@pytest.mark.parametrize("ragged", [False, True])
def test_model_detect_equals_predict_under_each_streams_settings(torch_cuda, ragged):
    rng = np.random.default_rng(60 + ragged)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    B = len(SETTINGS)
    d = streams_model(B, fi, max_chunks=3, audio_history=2.0)
    singles = [streams_model(1, fi, max_chunks=3) for _ in range(B)]
    for b, (own, _) in enumerate(SETTINGS):
        if own is not None:
            d.set_stream_detection([b], **own)
    n_events = 0
    for t in range(50):
        if ragged:
            xs = [rng.integers(-6000, 6000, [0, 500, 1280, 1024, 2560, 3000][int(rng.integers(0, 6))]).astype(np.int16)
                  for _ in range(B)]
            got = d.detect_ragged(xs, capture=0.5, **CALL)
            for s, lab, sc, audio, end in got:
                assert audio.shape == (8000,) and end > 0
            got = [g[:3] for g in got]
        else:
            x = rng.integers(-6000, 6000, (B, [1280, 2560, 640][t % 3])).astype(np.int16)
            xs = list(x)
            got = d.detect(x, **CALL)
        want = []
        for b, (_, kw) in enumerate(SETTINGS):
            res = singles[b].predict_ragged([xs[b]], **kw) if ragged else singles[b].predict(xs[b], **kw)
            want += _predict_events(singles[b], res, kw["threshold"], b)
        assert got == want, (t, got[:4], want[:4])
        n_events += len(got)
    assert n_events > 20
    # the settings move with the stream, into this Model and into another
    st = d.export_streams([1])
    e = streams_model(B, fi, max_chunks=3, audio_history=2.0)
    e.import_streams([3], st)
    d.import_streams([3], st)
    assert e.stream_detection(3) == d.stream_detection(3) == d.stream_detection(1)
    x = rng.integers(-6000, 6000, (B, 1280)).astype(np.int16)
    x[3] = x[1]
    got_d = [g for g in d.detect(x, **CALL) if g[0] in (1, 3)]
    got_e = [g for g in e.detect(x, **CALL) if g[0] == 3]
    assert [g[1:] for g in got_d if g[0] == 1] == [g[1:] for g in got_d if g[0] == 3] == [g[1:] for g in got_e]
