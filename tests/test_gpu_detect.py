"""-m gpu: detections on the device (oww_set_detector / oww_detect, csrc/detect.cu).

* The kernel against oracle/detect.py on hand-made score matrices - values on, just below and just above the thresholds,
  per-stream `prepared` from {-1, 0, 400, 1280, 2560, 5120}, with patience, with debounce and with neither - bit for bit:
  d_final, every event field, the count and the exported histories.
* The event list: ascending (stream, label) over many CTAs, truncation at max_events with the true count, NULL outputs.
* Skipped streams, resets of a subset (oww_reset, oww_reset_async), oww_set_streams, reconfiguration, refused arguments.
* End to end: Model.detect_ragged against a twin Model's thresholded predict_ragged, the engine loop with held streams,
  moving a stream's history to another handle, and a handle without a detector launching what it always launched."""
import os

import numpy as np
import pytest

from helpers import GOLDEN, TIMER_MAP, emb_weights, head
from oracle import detect as odet

pytestmark = pytest.mark.gpu
PREPARED = np.array([-1, 0, 400, 1280, 2560, 5120], np.int32)
NAN = float("nan")


@pytest.fixture(scope="module")
def torch_cuda(built_library):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


_engines = {}


def _engine(B, fresh=False):
    """alexa (1 column) + timer (7 columns): 8 score columns"""
    from openwakeword_b200.engine import StreamEngine
    if fresh or B not in _engines:
        eng = StreamEngine([head("alexa_v0.1"), head("timer_v0.1")], B, embedding=emb_weights(), max_chunks=2)
        if fresh:
            return eng
        _engines[B] = eng
    return _engines[B]


def _table(rng, L, n_cols, mode):
    rows = []
    for j in range(L):
        thr = [0.5, 0.25, None][int(rng.integers(0, 3))] if j else 0.5
        pat = 0
        if mode == "patience" and thr is not None:
            pat = [0, 1, 2, 3, 30][int(rng.integers(0, 5))] if j else 2
        rows.append((int(rng.integers(-1, n_cols)) if j else 0, bool(rng.integers(0, 2)) if j else True, thr, pat))
    return rows


def _edge_scores(rng, shape):
    """values on, one ulp below and one ulp above the thresholds, zeros, and uniform noise"""
    f = np.float32
    pool = np.array([0.5, np.nextafter(f(0.5), f(0)), np.nextafter(f(0.5), f(1)), 0.25, np.nextafter(f(0.25), f(0)),
                     np.nextafter(f(0.25), f(1)), 0.0, 0.9], np.float32)
    pick = rng.integers(0, pool.size + 3, shape)
    return np.where(pick < pool.size, pool[np.minimum(pick, pool.size - 1)], rng.uniform(0, 1, shape).astype(np.float32))


def _expected_events(final, table, counts):
    thr = np.array([NAN if t[2] is None else t[2] for t in table], np.float32)
    b, j = np.nonzero(final >= thr[None, :])             # row-major: ascending (stream, label); NaN never compares
    return b, j, final[b, j], counts[b]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("mode", ["none", "patience", "debounce"])
@pytest.mark.parametrize("L", [1, 11, 40])
@pytest.mark.parametrize("B", [1, 7, 257, 8192])
def test_kernel_equals_the_oracle(torch_cuda, B, L, mode):
    torch = torch_cuda
    rng = np.random.default_rng(1000 * B + 10 * L + len(mode))
    eng = _engine(B)
    ctx, n_cols = eng.ctx, eng.n_cols
    table = _table(rng, L, n_cols, mode)
    debounce = 0.5 if mode == "debounce" else 0.0
    eng.reset()
    ctx.set_detector([], 0.0)                            # a fresh detector whatever the test before configured
    ctx.set_detector(table, debounce)
    calls = 200
    # the oracle runs every stream of a small handle, and a sample (first, last, CTA edges, random) of a large one
    S = 256 // L
    watch = np.arange(B) if B <= 64 else np.unique(np.concatenate(
        [np.minimum([0, 1, B - 1, B - 2, S - 1, S, 2 * S - 1, 2 * S], B - 1), rng.integers(0, B, 24)]))
    oracles = {int(b): odet.StreamDetector([odet.Label(*r) for r in table], debounce) for b in watch}
    scores = torch.from_numpy(_edge_scores(rng, (calls, B, n_cols))).cuda()
    h_scores = scores.cpu().numpy()
    d_final = torch.empty((B, L), dtype=torch.float32, device="cuda")
    counts = np.zeros(B, np.int64)
    n_total = 0
    for t in range(calls):
        prep = PREPARED[rng.integers(0, PREPARED.size, B)] if t % 9 else np.full(B, 1280, np.int32)
        d_final.fill_(-7.0)
        ev, n = ctx.detect_events(scores[t], prep if t % 9 else 1280, d_final)
        final = d_final.cpu().numpy()
        live = prep >= 0
        assert (final[~live] == -7.0).all()              # rows of skipped streams are not written
        for b in watch:
            r = oracles[int(b)].detect(h_scores[t, b], int(prep[b]))
            if r is not None:
                assert (_bits(final[b]) == _bits(r[0])).all(), (t, b, final[b], r[0])
        eb, ej, es, ei = _expected_events(np.where(live[:, None], final, np.float32(NAN)), table, counts)
        assert n == eb.size == ev.size
        assert (ev["stream"] == eb).all() and (ev["label"] == ej).all() and (ev["index"] == ei).all()
        assert (_bits(ev["score"]) == _bits(es)).all()
        counts += live
        n_total += n
    assert n_total > 0 or mode == "patience"      # a label under patience never fires: its history holds final values
    hist, cnt = ctx.detector_history(np.arange(B))
    assert (cnt == counts).all()
    for b in watch:
        h, c = oracles[int(b)].export()
        assert c == counts[b] and (_bits(hist[b]) == _bits(h)).all()


def test_event_order_truncation_and_null_outputs(torch_cuda):
    torch = torch_cuda
    B, L = 8192, 11
    eng = _engine(B)
    ctx = eng.ctx
    eng.reset()
    ctx.set_detector([], 0.0)
    ctx.set_detector([(j % eng.n_cols, True, 0.0, 0) for j in range(L)], 0.0)
    scores = torch.ones((B, eng.n_cols), dtype=torch.float32, device="cuda")
    ev, n = ctx.detect_events(scores, 1280)              # 0.0 >= 0.0: every pair fires, from the first prediction on
    assert n == B * L == 90112 and ev.size == n
    assert (ev["stream"] == np.repeat(np.arange(B), L)).all() and (ev["label"] == np.tile(np.arange(L), B)).all()
    assert (ev["index"] == 0).all() and (ev["score"] == 0.0).all()
    # fewer slots than events: the true count, the prefix, and nothing behind it
    stream = torch.cuda.current_stream().cuda_stream
    buf = torch.full((1000 + 64, 4), -559038737, dtype=torch.int32, device="cuda")
    n_ev = torch.zeros(1, dtype=torch.int32, device="cuda")
    ctx.detect(scores, 1280, None, buf, 1000, n_ev, stream)
    got = buf.cpu().numpy()
    assert int(n_ev.item()) == B * L
    assert (got[:1000, 0] == np.repeat(np.arange(B), L)[:1000]).all() and (got[:1000, 3] == 1).all()
    assert (got[1000:] == -559038737).all()
    # no event list at all; no dense output; the count alone
    final = torch.empty((B, L), dtype=torch.float32, device="cuda")
    ctx.detect(scores, 1280, final, None, 0, None, stream)
    ctx.detect(scores, 1280, None, None, 0, n_ev, stream)
    assert int(n_ev.item()) == B * L and (final.cpu().numpy() == 0.0).all()
    # one event, in the last stream only
    ctx.set_detector([(j % eng.n_cols, True, 0.5, 0) for j in range(L)], 0.0)      # same labels: the counts stay at 4
    for _ in range(2):
        assert ctx.detect_events(scores * 0, 1280)[1] == 0
    one = torch.zeros((B, eng.n_cols), dtype=torch.float32, device="cuda")
    one[B - 1, 3] = 0.75
    ev, n = ctx.detect_events(one, 1280)
    assert n == 1 and ev.tolist() == [(B - 1, 3, 0.75, 6)]


def test_skips_resets_and_reconfiguration(torch_cuda):
    torch = torch_cuda
    B, L = 40, 3
    eng = _engine(B, fresh=True)
    ctx = eng.ctx
    table = [(0, True, 0.5, 0), (3, False, 0.25, 0), (-1, False, None, 0)]
    ctx.set_detector(table, 0.0)
    rng = np.random.default_rng(3)
    ids = np.arange(B)
    for t in range(8):
        ctx.detect_events(torch.from_numpy(_edge_scores(rng, (B, eng.n_cols))).cuda(), 1280)
    before, cnt = ctx.detector_history(ids)
    assert (cnt == 8).all() and before[:, :2, -3:].any()
    prep = np.where(ids % 2 == 0, -1, 1280).astype(np.int32)               # even streams are skipped
    ctx.detect_events(torch.from_numpy(_edge_scores(rng, (B, eng.n_cols))).cuda(), prep)
    after, cnt = ctx.detector_history(ids)
    assert (_bits(after[::2]) == _bits(before[::2])).all() and (cnt[::2] == 8).all() and (cnt[1::2] == 9).all()
    eng.reset(stream_ids=np.array([1, 5], np.int32))                       # oww_reset
    eng.reset_async(stream_ids=np.array([7], np.int32))                    # oww_reset_async
    torch.cuda.synchronize()
    h2, c2 = ctx.detector_history(ids)
    cleared = np.isin(ids, [1, 5, 7])
    assert (c2[cleared] == 0).all() and not h2[cleared].any()
    assert (_bits(h2[~cleared]) == _bits(after[~cleared])).all() and (c2[~cleared] == cnt[~cleared]).all()
    # new thresholds, patience or debounce under the same labels keep the histories; other labels clear them
    ctx.set_detector([(0, True, 0.1, 2), (3, False, None, 0), (-1, False, 0.3, 0)], 0.0)
    h3, c3 = ctx.detector_history(ids)
    assert (_bits(h3) == _bits(h2)).all() and (c3 == c2).all()
    ctx.set_detector([(0, True, 0.1, 0), (4, False, None, 0), (-1, False, 0.3, 0)], 0.0)
    h4, c4 = ctx.detector_history(ids)
    assert not h4.any() and not c4.any()
    ctx.detect_events(torch.ones((B, eng.n_cols), dtype=torch.float32, device="cuda"), 1280)
    eng.set_streams(24)                                                    # oww_set_streams: reallocated and cleared
    h5, c5 = ctx.detector_history(np.arange(24))
    assert h5.shape == (24, 3, 30) and not h5.any() and not c5.any()


def test_refused_arguments_enqueue_nothing(torch_cuda):
    torch = torch_cuda
    from openwakeword_b200._native import NativeError
    B = 7
    eng = _engine(B, fresh=True)
    ctx = eng.ctx
    stream = torch.cuda.current_stream().cuda_stream
    scores = torch.zeros((B, eng.n_cols), dtype=torch.float32, device="cuda")
    final = torch.zeros((B, 2), dtype=torch.float32, device="cuda")
    n_ev = torch.zeros(1, dtype=torch.int32, device="cuda")
    buf = torch.zeros((8, 4), dtype=torch.int32, device="cuda")
    launches = ctx.launch_count
    with pytest.raises(NativeError):
        ctx.detect(scores, 1280, final, None, 0, None, stream)            # no detector configured
    with pytest.raises(NativeError):
        ctx.detector_history([0])
    for bad, deb in (([(eng.n_cols, True, 0.5, 0)], 0.0), ([(-2, True, 0.5, 0)], 0.0), ([(0, True, 0.5, 31)], 0.0),
                     ([(0, True, 0.5, -1)], 0.0), ([(0, True, None, 2)], 0.0), ([(0, True, 0.5, 2)], 0.5),
                     ([(0, True, 0.5, 0)], -1.0)):
        with pytest.raises(NativeError):
            ctx.set_detector(bad, deb)
    ctx.set_detector([(0, True, 0.5, 0), (1, False, 0.5, 0)], 0.0)
    assert ctx.launch_count == launches
    for args in ((scores, 1280, final, buf, -1, n_ev), (scores, 1280, None, None, 0, None), (None, 1280, final, None, 0, None),
                 (scores, 1280, final, None, 4, n_ev), (scores, 1280, final, buf, 4, None)):
        with pytest.raises(NativeError):
            ctx.detect(*args, stream)
    with pytest.raises(ValueError):
        ctx.detect(scores, np.zeros(B + 1, np.int32), final, None, 0, None, stream)
    h = torch.zeros((2, 2, 30), dtype=torch.float32, device="cuda")
    c = torch.zeros(2, dtype=torch.int32, device="cuda")
    with pytest.raises(NativeError):
        ctx.detector_import([3, 3], h, c, stream)                         # a duplicate id
    with pytest.raises(NativeError):
        ctx.detector_import([3, B], h, c, stream)
    assert ctx.launch_count == launches
    ctx.detect(scores, 1280, final, buf, 8, n_ev, stream)
    assert ctx.launch_count == launches + 2
    ctx.detect(scores, 1280, final, None, 0, None, stream)
    assert ctx.launch_count == launches + 3


def test_a_handle_without_a_detector_is_unchanged(torch_cuda):
    """the same scores and the same launches per step with a detector configured, removed, or never there"""
    torch = torch_cuda
    rng = np.random.default_rng(5)
    B = 19
    pcm = torch.from_numpy(rng.integers(-3000, 3000, (B, 6 * 1280)).astype(np.int16)).cuda()
    runs = []
    for detector in (False, True):
        eng = _engine(B, fresh=True)
        if detector:
            eng.set_detector([(0, True), (1, False)], 0.5)
        out, launches = [], []
        for t in range(6):
            if detector and t == 3:
                eng.ctx.set_detector([], 0.0)
            n0 = eng.ctx.launch_count
            out.append(eng.step(pcm[:, t * 1280:(t + 1) * 1280]).cpu().numpy())
            launches.append(eng.ctx.launch_count - n0)
        runs.append((np.stack(out), launches))
    assert (_bits(runs[0][0]) == _bits(runs[1][0])).all() and runs[0][1] == runs[1][1]


def test_engine_loop_with_held_streams_and_a_moved_stream(torch_cuda):
    """step_ragged + detect with held streams (prepared -1) equals one oracle per stream fed only the calls the stream
    stepped; a stream whose records and history move to another engine continues with the same events"""
    torch = torch_cuda
    rng = np.random.default_rng(8)
    B, steps = 21, 40
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    labels = [(0, True)] + [(1 + k, False) for k in range(7)]
    thr = {0: 0.3, 2: 0.1, 3: 0.1, 7: 0.1}
    a, b = _engine(B, fresh=True), _engine(B, fresh=True)
    for e in (a, b):
        e.reset(fi)
        e.set_detector(labels, thr, debounce_time=0.2)
    table = [(c, r, thr.get(j), 0) for j, (c, r) in enumerate(labels)]
    oracles = [odet.StreamDetector([odet.Label(*r) for r in table], 0.2) for _ in range(B)]
    pcm = rng.integers(-8000, 8000, (B, steps, 2 * 1280)).astype(np.int16)
    src, dst = 4, 2
    n_events = 0
    for t in range(steps):
        if t == 25:                                      # stream 4 of `a` becomes stream 2 of `b`
            b.import_streams([dst], a.export_streams([src]))
            b.set_detector_history([dst], *a.detector_history([src]))
        chunks = rng.integers(0, 3, B).astype(np.int32)
        d = torch.from_numpy(np.ascontiguousarray(pcm[:, t])).cuda()
        scores = a.step_ragged(d, chunks)
        ev, n = a.detect(scores, np.where(chunks > 0, chunks * 1280, -1))
        h_scores = scores.cpu().numpy()
        want = []
        for s in range(B):
            if chunks[s]:
                want += [(s, j, sc, i) for j, sc, i in oracles[s].detect(h_scores[s], int(chunks[s]) * 1280)[1]]
        assert n == len(want) and ev.tolist() == [(s, j, float(sc), i) for s, j, sc, i in want], t
        n_events += n
        if t >= 25:
            cb = np.zeros(B, np.int32)
            cb[dst] = chunks[src]
            db = torch.zeros((B, 2 * 1280), dtype=torch.int16, device="cuda")
            db[dst] = d[src]
            sb = b.step_ragged(db, cb)
            evb, nb = b.detect(sb, np.where(cb > 0, cb * 1280, -1))
            mine = ev[ev["stream"] == src]
            assert nb == mine.size and (evb["label"] == mine["label"]).all() and (evb["index"] == mine["index"]).all()
            assert (_bits(evb["score"]) == _bits(mine["score"])).all()
    assert n_events > 20


def _twin_models(B, fi, **kw):
    import openwakeword_b200 as owb
    from openwakeword_b200 import weights as W
    specs = [{"name": "hey_jarvis_v0.1", "head": head("hey_jarvis_v0.1")},
             {"name": "timer_v0.1", "head": head("timer_v0.1"), "class_mapping": dict(TIMER_MAP)},
             {"name": "alexa_v0.1", "head": head("alexa_v0.1")}]
    users = {None: W.synthetic_head(seed=70), 3: W.synthetic_head(seed=71), 8: W.synthetic_head(seed=72)}
    return [owb.Model(wakeword_models=specs, embedding_model_path=emb_weights(), feature_init=fi, n_streams=B, max_chunks=3,
                      stream_models={"user": users}, **kw) for _ in range(2)]


def _thresholded(res, model, thr):
    out = []
    for s in range(model.n_streams):
        for lab in model.labels():
            t = thr.get(model.get_parent_model_from_label(lab))
            if t is not None and res[lab][s] >= np.float32(t):
                out.append((s, lab, float(res[lab][s])))
    return out


@pytest.mark.parametrize("verifiers", [False, True])
def test_model_detect_equals_thresholded_predict(torch_cuda, verifiers):
    """a gated pair, a multi-class head, a plain head and a head bank on 33 streams with ragged arrivals; with device
    verifier banks every stream steps in every call (a repeated prediction is where detect differs, below)"""
    rng = np.random.default_rng(21 + verifiers)
    B = 33
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    kw = dict(custom_verifier_models={"alexa_v0.1": os.path.join(GOLDEN, "verifier_alexa.pkl")},
              custom_verifier_threshold=0.05) if verifiers else {}
    p, d = _twin_models(B, fi, **kw)
    thr = {"hey_jarvis_v0.1": 0.05, "timer_v0.1": 0.12, "alexa_v0.1": 0.05, "user": 0.05}
    post = dict(debounce_time=0.25)
    sizes = [1280, 2560, 3000, 1500] if verifiers else [0, 500, 1280, 1024, 2560, 3000, 4500]
    n_events = 0
    for t in range(60):
        if t == 30 and not verifiers:
            p.reset_streams([2, 9])
            d.reset_streams([2, 9])
        if t == 45:
            post = dict(patience={"alexa_v0.1": 2, "user": 1})
        xs = [rng.integers(-6000, 6000, sizes[int(rng.integers(0, len(sizes)))]).astype(np.int16) for _ in range(B)]
        want = _thresholded(p.predict_ragged(xs, threshold=thr, **post), p, thr)
        got = d.detect_ragged(xs, thr, **post)
        assert got == want, (t, got[:4], want[:4])
        n_events += len(got)
    assert n_events > 50
    sp, sd = p.export_streams([0, 5]), d.export_streams([0, 5])
    for lab in p.labels():
        assert (_bits(sp.history[lab]) == _bits(sd.history[lab])).all() and (sp.counts[lab] == sd.counts[lab]).all()
    assert list(p.prediction_buffer["alexa_v0.1"]) == list(d.prediction_buffer["alexa_v0.1"])


def test_repeated_prediction_is_not_verified_again(torch_cuda):
    """The documented difference, in isolation: with a device verifier, a call below 1280 samples repeats the stored
    prediction in detect, while predict passes it through the stream's verifier once more - visible when the verifier
    has changed in between."""
    import openwakeword_b200 as owb
    rng = np.random.default_rng(33)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    from openwakeword_b200.custom_verifier_model import load_verifier
    v1 = os.path.join(GOLDEN, "verifier_alexa.pkl")
    v2 = load_verifier(v1)
    v2.steps[-1][1].intercept_ = v2.steps[-1][1].intercept_ + 1.0
    spec = [{"name": "alexa_v0.1", "head": head("alexa_v0.1")}]
    p, d = [owb.Model(wakeword_models=spec, embedding_model_path=emb_weights(), feature_init=fi, n_streams=2,
                      custom_verifier_models={"alexa_v0.1": v1}, custom_verifier_threshold=0.0) for _ in range(2)]
    thr = {"alexa_v0.1": 0.0}
    for t in range(7):
        x = rng.integers(-6000, 6000, (2, 1280)).astype(np.int16)
        want = p.predict(x, threshold=thr)
        got = d.detect(x, thr)
        assert [g[2] for g in got] == [float(v) for v in want["alexa_v0.1"]]
    stored = [g[2] for g in got]
    for m in (p, d):
        m.set_custom_verifier("alexa_v0.1", v2)
    x = rng.integers(-6000, 6000, (2, 640)).astype(np.int16)
    again = p.predict(x, threshold=thr)["alexa_v0.1"]
    assert [g[2] for g in d.detect(x, thr)] == stored
    assert all(float(a) != s for a, s in zip(again, stored))
