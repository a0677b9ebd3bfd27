"""Pipelined detection from host audio without a GPU (include/owwb200.h, oww_detect_host_submit / _collect) on the
stand-in of the C ABI: every refusal fails before anything changes - the streams' ingest state (rates, input and staged
counts, staged samples, filter history), detector histories, audio and capacities are the same afterwards - and the
ticket protocol (two in flight, a third refused, collects in submission order, an unknown or collected ticket refused).
``refusal_session`` is the scenario test_gpu_detect_host.py runs on the device.  The stand-in's two calls live in a
subclass here (fake_backend.FakeContext's public methods are the ones the scripted session of test_gpu_context_session
drives), checked against the binding's signatures as test_fake_backend checks the others."""
import inspect

import numpy as np
import pytest

import fake_backend
from helpers import emb_weights, head
from openwakeword_b200 import _native

CHUNK = 1280
H = 8 * CHUNK
RATES = (8000, 16000, 44100, 48000)


class DetectHostContext(fake_backend.FakeContext):
    """the stand-in with oww_detect_host_submit / _collect: the synchronous ingest + detect (+ capture) at submit, the
    results held for the collect; the ticket protocol and refusals of the library"""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self._det_q, self._det_next = [], 0     # tickets in flight, oldest first: (ticket, results); the next ticket

    def detect_host_submit(self, packets, offsets, max_events, capture=None, final=False):
        q = self._det_q
        if len(q) == 2:
            raise _native.NativeError("two detect tickets are in flight")
        if self._ing is None:
            raise _native.NativeError("no ingest state")
        if not self.det:
            raise _native.NativeError("no detector")
        cs = 0 if capture is None else int(capture)
        if cs < 0 or (cs and not 0 < cs <= self.audio_history):
            raise _native.NativeError("capture without an audio history, or above it")
        if max_events < 0:
            raise _native.NativeError("max_events is negative")
        off = np.asarray(offsets, np.int64).ravel()
        if off.size != self._n + 1 or off[0] < 0 or (np.diff(off) < 0).any() or off[-1] > np.size(packets):
            raise _native.NativeError("bad offsets")
        scores = self.new_scores()
        chunks, prepared = self.ingest_pcm(np.asarray(packets, np.int16), off, scores)   # refuses a packet over capacity
        fin = np.zeros((self._n, self.n_detect_labels), np.float32) if final else None
        events, n = self.detect_events(scores, prepared, fin, max_events)
        clips = ends = None
        if cs:
            s = events["stream"]
            clips, ends = self._clips(s, self.pos[s], cs), self.pos[s].copy()
        ticket, self._det_next = self._det_next, self._det_next ^ 1
        q.append((ticket, (events, n, chunks, prepared, clips, ends, fin)))
        return ticket

    def detect_host_collect(self, ticket):
        q = self._det_q
        if ticket not in [t for t, _ in q]:
            raise _native.NativeError(f"detect ticket {ticket} is not in flight")
        if q[0][0] != ticket:
            raise _native.NativeError(f"detect ticket {q[0][0]} was submitted before ticket {ticket}")
        return q.pop(0)[1]


@pytest.mark.parametrize("name", ["detect_host_submit", "detect_host_collect"])
def test_the_binding_has_the_stand_ins_calls(name):
    def params(f):
        return [p for p in inspect.signature(f).parameters if p != "self"]
    assert params(getattr(DetectHostContext, name)) == params(getattr(_native.Context, name))


def state(eng):
    """everything a refused call must leave as it was"""
    ids = np.arange(eng.n_streams)
    out = list(eng.ctx.ingest_state(ids)) + [eng.ingest_capacity()]
    if eng.ctx.n_detect_labels:
        out += list(eng.detector_history(ids))
    if eng.ctx.audio_history:
        out += list(eng.audio_history(ids))
    return out


def same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def packets(eng, rng, frac=0.5):
    """one packet per stream, a share `frac` of its capacity -> (int16 packets, offsets)"""
    n = (eng.ingest_capacity() * frac).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(n)])
    return rng.integers(-8000, 8000, int(off[-1])).astype(np.int16), off


def configure(eng, ingest=True, detector=True, history=True):
    if history:
        eng.set_audio_history(H)
    if ingest:
        # host state only: no stream argument (the engine's would ask torch for the current CUDA stream)
        eng.ctx.set_input_rates(None, np.array([RATES[b % len(RATES)] for b in range(eng.n_streams)], np.int32))
    if detector:
        eng.set_detector([(0, True)], 0.5)


def refusal_session(make_engine, rng):
    """make_engine(ingest, detector, history) -> a configured StreamEngine.  Every refusal of the submit, then the ticket
    protocol."""
    NE = _native.NativeError
    for kw, cap in ((dict(ingest=False), None), (dict(detector=False), None), (dict(history=False), CHUNK)):
        eng = make_engine(**kw)
        if kw.get("ingest") is False:
            with pytest.raises(NE):
                eng.submit_detect(np.zeros(eng.n_streams, np.int16), np.arange(eng.n_streams + 1))
            continue
        pk, off = packets(eng, rng)
        before = state(eng)
        with pytest.raises(NE):
            eng.submit_detect(pk, off, max_events=4, capture=cap)
        assert same(before, state(eng))

    eng = make_engine()
    B = eng.n_streams
    pk, off = packets(eng, rng)
    t = eng.submit_detect(pk, off)                     # something staged, so that the capacities are not the initial ones
    eng.collect_detect(t)
    before = state(eng)
    cap = eng.ingest_capacity()
    pk, off = packets(eng, rng)
    bad_off = off.copy()
    bad_off[B // 2] = bad_off[B // 2 + 1] + 1          # decreasing
    over = np.concatenate([[0], np.cumsum(cap + (np.arange(B) == B - 1))])
    for args, kw in (((pk, off), dict(max_events=-1)),
                     ((pk, off), dict(max_events=4, capture=-1)),
                     ((pk, off), dict(max_events=4, capture=H + CHUNK)),
                     ((pk, bad_off), {}),
                     ((pk, np.concatenate([[-1], off[1:]])), {}),
                     ((np.zeros(int(over[-1]), np.int16), over), {})):
        with pytest.raises(NE):
            eng.submit_detect(*args, **kw)
        assert same(before, state(eng)), kw

    # the capacity counts what a ticket in flight staged: exactly the capacity then is taken, one sample more is not
    t0 = eng.submit_detect(pk, off)
    cap = eng.ingest_capacity()
    mid = state(eng)
    over = np.concatenate([[0], np.cumsum(cap + (np.arange(B) == 0))])
    with pytest.raises(NE):
        eng.submit_detect(np.zeros(int(over[-1]), np.int16), over)
    assert same(mid, state(eng))
    full = np.concatenate([[0], np.cumsum(cap)])
    t1 = eng.submit_detect(np.zeros(int(full[-1]), np.int16), full)
    assert t0 != t1
    assert (eng.ingest_capacity() <= cap).all()
    mid = state(eng)
    with pytest.raises(NE):                            # a third ticket
        eng.submit_detect(np.zeros(0, np.int16), np.zeros(B + 1, np.int64))
    assert same(mid, state(eng))
    with pytest.raises(NE):                            # out of order
        eng.collect_detect(t1)
    r0 = eng.collect_detect(t0)
    r1 = eng.collect_detect(t1)
    assert len(r0) == len(r1) == 4
    for t in (t0, t1, 7, -1):                          # collected, or never submitted
        with pytest.raises(NE):
            eng.collect_detect(t)
    # the handle still serves calls
    t = eng.submit_detect(np.zeros(0, np.int16), np.zeros(B + 1, np.int64), final=True)
    ev, n, chunks, prepared, fin = eng.collect_detect(t)
    assert fin.shape == (B, 1) and chunks.shape == prepared.shape == (B,)


@pytest.fixture
def fake_engine(monkeypatch, built_library):
    monkeypatch.setattr(_native, "Context", DetectHostContext)
    from openwakeword_b200.engine import StreamEngine

    def make(ingest=True, detector=True, history=True):
        eng = StreamEngine([head("alexa_v0.1")], 5, embedding=emb_weights(), max_chunks=1)
        eng.ctx.features = False                      # audio only: the refusals and the protocol need no scores
        configure(eng, ingest, detector, history)
        return eng
    return make


def test_refusals_leave_every_stream_unchanged_and_the_ticket_protocol(fake_engine):
    refusal_session(fake_engine, np.random.default_rng(0))


def test_submit_equals_ingest_then_detect_on_the_stand_in(monkeypatch, built_library):
    """the stand-in's submit is its own synchronous ingest + detect (+ capture): the results a twin gets that way"""
    monkeypatch.setattr(_native, "Context", DetectHostContext)
    from openwakeword_b200.engine import StreamEngine
    engs = []
    for _ in range(2):
        e = StreamEngine([head("alexa_v0.1")], 3, embedding=emb_weights(), max_chunks=1)
        e.ctx.features = False
        configure(e)
        e.set_detector([(0, True)], 0.0)               # every prediction fires: events from the sixth call on
        engs.append(e)
    a, b = engs
    rng = np.random.default_rng(1)
    pending = []
    for k in range(9):
        pk, off = packets(a, rng, 0.6)
        pending.append(a.submit_detect(pk, off, max_events=2, capture=CHUNK, final=True))
        scores = b.ctx.new_scores()
        chunks, prepared = b.ctx.ingest_pcm(pk, off, scores)
        fin = np.zeros((3, 1), np.float32)
        ev, n = b.ctx.detect_events(scores, prepared, fin, 2)
        clips = b.ctx._clips(ev["stream"], b.ctx.pos[ev["stream"]], CHUNK)
        got = a.collect_detect(pending.pop(0)) if len(pending) == 2 else None
        if got is not None:
            assert len(got) == 7
        if k == 8:
            while pending:
                got = a.collect_detect(pending.pop(0))
            for x, y in zip(got, (ev, n, chunks, prepared, clips, b.ctx.pos[ev["stream"]], fin)):
                assert np.array_equal(x, y)
            assert n > 2 and len(got[0]) == 2
