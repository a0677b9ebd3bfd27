"""-m gpu: pipelined detection from host audio (oww_detect_host_submit / _collect, csrc/api.cu and the delivery kernel of
csrc/detect.cu) against the synchronous loop bit for bit.

Two handles of the same weights, heads (a gated pair, a 7-class head and a head bank), detector, rates and audio history
take the same packets: handle A through submit_detect / collect_detect with two tickets in flight, handle B through
ingest + oww_detect (+ oww_capture_events).  After every call the events, counts, chunks, prepared counts, final rows,
clips and ends are equal.  151 streams (not a multiple of the fused group size) at 8 / 16 / 44.1 / 48 kHz; packets of 0
samples, under one chunk, 80 ms and up to the capacity; held streams; max_events below the count and 0; 1 s clips; a
page-locked caller buffer and a pageable one (overwritten right after the submit).  Between two submits, while the
earlier ticket is in flight, both handles take the same per-stream settings (set and cleared), partial resets (blocking
and stream-ordered), moves of streams with their detector history, audio and ingest state, rate changes and head-bank
assignments: each applies to the later call only.  A few calls at the C3 shape (8192 streams, the bench's seven
networks).  Then the refusals and the ticket protocol of test_detect_host_host.refusal_session on the device."""
from collections import deque

import numpy as np
import pytest

from helpers import bank_heads, emb_weights, head, seven_heads
from test_detect_host_host import configure, refusal_session

pytestmark = pytest.mark.gpu
CHUNK = 1280
CLIP = 16000                          # 1 s clips
RATES = (8000, 16000, 44100, 48000)
FI = np.zeros((41, 96), np.float32)


@pytest.fixture(scope="module")
def torch_cuda(built_library):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _engine(B, heads, labels, threshold, bank, rates, H=2 * CLIP):
    from openwakeword_b200.engine import StreamEngine
    eng = StreamEngine(heads, B, embedding=emb_weights(), max_chunks=2 if bank else 1)
    if bank:
        cands = bank_heads()
        eng.bank = eng.add_head_bank(cands[0], len(cands))[0]
        for k, h in enumerate(cands):
            eng.load_bank_head(eng.bank, k, h)
        eng.assign_bank_head(eng.bank, (np.arange(B) % (len(cands) + 1) - 1).astype(np.int32))
    if H:
        eng.set_audio_history(H)
    eng.ctx.set_input_rates(None, np.asarray(rates, np.int32))
    eng.set_detector(labels, threshold)
    return eng


def _sync(eng, pk, off, M, cs, final):
    """the synchronous loop: ingest, oww_detect with prepared from it, oww_capture_events -> what collect_detect returns"""
    import torch
    from openwakeword_b200 import _native
    ctx, B, L = eng.ctx, eng.n_streams, eng.ctx.n_detect_labels
    dev = torch.device("cuda", eng.device_index)
    chunks, prepared = eng.ingest(torch.from_numpy(pk if pk.size else np.zeros(1, np.int16)).to(dev), off)
    s = ctx._current_stream()
    fin = torch.empty((B, L), dtype=torch.float32, device=dev)
    ev = torch.empty((max(M, 1), 4), dtype=torch.int32, device=dev)
    n_ev = torch.zeros(1, dtype=torch.int32, device=dev)
    ctx.detect(eng.ingest_scores, prepared, fin, ev if M else None, M, n_ev, s)
    if cs:
        clips = torch.empty((max(M, 1), cs), dtype=torch.int16, device=dev)
        ends = torch.empty(max(M, 1), dtype=torch.int64, device=dev)
        ctx.capture_events(ev, n_ev, M, cs, clips, ends, s)
    n = int(n_ev.item())
    k = min(n, M)
    out = (ev[:k].cpu().numpy().view(_native.EVENT_DTYPE).reshape(-1), n, chunks, prepared)
    if cs:
        out += (clips[:k].cpu().numpy(), ends[:k].cpu().numpy())
    if final:
        out += (fin.cpu().numpy(),)
    return out


def _equal(got, want, what):
    assert len(got) == len(want), what
    assert got[1] == want[1], (what, got[1], want[1])
    for i, (g, w) in enumerate(zip(got, want)):
        if i == 1:
            continue
        g, w = np.asarray(g), np.asarray(w)
        assert g.dtype == w.dtype and g.shape == w.shape and g.tobytes() == w.tobytes(), (what, i)


def _packets(k, cap, rates, rng):
    """stream b's packet of call k: 0 samples, under one chunk, 80 ms, random, its whole capacity or 80 ms again"""
    n = np.empty(cap.size, np.int64)
    for b in range(cap.size):
        kind = (b + k) % 6
        r = int(rates[b])
        n[b] = (0, r // 50, r * 8 // 100, int(rng.integers(0, cap[b] + 1)), cap[b], r * 8 // 100)[kind]
    n = np.minimum(n, cap)
    off = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    t = np.arange(int(off[-1]))
    pk = np.clip(rng.normal(0, 6000, t.size) * (1 + np.sin(t / 900.0)), -32768, 32767).astype(np.int16)
    return pk, off


def _run(torch, a, b, n_calls, rng, schedule, between=None):
    """n_calls submits on a (two in flight) against the synchronous loop on b; between(k, eng) runs on both handles
    before call k -> (events found, calls whose count exceeded max_events, clips delivered)"""
    pending = deque()
    stats = np.zeros(3, np.int64)

    def collect():
        t, want, what, _ = pending.popleft()
        got = a.collect_detect(t)
        _equal(got, want, what)
        stats[:] += (want[1], want[1] > len(want[0]), len(want[4]) if len(want) >= 6 else 0)

    for k in range(n_calls):
        if between is not None:
            between(k, a)
            between(k, b)
        cap = a.ingest_capacity()
        assert np.array_equal(cap, b.ingest_capacity()), k        # the staged samples of the ticket in flight count
        rates = a.ctx.ingest_state(np.arange(a.n_streams), samples=False)[0]
        pk, off = _packets(k, cap, rates, rng)
        M, cs, final = schedule(k)
        keep = None
        if k % 2:                                      # page-locked: read by the copy engine until the collect
            keep = torch.empty(max(pk.size, 1), dtype=torch.int16).pin_memory()
            x = keep.numpy()[:pk.size]
            x[:] = pk
        else:                                          # pageable: staged before the submit returns
            x = pk.copy()
        t = a.submit_detect(x, off, max_events=M, capture=cs or None, final=final)
        if keep is None:
            x[:] = rng.integers(-32768, 32767, x.size).astype(np.int16)
        pending.append((t, _sync(b, pk, off, M, cs, final), f"call {k}", keep))
        if len(pending) == 2:
            collect()
    while pending:
        collect()
    return stats


def test_submit_collect_equals_the_synchronous_loop_151_streams(torch_cuda):
    B = 151
    rates = np.array([RATES[b % 4] for b in range(B)], np.int32)
    heads = [head("alexa_v0.1"), head("hey_jarvis_v0.1"), head("timer_v0.1")]
    # columns: alexa 0, hey_jarvis 1 (its verifier's raw score 2), timer 3..9, the head bank 10
    labels = [(0, True), (1, True), (3, False), (4, False), (10, True)]
    thr = {0: 0.5, 1: 0.3, 2: 0.0, 4: 0.5}
    a, b = (_engine(B, heads, labels, thr, True, rates) for _ in range(2))
    L = len(labels)
    moved = np.array([3, 40, 77, 150])

    def between(k, eng):
        if k == 4:
            eng.set_stream_detection(np.arange(0, B, 3), threshold={0: 0.2, 1: None}, debounce_time=1.0)
            eng.set_stream_detection(np.arange(1, B, 3), patience={0: 2})
        elif k == 10:
            eng.clear_stream_detection(np.arange(0, B, 6))
        elif k in (7, 19):
            eng.reset(FI, np.arange(k % 5, B, 9))
        elif k == 13:
            eng.reset_async(FI, np.arange(2, B, 11))
        elif k == 16:                                  # streams move with their detector history, audio and ingest state
            rec = eng.export_streams(moved)
            hist, cnt = eng.detector_history(moved)
            aud, pos = eng.audio_history(moved)
            ing = eng.ctx.ingest_state(moved)
            dst = np.roll(moved, 1)
            eng.import_streams(dst, rec)
            eng.set_detector_history(dst, hist, cnt)
            eng.set_audio_history_state(dst, aud, pos)
            eng.ctx.set_ingest_state(dst, *ing)
        elif k == 22:
            ids = np.arange(5, B, 13)
            eng.ctx.set_input_rates(ids, np.array([RATES[(i + 1) % 4] for i in range(ids.size)], np.int32))
        elif k == 25:
            eng.assign_bank_head(eng.bank, np.full(20, 2, np.int32), stream_ids=np.arange(20))
        elif k == 28:
            eng.set_stream_detection(None, threshold=0.4, debounce_time=0.5)
        elif k == 33:
            eng.clear_stream_detection()

    def schedule(k):
        M = 2 if k % 5 == 3 else (0 if k % 7 == 4 else B * L)
        cs = CLIP if k % 3 == 1 else 0
        return (min(M, 64) if cs else M), cs, k % 2 == 0

    n_ev, truncated, clips = _run(torch_cuda, a, b, 40, np.random.default_rng(7), schedule, between)
    assert n_ev > 0 and truncated >= 3 and clips > 0, (n_ev, truncated, clips)


def test_submit_collect_at_c3(torch_cuda):
    """8192 streams x the bench's seven networks, 80 ms packets at 16 kHz and 48 kHz, threshold 0.5, then a 0.5 s
    debounce on every stream"""
    B = 8192
    rates = np.where(np.arange(B) % 2, 48000, 16000).astype(np.int32)
    # columns: heads 0, 1; the gated pair 2 (verifier 3); heads 4, 5; the timer 6..12
    labels = [(0, True), (1, True), (2, True), (4, True), (5, True), (7, False)]
    a, b = (_engine(B, seven_heads(), labels, 0.5, False, rates, H=13 * CHUNK) for _ in range(2))

    def between(k, eng):
        if k == 4:
            eng.set_stream_detection(None, debounce_time=0.5)

    def schedule(k):
        return (64, CLIP, True) if k == 5 else (B * len(labels), 0, k % 2 == 0)

    _run(torch_cuda, a, b, 8, np.random.default_rng(3), schedule, between)


def test_refusals_and_tickets_on_the_device(torch_cuda):
    from openwakeword_b200.engine import StreamEngine

    def make(ingest=True, detector=True, history=True):
        eng = StreamEngine([head("alexa_v0.1")], 37, embedding=emb_weights(), max_chunks=1)
        configure(eng, ingest, detector, history)
        return eng
    refusal_session(make, np.random.default_rng(5))
