"""-m gpu: long-running streams against twin streams.

Per-stream state that grows for the life of a stream - the mel and feature ring row counts, the detector's prediction
count, the audio history position and the resampler's input count - is set near or past its limit on a twin of a
control stream in the same handle.  Twin and control get the same samples, schedule, head-bank slot and verifier, and
no slot position or count value enters any arithmetic, so everything they produce is equal bit for bit; the counters
themselves (and the event indices and positions derived from them) equal the rules of tests/helpers.py.

1. Ring counts: twins at 2^30 - d mel / feature rows, so the rebase lands at every position inside 1-, 2- and 3-chunk
   calls and on call boundaries, just past a rebase, and imported at or past 2^30 (rebased on import); every split
   point of mode 3, modes 0 and 2, and mode 3 without the fused step.  After every call: score rows, stream records
   (outside the count words, which follow the rule) and, every fifth call, the host readers.
2. Detector: histories copied to twins at 2^30 - d and 2^31 - 1 predictions, with patience and with debounce.
3. Audio history: positions just below and across 2^31, 2^32 and 2^40, and a buffer of more than 2^31 samples.
4. Ingest: resampler input counts offset by a multiple of `down` near 2^31, 2^32 and 2^40 (bit for bit), and at
   2^32 + 1 against the float64 resampler.
5. max_chunks above OWW_MAX_CHUNKS is refused."""
import numpy as np
import pytest

from helpers import (COUNT_WRAP, bank_heads, det_count, det_imported, emb_weights, event_index, events_diff, head,
                     imported_count, judge_resampled, mixes, record_diff, record_words, ring_count, seven_heads)

pytestmark = pytest.mark.gpu
CHUNK = 1280
VER = "verifier_alexa.pkl"
M30 = 1 << 30


@pytest.fixture(scope="module")
def torch_cuda(built_library):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _fi(rng):
    return rng.normal(0, 1, (41, 96)).astype(np.float32)


# ---- 1. ring counts ------------------------------------------------------------------------------------------------
RING_CONFIGS = {
    "mode3_split3": dict(cnn_mode=3, split_from=3),
    "mode3_split7": dict(cnn_mode=3, split_from=7),
    "mode3_split11": dict(cnn_mode=3, split_from=11),
    "mode3_split15": dict(cnn_mode=3, split_from=15),
    "mode3_split20": dict(cnn_mode=3, split_from=20),
    "mode3_unfused": dict(cnn_mode=3, split_from=11, fuse_step=False),
    "mode0": dict(cnn_mode=0),
    "mode2": dict(cnn_mode=2),
}
# twin counts from the control's (m, f): 8 mel rows and 1 feature row per chunk
RING_TARGETS = (
    [(f"mel 2^30-{d}", lambda m, f, d=d: (M30 - d, f)) for d in (1, 3, 5, 8, 9, 16, 17, 24, 25)]
    + [(f"feature 2^30-{d}", lambda m, f, d=d: (m, M30 - d)) for d in (1, 2, 3)]
    + [("both 2^30-1", lambda m, f: (M30 - 1, M30 - 1)),
       ("feature only, 2^30-7", lambda m, f: (m, M30 - 7)),
       ("just past a rebase", lambda m, f: ((1 << 20) + 3, (1 << 20) + 1)),
       ("imported at 2^31-1", lambda m, f: (2 ** 31 - 1, 2 ** 31 - 1)),
       ("imported at 2^30+5", lambda m, f: (M30 + 5, M30 + 5))])
RING_P = 75                 # twin pairs: 151 streams give fused groups of more than one stream, the last one ragged
RING_MC = 3
RING_POST = (["rag", 1, "sub", 2, "rag", 3, 1, "rag", 2, "sub"] * 6)[:56]     # crossings in ragged and lockstep calls
RING_RESET_AT = 30


class RingHandle:
    """151 streams on the bench's seven networks (a gated pair among them): controls 0..P-1, twins P..2P-1 (so a pair
    never shares a fused group), stream 2P alone; outside mode 0 a head bank of three slots, and a verifier bank,
    assigned per pair."""

    def __init__(self, fi, **kw):
        from openwakeword_b200.engine import StreamEngine
        import os
        from helpers import GOLDEN
        self.P = RING_P
        self.B = 2 * self.P + 1
        self.eng = StreamEngine(seven_heads(), self.B, embedding=emb_weights(), feature_init=fi, max_chunks=RING_MC, **kw)
        vb = self.eng.add_verifier_bank(0, 1, 0.0)
        self.eng.load_verifier(vb, 0, os.path.join(GOLDEN, VER))
        pair = np.concatenate([np.arange(self.P), np.arange(self.P), [self.P]])
        self.eng.assign_verifier(vb, np.where(pair % 2 == 0, 0, -1).astype(np.int32))
        if kw.get("cnn_mode", 3) != 0:
            bh = bank_heads()
            hb, _, _ = self.eng.add_head_bank(bh[0], 3)
            for k, h in enumerate(bh):
                self.eng.load_bank_head(hb, k, h)
            self.eng.assign_bank_head(hb, (pair % 3).astype(np.int32))
        self.ctrl = np.arange(self.P)
        self.twin = self.ctrl + self.P


def _ring_call(torch, H, rng, kind):
    """one call of `kind` with the same samples and chunk count for both streams of each pair -> (score rows, chunks)"""
    B, P = H.B, H.P
    x = mixes(rng, B, RING_MC * CHUNK)
    x[H.twin] = x[H.ctrl]
    if isinstance(kind, int):
        d = torch.from_numpy(np.ascontiguousarray(x[:, :kind * CHUNK])).cuda()
        return H.eng.step(d, kind).cpu().numpy(), np.full(B, kind, np.int32)
    c = rng.integers(0, RING_MC + 1, B).astype(np.int32)
    c[rng.choice(P, 8, replace=False)] = 0                       # pairs held together
    c[H.twin] = c[H.ctrl]
    c[-1] = RING_MC
    if kind == "sub":
        return H.eng.collect(H.eng.submit_ragged(x, c)), c
    return H.eng.step_ragged(torch.from_numpy(x).cuda(), c).cpu().numpy(), c


def _readers_equal(ctx, a, b):
    for get in (lambda s: ctx.get_mel(s, 76), lambda s: ctx.get_features(s, 120), lambda s: ctx.get_features(s, 16, 3)):
        assert np.array_equal(get(a), get(b)), (a, b)


@pytest.mark.parametrize("config", list(RING_CONFIGS))
def test_ring_counts_across_the_rebase(torch_cuda, config):
    import time
    torch = torch_cuda
    t0 = time.time()
    kw = RING_CONFIGS[config]
    rng = np.random.default_rng(list(RING_CONFIGS).index(config) + 100)
    fi = _fi(rng)
    H = RingHandle(fi, **kw)
    P, ctx = H.P, H.eng.ctx
    for t in range(40):                                          # warm-up: every stream its own audio
        _ring_call(torch, H, rng, [1, 2, "rag", 3][t % 4])
    rec = H.eng.export_streams(H.ctrl).cpu().numpy()
    w = record_words(rec).reshape(P, -1)
    ctrl_counts = [(int(w[k, 5]), int(w[k, 6])) for k in range(P)]
    targets = [RING_TARGETS[k % len(RING_TARGETS)] for k in range(P)]
    raised = [fn(*ctrl_counts[k]) for k, (_, fn) in enumerate(targets)]
    w[:, 5] = [r[0] for r in raised]
    w[:, 6] = [r[1] for r in raised]
    H.eng.import_streams(H.twin, torch.from_numpy(rec))
    assert ctx.stream_state_rejected() == 0
    want_c = list(ctrl_counts)
    want_t = [(imported_count(m), imported_count(f)) for m, f in raised]
    crossed = {}                                                 # pair -> call of its first crossing
    kinds = (set(), set())                                       # kinds of call in which mel / feature counts crossed
    n_cmp = 0

    fresh = set()                                                # pairs reset: the twin's counts are the control's

    def check_records(t):
        nonlocal n_cmp
        r = H.eng.export_streams(np.arange(2 * P)).cpu().numpy()
        for k in range(P):
            wc = record_words(r[k])
            if k in fresh:
                want_c[k] = want_t[k] = (int(wc[5]), int(wc[6]))
            assert (int(wc[5]), int(wc[6])) == want_c[k], (t, k)
            bad = record_diff(r[k], r[P + k], want_t[k])
            assert not bad, (config, t, k, targets[k][0], bad)
        n_cmp += P

    check_records(-1)
    for t, kind in enumerate(RING_POST):
        if t == RING_RESET_AT:                                   # a reset pair: the twin is the control again
            ids = [0, P]
            H.eng.reset_async(fi, stream_ids=ids)
            fresh.add(0)
        out, c = _ring_call(torch, H, rng, kind)
        assert np.array_equal(out[H.ctrl], out[H.twin], equal_nan=True), \
            (config, t, kind, np.nonzero(~((out[H.ctrl] == out[H.twin]) | np.isnan(out[H.ctrl])))[0][:8])
        n_cmp += P
        for k in range(P):
            n = int(c[k])
            if n == 0 or k in fresh:
                continue
            want_c[k] = (ring_count(want_c[k][0], 8 * n), ring_count(want_c[k][1], n))
            m, f = want_t[k]
            if (m + 8 * n >= COUNT_WRAP or f + n >= COUNT_WRAP) and k not in crossed:
                crossed[k] = t
            for i, v in enumerate((m + 8 * n, f + n)):
                if v >= COUNT_WRAP:
                    kinds[i].add(kind if isinstance(kind, str) else "lockstep")
            want_t[k] = (ring_count(m, 8 * n), ring_count(f, n))
        check_records(t)
        if t % 5 == 4:
            for k in range(P):
                assert ctx.get_counts(int(H.ctrl[k])) == want_c[k] and ctx.get_counts(int(H.twin[k])) == want_t[k]
                _readers_equal(ctx, int(H.ctrl[k]), int(H.twin[k]))
            n_cmp += P
    should_cross = {k for k, (name, _) in enumerate(targets) if "2^30-" in name or "2^31-1" in name}
    assert should_cross <= set(crossed), sorted(should_cross - set(crossed))
    assert {"rag", "sub"} <= kinds[0] and {"rag", "sub"} <= kinds[1], kinds   # the ragged append's rebase
    last = max(crossed.values())
    assert len(RING_POST) - 1 - last >= 45, last
    by_target = {}
    for k, t in crossed.items():
        by_target.setdefault(targets[k][0], []).append(t)
    print(f"\n[{config}] {n_cmp} twin comparisons, {time.time() - t0:.1f} s; mel / feature crossings in {kinds}; calls "
          + "; ".join(f"{name}: {sorted(v)}" for name, v in by_target.items()))


# ---- 2. detector ---------------------------------------------------------------------------------------------------
DET_TARGETS = [M30 - 1, M30 - 2, M30 - 5, M30 - 30, 2 ** 31 - 1]


@pytest.mark.parametrize("post", ["patience", "debounce"])
def test_detector_counts_across_the_rebase(torch_cuda, post):
    import time
    torch = torch_cuda
    from openwakeword_b200.engine import StreamEngine
    t0 = time.time()
    rng = np.random.default_rng(7 if post == "patience" else 8)
    P = 2 * len(DET_TARGETS)
    B = 2 * P + 1
    ctrl, twin = np.arange(P), np.arange(P) + P
    eng = StreamEngine(seven_heads(), B, embedding=emb_weights(), feature_init=_fi(rng), max_chunks=3)
    eng.set_audio_history(3 * 3840)
    # columns: 0, 1 single heads; 2 the gated head (3 its verifier); 4, 5 single heads; 6..12 the 7-class head
    labels = [(0, True), (2, True), (4, True), (6, False), (8, False), (-1, False)]
    thr = {0: 0.3, 1: 0.5, 3: 0.1, 5: 0.0}                       # label 2 and 4 without one; 5 fires on every call
    if post == "patience":
        eng.set_detector(labels, thr, patience={0: 2, 3: 3})
    else:
        eng.set_detector(labels, thr, debounce_time=0.3)
    L = len(labels)

    def call(kind):
        x = mixes(rng, B, 3 * CHUNK)
        x[twin] = x[ctrl]
        if kind == "lock":
            n = int(rng.integers(1, 4))
            c = np.full(B, n, np.int32)
        else:
            c = rng.integers(0, 4, B).astype(np.int32)
            c[twin] = c[ctrl]
        scores = eng.step_ragged(torch.from_numpy(x).cuda(), c)
        prep = np.where(c > 0, c * CHUNK, -1).astype(np.int32)
        if kind == "rag":                                        # held pairs: skipped, or a short prepared count
            short = (c == 0) & (rng.random(B) < 0.5)
            prep[short] = rng.integers(0, CHUNK, int(short.sum()))
            prep[twin] = prep[ctrl]
        return scores, prep

    for _ in range(34):                                          # the controls past 30 predictions
        s, p = call("lock")
        eng.detect(s, p)
    hist, cnt = eng.detector_history(ctrl)
    assert (cnt >= 30).all(), cnt
    raised = np.array([DET_TARGETS[k % len(DET_TARGETS)] for k in range(P)], np.int64)
    eng.set_detector_history(twin, hist, raised.astype(np.int32))
    h2, c2 = eng.detector_history(twin)
    want = {int(s): int(v) for s, v in zip(ctrl, cnt)}
    want.update({int(twin[k]): det_imported(raised[k]) for k in range(P)})
    assert np.array_equal(h2, hist) and [int(v) for v in c2] == [want[int(s)] for s in twin]
    twin_of = {int(c): int(t) for c, t in zip(ctrl, twin)}
    crossed, n_cmp = {}, 0
    for t in range(48):
        scores, prep = call(["lock", "rag", "lock", "lock", "rag"][t % 5])
        index_of = {b: event_index(want[b]) for b in want}
        if t % 2:
            ev, n, clips, ends = eng.detect(scores, prep, capture=2 * CHUNK)
        else:
            final = torch.empty((B, L), dtype=torch.float32, device="cuda")
            ev, n = eng.detect(scores, prep, final=final)
            f = final.cpu().numpy()
            live = prep[ctrl] >= 0
            assert np.array_equal(f[ctrl][live].view(np.int32), f[twin][live].view(np.int32)), t
        assert n == len(ev)
        assert not events_diff(ev, ev, twin_of, index_of), (post, t, events_diff(ev, ev, twin_of, index_of))
        if t % 2:
            clips = clips.cpu().numpy()
            row = {(int(e["stream"]), int(e["label"])): i for i, e in enumerate(ev)}
            for (s, j), i in row.items():
                if s in twin_of:
                    k = row[(twin_of[s], j)]
                    assert np.array_equal(clips[i], clips[k]) and ends[i] == ends[k], (t, s, j)
                    n_cmp += 1
        for e in ev:                                             # the controls' indices follow the same rule
            if int(e["stream"]) in twin_of:
                assert int(e["index"]) == index_of[int(e["stream"])]
        n_cmp += P
        for b in list(want):
            if prep[b] >= 0:
                if det_count(want[b]) < want[b] and b not in crossed:
                    crossed[b] = t
                want[b] = det_count(want[b])
    _, c3 = eng.detector_history(np.concatenate([ctrl, twin]))
    assert [int(v) for v in c3] == [want[int(s)] for s in np.concatenate([ctrl, twin])]
    assert set(int(s) for s in twin) <= set(crossed), sorted(set(int(s) for s in twin) - set(crossed))
    print(f"\n[detector {post}] {n_cmp} twin comparisons, {time.time() - t0:.1f} s; crossings (twin: call) "
          + ", ".join(f"{DET_TARGETS[(s - P) % len(DET_TARGETS)]}: {t}" for s, t in sorted(crossed.items())))


# ---- 3. audio history ----------------------------------------------------------------------------------------------
AUDIO_MARKS = [2 ** 31, 2 ** 32, 2 ** 40]


def _audio_pairs(torch, eng, rng, ctrl, twin, marks, deltas, calls, n_read):
    """import the controls' histories into the twins at position mark - delta, step both, and compare -> comparisons"""
    B = eng.n_streams
    audio, pos = eng.audio_history(ctrl)
    shift = np.array([m - d for m, d in zip(marks, deltas)], np.int64) - pos
    eng.set_audio_history_state(twin, audio, pos + shift)
    n_cmp = 0
    for t in range(calls):
        x = mixes(rng, B, 3 * CHUNK)
        c = rng.integers(0, 4, B).astype(np.int32) if eng.ctx.max_chunks >= 3 else np.ones(B, np.int32)
        c = np.minimum(c, eng.ctx.max_chunks)
        x[twin], c[twin] = x[ctrl], c[ctrl]
        scores = eng.step_ragged(torch.from_numpy(np.ascontiguousarray(x[:, :eng.ctx.max_chunks * CHUNK])).cuda(), c)
        a_c, p_c = eng.audio_history(ctrl)
        a_t, p_t = eng.audio_history(twin)
        assert np.array_equal(a_c, a_t) and np.array_equal(p_t - p_c, shift), t
        # ends straddling each mark on the twin, the same samples on the control
        offs = np.array([-2 * CHUNK - 7, -1, 0, 1, 700, 2 * CHUNK + 3, 4 * CHUNK], np.int64)
        ends_t = (np.array(marks, np.int64)[:, None] + offs[None]).ravel()
        ends_c = ends_t - np.repeat(shift, offs.size)
        ids_c, ids_t = np.repeat(ctrl, offs.size), np.repeat(twin, offs.size)
        g_c, q_c = eng.get_audio(ids_c, n_read, ends_c)
        g_t, q_t = eng.get_audio(ids_t, n_read, ends_t)
        assert torch.equal(g_c, g_t), t
        assert np.array_equal(q_t.cpu().numpy() - q_c.cpu().numpy(), np.repeat(shift, offs.size))
        n_cmp += ids_c.size + len(ctrl)
        if eng.ctx.n_detect_labels:
            prep = np.where(c > 0, c * CHUNK, -1).astype(np.int32)
            ev, n, clips, ends = eng.detect(scores, prep, capture=n_read)
            clips = clips.cpu().numpy()
            row = {int(e["stream"]): i for i, e in enumerate(ev)}
            for k in range(len(ctrl)):
                if c[ctrl[k]]:
                    i, j = row[int(ctrl[k])], row[int(twin[k])]
                    assert np.array_equal(clips[i], clips[j]) and ends[j] - ends[i] == shift[k], (t, k)
                    n_cmp += 1
    return n_cmp, shift


@pytest.mark.parametrize("H", [3840, 160000])
def test_audio_positions_past_2_31(torch_cuda, H):
    torch = torch_cuda
    from openwakeword_b200.engine import StreamEngine
    rng = np.random.default_rng(H)
    marks = [m for m in AUDIO_MARKS for _ in range(2)]
    deltas = [1, 2 * CHUNK + 333] * len(AUDIO_MARKS)             # across on the first stepping call / a few calls later
    P = len(marks)
    B = 2 * P + 1
    ctrl, twin = np.arange(P), np.arange(P) + P
    eng = StreamEngine([head("alexa_v0.1")], B, embedding=emb_weights(), max_chunks=3)
    eng.set_audio_history(H)
    eng.set_detector([(-1, False)], {0: 0.0})                    # fires for every stream that predicts
    for _ in range(4):
        x = mixes(rng, B, 3 * CHUNK)
        x[twin] = x[ctrl]
        eng.step(torch.from_numpy(x).cuda(), 3)
    n_cmp, shift = _audio_pairs(torch, eng, rng, ctrl, twin, marks, deltas, 8, min(H, 5000))
    print(f"\n[audio H={H}] {n_cmp} twin comparisons; twin positions offset by {sorted(set(shift.tolist()))}")


def test_audio_buffer_past_2_31_samples(torch_cuda):
    """2304 streams x 960000 samples (4.4 GB): pairs at the first and last slots, whose rings start past 2^31 samples"""
    torch = torch_cuda
    from openwakeword_b200.engine import StreamEngine
    rng = np.random.default_rng(5)
    B, H = 2304, 960000
    assert (B - 1) * H > 2 ** 31
    eng = StreamEngine([head("alexa_v0.1")], B, embedding=emb_weights(), max_chunks=1)
    eng.set_audio_history(H)
    ctrl, twin = np.array([0, B - 2]), np.array([B - 1, 1])
    for _ in range(3):
        x = mixes(rng, B, CHUNK)
        x[twin] = x[ctrl]
        eng.step(torch.from_numpy(x).cuda(), 1)
    n_cmp, _ = _audio_pairs(torch, eng, rng, ctrl, twin, [2 ** 32, 2 ** 31], [CHUNK + 5, 1], 3, 3 * CHUNK)
    print(f"\n[audio 2304 x 960000] {n_cmp} twin comparisons")
    del eng
    torch.cuda.empty_cache()


# ---- 4. ingest -----------------------------------------------------------------------------------------------------
INGEST_RATES = [8000, 11025, 16000, 44100, 48000]


def test_ingest_counts_past_2_31(torch_cuda):
    torch = torch_cuda
    from openwakeword_b200 import _native
    from openwakeword_b200.engine import StreamEngine
    from oracle import resample as ores
    rng = np.random.default_rng(11)
    pairs = [(r, m) for r in INGEST_RATES for m in AUDIO_MARKS]
    P = len(pairs)
    ctrl, twin = np.arange(P), np.arange(P) + P
    f64 = np.arange(len(INGEST_RATES)) + 2 * P                  # one stream per rate against the float64 resampler
    B = 2 * P + len(INGEST_RATES)
    rates = np.array([r for r, _ in pairs] * 2 + INGEST_RATES, np.int32)
    eng = StreamEngine([head("alexa_v0.1"), head("timer_v0.1")], B, embedding=emb_weights(), max_chunks=2)
    eng.set_audio_history(160000)
    eng.set_input_rates(rates)
    sig = lambda r, n: np.clip(rng.normal(0, 6000, n), -32768, 32767).astype(np.int16)  # noqa: E731

    def feed(lengths):
        xs = [sig(int(rates[b]), int(lengths[b])) for b in range(B)]
        for k in range(P):
            xs[twin[k]] = xs[ctrl[k]]
        off = np.concatenate([[0], np.cumsum([x.size for x in xs])])
        chunks, prep = eng.ingest(torch.from_numpy(np.concatenate(xs)).cuda(), off)
        return xs, chunks, prep

    for _ in range(3):                                           # warm-up of the pairs
        cap = eng.ingest_capacity()
        n = np.minimum(cap, rng.integers(0, 4000, B))
        n[twin] = n[ctrl]
        n[f64] = 0
        feed(n)
    r_, S, staged, x, hist = eng.ctx.ingest_state(ctrl)
    downs = np.array([_native.resampler_taps(int(r))[2] for r in r_], np.int64)
    k = np.array([(m - int(s)) // d - 2 for (_, m), s, d in zip(pairs, S, downs)], np.int64)
    eng.ctx.set_ingest_state(twin, r_, S + k * downs, staged, x, hist)
    S0 = 2 ** 32 + 1
    h0 = sig(0, 128 * len(INGEST_RATES)).reshape(len(INGEST_RATES), 128)
    eng.ctx.set_ingest_state(f64, rates[f64], np.full(f64.size, S0, np.int64), np.zeros(f64.size, np.int32),
                             np.zeros((f64.size, 1), np.int16), h0)
    fed = [[] for _ in f64]
    n_cmp = 0
    for t in range(12):
        cap = eng.ingest_capacity()
        assert np.array_equal(cap[ctrl], cap[twin]), t
        n = cap if t == 0 else np.minimum(cap, rng.choice([0, 1, 13, 997, 2000, 5000, 10 ** 6], B))
        n[twin] = n[ctrl]
        xs, chunks, prep = feed(n)
        for i, b in enumerate(f64):
            fed[i].append(xs[b])
        assert np.array_equal(chunks[ctrl], chunks[twin]) and np.array_equal(prep[ctrl], prep[twin]), t
        sc = eng.ingest_scores.cpu().numpy()
        assert np.array_equal(sc[ctrl], sc[twin], equal_nan=True), t
        a, b = eng.ctx.ingest_state(ctrl), eng.ctx.ingest_state(twin)
        assert np.array_equal(a[0], b[0]) and np.array_equal(b[1] - a[1], k * downs), t
        for u, v in zip(a[2:], b[2:]):
            assert np.array_equal(u, v), t
        n_cmp += 4 * P
    assert (eng.ctx.ingest_state(twin, samples=False)[1] >= np.array([m for _, m in pairs])).all()     # crossed
    # the float64 streams: every 16 kHz sample made final since S0
    audio, pos = eng.audio_history(f64)
    _, S1, st, xx, _ = eng.ctx.ingest_state(f64)
    fracs = {}
    for i, b in enumerate(f64):
        rate = int(rates[b])
        got = np.concatenate((audio[i, audio.shape[1] - pos[i]:], xx[i, :st[i]]))
        x_all = np.concatenate(fed[i])
        assert S1[i] == S0 + x_all.size
        h32, up, down = _native.resampler_taps(rate)
        if up == down:
            assert np.array_equal(got, x_all)
            fracs[rate] = 1.0
            continue
        r = ores.StreamResampler(rate, h=h32.astype(np.float64))
        r.S = S0
        r.hist[-128:] = h0[i]                                    # zeros before: each phase reads K <= 61 taps
        y64, s = r.feed(x_all, abs_sum=True)
        assert y64.size == ores.final_outputs(S0 + x_all.size, up, down) - ores.final_outputs(S0, up, down)
        fracs[rate] = judge_resampled(got, y64, s, up, down, h32.size)
    print(f"\n[ingest] {n_cmp} twin comparisons; judged fractions at S0 = 2^32 + 1: {fracs}")
    assert min(fracs.values()) >= 0.75


# ---- 5. refusals ---------------------------------------------------------------------------------------------------
def test_max_chunks_limit(torch_cuda):
    from openwakeword_b200 import _native
    limit = _native.MAX_CHUNKS
    with pytest.raises(_native.NativeError, match="max_chunks"):
        _native.Context(max_chunks=limit + 1)
    with pytest.raises(_native.NativeError, match="max_chunks"):
        _native.Context(max_chunks=2 ** 31 - 1)
    c = _native.Context(max_chunks=limit)
    c.close()
