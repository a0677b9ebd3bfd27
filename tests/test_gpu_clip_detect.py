"""-m gpu: detections on the bulk clip path (oww_detect_clips, csrc/detect.cu).

* The kernel against the clip restatement (tests/clip_detect_ref.py) on random raw rows, bit for bit: up to 10 000 clips,
  up to 40 labels, every chunk size of the host tests (the engine's max_chunks * 1280 among them), thresholds of 0 and NaN, verifier rows at
  verifier thresholds 0 and 0.5, the final rows and every event field.
* End to end: predict_clips(..., patience / threshold / debounce_time) against the host loop predict_clip(**kw) after
  reset, with a verifier bank (at verifier thresholds 0.05 and 0, where re-verifying a repeat is not idempotent), stream
  models with stream verifiers through streams=, and clips at 48 kHz; detect_clips against the thresholded rows.
* N = 0, the refusals (nothing enqueued), and the launches of a plain predict_clips call."""
import numpy as np
import pytest

from clip_detect_ref import detect_clips as ref_detect_clips
from helpers import emb_weights, head
from oracle import detect as odet
from test_gpu_bulk_ragged import _rows, _signal, _verified_model
from test_gpu_detect import _edge_scores, _engine

pytestmark = pytest.mark.gpu
NAN = float("nan")


@pytest.fixture(scope="module")
def torch_cuda(built_library):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _table(rng, L, n_cols, mode):
    rows = []
    for j in range(L):
        thr = [0.5, 0.25, 0.0, None][int(rng.integers(0, 4))] if j else 0.5
        pat = [0, 1, 2, 5, 30][int(rng.integers(0, 5))] if mode == "patience" and thr is not None else 0
        rows.append((int(rng.integers(-1, n_cols)) if j else 0, bool(rng.integers(0, 2)) if j else True, thr, pat))
    return rows


def _events_of(final, row_off, table):
    """the event list of the final rows: (clip, label, score, call) in ascending (clip, label, call) order"""
    thr = np.array([NAN if t[2] is None else t[2] for t in table], np.float32)
    r, j = np.nonzero(final >= thr[None, :])
    clip = np.searchsorted(row_off, r, side="right") - 1
    o = np.lexsort((r, j, clip))
    return clip[o], j[o], final[r[o], j[o]], (r - row_off[clip])[o]


CHUNKS = [1, 400, 1024, 1280, 2000, 2560, 3840]          # 2560: max_chunks * 1280 of test_gpu_detect's engine


@pytest.mark.parametrize("vthr", [0.5, 0.0])
@pytest.mark.parametrize("L", [1, 11, 40])
@pytest.mark.parametrize("chunk", CHUNKS)
def test_kernel_equals_the_restatement(torch_cuda, chunk, L, vthr):
    torch = torch_cuda
    case = CHUNKS.index(chunk) * 6 + [1, 11, 40].index(L) * 2 + int(vthr == 0.0)
    rng = np.random.default_rng(case)
    mode = ["none", "patience", "debounce"][case % 3]
    debounce = 1.25 if mode == "debounce" else 0.0
    eng = _engine(1)
    ctx, n_cols = eng.ctx, eng.n_cols
    table = _table(rng, L, n_cols, mode)
    # clips of 0 to 60 s (calls capped at 2000 below 400 samples per call); 10 000 of them at L = 11
    n_clips = 10000 if L == 11 else 1500
    max_calls = min(60 * 16000 // chunk, 2000)
    calls = rng.integers(0, max_calls + 1, n_clips)
    calls[:4] = [0, 1, 5, max_calls]
    row_off = np.concatenate([[0], np.cumsum(calls)]).astype(np.int64)
    rows = int(row_off[-1])
    raw = _edge_scores(rng, (rows, n_cols))
    ver = rng.uniform(0, 1, (rows, L)).astype(np.float32)
    ver[:, rng.random(L) < 0.3] = NAN                      # labels without a verifier
    d_raw, d_ver = torch.from_numpy(raw).cuda(), torch.from_numpy(ver).cuda()
    d_final = torch.full((rows, L), -7.0, dtype=torch.float32, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int32, device="cuda")
    ctx.detect_clips(table, debounce, d_raw, d_ver, vthr, row_off, chunk, None, None, 0, d_n)      # the count only
    cap = int(d_n.item())
    d_ev = torch.empty((max(cap, 1), 4), dtype=torch.int32, device="cuda")
    ctx.detect_clips(table, debounce, d_raw, d_ver, vthr, row_off, chunk, d_final, d_ev, cap, d_n)
    final = d_final.cpu().numpy()
    n = int(d_n.item())
    ev = d_ev[:n].cpu().numpy().view(np.dtype([("stream", "<i4"), ("label", "<i4"), ("score", "<f4"),
                                                          ("index", "<i4")])).reshape(-1)
    # every clip: the events are the thresholded final rows, in order
    ec, ej, es, ei = _events_of(final, row_off, table)
    assert n == ec.size == cap
    assert (ev["stream"] == ec).all() and (ev["label"] == ej).all() and (ev["index"] == ei).all()
    assert (_bits(ev["score"]) == _bits(es)).all()
    # a sample of clips (the first, CTA edges, random): the final rows bit for bit against the restatement
    S = 256 // L
    watch = np.unique(np.concatenate([[0, 1, 2, 3, n_clips - 1, S - 1, S, 2 * S], rng.integers(0, n_clips, 12)]))
    watch = watch[watch < n_clips]
    labels = [odet.Label(*r) for r in table]
    for c in watch:
        a, b = int(row_off[c]), int(row_off[c + 1])
        want, _ = ref_detect_clips(labels, debounce, raw[a:b], np.array([0, b - a]), chunk, ver[a:b], np.float32(vthr))
        assert (_bits(final[a:b]) == _bits(want)).all(), (c, chunk, L)
    print(f"chunk {chunk} L {L} vthr {vthr} {mode}: {n_clips} clips, {rows} rows, {n} events")


def _thresholds_away(scores, names_of_cols, candidates, gap=1e-5):
    """per model the first candidate at least `gap` from every score of its labels, so that no comparison can flip"""
    out = {}
    for mdl, cols in names_of_cols.items():
        s = scores[:, cols].ravel()
        out[mdl] = next(t for t in candidates if s.size == 0 or np.abs(s - t).min() >= gap)
    return out


def _label_cols(m):
    labels = m.labels()
    cols = {}
    for j, lab in enumerate(labels):
        cols.setdefault(m.get_parent_model_from_label(lab), []).append(j)
    return cols


def _check_against_host_loop(m, clips, chunk, kw, **call):
    labels = m.labels()
    bulk = m.predict_clips(clips, padding=1, chunk_size=chunk, **call, **kw)
    for i, clip in enumerate(clips):
        m.reset()
        ref = _rows(m.predict_clip(clip, padding=1, chunk_size=chunk, sr=call.get("sr"), **kw), labels)
        got = _rows(bulk[i], labels)
        assert got.shape == ref.shape
        if ref.size:
            assert np.abs(got - ref).max() < 2e-6, (chunk, kw, i, np.abs(got - ref).max())
    return bulk


@pytest.mark.parametrize("vthr", [0.05, 0.0])
def test_predict_clips_kwargs_equal_the_host_loop(torch_cuda, vthr):
    m = _verified_model(3, vthr)
    labels = m.labels()
    rng = np.random.default_rng(31)
    clips = [_signal(rng, n) for n in (0, 300, 9000, 23456, 40000)]
    for chunk in (400, 1280, 2000):
        plain = np.concatenate([_rows(r, labels) for r in m.predict_clips(clips, padding=1, chunk_size=chunk)])
        thr = _thresholds_away(plain, _label_cols(m), [0.5, 0.3, 0.2, 0.1, 0.05, 0.02, 0.7, 0.9])
        for kw in (dict(threshold=thr, debounce_time=1.25), dict(threshold=thr, debounce_time=0.25),
                   dict(threshold=thr, patience={n: 3 for n in thr}), dict(threshold=thr)):
            bulk = _check_against_host_loop(m, clips, chunk, kw)
            events = m.detect_clips(clips, thr, patience=kw.get("patience", {}),
                                    debounce_time=kw.get("debounce_time", 0.0), padding=1, chunk_size=chunk)
            want = [(i, lab, j, r[lab]) for i, clip_rows in enumerate(bulk) for lab in labels
                    for j, r in enumerate(clip_rows) if r[lab] >= np.float32(thr[m.get_parent_model_from_label(lab)])]
            assert events == want, (chunk, kw)


def test_stream_models_and_verifiers_through_streams(torch_cuda):
    from openwakeword_b200 import Model
    from test_gpu_stream_verifiers import _cands, _setup
    rng = np.random.default_rng(41)
    B = 12
    cands, vers, fi = _cands(), _setup()[6], _setup()[7]
    sm = {b: cands[b % 3] for b in range(B) if b % 4 != 3}
    sv = {b: vers[b % 4] for b in range(B) if b % 5 != 4}
    m = Model(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")}], embedding_model_path=emb_weights(),
              feature_init=fi, n_streams=B, max_chunks=3, stream_models={"mine": sm}, stream_verifiers={"mine": sv},
              custom_verifier_threshold=0.0)
    clips = list(np.clip(rng.normal(0, 5000, (B, 30000)), -32768, 32767).astype(np.int16))
    streams = np.arange(B)
    labels = m.labels()
    for chunk in (640, 2000):
        plain = m.predict_clips(clips, padding=1, chunk_size=chunk, streams=streams)
        thr = _thresholds_away(np.concatenate([_rows(r, labels) for r in plain]), _label_cols(m), [0.5, 0.3, 0.7, 0.1])
        for kw in (dict(threshold=thr, debounce_time=1.25), dict(threshold=thr, patience={n: 2 for n in thr})):
            bulk = m.predict_clips(clips, padding=1, chunk_size=chunk, streams=streams, **kw)
            m.reset(fi)
            data = np.concatenate([np.zeros((B, 16000), np.int16), np.stack(clips), np.zeros((B, 16000), np.int16)], 1)
            for j, i in enumerate(range(0, data.shape[1] - chunk, chunk)):
                r = m.predict(data[:, i:i + chunk], **kw)
                for b in range(B):
                    for lab in labels:
                        assert abs(bulk[b][j][lab] - r[lab][b]) < 2e-6, (chunk, kw, j, b, lab)


def test_clips_at_48k(torch_cuda):
    m = _verified_model(3)
    labels = m.labels()
    rng = np.random.default_rng(51)
    clips = [_signal(rng, n) for n in (3000, 30000, 70001, 96000)]
    for chunk in (1024, 1280):
        plain = np.concatenate([_rows(r, labels) for r in m.predict_clips(clips, padding=1, chunk_size=chunk, sr=48000)])
        thr = _thresholds_away(plain, _label_cols(m), [0.5, 0.3, 0.2, 0.1, 0.7])
        _check_against_host_loop(m, clips, chunk, dict(threshold=thr, debounce_time=1.25), sr=48000)


def test_empty_batches_refusals_and_launches(torch_cuda):
    torch = torch_cuda
    from openwakeword_b200 import _native
    m = _verified_model(3)
    ctx = m.preprocessor.ctx
    kw = dict(threshold={"alexa_v0.1": 0.5}, debounce_time=1.25)
    assert m.predict_clips([], **kw) == [] and m.detect_clips([], 0.5) == []
    scores, row_off, labels = m.predict_clips_ragged(np.zeros(0, np.int16), [0], **kw)
    assert scores.shape == (0, len(labels)) and row_off.tolist() == [0]
    d_n = torch.full((1,), 7, dtype=torch.int32, device="cuda")
    table = [(0, True, 0.5, 0)]
    ctx.detect_clips(table, 0.0, None, None, 0.5, [0], 1280, None, None, 0, d_n)
    assert int(d_n.item()) == 0
    # refusals: nothing enqueued
    raw = torch.zeros((10, ctx.n_outputs), dtype=torch.float32, device="cuda")
    fin = torch.zeros((10, 1), dtype=torch.float32, device="cuda")
    l0 = ctx.launch_count
    bad = [dict(labels=[]), dict(labels=[(ctx.n_outputs, True, 0.5, 0)]), dict(labels=[(0, True, None, 2)]),
           dict(labels=[(0, True, 0.5, 2)], debounce=1.0), dict(labels=[(0, True, 0.5, 31)]), dict(off=[1, 10]),
           dict(off=[0, 6, 4, 10]), dict(chunk=0), dict(final=None), dict(debounce=-1.0), dict(scores=None)]
    for b in bad:
        with pytest.raises(_native.NativeError):
            ctx.detect_clips(b.get("labels", table), b.get("debounce", 0.0), b.get("scores", raw), None, 0.5,
                             b.get("off", [0, 4, 10]), b.get("chunk", 1280), b.get("final", fin), None, 0, None)
    with pytest.raises(ValueError, match="at least one model"):
        type(m).detect_clips.__get__(_NoLabels(m))([np.zeros(100, np.int16)], 0.5)
    assert ctx.launch_count == l0
    # a plain predict_clips call: the clip call's launches plus one detect_clips launch
    rng = np.random.default_rng(61)
    clips = [_signal(rng, n) for n in (9000, 23456, 40000)]
    for chunk in (1280, 400):
        m.predict_clips(clips, padding=1, chunk_size=chunk)             # warm
        l0 = ctx.launch_count
        m.predict_clips(clips, padding=1, chunk_size=chunk)
        whole = ctx.launch_count - l0
        l0 = ctx.launch_count
        m._clip_call(*_concat(clips), 1, chunk, None, None, True)
        device = ctx.launch_count - l0
        print(f"chunk {chunk}: a plain predict_clips call takes {whole} launches; the clip call and the verifier rows "
              f"take {device}, oww_detect_clips 1")
        assert whole == device + 1


def _concat(clips):
    from openwakeword_b200.model import _concat_clips
    return _concat_clips(clips)


class _NoLabels:
    """a Model view without models, for the refusal of detect_clips"""

    def __init__(self, m):
        self._m = m

    def labels(self):
        return []

    def __getattr__(self, name):
        return getattr(self._m, name)
