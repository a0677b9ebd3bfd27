"""not-gpu: the bookkeeping of test_gpu_fused_schedules on the CPU stand-in of the library (fake_backend.FakeContext).

The same schedule generator drives a StreamEngine on the stand-in through the same holds, partial resets and
per-stream counts, and the same segment -> clip and row mapping takes the reference rows, here from the NumPy oracle
(oracle.streaming) run on each segment's clip at chunk size c*1280.  Both sides run the oracle's arithmetic, so any
difference is the harness's: a held stream that was fed, a reset in the wrong place, rows mapped to the wrong call."""
import numpy as np
import pytest

import fake_backend
from helpers import emb_weights
from oracle import embedding as oemb, heads as oheads, streaming as ostream
from openwakeword_b200 import _native
from openwakeword_b200.engine import StreamEngine
from test_gpu_fused_schedules import CHUNK, MAX_C, Schedule, compare, heads, run_schedule, segment_clips, signals


def oracle_reference(hs, fi, sched, clips):
    """{(stream, segment): (score rows, feature rows)}: each clip through a fresh OracleAudioFeatures at chunk size
    c*1280, every call's score row the per-head max over its c windows (a gated pair: gated score, then the verifier's
    raw one, as the engine lays out its columns)"""
    w = emb_weights()
    out = {}
    for k, x in clips.items():
        c = sched.c[k]
        af = ostream.OracleAudioFeatures(w, feature_init=fi)
        rows, feats = [], []
        for j in range(x.size // (c * CHUNK)):
            assert af(x[j * c * CHUNK:(j + 1) * c * CHUNK]) == c * CHUNK
            cols = []
            for h in hs:
                for net in ([h, h["verifier"]] if "verifier" in h else [h]):
                    win = [oheads.forward(net, af.get_features(h["n_in"], -h["n_in"] - i))[0] for i in range(c)]
                    cols.append(np.max(np.stack(win), axis=0))
            rows.append(np.concatenate(cols))
            feats.append(af.feature_buffer[-c:])
        out[k] = (np.stack(rows), np.concatenate(feats))
    return out


def test_schedule_bookkeeping_on_the_cpu_stand_in(monkeypatch):
    # the oracle CNN is the slow part and runs on the same windows on both sides: compute each window once
    memo = {}
    embed = oemb.embed_windows

    def embed_once(weights, windows, *a, **kw):
        key = (np.ascontiguousarray(windows).tobytes(), a, tuple(sorted(kw.items())))
        if key not in memo:
            memo[key] = embed(weights, windows, *a, **kw)
        return memo[key].copy()
    monkeypatch.setattr(ostream._emb, "embed_windows", embed_once)

    n, G, S = 10, 3, 2
    sched = Schedule(n, G, S, seed=5)
    rng = np.random.default_rng(5)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    sig = signals(rng, n, int(sched.counts.sum(0).max()) * CHUNK)
    hs = heads()
    monkeypatch.setattr(_native, "Context", fake_backend.FakeContext)
    eng = StreamEngine(hs, n, embedding=emb_weights(), feature_init=fi, max_chunks=MAX_C)
    got = run_schedule(eng, sched, sig, fi)
    ref = oracle_reference(hs, fi, sched, segment_clips(sched, sig))
    assert len(ref) > n and {sched.c[k] for k in ref} == {1, 2, 3}
    assert compare(sched, got, ref, 0.0) == (0.0, 0.0)
    print(f"{n} streams, {len(ref)} segments, calls (fused, general) = {sched.kinds()}, hold runs {len(sched.runs)}, "
          f"coverage {sched.coverage()}")

    # the harness notices a stream fed while it should be held, and a reset that is skipped
    for break_it in ("feed_held", "skip_reset"):
        bad = Schedule(n, G, S, seed=5)
        if break_it == "feed_held":
            b, t0, _ = bad.runs[len(bad.runs) // 2]
            eng_counts = bad.counts.copy()
            eng_counts[t0, b] = bad.c[(b, int(bad.seg[t0, b]))]
            bad.counts = eng_counts
        else:
            t = min(bad.resets)
            bad.resets = {k: v for k, v in bad.resets.items() if k != t}
        eng = StreamEngine(hs, n, embedding=emb_weights(), feature_init=fi, max_chunks=MAX_C)
        got = run_schedule(eng, bad, sig, fi)
        with pytest.raises(AssertionError):
            compare(sched, got, ref, 0.0)
