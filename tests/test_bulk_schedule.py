"""not-gpu: the call schedule and the slab plan of the ragged bulk clip path (oww_clip_schedule, oww_clip_slab_plan;
pure host code in libowwb200) and the argument errors of oww_predict_clips_ragged.

The schedule is checked against a literal replay of the reference's AudioFeatures._streaming_features accumulation
(openwakeword/utils.py:409-452): remainder kept for the next call, melspectrogram and embeddings once the accumulated
samples are a non-zero multiple of 1280."""
import ctypes as C

import numpy as np
import pytest

from openwakeword_b200 import _native

OWW_EINVAL = -1


def replay(chunk_size, n_padded):
    """chunks stepped by each predict call of predict_clip(chunk_size) on n_padded samples, as the reference counts them"""
    acc, rem, out = 0, 0, []
    for _ in range(0, n_padded - chunk_size, chunk_size):
        x = rem + chunk_size
        rem = 0
        if acc + x >= 1280:
            r = (acc + x) % 1280
            acc += x - r
            rem = r
        else:
            acc += x
        if acc >= 1280 and acc % 1280 == 0:
            out.append(acc // 1280)
            acc = 0
        else:
            out.append(0)
    return out


def test_schedule_matches_streaming_replay(built_library):
    rng = np.random.default_rng(0)
    chunks = list(range(1, 3001)) + [3840, 4000, 5120, 7777, 10240]
    for c in chunks:
        for pad in (0, 1, 2):
            # lengths 0 .. 5 s: the edges around one and two calls, and a few seeded ones
            lens = {0, 1, c - 1, c, c + 1, 2 * c, 80000} | set(rng.integers(0, 80001, 3).tolist())
            for n in sorted(x for x in lens if 0 <= x <= 80000):
                L = n + 2 * 16000 * pad
                got = _native.clip_schedule(c, L)
                assert got.tolist() == replay(c, L), (c, pad, n)


def test_schedule_counts_and_errors(built_library):
    assert built_library.oww_clip_schedule(1280, 1280, None, 0) == 0
    assert built_library.oww_clip_schedule(1280, 1281, None, 0) == 1
    assert built_library.oww_clip_schedule(0, 5000, None, 0) == OWW_EINVAL
    assert built_library.oww_clip_schedule(400, -1, None, 0) == OWW_EINVAL
    buf = (C.c_int32 * 4)(*([-7] * 4))
    assert built_library.oww_clip_schedule(400, 16000, buf, 2) == 39     # writes only the first `max` counts
    assert list(buf) == [0, 0, -7, -7]


def test_slab_plan_overhead_on_mixed_lengths(built_library):
    """20 000 seeded lengths uniform over 0.5-4 s (1 s padding, 1280-sample calls): at most 10 % more steps computed
    than needed, and far fewer slabs than clips."""
    rng = np.random.default_rng(1)
    lens = rng.integers(8000, 64001, 20000)
    steps = np.array([_native.clip_schedule(1280, int(n) + 32000).sum() for n in lens], np.int32)
    n_slabs, done, need = _native.clip_slab_plan(steps)
    print(f"{n_slabs} slabs, {done} steps computed for {need} needed ({done / need - 1:.2%} padding)")
    assert need == int(steps.sum())
    assert need <= done <= 1.10 * need
    assert n_slabs < 200


def test_slab_plan_equal_lengths_and_zero_steps(built_library):
    n_slabs, done, need = _native.clip_slab_plan(np.full(1000, 31, np.int32))
    assert (done, need) == (31000, 31000) and n_slabs >= 1
    assert _native.clip_slab_plan(np.zeros(5, np.int32)) == (0, 0, 0)


def test_ragged_argument_errors(built_library):
    """oww_predict_clips_ragged validates its arguments before it touches the device (a NULL handle cannot get past
    the null check, so the checks run on a handle-less call only up to there; the geometry checks are exercised on a
    GPU handle in tests/test_gpu_bulk_ragged.py)."""
    off = np.array([0, 10], np.int64)
    rc = built_library.oww_predict_clips_ragged(None, None, off.ctypes.data, 1, 0, 1280, None, 0, None, None, None, None)
    assert rc == OWW_EINVAL
