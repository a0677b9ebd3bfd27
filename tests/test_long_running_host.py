"""The counter rules of long-running streams on the host, and the twin comparators of the GPU test.

* The ring rebase (OWW_COUNT_REBASE, oww_internal.h) keeps the slot count & (rows - 1) for every ring size a handle can
  have (2^7 .. 2^20 rows, max_chunks up to OWW_MAX_CHUNKS) and leaves the count >= the ring size; a count imported at
  any value below 2^31 is rebased so that no step overflows int.
* The detector rebase (DET_COUNT_REBASE, detect.cu) keeps count % 30, min(count, 30) and count < 5.
* Wrapping per chunk and per call give the same count; the event index is the count before the append in the frame
  after the call's rebase.
* The constants restated in tests/helpers.py are the library's, and the library refuses max_chunks above
  OWW_MAX_CHUNKS before it looks for a device.
* record_diff and events_diff accept a real twin pair (two stream records exported from a handle in which the twin
  crossed 2^30 mel rows) and fail on planted divergences: a feature row shifted by one slot, a count off by one, an
  unrebased count, an event index reported before the rebase."""
import os
import re

import numpy as np
import pytest

from helpers import (COUNT_REBASE, COUNT_WRAP, DET_REBASE, GOLDEN, REC_COUNT_WORDS, det_count, det_imported,
                     event_index, events_diff, imported_count, record_diff, record_words, ring_count)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "openwakeword_b200", "csrc")


def _define(path, name):
    src = open(path).read()
    m = re.search(rf"#define {name} (.+)", src)
    assert m, name
    return int(eval(m.group(1).split("/*")[0].split("//")[0]))


def _next_pow2(v):
    p = 1
    while p < v:
        p <<= 1
    return p


def test_constants_are_the_library_s():
    from openwakeword_b200 import _native
    assert _define(os.path.join(CSRC, "oww_internal.h"), "OWW_COUNT_WRAP") == COUNT_WRAP
    assert _define(os.path.join(CSRC, "oww_internal.h"), "OWW_COUNT_REBASE") == COUNT_REBASE
    assert _define(os.path.join(CSRC, "detect.cu"), "DET_COUNT_REBASE") == DET_REBASE
    limit = _define(os.path.join(ROOT, "include", "owwb200.h"), "OWW_MAX_CHUNKS")
    assert limit == _native.MAX_CHUNKS
    # the largest max_chunks whose mel ring (next_pow2(76 + 8 mc), api.cu) stays within 2^20 rows
    assert _next_pow2(76 + 8 * limit) == 1 << 20 and _next_pow2(76 + 8 * (limit + 1)) == 1 << 21
    assert _next_pow2(120 + limit) <= 1 << 20
    assert limit * 1280 < 2 ** 31


RING_SIZES = [1 << k for k in range(7, 21)]


def test_ring_rebase_keeps_every_slot():
    assert COUNT_REBASE % RING_SIZES[-1] == 0
    rng = np.random.default_rng(0)
    max_add = 8 * 131062
    c = np.concatenate([COUNT_WRAP - np.arange(1, 4096), COUNT_WRAP - rng.integers(1, max_add, 4096)]).astype(np.int64)
    add = np.concatenate([np.arange(1, 4096) + rng.integers(0, 64, 4095), rng.integers(1, max_add + 1, 4096)])
    for ci, ai in zip(c.tolist(), add.tolist()):
        w = ring_count(ci, ai)
        assert w >= 1 << 20                                      # >= every ring size, and far above 120 and 76
        for R in RING_SIZES:
            assert (w & (R - 1)) == ((ci + ai) & (R - 1))
    # below the wrap nothing changes; the rebased count never reaches the wrap again within one step
    assert ring_count(COUNT_WRAP - 9, 8) == COUNT_WRAP - 1
    assert ring_count(COUNT_WRAP - 1, 1) == 1 << 20
    assert ring_count(COUNT_WRAP - 1, max_add) + max_add < COUNT_WRAP


def test_imported_counts_never_overflow():
    max_add = 8 * 131062
    for c in [COUNT_WRAP, COUNT_WRAP + 5, 2 ** 31 - max_add - 1, 2 ** 31 - 8 * 3, 2 ** 31 - 1]:
        w = imported_count(c)
        assert 1 << 20 <= w and w + max_add < 2 ** 31
        assert w % (1 << 20) == c % (1 << 20)
        assert ring_count(w, max_add) < COUNT_WRAP                # the next step lands below 2^30
    assert imported_count(COUNT_WRAP - 1) == COUNT_WRAP - 1
    assert imported_count(2 ** 31 - 1) == 2 ** 30 + 2 ** 20 - 1


def test_detector_rebase_keeps_the_rule_inputs():
    assert DET_REBASE % 30 == 0 and DET_REBASE <= COUNT_WRAP - 30
    for c in list(range(COUNT_WRAP - 200, COUNT_WRAP)) + [2 ** 31 - 2]:
        w = det_count(c)
        assert w % 30 == (c + 1) % 30 and min(w, 30) == min(c + 1, 30) and (w < 5) == (c + 1 < 5)
    for c in [COUNT_WRAP, 2 ** 31 - 1]:
        w = det_imported(c)
        assert w % 30 == c % 30 and w >= 30 and det_count(w) < COUNT_WRAP
    assert det_imported(-5) == 0


@pytest.mark.parametrize("mc", [1, 2, 3, 8, 131062])
def test_where_the_wrap_fires_does_not_matter(mc):
    """a call of n chunks wraps once on its total (the fused and ragged paths) or per chunk (a path that appends chunk by
    chunk): the same count, for mel (8 rows per chunk) and feature (1 row) rings"""
    rng = np.random.default_rng(mc)
    for per in (8, 1):
        for start in range(COUNT_WRAP - 3 * per * min(mc, 4), COUNT_WRAP + 1):
            c_call = c_chunk = start if start < COUNT_WRAP else imported_count(start)
            for _ in range(6):
                n = int(rng.integers(0, min(mc, 4) + 1))
                c_call = ring_count(c_call, per * n)
                for _ in range(n):
                    c_chunk = ring_count(c_chunk, per)
                assert c_call == c_chunk, (per, start)


def test_event_index_rule():
    """index = the count before the append, in the count's frame after this call's rebase: 63 on the call that reaches
    2^30, the plain count before it, and the same residue mod 30 as the count before the append"""
    assert event_index(COUNT_WRAP - 2) == COUNT_WRAP - 2
    assert event_index(COUNT_WRAP - 1) == 63 == COUNT_WRAP - 1 - DET_REBASE
    assert event_index(0) == 0 and event_index(29) == 29
    for c in range(COUNT_WRAP - 100, COUNT_WRAP):
        assert event_index(c) % 30 == c % 30
        assert event_index(c) == det_count(c) - 1


def test_max_chunks_is_refused_before_the_device(built_library):
    """above the limit oww_create fails on max_chunks whatever the machine; at the limit it gets past that check"""
    from openwakeword_b200 import _native
    with pytest.raises(_native.NativeError, match="max_chunks"):
        _native.Context(max_chunks=_native.MAX_CHUNKS + 1)
    with pytest.raises(_native.NativeError, match="max_chunks"):
        _native.Context(max_chunks=2 ** 31 - 1)
    try:
        _native.Context(max_chunks=_native.MAX_CHUNKS).close()
    except _native.NativeError as e:                            # no GPU here: refused for that, not for max_chunks
        assert "max_chunks" not in str(e)


# ---- the comparators on real records ----
def _pair():
    z = np.load(os.path.join(GOLDEN, "long_running_records.npz"))
    return z["ctrl"], z["twin"], tuple(int(v) for v in z["twin_counts"]), tuple(int(v) for v in z["twin_before"])


def test_real_twin_pair_holds():
    ctrl, twin, counts, before = _pair()
    assert before[0] < COUNT_WRAP <= before[0] + 8 and counts[0] == ring_count(before[0], 8)
    assert not record_diff(ctrl, twin, counts)
    assert record_diff(ctrl, twin, before)                      # the count before the step is not the twin's count


REC_FEAT = 670 * 16                                             # byte offset of the 120 feature rows (api.cu layout)


def test_comparator_fails_on_a_shifted_feature_row():
    ctrl, twin, counts, _ = _pair()
    t = twin.copy()
    rows = t[REC_FEAT:REC_FEAT + 120 * 384].reshape(120, 384)
    assert not np.array_equal(rows[-1], rows[-2])
    rows[:] = np.roll(rows, 1, axis=0)                          # every row one slot late
    assert any("words differ" in m for m in record_diff(ctrl, t, counts))
    t = twin.copy()
    t[REC_FEAT + 119 * 384:REC_FEAT + 120 * 384] = twin[REC_FEAT + 118 * 384:REC_FEAT + 119 * 384]   # newest = previous
    assert record_diff(ctrl, t, counts)


@pytest.mark.parametrize("word", REC_COUNT_WORDS)
def test_comparator_fails_on_a_count_off_by_one(word):
    ctrl, twin, counts, _ = _pair()
    for d in (-1, 1):
        t = twin.copy()
        record_words(t)[word] += d
        assert any("counts" in m for m in record_diff(ctrl, t, counts))
    t = ctrl.copy()                                             # nor may the control's other words carry a count
    record_words(t)[REC_COUNT_WORDS[0] - 1] += 1                # seen
    assert any("words differ" in m for m in record_diff(ctrl, t, (int(record_words(t)[5]), int(record_words(t)[6]))))


def test_comparator_fails_on_an_unrebased_count():
    ctrl, twin, counts, before = _pair()
    t = twin.copy()
    record_words(t)[REC_COUNT_WORDS[0]] = before[0] + 8         # c + added without the rebase
    assert record_diff(ctrl, t, counts)
    assert not record_diff(ctrl, t, (before[0] + 8, counts[1]))  # ... which a rule without the rebase would accept


def test_events_comparator_fails_on_an_index_before_the_rebase():
    from openwakeword_b200._native import EVENT_DTYPE
    ev = np.zeros(4, EVENT_DTYPE)
    ev["stream"], ev["label"], ev["score"] = [0, 0, 2, 2], [0, 3, 0, 3], [0.5, 0.75, 0.5, 0.75]
    before = {0: 100, 2: COUNT_WRAP - 1}                         # control 0 at 100 predictions, its twin 2 at 2^30 - 1
    index_of = {b: event_index(c) for b, c in before.items()}
    ev["index"] = [index_of[0], index_of[0], index_of[2], index_of[2]]
    assert not events_diff(ev, ev, {0: 2}, index_of)
    bad = ev.copy()
    bad["index"][2:] = COUNT_WRAP - 1                           # the count before the append, before the rebase
    assert events_diff(bad, bad, {0: 2}, index_of)
    bad = ev.copy()
    bad["score"][3] = np.nextafter(np.float32(0.75), np.float32(1))
    assert events_diff(bad, bad, {0: 2}, index_of)
    assert events_diff(ev[:3], ev[:3], {0: 2}, index_of)          # a twin event missing
