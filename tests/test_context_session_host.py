"""not-gpu: the comparator of test_gpu_context_session on the CPU.  The session runs twice on the stand-in of the library
(fake_backend.FakeContext) and must pass; then one side is a stand-in with one planted divergence from the header's
rules, and the comparator must fail for each."""
import numpy as np
import pytest

import fake_backend
from test_gpu_context_session import (MAX_C, Judge, Mismatch, Recorder, Session, check_coverage, memo_embedding,
                                      public_names)


class GateAfterMax(fake_backend.FakeContext):
    """the gate applied to the max over the chunk windows instead of to every window"""

    def _gated(self, raw):
        return super()._gated(raw.max(axis=0, keepdims=True))


class VerifierAbove(fake_backend.FakeContext):
    """the verifier threshold compared with > instead of >="""

    @staticmethod
    def _verified(cols, thr):
        return cols > thr


class ResetKeepsPosition(fake_backend.FakeContext):
    """reset leaves the audio position"""

    def reset(self, stream_ids=None, feature_init=None):
        ids = self._ids(stream_ids)
        pos = self.pos[ids].copy()
        super().reset(stream_ids, feature_init)
        self.pos[ids] = pos


class BankColumnsSwapped(fake_backend.FakeContext):
    def _bank_scores(self, b, hb, chunks):
        return super()._bank_scores(b, hb, chunks)[::-1].copy()


class HeldRowsZeroed(fake_backend.FakeContext):
    def step_host_ragged(self, pcm, chunks, scores_out):
        super().step_host_ragged(pcm, chunks, scores_out)
        scores_out[np.asarray(chunks) == 0] = 0.0


class HistoryKeptOnNewColumns(fake_backend.FakeContext):
    """set_detector with other columns keeps the histories"""

    def set_detector(self, labels, debounce_time=0.0):
        old = self.det
        super().set_detector(labels, debounce_time)
        if old and len(old[0].labels) == len(labels):
            for d, o in zip(self.det, old):
                d.history, d.count = o.history, o.count


PLANTED = [GateAfterMax, VerifierAbove, ResetKeepsPosition, BankColumnsSwapped, HeldRowsZeroed, HistoryKeptOnNewColumns]


@pytest.fixture(scope="module")
def reference():
    """the stand-in's session log (the embedding memo stays in place for the module)"""
    with pytest.MonkeyPatch.context() as mp:
        memo_embedding(mp)
        rec = Recorder(fake_backend.FakeContext(max_chunks=MAX_C))
        yield Session().run(rec), rec.called


def test_two_stand_ins_agree(reference):
    log, called = reference
    rec = Recorder(fake_backend.FakeContext(max_chunks=MAX_C))
    j = Judge()
    Session().run(rec, ref=log, judge=j)
    print(j.report("stand-in vs stand-in"))
    assert j.worst == dict(score=0.0, feature=0.0, mel=0.0) and j.ties == 0 and j.audio_lsb == 0
    assert j.judged > 0
    check_coverage(called)
    check_coverage(rec.called)


def test_coverage_guard_notices_a_missing_call(reference):
    _, called = reference
    for name in sorted(public_names())[::7]:
        with pytest.raises(AssertionError, match=name):
            check_coverage(set(called) - {name})


@pytest.mark.parametrize("planted", PLANTED, ids=[c.__name__ for c in PLANTED])
def test_the_comparator_catches(reference, planted):
    log, _ = reference
    with pytest.raises(Mismatch) as e:
        Session().run(Recorder(planted(max_chunks=MAX_C)), ref=log, judge=Judge())
    print(f"{planted.__name__}: {e.value}")


def test_cnn_mode_0_refuses_head_banks():
    """the library refuses head banks in cnn_mode 0; so does the stand-in, and the session runs without them"""
    with pytest.MonkeyPatch.context() as mp:
        memo_embedding(mp)
        ctx = fake_backend.FakeContext(max_chunks=MAX_C, cnn_mode=0)
        rec = Recorder(ctx)
        Session(bank=False, seed=1).run(rec)
        assert not ctx.hbanks
