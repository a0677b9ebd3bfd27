"""-m gpu: the ragged bulk clip path (oww_predict_clips_ragged): clips of mixed lengths in one device call, any
chunk_size, bulk_predict on WAV files of all-distinct lengths, and bulk_predict with _get_positive_prediction_frames.

* Ragged equals equal-length bit for bit: every clip of a mixed batch (a 0-call clip, a 1-step clip, lengths on both
  sides of the 5 % slab split and of the grouped heads' 128-clip tiles, one clip longer than one 8192-step frontend
  segment) against the same clip alone through oww_predict_clips.  Clips share slabs with longer ones and run on over
  virtual zeros there, so this also pins the prefix property.
* Every chunk size against streaming: Model.predict_clips(list, chunk_size=c) against a fresh-stream predict_clip.
* The golden predict_clip cases at their own chunk sizes, through the bulk path.
* bulk_predict: one device call per batch of files, kwargs routed or dropped, and the positive-frame miner."""
import os
import wave

import numpy as np
import pytest

from helpers import (GOLDEN, VERIFIER_CASES, case_model as _model, class_mapping, emb_weights, golden_cases, head,
                     load_case)
from test_gpu_parity import SCORE_TOL, _gated_error

pytestmark = pytest.mark.gpu

CHUNK = 1280
NAMES = ["alexa_v0.1", "timer_v0.1", "hey_jarvis_v0.1"]          # binary, 7-class and gated heads


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _signal(rng, n):
    """noise at a random level with a few louder bursts, so scores move and the per-call clamp matters"""
    x = rng.normal(0, rng.uniform(200, 4000), n)
    for _ in range(max(1, n // 20000)):
        a = int(rng.integers(0, max(1, n - 4000)))
        x[a:a + 4000] += rng.normal(0, 9000, min(4000, n - a))
    return np.clip(x, -32768, 32767).astype(np.int16)


def _specs():
    return [{"name": n, "head": head(n), "class_mapping": class_mapping([n]).get(n)} for n in NAMES]


def _engine(mode, max_chunks=8):
    """handle with the three heads and a custom verifier bank on the binary head (clip slot 1; slot 0 is a decoy)"""
    from openwakeword_b200.engine import StreamEngine
    eng = StreamEngine([head(n) for n in NAMES], 1, embedding=emb_weights(), max_chunks=max_chunks, cnn_mode=mode)
    rng = np.random.default_rng(5)
    D = 16 * 96
    bank = eng.add_verifier_bank(0, 2, 0.05)
    mean, weight = rng.normal(0, 1, D).astype(np.float32), rng.normal(0, 0.03, D).astype(np.float32)
    eng.load_verifier(bank, 0, (mean + 1, -weight, -3.0))
    eng.load_verifier(bank, 1, (mean, weight, 0.2))
    eng.ctx.set_verifier_clip_slot(bank, 1)
    return eng


@pytest.mark.parametrize("mode", [0, 2, 3])
def test_ragged_equals_equal_length_bit_for_bit(torch_cuda, built_library, mode):
    torch = torch_cuda
    from openwakeword_b200 import _native
    rng = np.random.default_rng(mode)
    lens = [0, 1000, 2000, 1280 * 8201 + 77]                          # 0 calls, 0 calls, 1 step, > one 8192-step segment
    lens += [1280 * 41 + int(x) for x in rng.integers(1, 1280, 131)]  # 40 steps: 131 clips, past one 128-clip tile
    lens += [1280 * 39 + 5, 1280 * 38 + 9, 1280 * 37 + 700, 1280 * 31 + 1]   # within 5 % of 40 steps, and beyond it
    lens = [lens[i] for i in rng.permutation(len(lens))]
    clips = [_signal(rng, n) for n in lens]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    eng = _engine(mode)
    pcm = np.concatenate(clips)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    steps = [len(range(0, n - CHUNK, CHUNK)) for n in lens]
    rows = sum(steps)
    d = torch.from_numpy(pcm).cuda()
    got = torch.full((rows, eng.n_cols), np.nan, dtype=torch.float32, device="cuda")
    stepped = torch.zeros(rows, dtype=torch.uint8, device="cuda")
    l0 = eng.ctx.launch_count
    eng.ctx.predict_clips_ragged(d, off, 0, CHUNK, fi, got, stepped)
    torch.cuda.synchronize()
    print(f"mode {mode}: {len(lens)} clips, {rows} rows, {eng.ctx.launch_count - l0} launches")
    got = got.cpu().numpy()
    assert stepped.cpu().numpy().all()
    r0 = 0
    for i, n in enumerate(lens):
        if steps[i]:
            one = torch.full((steps[i], eng.n_cols), np.nan, dtype=torch.float32, device="cuda")
            eng.ctx.predict_clips(torch.from_numpy(clips[i]).cuda(), 1, n, 0, fi, one)
            ref = one.cpu().numpy()
            assert np.array_equal(ref, got[r0:r0 + steps[i]]), (i, n, np.abs(ref - got[r0:r0 + steps[i]]).max())
        r0 += steps[i]
    # argument errors
    with pytest.raises(_native.NativeError, match="monotone"):
        eng.ctx.predict_clips_ragged(d, np.array([0, 5000, 4000], np.int64), 0, CHUNK, fi, got, stepped)
    for bad in (0, 8 * CHUNK + 1):
        with pytest.raises(_native.NativeError, match="chunk_size"):
            eng.ctx.predict_clips_ragged(d, off[:3], 0, bad, fi, got, stepped)


def _verified_model(mode, thr=0.05):
    import openwakeword_b200 as owb
    fi = np.random.default_rng(3).normal(0, 1, (41, 96)).astype(np.float32)
    return owb.Model(wakeword_models=_specs(), embedding_model_path=emb_weights(), feature_init=fi, max_chunks=8,
                     cnn_mode=mode, custom_verifier_models={"alexa_v0.1": os.path.join(GOLDEN, "verifier_alexa.pkl")},
                     custom_verifier_threshold=thr)


def _rows(res, labels):
    return np.array([[r[lab] for lab in labels] for r in res], np.float32).reshape(len(res), len(labels))


@pytest.mark.parametrize("mode", [0, 3])
def test_every_chunk_size_against_streaming(torch_cuda, built_library, mode):
    """predict_clips(list, chunk_size=c) equals predict_clip(clip, chunk_size=c) on a fresh stream, per clip: calls that
    step no chunk (c < 1280) repeat or zero, the first 5 calls are zeroed, verified scores are re-verified."""
    m = _verified_model(mode)
    labels = m.labels()
    rng = np.random.default_rng(11)
    clips = [_signal(rng, n) for n in (300, 9000, 17003, 23456, 40000)]
    repeats = verified = 0
    for c in (400, 1024, 1280, 2000, 2048, 2560, 3840, 8 * CHUNK):
        res = m.predict_clips(clips, padding=1, chunk_size=c)
        assert len(res) == len(clips)
        for clip, got in zip(clips, res):
            m.reset()
            ref = _rows(m.predict_clip(clip, padding=1, chunk_size=c), labels)
            got = _rows(got, labels)
            assert got.shape == ref.shape
            err = np.abs(got - ref).max() if ref.size else 0.0
            assert err < 2e-6, (c, clip.size, err)
            assert not got[:5].any()
            if c < CHUNK:
                repeats += int((got[5:, 0][1:] == got[5:, 0][:-1]).sum())
            verified += int((got[:, 0] >= 0.05).sum())
    print(f"mode {mode}: {repeats} repeated rows, {verified} verified-range scores")
    assert repeats > 0 and verified > 0
    with pytest.raises(ValueError, match="max_chunks"):
        m.predict_clips(clips, chunk_size=8 * CHUNK + 1)


_CASES = [t for t in golden_cases("predict_clip") if not load_case(t)["kw"]] + VERIFIER_CASES


@pytest.mark.parametrize("tag", _CASES)
def test_golden_cases_through_the_bulk_path(torch_cuda, built_library, tag):
    c = load_case(tag)
    kw = {}
    if "parent" in c:
        kw = dict(custom_verifier_models={str(c["parent"]): os.path.join(GOLDEN, str(c["verifier"]))},
                  custom_verifier_threshold=float(c["threshold"]))
    m = _model(c, cnn_mode=3, **kw)
    res = m.predict_clips([c["pcm"]], padding=int(c["padding"]), chunk_size=int(c["chunk"]))[0]
    assert list(res[0].keys()) == c["labels"]
    got = _rows(res, c["labels"])
    err = np.abs(got - c["scores"])
    for j, name in enumerate(c["labels"]):
        if name in c["names"] and "verifier" in head(name):
            err[:, j] = _gated_error(c, name, got[:, j], err[:, j])
    print(tag, "max |bulk - golden| =", err.max())
    assert err.max() < SCORE_TOL


def _write_wav(path, pcm):
    with wave.open(str(path), "wb") as f:
        f.setnchannels(1); f.setsampwidth(2); f.setframerate(16000)
        f.writeframes(np.asarray(pcm, np.int16).tobytes())


@pytest.fixture
def wav_files(tmp_path):
    rng = np.random.default_rng(21)
    paths = []
    for i, n in enumerate((900, 7000, 12345, 20000, 31111, 47000, 100000)):   # all lengths distinct, one under a chunk
        p = tmp_path / f"clip_{i}.wav"
        _write_wav(p, _signal(rng, n))
        paths.append(str(p))
    return paths


def _spy(monkeypatch):
    from openwakeword_b200 import _native
    calls = []
    real = _native.Context.predict_clips_ragged

    def spy(self, *a, **k):
        calls.append(a[1].size - 1)
        return real(self, *a, **k)
    monkeypatch.setattr(_native.Context, "predict_clips_ragged", spy)
    return calls


def test_bulk_predict_distinct_lengths_one_device_call(torch_cuda, built_library, wav_files, monkeypatch):
    import openwakeword_b200 as owb
    from openwakeword_b200 import utils as U
    fi = np.random.default_rng(4).normal(0, 1, (41, 96)).astype(np.float32)
    m = owb.Model(wakeword_models=_specs(), embedding_model_path=emb_weights(), feature_init=fi)
    labels = m.labels()
    calls = _spy(monkeypatch)
    for kw in ({}, {"chunk_size": 2560, "padding": 2}, {"chunk_size": 400, "padding": 0}, {"no_such_argument": 1}):
        calls.clear()
        res = U.bulk_predict(wav_files, wakeword_models=_specs(), ncpu=2, embedding_model_path=emb_weights(),
                             feature_init=fi, **kw)
        assert calls == [len(wav_files)], calls                       # one device call covers the batch
        for p in wav_files:
            m.reset()
            ref = _rows(m.predict_clip(p, padding=kw.get("padding", 1), chunk_size=kw.get("chunk_size", CHUNK)), labels)
            got = _rows(res[p], labels)
            assert got.shape == ref.shape, (kw, p)
            assert got.size == 0 or np.abs(got - ref).max() < 2e-6, (kw, p, np.abs(got - ref).max())


@pytest.mark.parametrize("return_type", ["features", "audio"])
def test_bulk_predict_positive_prediction_frames(torch_cuda, built_library, wav_files, monkeypatch, return_type):
    import openwakeword_b200 as owb
    from openwakeword_b200 import utils as U
    fi = np.random.default_rng(4).normal(0, 1, (41, 96)).astype(np.float32)
    m = owb.Model(wakeword_models=_specs(), embedding_model_path=emb_weights(), feature_init=fi)
    # a threshold inside the widest gap of the alexa scores below the best score of a frame with 4 s of audio around it
    # (so both return types have hits), where last-bit differences cannot move a frame across it
    sc, row_off, labels = m.predict_clips_ragged(*owb.model._concat_clips([U._read_wav(p) for p in wav_files]), padding=0)
    a = sc[:, labels.index("alexa_v0.1")]
    last = a[row_off[-2]:row_off[-1]]                                 # the 100 000-sample file
    s = np.arange(last.size)
    target = last[(s * CHUNK >= 48000) & (s * CHUNK + 16000 <= 100000)].max()
    v = np.unique(a[(a > 0) & (a <= target)])
    gaps = np.diff(v)
    k = int(np.argmax(gaps))
    t = float((v[k] + v[k + 1]) / 2)
    calls = _spy(monkeypatch)
    res = U.bulk_predict(wav_files, wakeword_models=_specs(), prediction_function="_get_positive_prediction_frames",
                         embedding_model_path=emb_weights(), feature_init=fi, threshold=t, return_type=return_type)
    assert calls == [len(wav_files)]
    n_hits = 0
    for p in wav_files:
        m.reset()
        ref = m._get_positive_prediction_frames(p, threshold=t, return_type=return_type)
        assert set(res[p]) == set(ref), p
        for lab in ref:
            assert res[p][lab].shape == ref[lab].shape
            if return_type == "audio":
                assert np.array_equal(res[p][lab], ref[lab])
            else:
                assert np.abs(res[p][lab] - ref[lab]).max() < 1e-6
            n_hits += ref[lab].shape[0]
    print(f"threshold {t:.6f}: {n_hits} positive frames")
    assert n_hits > 0
    with pytest.raises(ValueError):
        U.bulk_predict(wav_files, wakeword_models=_specs(), prediction_function="predict",
                       embedding_model_path=emb_weights())
