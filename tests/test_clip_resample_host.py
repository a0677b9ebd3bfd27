"""Whole clips at any sample rate without a GPU (include/owwb200.h, oww_resample_clips):

* oww_resample_clip_plan against the definition A(S) + 2*pad for every rate, and its refusals;
* the float64 clip reference (clip_resample_ref.py) against scipy.signal.upfirdn on the zero-padded clip, and against the
  streaming oracle (oracle/resample.py) fed the padded clip in random packet splits; leading pad exactly 0, a short tail;
* the WAV reader at every rate of the table, and its refusals;
* routing of the clip and bulk paths on a stand-in of the C ABI: sr scalar and per clip, WAV headers, a header / sr
  mismatch, bulk_predict keeping sr away from the Model, 16 kHz calls never reaching the resampler, and the refusals of a
  device-ingest Model."""
import wave

import numpy as np
import pytest
import scipy.signal as ss

import clip_resample_ref as cref
import fake_backend
from helpers import emb_weights, head
from openwakeword_b200 import _native
from oracle import resample as ores

CHUNK = 1280
FI = np.zeros((41, 96), np.float32)
RESAMPLED = [r for r in ores.RATES if r != 16000]


def _K(rate):
    up, _ = ores.up_down(rate)
    return -(-ores.taps(rate).size // up) if rate != 16000 else 1


@pytest.mark.parametrize("rate", ores.RATES)
def test_plan_matches_the_definition(built_library, rate):
    K = _K(rate)
    for n_in in (0, 1, K - 1, K, K + 1, 1279, 1281, 10 ** 6):
        for pad in (0, 640, 16000):
            assert _native.resample_clip_plan(rate, n_in, pad) == cref.plan(rate, n_in, pad), (n_in, pad)
    up, _ = ores.up_down(rate)
    bad = [(rate, -1, 0), (rate, 0, -640)] + ([(rate, 10, up // 2)] if up > 1 else [])
    for r, n, p in bad + [(9000, 10, 0), (0, 10, 0), (96000, 10, 0)]:
        assert cref.plan(r, n, p) is None
        assert built_library.oww_resample_clip_plan(r, n, p, None) == -1
        with pytest.raises(ValueError, match="refused"):
            _native.resample_clip_plan(r, n, p)


@pytest.mark.parametrize("rate", RESAMPLED)
def test_reference_equals_upfirdn_and_streaming(rate):
    rng = np.random.default_rng(rate)
    up, down = ores.up_down(rate)
    K = _K(rate)
    for S in (0, 1, 20, K - 1, K + 1, 1279, 1281, int(rate * 0.7)):
        x = rng.normal(0, 5000, S)
        for pad in (0, 640, 16000):
            P = pad * down // up
            z = np.concatenate((np.zeros(P), x, np.zeros(P)))
            L = cref.plan(rate, S, pad)
            y = cref.resample_clip(x, rate, pad)
            assert y.size == L
            whole = ss.upfirdn(ores.taps(rate), z, up, down) if z.size else np.zeros(0)
            ref = np.zeros(L)
            ref[:min(L, whole.size)] = whole[:L]
            np.testing.assert_allclose(y, ref, rtol=0, atol=1e-9 * max(np.abs(ref).max(initial=0), 1.0))
            # a fresh stream fed the padded clip in random packets makes the same outputs final
            st = ores.StreamResampler(rate)
            pos, parts = 0, []
            while pos < z.size:
                k = int(rng.choice([1, 7, 97, 641, int(rng.integers(0, 4000))]))
                parts.append(st.feed(z[pos:pos + k]))
                pos += k
            got = np.concatenate(parts) if parts else np.zeros(0)
            assert got.size == L
            np.testing.assert_allclose(y, got, rtol=0, atol=1e-9 * max(np.abs(y).max(initial=0), 1.0))
            assert (y[:pad] == 0).all()
            tail = y[pad + ores.final_outputs(S, up, down):]
            assert np.count_nonzero(np.abs(tail) > 0) <= 39


def _write_wav(path, pcm, rate, channels=1, width=2):
    with wave.open(str(path), "wb") as f:
        f.setnchannels(channels); f.setsampwidth(width); f.setframerate(rate)
        f.writeframes(np.asarray(pcm).tobytes())
    return str(path)


def test_wav_reader(built_library, tmp_path):
    from openwakeword_b200.utils import _read_wav, _read_wav_rate, _read_wavs
    rng = np.random.default_rng(1)
    for r in ores.RATES:
        x = rng.integers(-3000, 3000, r // 10).astype(np.int16)
        p = _write_wav(tmp_path / f"a{r}.wav", x, r)
        pcm, rate = _read_wav_rate(p)
        assert rate == r and np.array_equal(pcm, x)
        if r == 16000:
            assert np.array_equal(_read_wav(p), x)
        else:
            with pytest.raises(ValueError, match="16 khz"):
                _read_wav(p)
    assert [r for _, r in _read_wavs([str(tmp_path / f"a{r}.wav") for r in ores.RATES], 3, _read_wav_rate)] == \
        list(ores.RATES)
    bad = [_write_wav(tmp_path / "w24.wav", np.zeros(96, np.uint8), 16000, width=3),
           _write_wav(tmp_path / "st.wav", np.zeros(64, np.int16), 48000, channels=2),
           _write_wav(tmp_path / "r9k.wav", np.zeros(64, np.int16), 9000)]
    for p in bad:
        with pytest.raises(ValueError, match=p.split("/")[-1]):
            _read_wav_rate(p)


# ---- routing on the stand-in ----
@pytest.fixture
def routed(monkeypatch):
    """the stand-in, the resampler's calls recorded, and _predict_ragged replaced by a recorder (the bulk path needs a
    GPU): it returns one zero row per call of each clip"""
    from openwakeword_b200 import Model, utils
    monkeypatch.setattr(_native, "Context", fake_backend.FakeContext)
    log = {"resample": [], "ragged": [], "init": []}

    def resample(self, pcm, offsets, rates, pad_samples=0):
        offsets = np.asarray(offsets, np.int64)
        rates = np.broadcast_to(np.asarray(rates, np.int64).ravel(), (offsets.size - 1,)).astype(np.int32)
        log["resample"].append((rates.copy(), int(pad_samples), offsets.copy()))
        n = [_native.resample_clip_plan(int(r), int(k), pad_samples) for r, k in zip(rates, np.diff(offsets))]
        out_off = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
        out = np.zeros(int(out_off[-1]), np.int16)
        self.ctx.resample_clips(np.asarray(pcm, np.int16), offsets, rates, pad_samples, out, out_off)
        import torch
        return torch.from_numpy(out), out_off

    def ragged(self, pcm, offsets, padding, chunk_size, feature_init, want_features=False, streams=None,
               check_ingest=True):
        if check_ingest:
            self._no_ingest("the bulk clip path (predict_clips_ragged, bulk_predict)")
        offsets = np.asarray(offsets, np.int64)
        log["ragged"].append((np.asarray(pcm).copy(), offsets.copy(), padding, chunk_size))
        calls = [_native.clip_schedule(chunk_size, int(k) + 2 * 16000 * int(padding)).size for k in np.diff(offsets)]
        row_off = np.concatenate([[0], np.cumsum(calls)]).astype(np.int64)
        steps = np.array(calls, np.int64) * chunk_size // CHUNK
        step_off = np.concatenate([[0], np.cumsum(steps)]).astype(np.int64)
        emb = np.zeros((int(step_off[-1]), 96), np.float32)
        return np.zeros((int(row_off[-1]), 1), np.float32), row_off, ["alexa"], emb, step_off, FI

    init = Model.__init__

    def record_init(self, *a, **kw):
        log["init"].append(dict(kw))
        init(self, *a, **kw)
    import torch

    class _HostTorch:                          # bulk_predict's page-locked staging needs a driver: plain host memory here
        def __getattr__(self, k):
            return getattr(torch, k)

        @staticmethod
        def empty(*a, pin_memory=False, **kw):
            return torch.empty(*a, **kw)
    monkeypatch.setattr(utils, "_torch", lambda: _HostTorch())
    monkeypatch.setattr(utils.AudioFeatures, "resample_clips", resample)
    monkeypatch.setattr(Model, "_predict_ragged", ragged)
    monkeypatch.setattr(Model, "__init__", record_init)
    yield log


def _model(sr=16000, n_streams=1):
    from openwakeword_b200 import Model
    return Model(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")}], embedding_model_path=emb_weights(),
                 feature_init=FI, n_streams=n_streams, max_chunks=2, sr=sr)


def test_clip_paths_route_through_the_resampler(routed):
    rng = np.random.default_rng(2)
    rates = [48000, 8000, 44100, 16000]
    clips = [rng.integers(-3000, 3000, int(r * 0.5)).astype(np.int16) for r in rates]
    m = _model()
    pcm = np.concatenate(clips)
    off = np.concatenate([[0], np.cumsum([c.size for c in clips])]).astype(np.int64)
    # per clip: one resample call with the padding, then the 16 kHz path on the padded clips with padding 0
    sc, row_off, labels = m.predict_clips_ragged(pcm, off, padding=1, chunk_size=2560, sr=rates)
    (r, pad, o), = routed["resample"]
    assert r.tolist() == rates and pad == 16000 and np.array_equal(o, off)
    x16, off16, padding, chunk = routed["ragged"][-1]
    assert padding == 0 and chunk == 2560
    assert np.diff(off16).tolist() == [cref.plan(r, c.size, 16000) for r, c in zip(rates, clips)]
    for i, (rt, c) in enumerate(zip(rates, clips)):
        h, _, _ = _native.resampler_taps(rt)
        ref = ores.to_int16(cref.resample_clip(c, rt, 16000, h=h.astype(np.float64) if h.size else None))
        assert np.array_equal(x16[off16[i]:off16[i + 1]], ref), rt
    assert np.diff(row_off).tolist() == [len(range(0, int(n) - 2560, 2560)) for n in np.diff(off16)]
    # one rate for every clip
    m.predict_clips([c[:4000] for c in clips], padding=0, sr=22050)
    assert routed["resample"][-1][0].tolist() == [22050] * 4 and routed["resample"][-1][1] == 0
    # positive frames: the audio context comes from the 16 kHz samples
    m._positive_frames_bulk(clips, return_type="audio", sr=rates)
    assert routed["resample"][-1][1] == 0 and routed["ragged"][-1][2] == 0
    # 16 kHz calls never reach the resampler
    n = len(routed["resample"])
    m.predict_clips_ragged(pcm, off, padding=1)
    m.predict_clips_ragged(pcm, off, padding=1, sr=16000)
    m.predict_clips([clips[3]], sr=[16000])
    m._positive_frames_bulk(clips)
    assert len(routed["resample"]) == n and routed["ragged"][-4][2] == 1
    with pytest.raises(ValueError, match="rates for"):
        m.predict_clips_ragged(pcm, off, sr=[48000, 8000])
    with pytest.raises(ValueError, match="not supported"):
        m.predict_clips_ragged(pcm, off, sr=9000)


def test_predict_clip_and_wav_headers(routed, tmp_path):
    rng = np.random.default_rng(3)
    x = rng.integers(-3000, 3000, 44100).astype(np.int16)
    p = _write_wav(tmp_path / "a.wav", x, 44100)
    m = _model()
    res = m.predict_clip(p, padding=1, chunk_size=1280)
    (r, pad, _), = routed["resample"]
    assert r.tolist() == [44100] and pad == 16000
    L = cref.plan(44100, x.size, 16000)
    assert len(res) == len(range(0, L - 1280, 1280))
    assert len(m.predict_clip(x, padding=0, sr=44100)) == len(range(0, cref.plan(44100, x.size, 0) - 1280, 1280))
    with pytest.raises(ValueError, match="header says 44100"):
        m.predict_clip(p, sr=48000)
    n = len(routed["resample"])
    m.predict_clip(p, sr=44100)
    p16 = _write_wav(tmp_path / "b.wav", x[:16000], 16000)
    m.predict_clip(p16)
    m.predict_clip(x[:16000])
    assert len(routed["resample"]) == n + 1
    m._get_positive_prediction_frames(p, threshold=2.0)
    assert routed["resample"][-1][1] == 0


def test_bulk_predict_reads_each_header(routed, tmp_path):
    from openwakeword_b200 import utils
    rng = np.random.default_rng(4)
    rates = [48000, 8000, 16000, 11025]
    paths = [_write_wav(tmp_path / f"c{i}.wav", rng.integers(-3000, 3000, int(r * 0.6)).astype(np.int16), r)
             for i, r in enumerate(rates)]
    kw = dict(embedding_model_path=emb_weights(), feature_init=FI, max_chunks=2)
    spec = [{"name": "alexa", "head": head("alexa_v0.1")}]
    out = utils.bulk_predict(paths, spec, **kw)
    assert list(out) == paths and routed["resample"][-1][0].tolist() == rates
    # sr is checked against every header and never reaches the Model (it would make a device-ingest Model)
    same = [_write_wav(tmp_path / f"s{i}.wav", rng.integers(-3000, 3000, 30000).astype(np.int16), 48000)
            for i in range(3)]
    utils.bulk_predict(same, spec, sr=48000, **kw)
    assert "sr" not in routed["init"][-1]
    with pytest.raises(ValueError, match="c0.wav"):
        utils.bulk_predict(paths, spec, sr=8000, **kw)
    utils.bulk_predict(same, spec, prediction_function="_get_positive_prediction_frames", **kw)
    assert routed["resample"][-1][0].tolist() == [48000] * 3
    # all 16 kHz: no resampling
    n = len(routed["resample"])
    utils.bulk_predict([paths[2]], spec, **kw)
    utils.bulk_predict([paths[2]], spec, prediction_function="_get_positive_prediction_frames", **kw)
    assert len(routed["resample"]) == n
    for name, pcm, r, ch in (("st.wav", np.zeros(64, np.int16), 48000, 2), ("r9k.wav", np.zeros(64, np.int16), 9000, 1)):
        bad = _write_wav(tmp_path / name, pcm, r, channels=ch)
        with pytest.raises(ValueError, match=name):
            utils.bulk_predict([paths[0], bad], spec, **kw)


def test_ingest_model_refusals(routed):
    m = _model(sr=48000)
    x = np.zeros(4000, np.int16)
    for call in (lambda: m.predict_clip(x),
                 lambda: m.predict_clips([x]),
                 lambda: m.predict_clips_ragged(x, [0, 4000]),
                 lambda: m.predict_clips_array(x[None]),
                 lambda: m._positive_frames_bulk([x])):
        with pytest.raises(ValueError, match="16 kHz clips"):
            call()
    # predict_clip is single-stream streaming: refused whatever sr
    for sr in (48000, 16000):
        with pytest.raises(ValueError, match="16 kHz clips"):
            m.predict_clip(x, sr=sr)
    assert not routed["resample"]
    # with the clips' rate given, the bulk paths take them
    m.predict_clips_ragged(x, [0, 4000], sr=48000)
    assert len(routed["resample"]) == 1
