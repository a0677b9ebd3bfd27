"""-m gpu: whole clips at any sample rate (oww_resample_clips, csrc/ingest.cu), every rate mixed in one call.

* Same bits as streaming ingest: each clip's outputs equal the samples a fresh ingest stream makes final for the padded
  clip fed in random packets (audio history + staged samples), clips of 0, 1, 20, K +- 1, 1279, 1281 samples, about 3 s,
  and one of more than 2^20 outputs, at padding 0 and 16000.  The clip call comes before oww_set_input_rates on the
  same handle, so streaming ingest is also checked to work after it.
* Float64 reference (clip_resample_ref.py) under test_gpu_ingest's bound gamma_K * sum |h32 * x|, with saturation.
* Scores: predict_clips_ragged(sr=...) equals the 16 kHz path on the device-resampled clips, and for chunk sizes 1280
  and 2560 a fresh Model(sr=rates) streaming the padded clips; predict_clip(x, sr=r) equals the same reference.
* bulk_predict on mixed-rate WAVs equals bulk_predict on 16 kHz WAVs of the resampled samples; embed_clips and
  compute_features_from_generator likewise.
* Launch counts of 16 kHz calls are unchanged, and refused arguments enqueue nothing."""
import os
import wave

import numpy as np
import pytest

import clip_resample_ref as cref
from helpers import GOLDEN, emb_weights, head
from oracle import resample as ores

pytestmark = pytest.mark.gpu
CHUNK = 1280
RATES = ores.RATES
FI = np.zeros((41, 96), np.float32)


@pytest.fixture(scope="module")
def torch_cuda(built_library):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _judge_bound(got, y64, s, K):
    """test_gpu_ingest's rule: outside the band gamma_K * sum |h32 * x| around a rounding boundary the int16 equals
    clip(rint(y64)), inside it differs by at most one -> fraction judged"""
    u = 2.0 ** -24
    band = K * u / (1 - K * u) * s
    ref = ores.to_int16(y64)
    near = np.abs(y64 - np.floor(y64) - 0.5) <= band
    sat = (y64 > 32767 + band) | (y64 < -32768 - band)
    judged = ~near | sat
    assert got.size == y64.size
    assert np.array_equal(got[judged], ref[judged]), np.nonzero(got[judged] != ref[judged])[0][:5]
    assert (np.abs(got.astype(np.int32) - ref) <= 1).all()
    return judged.mean()


def _K(rate):
    from openwakeword_b200 import _native
    h, up, _ = _native.resampler_taps(rate)
    return max(-(-h.size // up), 1)


def _signal(rng, n, full_scale=False):
    if full_scale:          # a square wave between the int16 extremes: its Gibbs overshoot saturates
        return np.where((np.arange(n) // 37) % 2 == 0, 32767, -32768).astype(np.int16)
    return np.clip(rng.normal(0, 6000, n), -32768, 32767).astype(np.int16)


def _device_resample(ctx, clips, rates, pad):
    import torch
    from openwakeword_b200 import _native
    off = np.concatenate([[0], np.cumsum([c.size for c in clips])]).astype(np.int64)
    n = [_native.resample_clip_plan(r, c.size, pad) for r, c in zip(rates, clips)]
    out_off = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    d_in = torch.from_numpy(np.concatenate(clips + [np.zeros(1, np.int16)])).cuda()
    d_out = torch.full((int(out_off[-1]) + 1,), 12345, dtype=torch.int16, device="cuda")
    ctx.resample_clips(d_in, off, np.asarray(rates, np.int32), pad, d_out, out_off)
    host = d_out.cpu().numpy()
    assert host[-1] == 12345                                  # nothing written past the last clip
    return [host[out_off[i]:out_off[i + 1]] for i in range(len(clips))]


def _padded(x, rate, pad):
    up, down = ores.up_down(rate)
    z = np.zeros(pad * down // up, np.int16)
    return np.concatenate((z, x, z))


def _stream_final16(eng, sigs, rng):
    """every 16 kHz sample a fresh ingest stream per signal makes final, fed in random packets"""
    import torch
    B, H = len(sigs), eng.ctx.audio_history
    pos, prev = np.zeros(B, np.int64), np.zeros(B, np.int64)
    got = [[] for _ in range(B)]
    while (pos < [s.size for s in sigs]).any():
        cap = eng.ingest_capacity()
        take = np.array([min(int(rng.integers(0, cap[b] + 1)), sigs[b].size - pos[b]) for b in range(B)], np.int64)
        off = np.concatenate([[0], np.cumsum(take)])
        pkt = np.concatenate([sigs[b][pos[b]:pos[b] + take[b]] for b in range(B)] + [np.zeros(1, np.int16)])
        eng.ingest(torch.from_numpy(pkt).cuda(), off)
        pos += take
        audio, p = eng.ctx.audio_state(np.arange(B))
        for b in range(B):
            d = int(p[b] - prev[b])
            assert d <= H
            if d:
                got[b].append(audio[b, H - d:])
        prev = p
    _, _, staged, x, _ = eng.ctx.ingest_state(np.arange(B))
    return [np.concatenate(got[b] + [x[b, :staged[b]]]) for b in range(B)]


def test_same_bits_as_streaming_ingest(torch_cuda):
    from openwakeword_b200.engine import StreamEngine
    rng = np.random.default_rng(0)
    rates, clips = [], []
    for r in RATES:
        K = _K(r)
        for n in (0, 1, 20, K - 1, K + 1, 1279, 1281, int(r * 3.1)):
            rates.append(r)
            clips.append(_signal(rng, n))
    rates.append(8000)
    clips.append(_signal(rng, 528000))                       # 66 s at 8 kHz: more than 2^20 outputs
    for pad in (0, 16000):
        eng = StreamEngine([head("alexa_v0.1")], len(clips), embedding=emb_weights(), max_chunks=8)
        eng.set_audio_history(8 * CHUNK)
        dev = _device_resample(eng.ctx, clips, rates, pad)   # a clip call first, then streaming ingest on the handle
        assert dev[-1].size > 2 ** 20
        eng.set_input_rates(np.asarray(rates, np.int32))
        ref = _stream_final16(eng, [_padded(c, r, pad) for c, r in zip(clips, rates)], rng)
        for i, (r, c) in enumerate(zip(rates, clips)):
            assert dev[i].size == cref.plan(r, c.size, pad)
            assert np.array_equal(dev[i], ref[i]), (r, c.size, pad)
            assert (dev[i][:pad] == 0).all()


def test_float64_reference(torch_cuda):
    from openwakeword_b200 import _native
    rng = np.random.default_rng(1)
    rates = [r for r in RATES for _ in range(3)]
    full = [i % 3 == 2 for i in range(len(rates))]
    clips = [_signal(rng, int(r * 1.3), fs) for r, fs in zip(rates, full)]
    ctx = _native.Context()
    dev = _device_resample(ctx, clips, rates, 16000)
    fracs = {}
    for i, r in enumerate(rates):
        h32, up, _ = _native.resampler_taps(r)
        y64, s = cref.resample_clip(clips[i], r, 16000, h=h32.astype(np.float64) if h32.size else None, abs_sum=True)
        fracs.setdefault(r, []).append(_judge_bound(dev[i], y64, s, max(-(-h32.size // up), 1)))
        if full[i] and r != 16000:
            assert (dev[i] == 32767).any() and (dev[i] == -32768).any(), r
    print("judged fractions:", {r: round(min(f), 4) for r, f in fracs.items()})
    assert min(min(f) for f in fracs.values()) >= 0.75


def _model_kw(n_streams):
    return dict(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")},
                                 {"name": "timer", "head": head("timer_v0.1")}],
                embedding_model_path=emb_weights(), feature_init=FI, n_streams=n_streams, max_chunks=3,
                custom_verifier_models={"alexa": os.path.join(GOLDEN, "verifier_alexa.pkl")},
                custom_verifier_threshold=0.0, stream_models={"bank": {None: head("big_v0.1")}})


def _streaming_reference(rates, clips, padding, chunk, labels):
    """a fresh Model(sr=rates) with one stream per clip fed the padded clips in chunk*r/16000-sample packets -> per clip
    the [calls, labels] rows of its own calls"""
    from openwakeword_b200 import Model, _native
    m = Model(sr=list(rates), **_model_kw(len(clips)))
    pads = [_padded(c, r, 16000 * padding) for c, r in zip(clips, rates)]
    calls = [_native.clip_schedule(chunk, _native.resample_clip_plan(r, c.size, 16000 * padding)).size
             for c, r in zip(clips, rates)]
    rows = [[] for _ in clips]
    for k in range(max(calls)):
        pk = [p[k * chunk * r // 16000:(k + 1) * chunk * r // 16000] if k < n else np.zeros(0, np.int16)
              for p, r, n in zip(pads, rates, calls)]
        res = m.predict_ragged(pk)
        for i in range(len(clips)):
            if k < calls[i]:
                rows[i].append([res[lab][i] for lab in labels])
    assert sorted(res) == sorted(labels)
    return [np.asarray(r, np.float32).reshape(-1, len(labels)) for r in rows]


def test_scores(torch_cuda):
    from openwakeword_b200 import Model
    rng = np.random.default_rng(2)
    rates = [48000, 44100, 8000, 11025, 16000, 22050, 24000, 32000, 12000, 48000]
    clips = [_signal(rng, int(r * s)) for r, s in zip(rates, (1.7, 2.3, 1.1, 0.4, 1.5, 0.9, 2.0, 0.05, 1.2, 0.0))]
    N = len(clips)
    pcm = np.concatenate(clips)
    off = np.concatenate([[0], np.cumsum([c.size for c in clips])]).astype(np.int64)
    m = Model(**_model_kw(N))
    for padding in (0, 1):
        d16, off16 = m.preprocessor.resample_clips(pcm, off, rates, 16000 * padding)
        for chunk in (1280, 2560, 1000):
            for streams in (None, np.arange(N)):       # the last: every clip scored as its own stream
                sc, row_off, labels = m.predict_clips_ragged(pcm, off, padding, chunk, streams=streams, sr=rates)
                s16, r16, l16 = m.predict_clips_ragged(d16, off16, 0, chunk, streams=streams)
                assert labels == l16 and np.array_equal(row_off, r16) and np.array_equal(sc, s16), (padding, chunk)
            if chunk == 1000:
                continue
            ref = _streaming_reference(rates, clips, padding, chunk, labels)
            for i in range(N):
                assert np.array_equal(sc[row_off[i]:row_off[i + 1]], ref[i]), (padding, chunk, rates[i])
    # predict_clip on a plain single-stream Model
    ref = _streaming_reference(rates[:3], clips[:3], 1, 1280, labels)
    for i in range(3):
        one = Model(**_model_kw(1))
        got = one.predict_clip(clips[i], padding=1, sr=rates[i])
        got = np.asarray([[d[lab] for lab in labels] for d in got], np.float32).reshape(-1, len(labels))
        assert np.array_equal(got, ref[i]), rates[i]


def _write_wav(path, pcm, rate):
    with wave.open(str(path), "wb") as f:
        f.setnchannels(1); f.setsampwidth(2); f.setframerate(rate)
        f.writeframes(np.asarray(pcm, np.int16).tobytes())
    return str(path)


def test_bulk_predict_mixed_rates(torch_cuda, tmp_path):
    from openwakeword_b200 import AudioFeatures
    from openwakeword_b200.utils import bulk_predict
    rng = np.random.default_rng(3)
    rates = [48000, 44100, 8000, 16000, 22050, 11025, 48000, 32000]
    clips = [_signal(rng, int(r * s)) for r, s in zip(rates, (2.1, 1.4, 3.0, 1.2, 0.7, 2.2, 0.3, 1.6))]
    paths = [_write_wav(tmp_path / f"m{i}.wav", c, r) for i, (c, r) in enumerate(zip(clips, rates))]
    af = AudioFeatures(embedding_model_path=emb_weights())
    kw = dict(embedding_model_path=emb_weights(), feature_init=FI, max_chunks=3)
    spec = [{"name": "alexa", "head": head("alexa_v0.1")}, {"name": "timer", "head": head("timer_v0.1")}]
    for fn, padding in (("predict_clip", 1), ("_get_positive_prediction_frames", 0)):
        off = np.concatenate([[0], np.cumsum([c.size for c in clips])]).astype(np.int64)
        d, o16 = af.resample_clips(np.concatenate(clips), off, rates, 16000 * padding)
        h = d.cpu().numpy()
        p16 = [_write_wav(tmp_path / f"r{fn}{i}.wav", h[o16[i]:o16[i + 1]], 16000) for i in range(len(clips))]
        fkw = dict(padding=padding) if fn == "predict_clip" else dict(threshold=0.0, return_type="features")
        a = bulk_predict(paths, spec, prediction_function=fn, **fkw, **kw)
        fkw16 = dict(padding=0) if fn == "predict_clip" else fkw
        b = bulk_predict(p16, spec, prediction_function=fn, **fkw16, **kw)
        assert len(a) == len(b) == len(clips)
        for pa, pb in zip(paths, p16):
            if fn == "predict_clip":
                assert a[pa] == b[pb], pa
            else:
                assert a[pa].keys() == b[pb].keys() and all(np.array_equal(a[pa][k], b[pb][k]) for k in a[pa]), pa


def test_feature_extraction(torch_cuda, tmp_path):
    from openwakeword_b200 import AudioFeatures
    from openwakeword_b200.utils import compute_features_from_generator
    rng = np.random.default_rng(4)
    af = AudioFeatures(embedding_model_path=emb_weights())
    for r in (48000, 44100, 8000, 22050):
        S = int(r * 1.9)
        x = np.stack([_signal(rng, S) for _ in range(5)])
        d, _ = af.resample_clips(x.reshape(-1), np.arange(6, dtype=np.int64) * S, r, 0)
        x16 = d.cpu().numpy().reshape(5, -1)
        assert np.array_equal(af.embed_clips(x, sr=r), af.embed_clips(x16))
        out, out16 = str(tmp_path / f"f{r}.npy"), str(tmp_path / f"g{r}.npy")
        compute_features_from_generator(iter([x[:3], x[3:]]), 5, S, out, audio_features=af, sr=r)
        compute_features_from_generator(iter([x16[:3], x16[3:]]), 5, x16.shape[1], out16, audio_features=af)
        assert np.array_equal(np.load(out), np.load(out16))


def test_launch_counts_and_refusals(torch_cuda, tmp_path, monkeypatch):
    import torch
    from openwakeword_b200 import Model, _native
    from openwakeword_b200.utils import bulk_predict
    rng = np.random.default_rng(5)
    clips = [_signal(rng, n) for n in (16000, 23456, 8000)]
    pcm = np.concatenate(clips)
    off = np.concatenate([[0], np.cumsum([c.size for c in clips])]).astype(np.int64)
    m = Model(**_model_kw(1))
    ctx = m.preprocessor.ctx
    m.predict_clips_ragged(pcm, off)
    deltas = []
    for sr in (None, 16000, [16000] * 3, 48000):
        n0 = ctx.launch_count
        m.predict_clips_ragged(pcm, off, sr=sr)
        torch.cuda.synchronize()
        deltas.append(ctx.launch_count - n0)
    assert deltas[0] == deltas[1] == deltas[2] and deltas[3] == deltas[0] + 1, deltas
    # an all-16 kHz bulk_predict batch never reaches the resampler
    paths = [_write_wav(tmp_path / f"s{i}.wav", c, 16000) for i, c in enumerate(clips)]

    def refuse(*a, **k):
        raise AssertionError("resampled a 16 kHz batch")
    monkeypatch.setattr(_native.Context, "resample_clips", refuse)
    kw = dict(embedding_model_path=emb_weights(), feature_init=FI, max_chunks=3)
    bulk_predict(paths, [{"name": "alexa", "head": head("alexa_v0.1")}], **kw)
    bulk_predict(paths, [{"name": "alexa", "head": head("alexa_v0.1")}],
                 prediction_function="_get_positive_prediction_frames", **kw)
    monkeypatch.undo()
    # refused arguments enqueue nothing
    d_in = torch.zeros(100, dtype=torch.int16, device="cuda")
    d_out = torch.zeros(100000, dtype=torch.int16, device="cuda")
    n0 = ctx.launch_count
    good = _native.resample_clip_plan(44100, 100, 0)
    for in_off, rates, pad, out_off in (([0, 100], [9000], 0, [0, 100]),               # rate outside the table
                                        ([0, 100], [44100], 16, [0, good + 32]),       # pad the up factor does not divide
                                        ([0, 100], [44100], 0, [0, good + 1]),         # output offsets off the plan
                                        ([50, 10], [44100], 0, [0, 0]),                # decreasing input offsets
                                        ([0, 100], [44100], -160, [0, good])):         # negative pad
        with pytest.raises(_native.NativeError):
            ctx.resample_clips(d_in, in_off, rates, pad, d_out, out_off)
    assert ctx.launch_count == n0
