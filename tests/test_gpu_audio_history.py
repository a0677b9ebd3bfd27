"""-m gpu: stream audio on the device (oww_set_audio_history and the calls after it, csrc/audio.cu).

* ``AudioFeatures.raw_data_buffer`` equals the unmodified reference's deque (tests/golden/raw_buffer.npz) bit for bit at
  H = 160000, on the lockstep and the ragged accumulation paths.
* Against a host copy of everything each stream stepped: every step entry point of the engine (device, host, submitted,
  ragged with held streams) and of Model (predict, predict_ragged, detect, detect_ragged), at an H that wraps often and
  at 10 s, in cnn_mode 0 and 3, on the fused single-chunk path and the multi-chunk path, across resets and set_streams.
* PCM rows as column slices at strides that are not a multiple of 8 samples.
* Windows before the history, partly overwritten or past the position give zeros exactly where samples are absent;
  post-roll after a detection.
* Capture of detections: clips and ends against the host copy, truncation at max_events, zero events.
* Moving streams between slots, Models and a grown engine; refused imports.
* History changes nothing else: scores and events bit-identical with it on and off, and one more launch per step."""
import os

import numpy as np
import pytest

from helpers import GOLDEN, emb_weights, head

pytestmark = pytest.mark.gpu
CHUNK = 1280


@pytest.fixture(scope="module")
def torch_cuda(built_library):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _engine(B, H, cnn_mode=3, max_chunks=4, **kw):
    from openwakeword_b200.engine import StreamEngine
    eng = StreamEngine([head("alexa_v0.1"), head("timer_v0.1")], B, embedding=emb_weights(), max_chunks=max_chunks,
                       cnn_mode=cnn_mode, **kw)
    if H:
        eng.set_audio_history(H)
    return eng


def _expect(stepped, H, e, n):
    """samples [e - n, e) of a stream that stepped `stepped`, as a history of H samples gives them"""
    q = np.arange(e - n, e)
    p = stepped.size
    ok = (q >= max(p - H, 0)) & (q < p)
    out = np.zeros(n, np.int16)
    out[ok] = stepped[q[ok]]
    return out


def _check_engine(eng, host, H, rng=None):
    ids = np.arange(eng.n_streams)
    clips, pos = eng.get_audio(ids, H)
    clips, pos = clips.cpu().numpy(), pos.cpu().numpy()
    for b in ids:
        assert pos[b] == host[b].size, b
        assert np.array_equal(clips[b], _expect(host[b], H, host[b].size, H)), b
    if rng is not None:                     # random windows, duplicate ids, explicit ends
        sel = rng.integers(0, eng.n_streams, 7)
        n = int(rng.integers(1, H + 1))
        ends = np.array([int(rng.integers(-1, host[b].size + 2 * n + 1)) for b in sel], np.int64)
        c, p = eng.get_audio(sel, n, ends)
        c = c.cpu().numpy()
        for i, b in enumerate(sel):
            e = host[b].size if ends[i] < 0 else ends[i]
            assert np.array_equal(c[i], _expect(host[b], H, e, n)), (i, b, e, n)


def _pcm(rng, B, n):
    return rng.integers(-32768, 32768, (B, n)).astype(np.int16)


# ---- the reference's raw_data_buffer ----
def test_raw_data_buffer_equals_the_reference(torch_cuda):
    from openwakeword_b200.utils import AudioFeatures
    z = np.load(os.path.join(GOLDEN, "raw_buffer.npz"))
    sig = z["signal"]
    one = AudioFeatures(embedding_model_path=emb_weights(), feature_init=np.zeros((41, 96), np.float32), audio_history=10)
    two = AudioFeatures(embedding_model_path=emb_weights(), n_streams=2, feature_init=np.zeros((41, 96), np.float32),
                        audio_history=10)
    rng = np.random.default_rng(1)
    scores = np.zeros((2, 1), np.float32)
    off = 0
    for k, c in enumerate(z["calls"]):
        if c < 0:
            one.reset()
            two.reset(stream_ids=[0])
        else:
            assert one(sig[off:off + c]) == z["ret"][k]
            other = rng.integers(-2000, 2000, int(rng.integers(0, 3000))).astype(np.int16)
            assert two._streaming_features_ragged([sig[off:off + c], other], scores)[0][0] == z["ret"][k]
            off += c
        want = sig[z["raw_lo"][k]:z["raw_hi"][k]]
        for af in (one, two):
            buf = af.raw_data_buffer
            assert buf.maxlen == 160000
            assert np.array_equal(np.array(buf, np.int16), want), k


# ---- every engine entry point against the host copy ----
@pytest.mark.parametrize("H", [3840, 160000])
@pytest.mark.parametrize("cnn_mode", [0, 3])
def test_engine_steps_against_the_host_copy(torch_cuda, H, cnn_mode):
    torch = torch_cuda
    B, mc = 5, 4
    eng = _engine(B, H, cnn_mode, mc)
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(H + cnn_mode)
    host = [np.zeros(0, np.int16) for _ in range(B)]
    kinds = ["step1", "step", "step_host", "submit", "ragged", "host_ragged", "submit_ragged"]
    n_iter = 90 if H > 100000 else 30
    for it in range(n_iter):
        kind = kinds[it % len(kinds)]
        if kind in ("step1", "step", "step_host", "submit"):
            n = 1 if kind == "step1" else int(rng.integers(1, mc + 1))
            pcm = _pcm(rng, B, n * CHUNK)
            chunks = np.full(B, n)
            if kind in ("step1", "step"):
                eng.step(torch.from_numpy(pcm).to(dev), n)
            elif kind == "step_host":
                eng.step_host(pcm, n)
            else:
                eng.collect(eng.submit(pcm, n))
        else:
            chunks = rng.integers(0, mc + 1, B).astype(np.int32)
            chunks[rng.integers(0, B)] = 0                   # a held stream
            chunks[rng.integers(0, B)] = 1                   # a stream on the single-chunk launch
            pcm = _pcm(rng, B, max(int(chunks.max()), 1) * CHUNK)
            if kind == "ragged":
                eng.step_ragged(torch.from_numpy(pcm).to(dev), chunks)
            elif kind == "host_ragged":
                eng.step_host_ragged(pcm, chunks)
            else:
                eng.collect(eng.submit_ragged(pcm, chunks))
        for b in range(B):
            host[b] = np.concatenate((host[b], pcm[b, :int(chunks[b]) * CHUNK]))
        if it % 3 == 0 or it == n_iter - 1:
            _check_engine(eng, host, H, rng)
    assert max(h.size for h in host) > H                     # the rings wrapped
    eng.reset(stream_ids=[1, 3])
    host[1] = host[3] = np.zeros(0, np.int16)
    _check_engine(eng, host, H, rng)
    eng.reset_async(stream_ids=[0])
    host[0] = np.zeros(0, np.int16)
    pcm = _pcm(rng, B, CHUNK)
    eng.step(torch.from_numpy(pcm).to(dev), 1)
    host = [np.concatenate((h, pcm[b])) for b, h in enumerate(host)]
    _check_engine(eng, host, H, rng)
    eng.set_streams(B + 2)
    host = [np.zeros(0, np.int16) for _ in range(B + 2)]
    _check_engine(eng, host, H)
    pcm = _pcm(rng, B + 2, 2 * CHUNK)
    eng.step_host(pcm, 2)
    _check_engine(eng, [p for p in pcm], H, rng)


@pytest.mark.parametrize("cnn_mode", [0, 3])
def test_model_paths_against_the_host_copy(torch_cuda, cnn_mode):
    import openwakeword_b200 as owb
    B = 4
    m = owb.Model(wakeword_models=[{"name": "alexa_v0.1", "head": head("alexa_v0.1")}], embedding_model_path=emb_weights(),
                  feature_init=np.zeros((41, 96), np.float32), n_streams=B, max_chunks=2, cnn_mode=cnn_mode,
                  audio_history=0.24)
    H = 3840
    rng = np.random.default_rng(cnn_mode)
    host = [np.zeros(0, np.int16) for _ in range(B)]
    pre = m.preprocessor
    for it in range(24):
        held, lens0 = pre._ragged_pending()
        kind = it % 4
        if kind == 0:
            x = rng.integers(-3000, 3000, (B, int(rng.integers(0, 7000)))).astype(np.int16)
            xs = list(x)
            m.predict(x)
        elif kind == 1:
            xs = [rng.integers(-3000, 3000, int(rng.integers(0, 4500))).astype(np.int16) for _ in range(B)]
            m.predict_ragged(xs)
        elif kind == 2:
            x = rng.integers(-3000, 3000, (B, int(rng.integers(0, 2600)))).astype(np.int16)
            xs = list(x)
            m.detect(x, threshold=0.5)
        else:
            xs = [rng.integers(-3000, 3000, int(rng.integers(0, 2600))).astype(np.int16) for _ in range(B)]
            m.detect_ragged(xs, threshold=0.5)
        lens = pre._ragged_pending()[1]
        for b in range(B):
            allx = np.concatenate((held[b, :lens0[b]], xs[b]))
            host[b] = np.concatenate((host[b], allx[:allx.size - lens[b]]))
        clips, ends = m.get_audio(np.arange(B), H / 16000)
        for b in range(B):
            assert ends[b] == host[b].size
            assert np.array_equal(clips[b], _expect(host[b], H, host[b].size, H)), (it, b)
        if it == 12:
            m.reset_streams([2])
            host[2] = np.zeros(0, np.int16)
    m.reset()
    clips, ends = m.get_audio(np.arange(B), 0.08)
    assert not ends.any() and not clips.any()


def test_odd_strides_append_correctly(torch_cuda):
    torch = torch_cuda
    B, H = 3, 6400
    eng = _engine(B, H, 3, 2)
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(7)
    host = [np.zeros(0, np.int16) for _ in range(B)]
    # row starts off 16 bytes in most rows (stride not a multiple of 8 samples, or an odd column), one aligned layout
    for it, (width, col) in enumerate([(2 * CHUNK + 3, 3), (2 * CHUNK + 5, 1), (2 * CHUNK + 8, 8), (2 * CHUNK + 1, 0)]):
        big = _pcm(rng, B, width)
        view = torch.from_numpy(big).to(dev)[:, col:col + 2 * CHUNK]
        if it % 2:
            chunks = np.array([2, 0, 1], np.int32)
            eng.step_ragged(view, chunks)
        else:
            chunks = np.array([1, 1, 1], np.int32)
            eng.step(view[:, :CHUNK], 1)
        for b in range(B):
            host[b] = np.concatenate((host[b], big[b, col:col + int(chunks[b]) * CHUNK]))
        _check_engine(eng, host, H, rng)


def test_windows_outside_the_ring_and_post_roll(torch_cuda):
    torch = torch_cuda
    B, H = 2, 3840
    eng = _engine(B, H, 3, 4)
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(9)
    pcm = _pcm(rng, B, 5 * CHUNK)
    eng.step(torch.from_numpy(pcm[:, :4 * CHUNK]).to(dev), 4)
    eng.step(torch.from_numpy(pcm[:, 4 * CHUNK:]).to(dev), 1)          # the ring holds [2560, 6400)
    cases = [(2000, 1000), (3000, 1280), (2560, 2560), (7000, 2000), (6400, 3840), (20000, 100), (1, 1), (6401, 2)]
    for e, n in cases:
        c, p = eng.get_audio([0, 1], n, np.array([e, e], np.int64))
        c = c.cpu().numpy()
        assert (p.cpu().numpy() == 6400).all()
        for b in range(B):
            assert np.array_equal(c[b], _expect(pcm[b], H, e, n)), (e, n)
    q = np.arange(3000 - 1280, 3000)
    c = eng.get_audio([0], 1280, np.array([3000], np.int64))[0].cpu().numpy()[0]
    assert not c[q < 2560].any() and np.array_equal(c[q >= 2560], pcm[0, 2560:3000])
    with pytest.raises(Exception, match="n_samples"):
        eng.get_audio([0], H + 1)
    # post-roll: audio after a detection, read once the stream has advanced a second
    eng2 = _engine(B, 160000, 3, 4)
    eng2.set_detector([(0, True)], threshold=0.0)
    host = [np.zeros(0, np.int16) for _ in range(B)]
    for it in range(6):
        pcm = _pcm(rng, B, CHUNK)
        sc = eng2.step(torch.from_numpy(pcm).to(dev), 1)
        host = [np.concatenate((h, pcm[b])) for b, h in enumerate(host)]
    ev, n, clips, ends = eng2.detect(sc, 1280, capture=16000)
    assert n == B and (ends == host[0].size).all()
    for _ in range(4):
        pcm = _pcm(rng, B, 4 * CHUNK)
        eng2.step(torch.from_numpy(pcm).to(dev), 4)
        host = [np.concatenate((h, pcm[b])) for b, h in enumerate(host)]
    e = ends + 16000
    c, p = eng2.get_audio(ev["stream"], 32000, e)
    c = c.cpu().numpy()
    for i, b in enumerate(ev["stream"]):
        assert np.array_equal(c[i], _expect(host[b], 160000, e[i], 32000))
        assert np.array_equal(c[i, :16000], clips[i].cpu().numpy())


def test_capture_events(torch_cuda):
    torch = torch_cuda
    B, H = 40, 16640
    eng = _engine(B, H, 3, 2)
    dev = torch.device("cuda", 0)
    eng.set_detector([(0, True), (3, False), (5, False)], threshold={0: 0.5, 1: 0.25, 2: 0.9})
    rng = np.random.default_rng(11)
    host = [np.zeros(0, np.int16) for _ in range(B)]
    zeros = torch.zeros((B, eng.n_cols), dtype=torch.float32, device=dev)
    for it in range(7):
        chunks = rng.integers(1, 3, B).astype(np.int32)
        pcm = _pcm(rng, B, 2 * CHUNK)
        eng.step_ragged(torch.from_numpy(pcm).to(dev), chunks)
        host = [np.concatenate((h, pcm[b, :chunks[b] * CHUNK])) for b, h in enumerate(host)]
        ev, n = eng.detect(zeros, chunks * CHUNK)          # fills the first five predictions
        assert n == 0
    scores = np.zeros((B, eng.n_cols), np.float32)
    fire = [(2, 0), (2, 1), (7, 2), (13, 0), (39, 1), (39, 2)]
    col = {0: 0, 1: 3, 2: 5}
    for b, j in fire:
        scores[b, col[j]] = 0.95
    d_scores = torch.from_numpy(scores).to(dev)
    for max_events in (None, 64, 3):                # no debounce: the same scores fire again at each call
        ev, n, clips, ends = eng.detect(d_scores, 1280, max_events=max_events, capture=4000)
        k = len(fire) if max_events is None else min(len(fire), max_events)
        assert n == len(fire) and len(ev) == k and tuple(clips.shape) == (k, 4000) and ends.shape == (k,)
        assert [(int(s), int(j)) for s, j in zip(ev["stream"], ev["label"])] == fire[:k]
        c = clips.cpu().numpy()
        for i in range(k):
            b = int(ev["stream"][i])
            assert ends[i] == host[b].size
            assert np.array_equal(c[i], host[b][-4000:]), i
    ev, n, clips, ends = eng.detect(zeros, 1280, max_events=16, capture=4000)
    assert n == 0 and len(ev) == 0 and tuple(clips.shape) == (0, 4000) and ends.size == 0
    # the raw call: rows past the count are not written
    ctx = eng.ctx
    evbuf = torch.zeros((8, 4), dtype=torch.int32, device=dev)
    evbuf[:, 0] = torch.arange(8, dtype=torch.int32)
    n_ev = torch.tensor([3], dtype=torch.int32, device=dev)
    out = torch.full((8, 100), 7, dtype=torch.int16, device=dev)
    pos = torch.full((8,), -5, dtype=torch.int64, device=dev)
    ctx.capture_events(evbuf, n_ev, 8, 100, out, pos, torch.cuda.current_stream(dev).cuda_stream)
    o, p = out.cpu().numpy(), pos.cpu().numpy()
    assert (o[3:] == 7).all() and (p[3:] == -5).all()
    for i in range(3):
        assert p[i] == host[i].size and np.array_equal(o[i], host[i][-100:])


def test_moving_streams(torch_cuda):
    torch = torch_cuda
    import openwakeword_b200 as owb
    from openwakeword_b200 import _native

    def model(B, secs):
        return owb.Model(wakeword_models=[{"name": "alexa_v0.1", "head": head("alexa_v0.1")}],
                         embedding_model_path=emb_weights(), feature_init=np.zeros((41, 96), np.float32), n_streams=B,
                         max_chunks=2, audio_history=secs)

    rng = np.random.default_rng(13)
    a, b2, other, off = model(3, 0.48), model(4, 0.48), model(4, 0.32), model(4, 0)
    for _ in range(5):
        a.predict_ragged([rng.integers(-3000, 3000, int(rng.integers(0, 3000))).astype(np.int16) for _ in range(3)])
    st = a.export_streams([1])
    b2.import_streams([3], st)
    ca, ea = a.get_audio([1], 0.48)
    cb, eb = b2.get_audio([3], 0.48)
    assert np.array_equal(ca, cb) and ea[0] == eb[0]
    x = rng.integers(-3000, 3000, 3333).astype(np.int16)
    xa = [np.zeros(0, np.int16)] * 3
    xa[1] = x
    xb = [np.zeros(0, np.int16)] * 4
    xb[3] = x
    a.predict_ragged(xa)
    b2.predict_ragged(xb)
    ca, ea = a.get_audio([1], 0.48)
    cb, eb = b2.get_audio([3], 0.48)
    assert np.array_equal(ca, cb) and ea[0] == eb[0] and ea[0] > 0
    for dst in (other, off):
        with pytest.raises(ValueError, match="audio history"):
            dst.import_streams([0], st)
    with pytest.raises(ValueError, match="audio history"):
        b2.import_streams([0], off.export_streams([0]))
    # engine calls across a grown engine
    dev = torch.device("cuda", 0)
    B, H = 3, 5120
    eng = _engine(B, H, 3, 2)
    host = [np.zeros(0, np.int16) for _ in range(B)]
    for _ in range(6):
        pcm = _pcm(rng, B, 2 * CHUNK)
        eng.step(torch.from_numpy(pcm).to(dev), 2)
        host = [np.concatenate((h, pcm[i])) for i, h in enumerate(host)]
    audio, pos = eng.audio_history([2, 0])
    assert audio.shape == (2, H) and (pos == 12 * CHUNK).all()
    assert np.array_equal(audio[0], host[2][-H:])
    records = eng.export_streams([2, 0])
    eng.set_streams(B + 3)
    eng.import_streams([4, 5], records)
    eng.set_audio_history_state([4, 5], audio, pos)
    host = [np.zeros(0, np.int16) for _ in range(4)] + [host[2], host[0]]
    pcm = _pcm(rng, B + 3, CHUNK)
    eng.step(torch.from_numpy(pcm).to(dev), 1)
    host = [np.concatenate((h, pcm[i])) for i, h in enumerate(host)]
    _check_engine(eng, host, H, rng)
    with pytest.raises(_native.NativeError, match="error -1"):
        eng.set_audio_history_state([1, 1], audio, pos)
    with pytest.raises(_native.NativeError, match="error -1"):
        eng.get_audio([B + 3], 10)


def test_history_changes_nothing_else(torch_cuda):
    torch = torch_cuda
    B = 24
    dev = torch.device("cuda", 0)
    engs = [_engine(B, 0, 3, 3), _engine(B, 160000, 3, 3)]
    for e in engs:
        e.set_detector([(0, True), (2, False)], threshold={0: 0.3, 1: 0.1})
    rng = np.random.default_rng(17)
    host_out = np.zeros((B, engs[0].n_cols), np.float32)
    for it in range(16):
        kind = it % 5
        pcm = _pcm(rng, B, 3 * CHUNK)
        chunks = rng.integers(0, 4, B).astype(np.int32)
        chunks[0], chunks[1] = 0, 1
        res, deltas = [], []
        for e in engs:
            n0 = e.ctx.launch_count
            if kind == 0:
                s = e.step(torch.from_numpy(pcm).to(dev), 1).cpu().numpy()
                prep = 1280
            elif kind == 1:
                s = e.step(torch.from_numpy(pcm).to(dev), 3).cpu().numpy()
                prep = 3 * 1280
            elif kind == 2:
                s = e.step_ragged(torch.from_numpy(pcm).to(dev), chunks).cpu().numpy()
                prep = np.where(chunks > 0, chunks * 1280, -1)
            elif kind == 3:
                s = e.step_host(pcm[:, :2 * CHUNK].copy(), 2)
                prep = 2 * 1280
            else:
                s = e.collect(e.submit_ragged(pcm, chunks), host_out.copy())
                prep = np.where(chunks > 0, chunks * 1280, -1)
            deltas.append(e.ctx.launch_count - n0)
            ev, n = e.detect(torch.from_numpy(np.nan_to_num(s)).to(dev), prep)
            res.append((s, ev.tobytes(), n))
        assert deltas[1] == deltas[0] + 1, (kind, deltas)
        assert np.array_equal(res[0][0], res[1][0], equal_nan=True), kind
        assert res[0][1:] == res[1][1:], kind
