"""Packets at any sample rate without a GPU (include/owwb200.h, oww_set_input_rates / oww_ingest):

* the fp32 taps of the built library (oww_resampler_taps) against scipy.signal.firwin for every rate of the table, and
  the refusal of other rates;
* the float64 streaming oracle (oracle/resample.py) against scipy.signal.upfirdn over random packet splits, with empty,
  1-sample and prime-length packets, and its final-output count against A(S) = ceil(S*up/down);
* the library's pure-host arithmetic (oww_ingest_plan, which oww_ingest and oww_ingest_capacity run) against the oracle;
* Model routing, splitting of long calls, refusals and export / import of the ingest state, on the stand-in of the C
  ABI (ingest through the oracle)."""
import numpy as np
import pytest
import scipy.signal as ss

import fake_backend
from helpers import emb_weights, head
from openwakeword_b200 import _native
from oracle import resample as ores

CHUNK = 1280
FI = np.zeros((41, 96), np.float32)


def test_taps_equal_scipy_firwin(built_library):
    for r in ores.RATES:
        h, up, down = _native.resampler_taps(r)
        assert (up, down) == ores.up_down(r)
        if r == 16000:
            assert h.size == 0 and up == down == 1
            continue
        mr = max(up, down)
        f = ss.firwin(20 * mr + 1, 1.0 / mr, window=("kaiser", 5.0)) * up
        assert h.dtype == np.float32 and h.size == f.size
        assert np.abs(h.astype(np.float64) - f).max() <= 2.0 ** -24 * np.abs(f).max(), r
        assert np.abs(ores.taps(r) - f).max() <= 1e-15, r
        assert -(-h.size // up) <= 61
    for bad in (0, 1, 7999, 16001, 96000, -16000):
        with pytest.raises(ValueError, match="not supported"):
            _native.resampler_taps(bad)
        assert built_library.oww_resampler_taps(bad, None, 0, None, None) == -1


def _packets(rng, n):
    out, pos = [], 0
    while pos < n:
        k = int(rng.choice([0, 1, 2, 3, 5, 7, 13, 97, 641, 1279, 1280, 3841, int(rng.integers(0, 6000))]))
        out.append((pos, min(n, pos + k)))
        pos = min(n, pos + k)
    return out


@pytest.mark.parametrize("rate", [r for r in ores.RATES if r != 16000])
def test_streaming_oracle_equals_upfirdn(rate):
    rng = np.random.default_rng(rate)
    x = rng.normal(0, 5000, int(rate * 0.3))
    up, down = ores.up_down(rate)
    whole = ss.upfirdn(ores.taps(rate), x, up, down)
    r = ores.StreamResampler(rate)
    got = []
    for a, b in _packets(rng, x.size):
        y = r.feed(x[a:b])
        assert y.size == ores.final_outputs(b, up, down) - ores.final_outputs(a, up, down)
        got.append(y)
    got = np.concatenate(got)
    assert got.size == ores.final_outputs(x.size, up, down) == -(-x.size * up // down)
    np.testing.assert_allclose(got, whole[:got.size], rtol=0, atol=1e-9 * np.abs(whole).max())
    # the outputs past A(S) read input sample S or later: a different next sample changes them
    longer = ss.upfirdn(ores.taps(rate), np.concatenate((x, rng.normal(0, 5000, 64))), up, down)
    assert np.array_equal(longer[:got.size], whole[:got.size])
    assert np.abs(longer[got.size:got.size + 8] - whole[got.size:got.size + 8]).max() > 1.0


@pytest.mark.parametrize("rate", ores.RATES)
def test_library_plan_matches_the_oracle(built_library, rate):
    up, down = ores.up_down(rate)
    rng = np.random.default_rng(rate + 1)
    for max_chunks in (1, 2, 3):
        cap = max_chunks * CHUNK + CHUNK - 1
        for _ in range(200):
            S, staged = int(rng.integers(0, 10 ** 7)), int(rng.integers(0, CHUNK))
            n_out, chunks, after, max_in = _native.ingest_plan(rate, max_chunks, S, staged, 0)
            assert n_out == 0 and chunks == staged // CHUNK
            A = lambda n: ores.final_outputs(S + n, up, down) - ores.final_outputs(S, up, down)   # noqa: E731
            assert staged + A(max_in) <= cap < staged + A(max_in + 1)
            n = int(rng.integers(0, max_in + 1))
            n_out, chunks, after, _ = _native.ingest_plan(rate, max_chunks, S, staged, n)
            assert n_out == A(n) and chunks == (staged + n_out) // CHUNK and after == (staged + n_out) % CHUNK
            assert chunks <= max_chunks
            assert _native.ingest_plan(rate, max_chunks, S, staged, max_in + 1)[0] is None
        n_out, chunks, _, _ = _native.ingest_plan(rate, max_chunks, 0, 0, rate * 8 // 100)   # an 80 ms packet
        assert n_out == CHUNK and chunks == 1


@pytest.fixture
def ingest_ctx(monkeypatch):
    monkeypatch.setattr(_native, "Context", fake_backend.FakeContext)


def _model(B, sr, **kw):
    from openwakeword_b200 import Model
    return Model(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")}], embedding_model_path=emb_weights(),
                 feature_init=FI, n_streams=B, max_chunks=2, sr=sr, **kw)


def test_model_routing_and_splitting(ingest_ctx):
    rng = np.random.default_rng(7)
    m = _model(3, [48000, 8000, 16000])
    assert m.preprocessor.ingest and m.preprocessor.pending_ragged
    assert not _model(2, 16000).preprocessor.ingest
    m.preprocessor._ensure_streams()
    ctx = m.preprocessor.ctx
    # one call longer than the capacity runs as several ingest calls; the result is that of the same audio in 80 ms
    # packets, which step one chunk each
    xs = [rng.integers(-3000, 3000, int(r * 0.4)).astype(np.int16) for r in (48000, 8000, 16000)]
    assert (np.array([x.size for x in xs]) > ctx.ingest_capacity()).any()
    out = m.predict_ragged(xs)
    ref = _model(3, [48000, 8000, 16000])
    for k in range(5):
        last = ref.predict_ragged([x[k * x.size // 5:(k + 1) * x.size // 5] for x in xs])
    assert np.array_equal(np.stack([s.size for s in ctx._ing["staged"]]),
                          np.stack([s.size for s in ref.preprocessor.ctx._ing["staged"]]))
    assert out["alexa"].shape == (3,) and np.isfinite(out["alexa"]).all()
    assert ref.preprocessor.ctx._ing["S"].tolist() == ctx._ing["S"].tolist() == [x.size for x in xs]
    # a call below a chunk prepares the staged samples and steps nothing
    n_prep, n_chunks, split = m.preprocessor._ingest_features([np.zeros(3, np.int16)] * 3, np.zeros((3, 1), np.float32))
    assert (n_chunks == 0).all() and not split
    assert n_prep.tolist() == [s.size for s in ctx._ing["staged"]]
    assert m.preprocessor._held_in_raw.all()
    # the lockstep call form goes the same way
    r = m.predict(np.zeros((3, 3840), np.int16))
    assert r["alexa"].shape == (3,)
    del last


def test_rates_and_refusals(ingest_ctx):
    from openwakeword_b200.utils import input_rates
    assert input_rates(16000, 3) is None
    assert input_rates(48000, 2).tolist() == [48000, 48000]
    assert input_rates([8000, 16000], 2).tolist() == [8000, 16000]
    for bad in (9000, [48000, 7000]):
        with pytest.raises(ValueError, match="not supported"):
            _model(2, bad)
    with pytest.raises(ValueError, match="rates for"):
        _model(2, [48000])
    plain = _model(2, 16000)
    with pytest.raises(ValueError, match="ingest"):
        plain.set_sample_rates([0], 48000)
    m = _model(1, 48000)
    for call in (lambda: m.predict_clip(np.zeros(4000, np.int16)),
                 lambda: m.predict_clips([np.zeros(4000, np.int16)]),
                 lambda: m.predict_clips_ragged(np.zeros(4000, np.int16), [0, 4000]),
                 lambda: m.predict_clips_array(np.zeros((1, 4000), np.int16)),
                 lambda: m._positive_frames_bulk([np.zeros(4000, np.int16)])):
        with pytest.raises(ValueError, match="16 kHz clips"):
            call()
    with pytest.raises(ValueError, match="not supported"):
        m.set_sample_rates([0], 12345)
    m.set_sample_rates([0], 44100)
    assert m.preprocessor.sample_rates.tolist() == [44100]


def test_speex_refusal(ingest_ctx, monkeypatch):
    import sys
    import types

    class _NS:
        @staticmethod
        def create(*a):
            return _NS()

        def process(self, b):
            return b
    monkeypatch.setitem(sys.modules, "speexdsp_ns", types.SimpleNamespace(NoiseSuppression=_NS))
    with pytest.raises(ValueError, match="Speex"):
        _model(1, 48000, enable_speex_noise_suppression=True)
    m = _model(1, [16000], enable_speex_noise_suppression=True)
    with pytest.raises(ValueError, match="Speex"):
        m.set_sample_rates([0], 8000)


def test_export_import_carries_the_ingest_state(ingest_ctx):
    rng = np.random.default_rng(9)
    rates = [48000, 8000, 44100]
    a, b = _model(3, rates), _model(3, rates)
    xs = [rng.integers(-3000, 3000, int(r * 0.13)).astype(np.int16) for r in rates]
    a.predict_ragged(xs)
    st = a.export_streams([0, 2])
    assert st.ingest[0].tolist() == [48000, 44100] and st.ingest[1].tolist() == [xs[0].size, xs[2].size]
    b.import_streams([2, 1], st)
    g = b.preprocessor.ctx._ing
    assert g["rate"].tolist() == [48000, 44100, 48000]
    assert np.array_equal(g["staged"][2], a.preprocessor.ctx._ing["staged"][0])
    more = [rng.integers(-3000, 3000, int(r * 0.05)).astype(np.int16) for r in rates]
    ra = a.predict_ragged([more[0], np.zeros(0, np.int16), more[2]])
    rb = b.predict_ragged([np.zeros(0, np.int16), more[2], more[0]])
    assert ra["alexa"][0] == rb["alexa"][2] and ra["alexa"][2] == rb["alexa"][1]
    assert np.array_equal(a.preprocessor.ctx._ing["staged"][0], b.preprocessor.ctx._ing["staged"][2])
    with pytest.raises(ValueError, match="device ingest"):
        _model(3, 16000).import_streams([0, 1], st)
    a.reset_streams([0])
    assert a.preprocessor.ctx._ing["S"][0] == 0 and a.preprocessor.ctx._ing["staged"][0].size == 0
    assert a.preprocessor.ctx._ing["rate"][0] == 48000
