"""-m gpu: packets at any sample rate (oww_set_input_rates / oww_ingest, csrc/ingest.cu), with mixed rates in one handle
and two or more streams per rate.

* Samples: the 16 kHz samples the device made final (audio history + exported staged samples) against the float64
  oracle (oracle/resample.py) under the per-element bound |y - y64| <= gamma_K * sum |h32 * x|; outside the bound's band
  around a rounding boundary the int16 equals clip(rint(y64)) exactly, inside it differs by at most one; at least 75% of
  the samples are judged.  Full-scale alternating input covers saturation.
* Split invariance: the same audio in three packet splits (80 ms packets, random lengths, packets that fill the capacity
  and so cross max_chunks) gives the same samples bit for bit.
* Scores and detections: a 16 kHz Model fed, through predict_ragged / detect_ragged, exactly the samples each ingest
  call made final gives the same predictions and events bit for bit, with a custom verifier, a head bank and debounce.
* 16 kHz streams on an ingest handle equal the host remainder path bit for bit, zero-length packets included.
* State changes: rate changes mid-stream, reset_streams, export / import to another Model, set_streams.
* Refusals fail before anything is enqueued."""
import os

import numpy as np
import pytest

from helpers import GOLDEN, emb_weights, head, judge_resampled
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


def _engine(rates, max_chunks=2, H=160000):
    from openwakeword_b200.engine import StreamEngine
    eng = StreamEngine([head("alexa_v0.1"), head("timer_v0.1")], len(rates), embedding=emb_weights(),
                       max_chunks=max_chunks)
    eng.set_audio_history(H)
    eng.set_input_rates(np.asarray(rates, np.int32))
    return eng


def _signal(rng, rate, seconds, full_scale=False):
    n = int(rate * seconds)
    if full_scale:          # a 400 Hz square wave between the int16 extremes: its Gibbs overshoot saturates
        return np.where((np.arange(n) // (rate // 800)) % 2 == 0, 32767, -32768).astype(np.int16)
    return np.clip(rng.normal(0, 6000, n), -32768, 32767).astype(np.int16)


def _feed_engine(eng, sigs, lengths):
    """feed sigs[b] in packets of lengths(b, k, capacity) samples until every signal is consumed"""
    import torch
    B = len(sigs)
    pos = np.zeros(B, np.int64)
    k = 0
    while (pos < [s.size for s in sigs]).any():
        cap = eng.ingest_capacity()
        take = np.array([min(lengths(b, k, int(cap[b])), sigs[b].size - pos[b]) for b in range(B)], np.int64)
        off = np.concatenate([[0], np.cumsum(take)])
        pkt = np.concatenate([sigs[b][pos[b]:pos[b] + take[b]] for b in range(B)])
        eng.ingest(torch.from_numpy(pkt).cuda(), off)
        pos += take
        k += 1


def _final16(ctx, B):
    """per stream: every 16 kHz sample the device made final (stepped, from the audio history, then staged)"""
    audio, pos = ctx.audio_state(np.arange(B))
    _, _, staged, x, _ = ctx.ingest_state(np.arange(B))
    H = audio.shape[1]
    out = []
    for b in range(B):
        assert pos[b] <= H
        out.append(np.concatenate((audio[b, H - pos[b]:], x[b, :staged[b]])))
    return out


def _judge(got, x, rate):
    """got (int16) against the oracle on input x under the round-off bound -> fraction judged"""
    from openwakeword_b200 import _native
    h32, up, down = _native.resampler_taps(rate)
    if up == down:
        assert np.array_equal(got, x)
        return 1.0
    y64, s = ores.StreamResampler(rate, h=h32.astype(np.float64)).feed(x, abs_sum=True)
    assert got.size == y64.size == ores.final_outputs(x.size, up, down)
    return judge_resampled(got, y64, s, up, down, h32.size)


def test_samples_against_the_float64_oracle(torch_cuda):
    rng = np.random.default_rng(0)
    rates = [r for r in RATES for _ in range(3)]
    full = [i % 3 == 2 for i in range(len(rates))]             # one full-scale alternating stream per rate
    sigs = [_signal(rng, r, 1.3, fs) for r, fs in zip(rates, full)]
    eng = _engine(rates)
    _feed_engine(eng, sigs, lambda b, k, cap: int(rng.integers(0, min(cap, 5000) + 1)))
    got = _final16(eng.ctx, len(rates))
    fracs = []
    for b, r in enumerate(rates):
        fracs.append(_judge(got[b], sigs[b], r))
        if full[b] and r != 16000:
            assert (got[b] == 32767).any() and (got[b] == -32768).any(), r
    print("judged fractions:", dict(zip(rates, np.round(fracs, 4))))
    assert min(fracs) >= 0.75


def test_80ms_packets_step_one_chunk_per_call(torch_cuda):
    import torch
    rates = [r for r in RATES for _ in range(2)]
    eng = _engine(rates)
    rng = np.random.default_rng(1)
    for _ in range(3):
        pk = [_signal(rng, r, 0.08) for r in rates]
        off = np.concatenate([[0], np.cumsum([p.size for p in pk])])
        chunks, prepared = eng.ingest(torch.from_numpy(np.concatenate(pk)).cuda(), off)
        assert (chunks == 1).all() and (prepared == 1280).all()


def test_split_invariance(torch_cuda):
    from openwakeword_b200 import Model
    rng = np.random.default_rng(2)
    rates = [r for r in RATES for _ in range(2)]
    sigs = [_signal(rng, r, 1.0) for r in rates]
    outs = []
    splits = [lambda b, k, cap: rates[b] * 8 // 100,                          # 80 ms
              lambda b, k, cap: int(rng.choice([0, 1, 7, 13, 997, cap])),      # empty, 1, prime, full
              lambda b, k, cap: cap]                                           # every call at capacity
    for split in splits:
        eng = _engine(rates)
        _feed_engine(eng, sigs, split)
        outs.append(_final16(eng.ctx, len(rates)))
    # a Model call longer than the capacity runs as several ingest calls
    m = Model(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")}], embedding_model_path=emb_weights(),
              feature_init=FI, n_streams=len(rates), sr=rates, max_chunks=2, audio_history=10)
    for k in range(2):
        m.predict_ragged([s[k * s.size // 2:(k + 1) * s.size // 2] for s in sigs])
    outs.append(_final16(m.preprocessor.ctx, len(rates)))
    for o in outs[1:]:
        for b in range(len(rates)):
            assert np.array_equal(o[b], outs[0][b]), (rates[b], o[b].size, outs[0][b].size)


def test_scores_and_detections_equal_a_16k_model(torch_cuda):
    from openwakeword_b200 import Model
    rng = np.random.default_rng(3)
    rates = [48000, 48000, 44100, 44100, 8000, 8000, 16000, 16000, 22050, 11025]
    B = len(rates)
    kw = dict(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")},
                               {"name": "timer", "head": head("timer_v0.1")}],
              embedding_model_path=emb_weights(), feature_init=FI, n_streams=B, max_chunks=3, audio_history=10,
              custom_verifier_models={"alexa": os.path.join(GOLDEN, "verifier_alexa.pkl")}, custom_verifier_threshold=0.0,
              stream_models={"bank": {None: head("big_v0.1")}})
    a = Model(sr=rates, **kw)
    b16 = Model(**kw)
    made = [np.zeros(0, np.int16) for _ in range(B)]
    for k in range(24):
        xs = [_signal(rng, r, float(rng.choice([0.0, 0.013, 0.08, 0.11, 0.2]))) for r in rates]
        cap = a.preprocessor.ctx.ingest_capacity()
        xs = [x[:c] for x, c in zip(xs, cap)]
        if k % 2:
            ra = a.predict_ragged(xs)
        else:
            ra = a.detect_ragged(xs, threshold=0.3, debounce_time=0.5)
        now = _final16(a.preprocessor.ctx, B)
        new = [now[b][made[b].size:] for b in range(B)]
        assert all(np.array_equal(now[b][:made[b].size], made[b]) for b in range(B))
        made = now
        rb = b16.predict_ragged(new) if k % 2 else b16.detect_ragged(new, threshold=0.3, debounce_time=0.5)
        if k % 2:
            assert ra.keys() == rb.keys()
            for lab in ra:
                assert np.array_equal(ra[lab], rb[lab]), (k, lab)
        else:
            assert ra == rb, k


def test_16k_streams_equal_the_host_path(torch_cuda):
    from openwakeword_b200 import Model
    rng = np.random.default_rng(4)
    B = 4
    kw = dict(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")}], embedding_model_path=emb_weights(),
              feature_init=FI, n_streams=B, max_chunks=2)
    a = Model(sr=[16000] * B, **kw)
    h = Model(**kw)
    assert a.preprocessor.ingest and not h.preprocessor.ingest
    for k in range(20):
        xs = [_signal(rng, 16000, float(rng.choice([0.0, 0.001, 0.05, 0.08, 0.15]))) for _ in range(B)]
        ra, rh = a.predict_ragged(xs), h.predict_ragged(xs)
        for lab in ra:
            assert np.array_equal(ra[lab], rh[lab]), (k, lab)
        assert np.array_equal(a.preprocessor._held_in_raw, h.preprocessor._held_in_raw)


def test_state_changes(torch_cuda):
    from openwakeword_b200 import Model
    rng = np.random.default_rng(5)
    rates = [48000, 48000, 8000, 8000, 44100, 44100]
    B = len(rates)
    mk = lambda: Model(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")}],   # noqa: E731
                       embedding_model_path=emb_weights(), feature_init=FI, n_streams=B, sr=list(rates), max_chunks=2,
                       audio_history=10)
    m = mk()
    sigs = [_signal(rng, r, 0.4) for r in rates]
    m.predict_ragged([s[:s.size // 2] for s in sigs])
    # rate change mid-stream: staged samples kept, the resampler restarts at the new rate
    staged_before = _final16(m.preprocessor.ctx, B)
    m.set_sample_rates([0, 2], [22050, 24000])
    tail = [_signal(rng, 22050, 0.2), None, _signal(rng, 24000, 0.2)]
    xs = [tail[0], sigs[1][sigs[1].size // 2:], tail[2]] + [s[s.size // 2:] for s in sigs[3:]]
    m.predict_ragged(xs)
    after = _final16(m.preprocessor.ctx, B)
    from openwakeword_b200 import _native
    for b, r in ((0, 22050), (2, 24000)):
        h32, up, down = _native.resampler_taps(r)
        y = ores.to_int16(ores.StreamResampler(r, h=h32.astype(np.float64)).feed(xs[b]))
        assert np.array_equal(after[b][:staged_before[b].size], staged_before[b])
        assert np.abs(after[b][staged_before[b].size:].astype(np.int32) - y).max() <= 1
    # export / import into another Model: the moved stream continues bit for bit
    st = m.export_streams([1, 4])
    m2 = mk()
    m2.import_streams([3, 0], st)
    more = [_signal(rng, rates[1], 0.3), _signal(rng, rates[4], 0.3)]
    xa = [np.zeros(0, np.int16)] * B
    xa[1], xa[4] = more
    xb = [np.zeros(0, np.int16)] * B
    xb[3], xb[0] = more
    ra, rb = m.predict_ragged(xa), m2.predict_ragged(xb)
    fa, fb = _final16(m.preprocessor.ctx, B), _final16(m2.preprocessor.ctx, B)
    assert ra["alexa"][1] == rb["alexa"][3] and ra["alexa"][4] == rb["alexa"][0]
    ea, eb = m.preprocessor.ctx.ingest_state([1, 4]), m2.preprocessor.ctx.ingest_state([3, 0])
    for u, v in zip(ea, eb):
        assert np.array_equal(u, v)
    assert np.array_equal(fa[1], fb[3]) and np.array_equal(fa[4], fb[0])
    # reset_streams: staged samples and history gone, rates kept
    m.reset_streams([4])
    r, S, staged, _, _ = m.preprocessor.ctx.ingest_state([4])
    assert r[0] == 44100 and S[0] == 0 and staged[0] == 0
    # set_streams sets every rate back to 16000
    ctx = m.preprocessor.ctx
    ctx.set_streams(B)
    r, S, staged, _, _ = ctx.ingest_state(np.arange(B))
    assert (r == 16000).all() and (S == 0).all() and (staged == 0).all()


def test_refusals_enqueue_nothing(torch_cuda):
    import torch
    from openwakeword_b200 import Model, _native
    eng = _engine([48000, 48000, 8000])
    eng.ingest(torch.zeros(1, dtype=torch.int16, device="cuda"), [0, 0, 0, 0])
    n0 = eng.ctx.launch_count
    cap = eng.ingest_capacity()
    big = torch.zeros(int(cap[0]) + 1, dtype=torch.int16, device="cuda")
    with pytest.raises(_native.NativeError, match="capacity"):
        eng.ingest(big, [0, big.numel(), big.numel(), big.numel()])
    with pytest.raises(_native.NativeError):
        eng.ctx.ingest(big, np.array([0, 5, 3, 6]), eng.ingest_scores)          # decreasing offsets
    with pytest.raises(ValueError):
        eng.set_input_rates([9000], [0])
    with pytest.raises(_native.NativeError):
        eng.ctx.set_input_rates([7], [16000])
    assert eng.ctx.launch_count == n0
    assert (eng.ctx.ingest_state(np.arange(3), samples=False)[1] == 0).all()
    plain = Model(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")}], embedding_model_path=emb_weights(),
                  feature_init=FI, n_streams=2)
    with pytest.raises(ValueError, match="ingest"):
        plain.set_sample_rates([0], [48000])
    m = Model(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")}], embedding_model_path=emb_weights(),
              feature_init=FI, sr=48000)
    with pytest.raises(ValueError, match="16 kHz"):
        m.predict_clip(np.zeros(16000, np.int16))
    with pytest.raises(ValueError, match="16 kHz"):
        m.predict_clips([np.zeros(16000, np.int16)])
