"""-m gpu: clip mixing on the device (oww_mix_clips, csrc/mix.cu) against the float64 restatement of its definition
(tests/mix_ref.py).  The int16 rows must equal the restatement's except where its value lies within the round-off bound
tau of a truncation boundary, where they may differ by one; the valid flags must be equal.

* RIRs of 1 tap and of N taps, direct paths at tap 0 and at tap L - 1, 1 / 16 / one RIR per mixture interleaved, rows of
  more than one 4096-sample tile and a partial last tile; foregrounds ending at sample N; backgrounds shorter than
  (non-integer tilings), as long as and longer than N; silent foregrounds and backgrounds; a non-positive signed
  maximum under the volume rule; negative peaks that saturate.
* n_mix = 0 and refused arguments launch nothing.
* detect_clips and predict_clips_ragged on the mixture tensor equal the same calls on its host copy; a seeded
  mix_clips_batch on the device matches the restatement run within one step."""
import numpy as np
import pytest

from helpers import emb_weights, head
from mix_ref import assert_int16_match, mix_ref
from openwakeword_b200 import _native

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda(built_library):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


@pytest.fixture(scope="module")
def af(torch_cuda):
    from openwakeword_b200.utils import AudioFeatures
    return AudioFeatures(embedding_model_path=emb_weights())


def noise(rng, n, scale=6000):
    return np.clip(rng.normal(0, scale, n), -32768, 32767).astype(np.int16)


def decaying_rir(rng, L, peak):
    h = (rng.normal(0, 1, L) * np.exp(-np.arange(L) / max(L / 6, 1))).astype(np.float32)
    h[peak] = np.float32(4.0) * (1 if rng.random() < 0.5 else -1)
    return h


def recs(rows):
    p = np.zeros(len(rows), _native.MIX_DTYPE)
    for i, r in enumerate(rows):
        base = dict(fg=0, bg=0, rir=-1, fg_start=0, fg_len=0, bg_offset=0, start=0, snr_db=0.0, volume=-1.0)
        base.update(r)
        for k, v in base.items():
            p[i][k] = v
    return p


def check(af, fg, bg, rirs, params, N, what):
    out, valid = af.mix_clips(fg, bg, N, params, rirs)
    q, v_ok, v, tau = mix_ref(fg, bg, rirs, params, N)
    dev = out.cpu().numpy()
    np.testing.assert_array_equal(valid.cpu().numpy(), v_ok, err_msg=what)
    near = assert_int16_match(dev, q, v, tau, what)
    return dev, near


def edge_case_call(rng, N):
    fg = [noise(rng, 3000), noise(rng, N), np.zeros(800, np.int16), noise(rng, 1)]
    bg = [noise(rng, 777, 2000), noise(rng, N, 2000), noise(rng, 3 * N + 5, 2000), np.zeros(50, np.int16),
          np.full(333, -1000, np.int16)]
    spike = np.full(N, 40, np.int16)
    spike[N // 3] = -30000
    bg.append(spike)                                    # bg 5: a small positive floor and one deep negative peak
    neg_fg = np.full(200, -3000, np.int16)
    fg.append(neg_fg)                                   # fg 4
    rirs = [np.array([0.7], np.float32), decaying_rir(rng, N, 0), decaying_rir(rng, 300, 0),
            decaying_rir(rng, 300, 299), decaying_rir(rng, 64, 17), decaying_rir(rng, 65, 64), decaying_rir(rng, min(4097, N - 1), 2000)]
    rows = []
    for rir in range(-1, len(rirs)):
        for vol in (-1.0, 0.6):
            rows += [dict(fg=0, fg_start=100, fg_len=2500, bg=0, bg_offset=500, start=N - 2500, snr_db=5.0, rir=rir, volume=vol),
                     dict(fg=1, fg_start=0, fg_len=N, bg=1, bg_offset=0, start=0, snr_db=-3.0, rir=rir, volume=vol),
                     dict(fg=0, fg_start=0, fg_len=3000, bg=2, bg_offset=3 * N + 4, start=17, snr_db=25.0, rir=rir, volume=vol),
                     dict(fg=3, fg_start=0, fg_len=1, bg=0, bg_offset=776, start=N - 1, snr_db=0.0, rir=rir, volume=vol)]
        rows += [dict(fg=2, fg_len=800, bg=1, start=5, rir=rir, volume=0.5),                 # silent foreground
                 dict(fg=0, fg_len=0, bg=1, start=5, rir=rir),                               # empty window
                 dict(fg=0, fg_len=3000, bg=3, bg_offset=7, start=5, rir=rir, volume=0.5),   # silent background
                 dict(fg=4, fg_len=200, bg=4, start=5, snr_db=-20.0, rir=-1, volume=0.5),    # signed max < 0
                 dict(fg=0, fg_len=1000, bg=5, start=N // 2, snr_db=-30.0, rir=-1, volume=0.9),   # saturating peak
                 dict(fg=0, fg_len=1000, bg=5, start=N // 2, snr_db=-30.0, rir=-1, volume=0.05)]
    return fg, bg, rirs, recs(rows)


@pytest.mark.parametrize("N", [4096, 9000])
def test_edge_cases_match_the_restatement(af, N):
    rng = np.random.default_rng(N)
    fg, bg, rirs, params = edge_case_call(rng, N)
    dev, near = check(af, fg, bg, rirs, params, N, f"N={N}")
    assert (dev[-2] == -32768).any(), "the saturating case did not saturate"
    assert not dev[-3].any()                           # signed maximum < 0: invalid, written as zeros
    print(f"N={N}: {params.size} mixtures, {near} samples within tau of a boundary")


@pytest.mark.parametrize("n_rirs", [1, 16, 0])
def test_many_rirs_interleaved(af, n_rirs):
    rng = np.random.default_rng(7 + n_rirs)
    N, n = 16000, 70
    n_rirs = n_rirs or n
    fg = [noise(rng, int(rng.integers(4000, 12000))) for _ in range(8)]
    bg = [noise(rng, int(rng.integers(3000, 40000)), 1500) for _ in range(8)]
    rirs = [decaying_rir(rng, int(rng.integers(1, 4000)), 0) for _ in range(n_rirs)]
    for h in rirs:
        h[int(rng.integers(0, h.size))] = 3.0
    rows = []
    for i in range(n):
        f, b = int(rng.integers(0, 8)), int(rng.integers(0, 8))
        fl = int(rng.integers(1, fg[f].size))
        rows.append(dict(fg=f, fg_start=int(rng.integers(0, fg[f].size - fl + 1)), fg_len=fl, bg=b,
                         bg_offset=int(rng.integers(0, bg[b].size)), start=int(rng.integers(0, N - fl + 1)),
                         snr_db=float(rng.uniform(-5, 20)), rir=int(rng.integers(-1, n_rirs)) if i % 5 else -1,
                         volume=float(rng.uniform(0.02, 1.0)) if i % 3 else -1.0))
    check(af, fg, bg, rirs, recs(rows), N, f"{n_rirs} rirs")


def test_nothing_launches_for_no_mixtures_and_refusals(af, torch_cuda):
    torch = torch_cuda
    rng = np.random.default_rng(3)
    fg, bg, rirs = [noise(rng, 100)], [noise(rng, 100)], [decaying_rir(rng, 50, 0)]
    N = 200
    ctx = af.ctx
    out = torch.full((1, N), 7, dtype=torch.int16, device="cuda")
    valid = torch.full((1,), 9, dtype=torch.uint8, device="cuda")
    d_fg = torch.from_numpy(fg[0]).cuda(); d_bg = torch.from_numpy(bg[0]).cuda(); d_rir = torch.from_numpy(rirs[0]).cuda()
    off = [0, 100]
    n0 = ctx.launch_count
    ctx.mix_clips(d_fg, off, d_bg, off, d_rir, [0, 50], recs([]), N, out, valid)
    assert ctx.launch_count == n0
    good = dict(fg=0, fg_len=50, bg=0, start=0, rir=0)
    bad_cases = [dict(fg=1), dict(bg=-1), dict(rir=1), dict(fg_start=60), dict(bg_offset=100), dict(start=151),
                 dict(start=-1), dict(snr_db=np.nan), dict(volume=np.inf)]
    for kw in bad_cases:
        with pytest.raises(_native.NativeError):
            ctx.mix_clips(d_fg, off, d_bg, off, d_rir, [0, 50], recs([dict(good, **kw)]), N, out, valid)
    for n_samples, rir_off in ((0, [0, 50]), (-5, [0, 50]), (40, [0, 50]), (N, [0, 0])):      # N <= 0, L > N, empty RIR
        with pytest.raises(_native.NativeError):
            ctx.mix_clips(d_fg, off, d_bg, off, d_rir, rir_off, recs([good]), n_samples, out, valid)
    with pytest.raises(_native.NativeError):                                              # empty background
        ctx.mix_clips(d_fg, off, d_bg, [0, 0], d_rir, [0, 50], recs([good]), N, out, valid)
    with pytest.raises(_native.NativeError):                                              # decreasing offsets
        ctx.mix_clips(d_fg, [50, 10], d_bg, off, d_rir, [0, 50], recs([good]), N, out, valid)
    torch.cuda.synchronize()
    assert ctx.launch_count == n0
    assert (out == 7).all() and (valid == 9).all()
    ctx.mix_clips(d_fg, off, d_bg, off, d_rir, [0, 50], recs([good]), N, out, valid)
    assert ctx.launch_count == n0 + 3
    ctx.mix_clips(d_fg, off, d_bg, off, d_rir, [0, 50], recs([dict(good, rir=-1)]), N, out, valid)
    assert ctx.launch_count == n0 + 5


def test_mixtures_feed_the_clip_paths_without_a_copy(af, torch_cuda):
    from openwakeword_b200 import Model
    rng = np.random.default_rng(5)
    N, n = 32000, 24
    fg = [noise(rng, 16000, 8000) for _ in range(4)]
    bg = [noise(rng, 50000, 1000)]
    rirs = [decaying_rir(rng, 4000, 3)]
    params = recs([dict(fg=i % 4, fg_len=16000, bg=0, bg_offset=int(rng.integers(0, 50000)), start=8000,
                        snr_db=float(rng.uniform(0, 20)), rir=0 if i % 2 else -1, volume=float(rng.uniform(0.1, 1)))
                   for i in range(n)])
    out, valid = af.mix_clips(fg, bg, N, params, rirs)
    host = out.cpu().numpy()
    m = Model(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")}], embedding_model_path=emb_weights(),
              feature_init=np.zeros((41, 96), np.float32))
    off = np.arange(n + 1, dtype=np.int64) * N
    a = m.predict_clips_ragged(out.reshape(-1), off)
    b = m.predict_clips_ragged(host.reshape(-1), off)
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1], b[1])
    thr = float(np.quantile(a[0][:, 0], 0.9))
    assert m.detect_clips(out, thr) == m.detect_clips(host, thr)


def test_seeded_mix_clips_batch_matches_the_restatement(af, monkeypatch):
    import random
    from openwakeword_b200 import data
    rng = np.random.default_rng(11)
    clips = {f"fg{i}": noise(rng, int(rng.integers(5000, 20000)), 8000) for i in range(10)}
    clips.update({f"bg{i}": noise(rng, int(rng.integers(2000, 60000)), 1500) for i in range(6)})
    rir_files = {f"rir{i}": decaying_rir(rng, 3000 + 500 * i, 2 * i)[None] for i in range(3)}
    monkeypatch.setattr(data, "_read_clip", lambda p: clips[p])
    monkeypatch.setattr(data, "_read_rir", lambda p: rir_files[p])

    class Restated:
        def mix_clips(self, fg, bg, n_samples, params, rirs=None):
            q, v, _, _ = mix_ref(fg, bg, rirs, params, n_samples)
            return q, v

    kw = dict(foreground_clips=[f"fg{i}" for i in range(10)], background_clips=[f"bg{i}" for i in range(6)],
              combined_size=32000, batch_size=4, snr_low=0, snr_high=15, start_index=[4000] * 10,
              foreground_durations=[1.0] * 10, rirs=list(rir_files), rir_probability=0.7,
              return_background_clips=True, return_background_clips_delay=(0, 100), seed=21)
    got = list(data.mix_clips_batch(audio_features=af, **kw))
    state = (np.random.get_state()[1].copy(), random.getstate())
    want = list(data.mix_clips_batch(audio_features=Restated(), **kw))
    assert np.array_equal(np.random.get_state()[1], state[0]) and random.getstate() == state[1]
    assert len(got) == len(want) == 3
    for (x, y, d), (x2, y2, d2) in zip(got, want):
        assert x.shape == x2.shape
        assert np.abs(x.astype(np.int64) - x2).max() <= 1
        np.testing.assert_array_equal(y, y2)
        np.testing.assert_array_equal(d, d2)
