"""CPU tests of clip mixing (no GPU): the float64 restatement (tests/mix_ref.py) against mixtures the unmodified reference
made (tests/golden/mix.npz, tests/golden/make_mix_golden.py), mix_clips_batch's random draws and RNG states against the
reference's, frame labels and truncation windows, and the host-side refusals."""
import os
import random

import numpy as np
import pytest

from mix_ref import check_record, mix_ref, mixture
from openwakeword_b200 import _native, data

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "mix.npz")
Z = np.load(GOLDEN)
N = int(Z["N"])
NAMES = [str(s) for s in Z["config_names"]]
FGS = ["fg0.wav", "fg1.wav", "fg2.wav", "fg3.wav", "fg4.wav", "fg5.wav"]
BGS = ["bg0.wav", "bg1.wav", "bg2.wav", "bg3.wav", "bg4.wav", "bg5.wav"]
# the keyword arguments of tests/golden/make_mix_golden.py's configurations
CONFIGS = {
    "shuffle_random_rir": dict(foreground_clips=FGS, batch_size=4, snr_low=-5, snr_high=15, start_index=[100, 0, 2000, 50, 1000, 30],
                               foreground_durations=[0.3, 0.5, 0.2, 0.4, 0.6, 0.1], foreground_truncate_strategy="random",
                               rirs=["rir_mono.wav", "rir_stereo.wav"], rir_probability=1, shuffle=True,
                               return_background_clips=True, return_background_clips_delay=(10, 200), seed=3),
    "noshuffle_start_norir": dict(foreground_clips=FGS, batch_size=4, snr_low=0, snr_high=10, start_index=[0, 10, 20, 30, 40, 50],
                                  foreground_durations=[0.3, 0.5, 0.2, 0.4, 0.6, 0.1], foreground_truncate_strategy="truncate_start",
                                  rirs=["rir_mono.wav"], rir_probability=0, volume_augmentation=False, shuffle=False,
                                  return_sequence_labels=True, return_background_clips=True,
                                  return_background_clips_delay=(0, 0), seed=5),
    "shuffle_end_stereo": dict(foreground_clips=FGS, batch_size=4, snr_low=5, snr_high=6, start_index=[7, 8, 9, 10, 11, 12],
                               foreground_durations=[0.25] * 6, foreground_truncate_strategy="truncate_end",
                               rirs=["rir_stereo.wav"], rir_probability=1, shuffle=True, return_sequence_labels=True,
                               return_background_clips=True, return_background_clips_delay=(10, 200), seed=11),
    "noshuffle_both": dict(foreground_clips=FGS, batch_size=4, snr_low=10, snr_high=10, start_index=[500, 600, 700, 800, 900, 1000],
                           foreground_durations=[0.3, 0.5, 0.2, 0.46875, 0.6, 0.1], foreground_truncate_strategy="truncate_both",
                           shuffle=False, volume_augmentation=False, return_background_clips=True,
                           return_background_clips_delay=(0, 0), seed=7),
    "short_batch_full_clips": dict(foreground_clips=["fg1.wav", "fg_silent.wav"], batch_size=5, snr_low=-10, snr_high=20,
                                   start_index=[3000, 1], labels=[1, 0], rirs=["rir_mono.wav", "rir_stereo.wav"],
                                   rir_probability=1, shuffle=True, seed=13),
}
TRUNC_METHODS = ["truncate_start", "truncate_end", "truncate_both", "random", "other"]


class FakeMixer:
    """oww_mix_clips computed by the float64 restatement; records every call"""

    def __init__(self):
        self.calls = []

    def mix_clips(self, fg, bg, n_samples, params, rirs=None):
        params = np.array(params, _native.MIX_DTYPE)
        self.calls.append((list(fg), list(bg), n_samples, params, rirs, [f"{len(x)}" for x in fg]))
        q, valid, _, _ = mix_ref(fg, bg, rirs, params, n_samples)
        return q, valid


@pytest.fixture
def golden_files(monkeypatch):
    reads = []

    def read_clip(path):
        reads.append(path)
        return Z[f"clip/{path}"]

    monkeypatch.setattr(data, "_read_clip", read_clip)
    monkeypatch.setattr(data, "_read_rir", lambda path: Z[f"rir/{path}"].astype(np.float32) / np.float32(32768))
    return reads


def run_config(name, mixer):
    gen = data.mix_clips_batch(background_clips=BGS, combined_size=N, audio_features=mixer, **CONFIGS[name])
    return next(gen)


def test_configurations_match_the_generator():
    assert sorted(NAMES) == sorted(CONFIGS)


@pytest.mark.parametrize("name", NAMES)
def test_draws_and_rng_states_match_the_reference(name, golden_files):
    mixer = FakeMixer()
    out, y, delayed = run_config(name, mixer)
    g = lambda k: Z[f"{name}/{k}"]
    assert golden_files == [str(s) for s in g("reads")]
    fg, bg, n, params, rirs, _ = mixer.calls[0]
    assert n == N and params.size == g("fg_len").size
    np.testing.assert_array_equal(params["fg_len"], g("fg_len"))
    np.testing.assert_array_equal(np.where(params["fg_len"] > 0, params["fg_start"], -1), g("fg_off"))
    np.testing.assert_array_equal(params["bg_offset"], g("bg_off"))
    np.testing.assert_array_equal(params["fg"], np.arange(params.size))
    np.testing.assert_array_equal(params["bg"], np.arange(params.size))
    np.testing.assert_array_equal(params["snr_db"], g("snr"))
    np.testing.assert_array_equal(params["start"], g("start"))
    if g("volume").size:
        np.testing.assert_array_equal(params["volume"], g("volume"))
    else:
        assert (params["volume"] < 0).all()
    if int(g("n_reverb")):
        assert (params["rir"] == 0).all() and len(rirs) == 1
        np.testing.assert_array_equal(rirs[0], g("rir").reshape(-1))
    else:
        assert (params["rir"] == -1).all() and rirs is None
    np.testing.assert_array_equal(np.random.get_state()[1], g("np_state"))
    assert np.random.get_state()[2] == int(g("np_pos"))
    assert random.getstate()[1] == tuple(int(v) for v in g("py_state"))
    # labels / frame labels of the kept rows
    valid = mix_ref(fg, bg, rirs, params, N)[1]
    want = g("sequence_labels") if CONFIGS[name].get("return_sequence_labels") else g("labels")
    np.testing.assert_array_equal(y, want[:params.size][valid])
    # delayed backgrounds: the reference gives none for a background exactly N + delay long (module docstring)
    if CONFIGS[name].get("return_background_clips"):
        delay = int(g("delay"))
        lens = np.array([len(x) for x in bg])
        has = lens != N + delay
        edge = g("delayed").shape[1] // 2
        mine = delayed if delayed is not None else np.zeros((0, N), np.int16)
        ref_rows = g("delayed")[:has.size][np.cumsum(has[:params.size]) - 1]        # the reference's list skips them
        for k in np.flatnonzero(valid):
            seg = mine[np.flatnonzero(valid).tolist().index(k)]
            if has[k]:
                np.testing.assert_array_equal(np.concatenate([seg[:edge], seg[-edge:]]), ref_rows[k])
            else:
                x = bg[k]
                np.testing.assert_array_equal(seg, ((x[delay:delay + N].astype(np.float32) / np.float32(32768))
                                                    * np.float32(32767)).astype(np.int16))
    else:
        assert delayed is None
    assert out.shape == (int(valid.sum()), N)


@pytest.mark.parametrize("name", NAMES)
def test_restatement_matches_the_reference_mixtures(name, golden_files):
    """Stage 3 of the contract against mix_clip's float32 outputs, within float32 round-off; and the whole row against
    the reference's int16 batch where it kept one (no reverb)"""
    mixer = FakeMixer()
    run_config(name, mixer)
    fg, bg, _, params, rirs, _ = mixer.calls[0]
    for k, p in enumerate(params):
        m, bad = mixture(fg[p["fg"]], bg[p["bg"]], N, p)
        assert bad == (p["fg_len"] == 0 or not np.any(fg[p["fg"]][p["fg_start"]:p["fg_start"] + p["fg_len"]]))
    if f"{name}/mixed" not in Z.files:
        return
    mixed, i16 = Z[f"{name}/mixed"], Z[f"{name}/int16"]
    q, valid, v, tau = mix_ref(fg, bg, rirs, params, N)
    for k, p in enumerate(params):
        m, _ = mixture(fg[p["fg"]], bg[p["bg"]], N, p)
        b = np.abs(bg[p["bg"]][(p["bg_offset"] + np.arange(N)) % len(bg[p["bg"]])] / 32768.0)
        np.testing.assert_array_less(np.abs(m - mixed[k]), 4 * 2.0 ** -24 * (b + 2 * np.abs(m)) + 1e-30)
        # the reference levels and truncates in float32: one step apart at most, where no int16 wrapped
        d = np.abs(q[k].astype(np.int64) - i16[k])
        assert d.max() <= 1 and (d == 0).mean() > 0.99


def test_truncation_windows_match_truncate_clip():
    for method_i, n, mx, first, count in Z["truncate"]:
        np.random.seed(int(n) * 1000 + int(mx))
        f, c = data.truncation_window(int(n), int(mx), TRUNC_METHODS[int(method_i)])
        assert c == count and (f == first or count == 0), (TRUNC_METHODS[int(method_i)], n, mx)


def test_frame_labels_are_exact():
    off = np.concatenate([[0], np.cumsum(Z["frame_len"])])
    for i, (cs, s, e) in enumerate(zip(Z["frame_cs"], Z["frame_s"], Z["frame_e"])):
        got = data.get_frame_labels(int(cs), int(s), int(e))
        want = Z["frame_labels"][off[i]:off[i + 1]]
        assert got.dtype == want.dtype
        np.testing.assert_array_equal(got, want)


def test_mix_clips_batch_refusals(golden_files, tmp_path):
    kw = dict(CONFIGS["noshuffle_start_norir"])
    with pytest.raises(ValueError, match="acoustics"):
        next(data.mix_clips_batch(background_clips=BGS, combined_size=N, audio_features=FakeMixer(),
                                  generated_noise_augmentation=0.5, **kw))
    kw["start_index"] = [0, -1, 0, 0, 0, 0]
    with pytest.raises(ValueError, match="start_index"):
        next(data.mix_clips_batch(background_clips=BGS, combined_size=N, audio_features=FakeMixer(), **kw))
    kw = dict(CONFIGS["noshuffle_start_norir"], start_index=[N - 100] * 6)     # the foreground runs past N
    with pytest.raises(ValueError, match="start"):
        next(data.mix_clips_batch(background_clips=BGS, combined_size=N, audio_features=FakeMixer(), **kw))


def test_rir_files_at_other_rates_are_refused(tmp_path):
    import wave
    for rate, ok in ((16000, True), (48000, False)):
        p = tmp_path / f"rir{rate}.wav"
        with wave.open(str(p), "wb") as w:
            w.setnchannels(2); w.setsampwidth(2); w.setframerate(rate)
            w.writeframes(np.arange(-20, 20, dtype="<i2").tobytes())
        if ok:
            h = data._read_rir(p)
            assert h.shape == (2, 20) and h[0, 0] == np.float32(-20 / 32768) and h[1, 0] == np.float32(-19 / 32768)
        else:
            with pytest.raises(ValueError, match="16 kHz"):
                data._read_rir(p)


def rec(**kw):
    p = np.zeros((), _native.MIX_DTYPE)
    base = dict(fg=0, bg=0, rir=-1, fg_start=0, fg_len=10, bg_offset=0, start=0, snr_db=0.0, volume=-1.0)
    base.update(kw)
    for k, v in base.items():
        p[k] = v
    return p


@pytest.mark.parametrize("kw", [dict(fg=1), dict(fg=-1), dict(bg=1), dict(rir=1), dict(rir=-2), dict(fg_start=-1),
                                dict(fg_len=21), dict(fg_start=15), dict(bg_offset=30), dict(bg_offset=-1),
                                dict(start=-1), dict(start=91), dict(rir=0, volume=np.nan), dict(snr_db=np.inf)])
def test_restatement_refusals(kw):
    p = rec(**kw)
    with pytest.raises(ValueError):
        check_record(p, [20], [30], [5], 100)
    check_record(rec(), [20], [30], [5], 100)


def test_restatement_refuses_long_and_empty_rirs():
    with pytest.raises(ValueError):
        check_record(rec(rir=0), [20], [30], [101], 100)
    with pytest.raises(ValueError):
        check_record(rec(rir=0), [20], [30], [0], 100)
    with pytest.raises(ValueError):
        check_record(rec(), [20], [0], [], 100)
    check_record(rec(rir=0, start=90), [20], [30], [100], 100)


def test_mix_dtype_is_the_c_record():
    assert _native.MIX_DTYPE.itemsize == 64
    assert [_native.MIX_DTYPE.fields[k][1] for k in ("fg", "bg", "rir", "fg_start", "fg_len", "bg_offset", "start",
                                                     "snr_db", "volume")] == [0, 4, 8, 16, 24, 32, 40, 48, 56]
