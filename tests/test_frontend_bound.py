"""CPU: a round-off bound for the log-mel frontend against the float64 yardstick (oracle.mel.mel_power_f64).

The flat 5e-3 tolerance of the parity tests (x/10+2 scale, 0.05 dB) is set by the float32 dense-DFT oracle's noise in
quiet bins and accepts a frontend whose filterbank is 0.1 % off.  The bound here scales with each element's level:
for frame t and filter j, with m the float64 mel power and E the frame energy over all 257 bins,

    d   = 10 log10(max(m, 1e-10))
    tau = (10 / ln 10) C eps32 (1 + sqrt(E / max(m, 1e-10))) + 8 ulp32(max(|d|, 1))

An FFT's absolute error per bin scales with sqrt(E), so a bin's relative power error scales with sqrt(E / m).  The
reference is r = max(d, D - 80) with D the call's maximum of d, and an element passes when |dev - r| <= max(tau,
tau at the argmax of d): max is 1-Lipschitz, so a clamped element carries the error of the call maximum.

This module checks that a float32 emulation of the frontend (scipy's rfft) passes the bound at the constant C the
kernels are held to, and that four small perturbations of the constants fail it by at least 2x.  tests/test_gpu_frontend.py
applies the same bound and guards to the CUDA frontend."""
import numpy as np
import pytest
import scipy.fft

from oracle import mel as M

EPS32 = 2.0 ** -23
# Round-off constant of the bound: the smallest power of two at least 4x the worst ratio the CUDA frontend reaches at
# C = 1 on the signal zoo.  Measured on an H100 80GB HBM3 (400 W limit): 0.19, so C = 1 (tests/test_gpu_frontend.py
# prints it and fails once the headroom is gone).  Above 16 the fp16-filterbank guard would lose its 2x margin.
C_ROUNDOFF = 1.0
GUARD_MARGIN = 2.0


def bound_ratio(dev_db, m, E, C=C_ROUNDOFF):
    """Worst |dev - r| / tolerance of ONE call (one clamp group): dev_db [T, 32] raw dB as the frontend returns it
    (clamped, before x/10+2); m [T, 32], E [T] from oracle.mel.mel_power_f64.  <= 1 passes."""
    dev = np.asarray(dev_db, np.float64)
    mc = np.maximum(np.asarray(m, np.float64), M.AMIN)
    d = 10.0 * np.log10(mc)
    ulp = np.spacing(np.maximum(np.abs(d), 1.0).astype(np.float32)).astype(np.float64)
    tau = (10.0 / np.log(10.0)) * C * EPS32 * (1.0 + np.sqrt(np.asarray(E, np.float64)[:, None] / mc)) + 8.0 * ulp
    top = np.unravel_index(np.argmax(d), d.shape)
    r = np.maximum(d, d[top] - M.TOP_DB)
    return float((np.abs(dev - r) / np.maximum(tau, tau[top])).max())


def default_constants():
    """The built-in constants as oww_load_mel holds them: float32 window [512] and filterbank [257, 32]."""
    return M.hann_window_padded().astype(np.float32), M.mel_filterbank()


def perturbations():
    """name -> (window, filterbank): small errors the bound must catch, each against the UNperturbed reference."""
    win, fb = default_constants()
    f7 = fb.copy()
    f7[:, 7] *= np.float32(1.01)
    n = np.arange(M.WIN, dtype=np.float64)
    sym = np.zeros(M.N_FFT, np.float32)
    sym[56:456] = 0.5 - 0.5 * np.cos(2.0 * np.pi * n / (M.WIN - 1))
    return {"filter7_x1.01": (win, f7),
            "fp16_filterbank": (win, fb.astype(np.float16).astype(np.float32)),
            "symmetric_hann": (sym, fb),
            "window_shift_1": (np.roll(win, 1), fb)}


def corner_frequencies():
    """The 34 corner frequencies of the Slaney filterbank (60 .. 3800 Hz)."""
    return M._mel_to_hz(np.linspace(M._hz_to_mel(M.FMIN), M._hz_to_mel(M.FMAX), M.N_MELS + 2))


def _tone(L, hz, amp, phase):
    return amp * np.cos(2.0 * np.pi * hz * np.arange(L) / M.SR + phase)


def zoo(L, seed=0):
    """The signal zoo at length L: list of (group, int16 [L]).  Bin tones sit exactly on FFT bins (k * 31.25 Hz)."""
    rng = np.random.default_rng(seed)
    n = np.arange(L)
    out = [("square", np.where((n // 8) % 2 == 0, 32767, -32768)),
           ("square", np.where((n // 25) % 2 == 0, -32768, 32767)),
           ("dc_-32768", np.full(L, -32768)),
           ("silence", np.zeros(L))]
    for pos in (2 * ((L // 3) // 2), 2 * ((L // 3) // 2) + 1, 0, L - 1):       # even and odd positions, both ends
        x = np.zeros(L)
        x[pos] = -32768 if pos % 2 else 32767
        out.append(("impulse_odd" if pos % 2 else "impulse_even", x))
    for k in (0, 1, 2, 37, 128, 200, 255, 256):
        out.append(("bin_tone", _tone(L, k * M.SR / M.N_FFT, 30000.0, rng.uniform(0, 2 * np.pi))))
    cf = corner_frequencies()
    for hz in cf[rng.choice(cf.size, 4, replace=False)]:
        out.append(("corner_tone", _tone(L, hz, 20000.0, rng.uniform(0, 2 * np.pi))))
    for hz in (3810.0, 4500.0, 7000.0, 7990.0):
        out.append(("tone_above_3800", _tone(L, hz, 32000.0, rng.uniform(0, 2 * np.pi))))
    out.append(("chirp", 30000.0 * np.cos(np.pi * (M.SR / 2) * n ** 2 / (M.SR * max(L, 1)))))
    out.append(("lsb_noise", rng.integers(-1, 2, L)))
    x = rng.integers(-1, 2, L).astype(np.float64)
    p = int(rng.integers(0, L - 511))
    x[p:p + 512] = rng.integers(-32768, 32768, 512)
    out.append(("lsb_noise_one_loud_frame", x))
    out.append(("full_scale_noise", rng.integers(-32768, 32768, L)))
    return [(g, np.clip(np.round(x), -32768, 32767).astype(np.int16)) for g, x in out]


def bin_sweep(L, seed=0):
    """One tone exactly on each FFT bin 0..256 and one on each filter corner: (groups, int16 [291, L])."""
    rng = np.random.default_rng(seed)
    hz = np.concatenate([np.arange(M.N_BINS) * M.SR / M.N_FFT, corner_frequencies()])
    x = np.stack([_tone(L, f, 25000.0, rng.uniform(0, 2 * np.pi)) for f in hz])
    groups = ["bin_tone"] * M.N_BINS + ["corner_tone"] * (hz.size - M.N_BINS)
    return groups, np.clip(np.round(x), -32768, 32767).astype(np.int16)


def emulate_f32(x, window, mel_fb):
    """The frontend in float32 on the CPU (scipy rfft), raw dB with the per-call clamp: [T, 32]."""
    T = M.n_frames(x.shape[0])
    idx = np.arange(T)[:, None] * M.HOP + np.arange(M.N_FFT)[None, :]
    X = scipy.fft.rfft(x.astype(np.float32)[idx] * np.asarray(window, np.float32)[None, :], axis=1)
    p = X.real * X.real + X.imag * X.imag
    mel = p.astype(np.float32) @ np.asarray(mel_fb, np.float32)
    db = np.float32(10.0) * np.log10(np.maximum(mel, np.float32(M.AMIN)))
    return np.maximum(db, db.max() - np.float32(M.TOP_DB))


def _cases():
    cases = [zg for L in (512, 1761, 16000) for zg in zoo(L, seed=L)]
    g, x = bin_sweep(1761)
    return cases + list(zip(g, x))


@pytest.fixture(scope="module")
def references():
    win, fb = default_constants()
    return [(g, x, M.mel_power_f64(x, win, fb)) for g, x in _cases()]


def _worst(refs, window, mel_fb, C):
    return max(bound_ratio(emulate_f32(x, window, mel_fb), m, E, C) for _, x, (m, E) in refs)


def test_float32_fft_passes_the_bound(references):
    win, fb = default_constants()
    per = {}
    for g, x, (m, E) in references:
        per[g] = max(per.get(g, 0.0), bound_ratio(emulate_f32(x, win, fb), m, E, 1.0))
    print("\nscipy float32 frontend, worst ratio at C = 1:", {g: round(v, 4) for g, v in per.items()})
    assert _worst(references, win, fb, C_ROUNDOFF) <= 1.0, per


@pytest.mark.parametrize("name", sorted(perturbations()))
def test_perturbed_constants_fail_the_bound(references, name):
    win, fb = perturbations()[name]
    r = _worst(references, win, fb, C_ROUNDOFF)
    print(f"\n{name}: worst ratio {r:.3g} at C = {C_ROUNDOFF:g}")
    assert r >= GUARD_MARGIN, (name, r)


def test_f64_power_matches_the_dense_dft_oracle():
    """mel_power_f64 (rfft) and melspectrogram_raw in float64 (dense DFT) are the same frontend, custom constants too."""
    rng = np.random.default_rng(3)
    x = rng.integers(-20000, 20000, 4000).astype(np.int16)
    for win, fb in [(None, None)] + list(perturbations().values()):
        m, _ = M.mel_power_f64(x, win, fb)
        d = 10.0 * np.log10(np.maximum(m, M.AMIN))
        ref = np.maximum(d, d.max() - M.TOP_DB)
        got = M.melspectrogram_raw(x, np.float64, window=win, mel_fb=fb)
        np.testing.assert_allclose(got, ref.astype(np.float32), rtol=0, atol=1e-4)


def test_oracle_defaults_are_unchanged():
    """Passing nothing is the built-in graph; the built-in constants passed explicitly stay within float32 rounding."""
    rng = np.random.default_rng(4)
    x = rng.integers(-3000, 3000, 16000).astype(np.int16)
    a = M.melspectrogram_raw(x)
    assert np.array_equal(a, M.melspectrogram_raw(x, np.float32, None, None))
    np.testing.assert_allclose(M.melspectrogram_raw(x, np.float32, *default_constants()), a, rtol=0, atol=2e-4)
    with pytest.raises(ValueError):
        M.melspectrogram_raw(x, window=np.ones(400))
    with pytest.raises(ValueError):
        M.mel_power_f64(x, mel_fb=np.ones((32, 257)))
