"""Log-mel frontend restatement (the graph inside ``melspectrogram.onnx``).

Follows notebooks/converting_google_speech_embedding_model.ipynb
lines 426-477 (torchlibrosa ``Spectrogram(center=False, n_fft=512, hop=160,
win=400)`` -> ``LogmelFilterBank(sr=16000, n_mels=32, fmin=60, fmax=3800)`` with
the patched ``power_to_db``) and openwakeword/utils.py:180-208
(int16 -> float32 *unscaled* in, ``x/10 + 2`` out).  torchlibrosa evaluates the
STFT as a conv1d with windowed DFT filters in float32; ``dtype`` selects that
(float32, faithful) or float64 (round-off yardstick).
"""
import numpy as np

N_FFT = 512
HOP = 160
WIN = 400
N_MELS = 32
SR = 16000
FMIN = 60.0
FMAX = 3800.0
AMIN = 1e-10
TOP_DB = 80.0
N_BINS = N_FFT // 2 + 1


def hann_window_padded():
    """Periodic Hann(400) centred in 512 samples (56 zeros each side).
    scipy.signal.get_window('hann', 400, fftbins=True) == 0.5-0.5cos(2*pi*n/400);
    librosa.util.pad_center -> lpad = (512-400)//2 (nb/conv:434,437)."""
    n = np.arange(WIN, dtype=np.float64)
    w = 0.5 - 0.5 * np.cos(2.0 * np.pi * n / WIN)
    out = np.zeros(N_FFT, dtype=np.float64)
    lpad = (N_FFT - WIN) // 2
    out[lpad:lpad + WIN] = w
    return out


def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    with np.errstate(divide="ignore", invalid="ignore"):
        log_t = min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep
    return np.where(f >= min_log_hz, log_t, mels)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    freqs = f_sp * m
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), freqs)


def mel_filterbank():
    """Slaney-scale, Slaney-normalised triangular filterbank, [257, 32] float32
    (librosa.filters.mel(sr=16000, n_fft=512, n_mels=32, fmin=60, fmax=3800).T,
    nb/conv:463-470; SURVEY.md Appendix A.5)."""
    fftfreqs = np.linspace(0.0, SR / 2.0, N_BINS)
    mel_pts = np.linspace(_hz_to_mel(FMIN), _hz_to_mel(FMAX), N_MELS + 2)
    mel_f = _mel_to_hz(mel_pts)
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    W = np.zeros((N_MELS, N_BINS), dtype=np.float64)
    for i in range(N_MELS):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        W[i] = np.maximum(0.0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:N_MELS + 2] - mel_f[:N_MELS])
    W *= enorm[:, None]
    return W.T.astype(np.float32)


def dft_filters(dtype=np.float32):
    """Windowed DFT filters as torchlibrosa builds them: real/imag [512, 257]."""
    n = np.arange(N_FFT, dtype=np.float64)[:, None]
    k = np.arange(N_BINS, dtype=np.float64)[None, :]
    ang = -2.0 * np.pi * n * k / N_FFT
    w = hann_window_padded()[:, None]
    return (np.cos(ang) * w).astype(dtype), (np.sin(ang) * w).astype(dtype)


_CACHE = {}


def _consts(dtype):
    key = np.dtype(dtype).name
    if key not in _CACHE:
        cr, ci = dft_filters(dtype)
        _CACHE[key] = (cr, ci, mel_filterbank().astype(dtype))
    return _CACHE[key]


def n_frames(n_samples):
    return (n_samples - N_FFT) // HOP + 1 if n_samples >= N_FFT else 0


def melspectrogram_raw(x, dtype=np.float32):
    """One ``melspec_model_predict`` call on ONE clip: x int16/float [n] ->
    dB log-mel [T, 32] *before* the x/10+2 affine.  The ``top_db`` clamp uses the
    max over the whole output of this call (nb/conv:449-452; SURVEY.md F7)."""
    x = np.asarray(x)
    if x.ndim != 1:
        raise ValueError("melspectrogram_raw takes one 1-D clip")
    T = n_frames(x.shape[0])
    if T <= 0:
        raise ValueError("need at least 512 samples")
    cr, ci, melW = _consts(dtype)
    xf = x.astype(np.float32).astype(dtype)           # utils.py:199 - no scaling
    idx = np.arange(T)[:, None] * HOP + np.arange(N_FFT)[None, :]
    frames = xf[idx]                                  # [T, 512]
    re = frames @ cr
    im = frames @ ci
    power = re * re + im * im                         # power=2
    mel = power @ melW                                # [T, 32]
    ten = dtype(10.0)
    log_spec = ten * np.log(np.maximum(mel, dtype(AMIN))) / np.log(ten)
    log_spec = log_spec - ten * np.log(np.maximum(dtype(AMIN), dtype(1.0))) / np.log(ten)
    log_spec = np.maximum(log_spec, log_spec.max() - dtype(TOP_DB))
    return log_spec.astype(np.float32)


def melspectrogram(x, dtype=np.float32):
    """``AudioFeatures._get_melspectrogram`` on one clip (utils.py:180-208):
    raw dB mel then ``spec/10 + 2``."""
    return (melspectrogram_raw(x, dtype) / np.float32(10.0) + np.float32(2.0)).astype(np.float32)
