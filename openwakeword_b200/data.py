"""Evaluation clips on the device: the reference's ``openwakeword.data.mix_clips_batch`` (data.py:294-478), which mixes
clean positive clips with background noise at a random SNR, reverberates them with a room impulse response (RIR) and
levels them, the test data of a false-reject evaluation (README "Performance and Evaluation"; docs/models/alexa.md:72).

Each batch is one ``oww_mix_clips`` call (include/owwb200.h); the host only reads files and draws the random values,
with ``np.random`` / ``random`` in the reference's order, so a seeded call picks the same clips, windows, offsets, SNRs,
RIRs and volumes.  Two defects of the reference are not reproduced:

- data.py:466 calls ``ndarray.max(dim=1)`` on the int16 batch, which NumPy refuses (TypeError), so the reference never
  yields a batch.  Here the rows whose largest sample is 0 are dropped, which is what the line means to do, together
  with the rows ``oww_mix_clips`` marks invalid (a silent foreground or background, or a non-positive maximum under the
  volume rule).
- A background exactly ``combined_size + delay`` samples long gets no delayed segment in the reference (neither branch
  of data.py:410-419 runs), so the returned segments no longer line up with the clips; with a delay it then fails its
  own length check.  Here such a background is mixed from its start and its delayed segment is
  ``bg[delay:delay + combined_size]``.

Without ``start_index`` every foreground starts at sample 0 (the reference builds ``batch_size`` zeros, which fails to
index when there are more foreground clips than that).  Out-of-range int16 values saturate instead of wrapping
(include/owwb200.h).  ``generated_noise_augmentation > 0`` raises ValueError: colored noise needs ``acoustics``.
"""
import random
import wave

import numpy as np

from . import _native, utils

_SR = 16000
_MIXER = None


class _ContextMixer:
    """oww_mix_clips on a bare handle: mixing needs no model weights"""

    def __init__(self, device_index=0):
        self.ctx = _native.Context(device=device_index)
        self.device_index = device_index

    def mix_clips(self, fg, bg, n_samples, params, rirs=None):
        return utils._mix_clips_on(self.ctx, self.device_index, fg, bg, n_samples, params, rirs)


def _default_mixer():
    global _MIXER
    if _MIXER is None:
        _MIXER = _ContextMixer()
    return _MIXER


def _read_clip(path):
    """16-bit, 16 kHz, single-channel WAV -> int16 samples"""
    return utils._read_wav(path)


def _read_rir(path):
    """16-bit WAV at 16 kHz, any channel count -> float32 [channels, taps] (s / 32768, as torchaudio.load reads it).
    The reference ignores an RIR's rate; one at another rate would reverberate at the wrong time scale, so it is
    refused."""
    with wave.open(str(path), mode="rb") as f:
        if f.getsampwidth() != 2:
            raise ValueError(f"{path}: expected a 16-bit WAV room impulse response")
        if f.getframerate() != _SR:
            raise ValueError(f"{path}: room impulse responses must be 16 kHz, this one is {f.getframerate()} Hz")
        c = f.getnchannels()
        pcm = np.frombuffer(f.readframes(f.getnframes()), dtype="<i2").reshape(-1, c).T
    return (pcm.astype(np.float32) / np.float32(32768)).astype(np.float32)


def truncation_window(n, max_size, method="truncate_start"):
    """The samples ``truncate_clip(x, max_size, method)`` (data.py:499-527) keeps of a clip of n samples, as
    (first, count); "random" draws its ``np.random.randint`` as the reference does."""
    if n <= max_size:
        return 0, n
    if method == "truncate_start":
        return n - max_size, max_size
    if method == "truncate_end":
        return 0, max_size
    if method == "truncate_both":
        k = int(np.ceil(n - max_size) / 2)
        return (k, min(max_size, n - 2 * k)) if k > 0 else (0, 0)     # x[k:-k] is empty for k = 0
    if method == "random":
        first = np.random.randint(0, n - max_size)
        return first, max_size
    return 0, n


def get_frame_labels(combined_size, start, end, buffer=1):
    """Frame labels of a clip of combined_size samples whose foreground spans [start, end): the embedding frames
    (every 1280 samples from sample 12400) nearest the start and the end are marked, two frames each (data.py:481-488,
    ``buffer`` is unused there too)."""
    frames = np.arange(12400, combined_size, 1280)
    labels = np.zeros(np.ceil((combined_size - 12400) / 1280).astype(int))
    first = np.argmin(abs(frames - start))
    last = np.argmin(abs(frames - end))
    labels[first:first + 2] = 1
    labels[last - 1:last + 1] = 1          # Python slicing: with last = 0 this marks nothing unless there is one frame
    return labels


def _background_window(n, combined_size, delay):
    """(offset of the mixed segment, offset of the delayed segment) of a background of n samples; draws the crop's
    ``np.random.randint`` as data.py:410-419 does.  Offsets are taken modulo n (the reference tiles short clips)."""
    if n < combined_size + delay:
        return 0, delay % n
    if n > combined_size + delay:
        r = np.random.randint(0, max(1, n - combined_size - delay))
        return r, r + delay
    return 0, delay


def mix_clips_batch(foreground_clips, background_clips, combined_size, labels=[], batch_size=32, snr_low=0, snr_high=0,
                    start_index=[], foreground_durations=[], foreground_truncate_strategy="random", rirs=[],
                    rir_probability=1, volume_augmentation=True, generated_noise_augmentation=0.0, shuffle=True,
                    return_sequence_labels=False, return_background_clips=False, return_background_clips_delay=(0, 0),
                    seed=0, audio_features=None):
    """The reference's generator (data.py:294-478) with each batch mixed on the device in one call.  Yields
    (int16 [n, combined_size], labels [n] or frame labels [n, frames], int16 delayed background segments [n,
    combined_size] or None), host arrays, without the rows the device marks invalid.  ``audio_features``: an
    ``AudioFeatures`` (or anything with its ``mix_clips``) to mix on; default a handle on cuda:0."""
    if generated_noise_augmentation > 0:
        raise ValueError("generated_noise_augmentation needs colored noise from the `acoustics` package, which is not "
                         "provided; use 0.0")
    mixer = audio_features if audio_features is not None else _default_mixer()
    if seed:
        np.random.seed(seed)
        random.seed(seed)
    N = int(combined_size)
    n_fg = len(foreground_clips)
    if not start_index:
        start_index = [0] * n_fg
    elif min(start_index) < 0:
        raise ValueError("Error! At least one value of the `start_index` argument is <0. Check your inputs.")
    if not labels:
        labels = [0] * n_fg
    fg_paths = list(foreground_clips)
    if shuffle:
        p = np.random.permutation(n_fg)
        fg_paths = np.array(fg_paths)[p].tolist()
        start_index = np.array(start_index)[p].tolist()
        labels = np.array(labels)[p].tolist()
        if foreground_durations:
            foreground_durations = np.array(foreground_durations)[p].tolist()

    for i in range(0, n_fg, batch_size):
        starts = start_index[i:i + batch_size]
        fg = [_read_clip(f) for f in fg_paths[i:i + batch_size]]
        if foreground_durations:
            windows = [truncation_window(len(x), int(k * _SR), foreground_truncate_strategy)
                       for x, k in zip(fg, foreground_durations[i:i + batch_size])]
        else:
            windows = [(0, len(x)) for x in fg]
        labels_batch = np.array(labels[i:i + batch_size])

        bg = [_read_clip(b) for b in random.sample(background_clips, batch_size)]
        delay = np.random.randint(return_background_clips_delay[0], return_background_clips_delay[1] + 1)
        bg_windows = [_background_window(len(x), N, delay) for x in bg]
        snrs_db = np.random.uniform(snr_low, snr_high, batch_size)
        n = min(len(windows), len(starts))
        params = np.zeros(n, _native.MIX_DTYPE)
        sequence_labels = []
        for k in range(n):
            first, count = windows[k]
            params[k] = (k, k, -1, 0, first, count, bg_windows[k][0], starts[k], snrs_db[k], -1.0)
            sequence_labels.append(get_frame_labels(N, starts[k], starts[k] + count))
            np.random.random()             # the colored-noise draw, made whatever its probability
        rir = None
        if rirs and np.random.random() <= rir_probability:
            h = _read_rir(random.choice(rirs))
            h = h[random.randint(0, h.shape[0] - 1)] if h.shape[0] > 1 else h[0]
            rir = [h]
            params["rir"] = 0
        if volume_augmentation:
            params["volume"] = np.random.uniform(0.02, 1.0, n)
        out, valid = mixer.mix_clips(fg[:n], bg, N, params, rir)
        out = out.cpu().numpy() if hasattr(out, "cpu") else np.asarray(out)
        keep = np.flatnonzero(valid.cpu().numpy() if hasattr(valid, "cpu") else np.asarray(valid))
        if return_sequence_labels:
            y = np.vstack(sequence_labels)[keep] if sequence_labels else np.zeros((0, 0))
        else:
            y = labels_batch[keep]
        delayed = None
        if return_background_clips:
            seg = np.stack([np.take(x, np.arange(o, o + N), mode="wrap") for x, (_, o) in zip(bg[:n], bg_windows)])
            delayed = ((seg.astype(np.float32) / np.float32(32768)) * np.float32(32767)).astype(np.int16)[keep]
        yield out[keep], y, delayed
