"""Generate tests/golden/mix.npz from the UNMODIFIED reference data.py (openwakeword/data.py of the original openWakeWord
project, OWW_REFERENCE = its root directory):
    OWW_REFERENCE=/path/to/openWakeWord python tests/golden/make_mix_golden.py

Stub modules stand in for data.py's imports that are not installed (pronouncing, audiomentations, torch_audiomentations,
speechbrain, mutagen, acoustics) and for torchaudio.load.  ``read_audio`` serves seeded int16 clips / 32768 by path and
logs the order of its calls; ``reverberate`` records its batch and RIR and returns the batch unchanged (speechbrain's
reverb is not compared); ``data.mix_clip`` is wrapped to record its inputs and output.  mix_clips_batch stops at
data.py:466 with TypeError on its first batch; the generator's frame at that point holds the volumes, labels, frame
labels and delayed backgrounds, and the RNG states then are those after the batch.  Also records truncate_clip and
get_frame_labels over a grid."""
import importlib.util
import os
import random
import sys
import types
import zlib

import numpy as np
import torch

N = 14000
SR = 16000


def clip(path, n):
    rng = np.random.default_rng(zlib.crc32(path.encode()))
    return rng.integers(-12000, 12000, n).astype(np.int16)


FG = {f"fg{i}.wav": clip(f"fg{i}.wav", n) for i, n in enumerate([6000, 9000, 4000, 7501, 12000, 3000])}
FG["fg_silent.wav"] = np.zeros(5000, np.int16)
BG = {f"bg{i}.wav": clip(f"bg{i}.wav", n) for i, n in enumerate([3000, 5500, N, 15000, 16000, 14100])}
RIR = {"rir_mono.wav": clip("rir_mono.wav", 700)[None], "rir_stereo.wav": clip("rir_stereo.wav", 2 * 900).reshape(2, 900)}
for r in RIR.values():          # a decaying response with its peak a few taps in
    r[...] = (r * np.exp(-np.arange(r.shape[1]) / 150.0)).astype(np.int16)
    r[:, 5] = 30000

READS, MIXES, REVERBS = [], [], []


def read_audio(path):
    READS.append(path)
    x = FG.get(path, BG.get(path))
    return torch.from_numpy(x.astype(np.float32) / np.float32(32768))


def reverberate(x, h, rescale_amp="avg"):
    REVERBS.append((x.numpy().copy(), np.asarray(h, np.float32).copy()))
    return x


def torchaudio_load(path):
    return torch.from_numpy(RIR[path].astype(np.float32) / np.float32(32768)), SR


def stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


for name in ("pronouncing", "audiomentations", "torch_audiomentations", "mutagen", "acoustics", "speechbrain",
             "speechbrain.dataio", "speechbrain.processing"):
    stub(name)
stub("speechbrain.dataio.dataio", read_audio=read_audio)
stub("speechbrain.processing.signal_processing", reverberate=reverberate)
stub("torchaudio", load=torchaudio_load)

spec = importlib.util.spec_from_file_location("ref_data", os.path.join(os.environ["OWW_REFERENCE"], "openwakeword", "data.py"))
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)
_mix_clip = ref.mix_clip


def mix_clip(fg, bg, snr, start):
    fg_in, bg_in = fg.numpy().copy(), bg.numpy().copy()
    out = _mix_clip(fg, bg, snr, start)
    MIXES.append((fg_in, bg_in, float(snr), int(start), out.numpy().copy()))
    return out


ref.mix_clip = mix_clip

FGS = ["fg0.wav", "fg1.wav", "fg2.wav", "fg3.wav", "fg4.wav", "fg5.wav"]
BGS = list(BG)
CONFIGS = [   # (name, keyword arguments of mix_clips_batch); every call draws batch_size backgrounds
    ("shuffle_random_rir", dict(foreground_clips=FGS, batch_size=4, snr_low=-5, snr_high=15, start_index=[100, 0, 2000, 50, 1000, 30],
                                foreground_durations=[0.3, 0.5, 0.2, 0.4, 0.6, 0.1], foreground_truncate_strategy="random",
                                rirs=["rir_mono.wav", "rir_stereo.wav"], rir_probability=1, shuffle=True,
                                return_background_clips=True, return_background_clips_delay=(10, 200), seed=3)),
    ("noshuffle_start_norir", dict(foreground_clips=FGS, batch_size=4, snr_low=0, snr_high=10, start_index=[0, 10, 20, 30, 40, 50],
                                   foreground_durations=[0.3, 0.5, 0.2, 0.4, 0.6, 0.1], foreground_truncate_strategy="truncate_start",
                                   rirs=["rir_mono.wav"], rir_probability=0, volume_augmentation=False, shuffle=False,
                                   return_sequence_labels=True, return_background_clips=True,
                                   return_background_clips_delay=(0, 0), seed=5)),
    ("shuffle_end_stereo", dict(foreground_clips=FGS, batch_size=4, snr_low=5, snr_high=6, start_index=[7, 8, 9, 10, 11, 12],
                                foreground_durations=[0.25, 0.25, 0.25, 0.25, 0.25, 0.25], foreground_truncate_strategy="truncate_end",
                                rirs=["rir_stereo.wav"], rir_probability=1, shuffle=True, return_sequence_labels=True,
                                return_background_clips=True, return_background_clips_delay=(10, 200), seed=11)),
    ("noshuffle_both", dict(foreground_clips=FGS, batch_size=4, snr_low=10, snr_high=10, start_index=[500, 600, 700, 800, 900, 1000],
                            foreground_durations=[0.3, 0.5, 0.2, 0.46875, 0.6, 0.1], foreground_truncate_strategy="truncate_both",
                            shuffle=False, volume_augmentation=False, return_background_clips=True,
                            return_background_clips_delay=(0, 0), seed=7)),
    ("short_batch_full_clips", dict(foreground_clips=["fg1.wav", "fg_silent.wav"], batch_size=5, snr_low=-10, snr_high=20,
                                    start_index=[3000, 1], labels=[1, 0], rirs=["rir_mono.wav", "rir_stereo.wav"],
                                    rir_probability=1, shuffle=True, seed=13)),
]


KEEP_MIXED = ("noshuffle_start_norir",)     # mix_clip outputs and the int16 batch kept for these configurations
EDGE = 256                                  # samples kept of each end of a delayed background segment


def locate(seg, x, wrap=False):
    """offset of the float32 segment seg (samples / 32768) in the int16 clip x, modulo len(x) when wrap; -1: empty"""
    if seg.size == 0:
        return -1
    s = np.round(seg * 32768).astype(np.int64)
    n = x.size
    for o in range(n):
        idx = (o + np.arange(min(s.size, 64))) % n if wrap else o + np.arange(min(s.size, 64))
        if (wrap or o + s.size <= n) and np.array_equal(x[idx], s[:idx.size]):
            full = x[(o + np.arange(s.size)) % n] if wrap else x[o:o + s.size]
            if np.array_equal(full, s):
                return o
    raise SystemExit("segment not found")


def run(kw):
    READS.clear(); MIXES.clear(); REVERBS.clear()
    gen = ref.mix_clips_batch(background_clips=BGS, combined_size=N, **kw)
    try:
        next(gen)
        raise SystemExit("the reference yielded a batch: data.py:466 no longer fails, regenerate by hand")
    except TypeError:
        tb = sys.exc_info()[2]
        while tb.tb_next is not None and tb.tb_frame.f_code.co_name != "mix_clips_batch":
            tb = tb.tb_next
        loc = tb.tb_frame.f_locals
    return loc


def main():
    out = {"N": N}
    for k, v in list(FG.items()) + list(BG.items()):
        out[f"clip/{k}"] = v
    for k, v in RIR.items():
        out[f"rir/{k}"] = v
    out["config_names"] = np.array([c[0] for c in CONFIGS])
    for name, kw in CONFIGS:
        loc = run(kw)
        p = f"{name}/"
        out[p + "reads"] = np.array(READS)
        out[p + "fg_len"] = np.array([m[0].size for m in MIXES])
        out[p + "fg_off"] = np.array([locate(m[0], FG[path]) for m, path in zip(MIXES, READS)])
        out[p + "bg_off"] = np.array([locate(m[1], BG[path], wrap=True) for m, path in zip(MIXES, READS[len(MIXES):])])
        out[p + "snr"] = np.array([m[2] for m in MIXES])
        out[p + "start"] = np.array([m[3] for m in MIXES])
        if name in KEEP_MIXED:
            out[p + "mixed"] = np.stack([m[4] for m in MIXES]).astype(np.float32)
            out[p + "int16"] = loc["mixed_clips_batch"]
        out[p + "rir"] = REVERBS[0][1] if REVERBS else np.zeros(0, np.float32)
        out[p + "n_reverb"] = len(REVERBS)
        out[p + "delay"] = int(loc["delay"])
        d = loc["background_clips_batch_delayed"]       # what data.py:474-475 makes of it
        d = (np.stack([t.numpy() for t in d]) * 32767).astype(np.int16) if d else np.zeros((0, N), np.int16)
        out[p + "delayed"] = np.concatenate([d[:, :EDGE], d[:, -EDGE:]], axis=1)     # its two ends pin each segment
        out[p + "volume"] = loc["volume_levels"] if "volume_levels" in loc else np.zeros(0)
        out[p + "labels"] = loc["labels_batch"]
        out[p + "sequence_labels"] = loc["sequence_labels_batch"].numpy()
        st = np.random.get_state()
        out[p + "np_state"] = st[1]
        out[p + "np_pos"] = st[2]
        out[p + "py_state"] = np.array(random.getstate()[1])
    # truncate_clip and get_frame_labels over a grid
    trunc = []
    for method in ("truncate_start", "truncate_end", "truncate_both", "random", "other"):
        for n in (1, 5, 6, 7, 8, 100, 101):
            for mx in (0, 1, 5, 6, 50, 99, 100, 120):
                np.random.seed(n * 1000 + mx)
                x = np.arange(n)
                y = ref.truncate_clip(x, mx, method)
                trunc.append((["truncate_start", "truncate_end", "truncate_both", "random", "other"].index(method), n, mx,
                              int(y[0]) if y.size else -1, y.size))
    out["truncate"] = np.array(trunc, np.int64)
    fl = []
    for cs in (12401, 13680, 13681, 14000, 16000, 32000):
        for s in (0, 1, 639, 640, 641, 12400, 13040, 13041, 20000):
            for e in (s, s + 1, s + 640, s + 1280, s + 5000, cs):
                fl.append((cs, s, e, ref.get_frame_labels(cs, s, e)))
    out["frame_cs"] = np.array([f[0] for f in fl])
    out["frame_s"] = np.array([f[1] for f in fl])
    out["frame_e"] = np.array([f[2] for f in fl])
    out["frame_labels"] = np.concatenate([f[3] for f in fl])
    out["frame_len"] = np.array([f[3].size for f in fl])
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mix.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
