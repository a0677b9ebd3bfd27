"""The detector's rules (openwakeword/model.py:328-363; include/owwb200.h, oww_detect) restated in float64 NumPy over all
streams at once, with every parameter per (stream, label): threshold, patience, and a debounce per stream.  The
threshold is taken at fp32 (as the handle stores it) and compared in float64, which orders fp32 values as fp32 does,
so the restatement must equal the device bit for bit: the rules only select and copy values."""
import numpy as np

HISTORY = 30
ZEROED = 5


class StreamRules:
    """B streams of L labels: columns int [L] (-1: always 0.0), repeats bool [L]; the history hist float64 [B, L, 30]
    (newest last, zeros before the first prediction) and count int64 [B] (predictions appended since the reset)."""

    def __init__(self, B, columns, repeats):
        self.columns, self.repeats = np.asarray(columns, np.int64), np.asarray(repeats, bool)
        self.hist = np.zeros((B, self.columns.size, HISTORY))
        self.count = np.zeros(B, np.int64)

    def step(self, scores, prepared, threshold, patience, debounce):
        """scores [B, columns] (not read for prepared < 1280), prepared int [B] (< 0: skipped), threshold [B, L] (NaN:
        none), patience int [B, L] (0: none), debounce [B] seconds (0: off) -> (final float64 [B, L], NaN in skipped
        rows; fired bool [B, L])."""
        B, L = self.hist.shape[:2]
        prepared = np.broadcast_to(np.asarray(prepared, np.int64), (B,))
        thr = np.asarray(threshold, np.float32).astype(np.float64)
        pat = np.asarray(patience, np.int64)
        deb = np.broadcast_to(np.asarray(debounce, np.float64), (B,))
        c = self.count
        n = np.minimum(c, HISTORY)
        age = np.arange(HISTORY)[::-1]                               # slot k of hist holds the entry of age 29 - k
        sc = np.asarray(scores, np.float32).astype(np.float64)[:, np.maximum(self.columns, 0)]
        sc = np.where(self.columns[None] >= 0, sc, 0.0)
        prev = np.where((c[:, None] > 0) & self.repeats[None], self.hist[:, :, -1], 0.0)
        pred = np.where((prepared >= 1280)[:, None], sc, prev)
        pred = np.where((c < ZEROED)[:, None], 0.0, pred)
        ge = self.hist >= thr[:, :, None]                            # NaN: never
        # patience: fewer than `patience` of the last min(patience, count) entries are >= the threshold
        win = age[None, None, :] < np.minimum(pat, n[:, None])[:, :, None]
        p_zero = (pred != 0.0) & ((ge & win).sum(-1) < pat)
        # debounce: one of the last min(count, ceil(debounce / (prepared / 16000))) entries (all of them at 0) is >= it
        with np.errstate(divide="ignore", invalid="ignore"):
            frames = np.where(prepared > 0, np.ceil(deb / (np.maximum(prepared, 1) / 16000.0)), np.inf)
        win = age[None, None, :] < np.minimum(n, frames)[:, None, None]
        d_zero = ((deb > 0.0)[:, None] & ~np.isnan(thr) & (pred != 0.0) & (pred >= thr) & (ge & win).any(-1))
        final = np.where(np.where(pat > 0, p_zero, d_zero), 0.0, pred)
        live = prepared >= 0
        self.hist[live] = np.concatenate((self.hist[live, :, 1:], final[live, :, None]), axis=2)
        self.count = c + live
        fired = live[:, None] & (final >= thr)
        return np.where(live[:, None], final, np.nan), fired


def events(final, fired, counts_before):
    """the event list oww_detect writes: (stream, label, score, index) ascending by stream, then label"""
    b, j = np.nonzero(fired)
    return [(int(s), int(l), np.float32(final[s, l]), int(counts_before[s])) for s, l in zip(b, j)]
