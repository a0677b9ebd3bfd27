"""Per-stream restatement of the detector (include/owwb200.h, oww_set_detector / oww_detect): what turns the scores of
a step into detections.  One ``StreamDetector`` is one stream: a ``deque(maxlen=30)`` of final predictions per label and
the number of predictions appended since the reset.  Plain Python on float32 scalars; the device kernel
(csrc/detect.cu) must equal it bit for bit, since the rules only select and copy values."""
import math
from collections import deque

import numpy as np

CHUNK = 1280
HISTORY = 30
ZEROED = 5          # predictions zeroed after a reset


class Label:
    """column of the score row (-1: always 0.0), repeats (a single-output head's label), threshold (None or NaN: none),
    patience (0: none)."""

    def __init__(self, column, repeats=True, threshold=None, patience=0):
        self.column, self.repeats, self.patience = int(column), bool(repeats), int(patience)
        self.threshold = None if threshold is None or math.isnan(threshold) else np.float32(threshold)
        if not 0 <= self.patience <= HISTORY:
            raise ValueError("patience outside 0..30")
        if self.patience and self.threshold is None:
            raise ValueError("patience needs a threshold")


def check(labels, debounce_time):
    if debounce_time > 0 and any(lab.patience for lab in labels):
        raise ValueError("patience and debounce_time cannot be used together")


class StreamDetector:
    def __init__(self, labels, debounce_time=0.0):
        check(labels, debounce_time)
        self.labels, self.debounce_time = list(labels), float(debounce_time)
        self.reset()

    def reset(self):
        self.history = [deque(maxlen=HISTORY) for _ in self.labels]
        self.count = 0

    def configure(self, labels, debounce_time=0.0):
        """new thresholds / patience / debounce under the same label set: the history stays"""
        check(labels, debounce_time)
        assert [(a.column, a.repeats) for a in labels] == [(a.column, a.repeats) for a in self.labels]
        self.labels, self.debounce_time = list(labels), float(debounce_time)

    def detect(self, scores, prepared):
        """scores: the stream's row of the step's score matrix (not read below 1280 prepared samples); prepared: samples
        the stream prepared in this call, < 0 = skipped.  -> (final predictions float32 [n_labels], events [(label index,
        score, index of the prediction since the reset)]), or None for a skipped stream."""
        if prepared < 0:
            return None
        final = np.zeros(len(self.labels), np.float32)
        events = []
        for j, lab in enumerate(self.labels):
            hist = self.history[j]
            if prepared >= CHUNK:
                pred = np.float32(scores[lab.column]) if lab.column >= 0 else np.float32(0.0)
            elif lab.repeats and len(hist):
                pred = hist[-1]
            else:
                pred = np.float32(0.0)
            if self.count < ZEROED:
                pred = np.float32(0.0)
            if lab.patience:
                recent = list(hist)[-lab.patience:]
                if pred != 0.0 and sum(1 for v in recent if v >= lab.threshold) < lab.patience:
                    pred = np.float32(0.0)
            elif self.debounce_time > 0 and lab.threshold is not None and pred != 0.0 and pred >= lab.threshold:
                n_frames = HISTORY if prepared == 0 else min(HISTORY, math.ceil(self.debounce_time / (prepared / 16000)))
                if any(v >= lab.threshold for v in list(hist)[-n_frames:]):
                    pred = np.float32(0.0)
            final[j] = pred
            if lab.threshold is not None and pred >= lab.threshold:
                events.append((j, pred, self.count))
        for j in range(len(self.labels)):
            self.history[j].append(final[j])
        self.count += 1
        return final, events

    def export(self):
        """-> (float32 [n_labels, 30] oldest first, zeros before the first prediction; count)"""
        out = np.zeros((len(self.labels), HISTORY), np.float32)
        for j, hist in enumerate(self.history):
            if len(hist):
                out[j, HISTORY - len(hist):] = np.array(hist, np.float32)
        return out, self.count

    def load(self, hist, count):
        self.count = int(count)
        n = min(self.count, HISTORY)
        self.history = [deque([np.float32(v) for v in (row[HISTORY - n:] if n else [])], maxlen=HISTORY) for row in hist]
