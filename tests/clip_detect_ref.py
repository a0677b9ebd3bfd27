"""Clip restatement of the detector of the bulk path (include/owwb200.h, oww_detect_clips): what predict_clip(clip,
padding, chunk_size, patience=..., threshold=..., debounce_time=...) returns after a reset, from the raw score rows of
its calls.  One oracle ``StreamDetector`` per clip, fresh for every clip; call j prepares what the reference's
_streaming_features returns (1280 k samples when it steps k >= 1 chunks, else ((j + 1) chunk_size) mod 1280), and on a
call that steps nothing a label with a verifier p takes p when its prediction is >= the verifier threshold, as
Model.predict re-verifies a repeated prediction."""
import math

import numpy as np

from oracle import detect as odet

CHUNK = odet.CHUNK


def chunks_of_call(j, chunk_size):
    return (j + 1) * chunk_size // CHUNK - j * chunk_size // CHUNK


def prepared_of_call(j, chunk_size):
    k = chunks_of_call(j, chunk_size)
    return CHUNK * k if k else (j + 1) * chunk_size % CHUNK


class ClipDetector(odet.StreamDetector):
    """StreamDetector.detect plus the verifier rule of a repeated prediction (p: float32 [n_labels], NaN = none)"""

    def detect_call(self, scores, prepared, p=None, vthr=None):
        if p is None or prepared >= CHUNK:
            return self.detect(scores, prepared)
        final = np.zeros(len(self.labels), np.float32)
        events = []
        for j, lab in enumerate(self.labels):
            hist = self.history[j]
            pred = hist[-1] if lab.repeats and len(hist) else np.float32(0.0)
            if not math.isnan(p[j]) and pred >= vthr:
                pred = np.float32(p[j])
            if self.count < odet.ZEROED:
                pred = np.float32(0.0)
            if lab.patience:
                recent = list(hist)[-lab.patience:]
                if pred != 0.0 and sum(1 for v in recent if v >= lab.threshold) < lab.patience:
                    pred = np.float32(0.0)
            elif self.debounce_time > 0 and lab.threshold is not None and pred != 0.0 and pred >= lab.threshold:
                n_frames = odet.HISTORY if prepared == 0 else min(odet.HISTORY,
                                                                  math.ceil(self.debounce_time / (prepared / 16000)))
                if any(v >= lab.threshold for v in list(hist)[-n_frames:]):
                    pred = np.float32(0.0)
            final[j] = pred
            if lab.threshold is not None and pred >= lab.threshold:
                events.append((j, pred, self.count))
        for j in range(len(self.labels)):
            self.history[j].append(final[j])
        self.count += 1
        return final, events


def detect_clips(labels, debounce_time, raw, row_off, chunk_size, verified=None, vthr=None):
    """raw float32 [rows][n_out] (read on calls that step), row_off int64 [N + 1], verified float32 [rows][n_labels] or
    None -> (final float32 [rows][n_labels], events [(clip, label, score, call)] in (clip, label, call) order)"""
    final = np.zeros((int(row_off[-1]), len(labels)), np.float32)
    events = []
    for c in range(len(row_off) - 1):
        det = ClipDetector(labels, debounce_time)
        ev = []
        for j in range(int(row_off[c + 1] - row_off[c])):
            r = int(row_off[c]) + j
            final[r], e = det.detect_call(raw[r], prepared_of_call(j, chunk_size),
                                          None if verified is None else verified[r], vthr)
            ev += [(c, lab, s, i) for lab, s, i in e]
        events += sorted(ev, key=lambda t: (t[1], t[3]))
    return final, events
