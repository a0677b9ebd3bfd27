"""The CPU stand-in for ``_native.Context`` of the not-gpu tests of the host-side logic (and the oracle of two GPU
tests): the C-ABI semantics of include/owwb200.h restated with the NumPy oracle; the product never sees it.  Every step
entry runs the per-stream core ``_step``; each area's state stays empty until its first call, as on the handle."""
import hashlib
import pickle

import numpy as np
import torch

import clip_resample_ref as cref
from helpers import kernel_order_proba
from oracle import detect as odet, heads as oheads, resample as ores, streaming as ostream
from openwakeword_b200 import _native, weights as W

CHUNK = 1280
_FIELDS = ("raw", "melspectrogram_buffer", "accumulated_samples", "remainder", "feature_buffer")


def unpack_embedding_blob(blob):
    conv, scale, bias = [], [], []
    off = 0
    for (kh, kw, cin, cout, _, _) in W.EMBEDDING_LAYERS:
        n = kh * kw * cin * cout
        conv.append(blob[off:off + n].reshape(kh, kw, cin, cout)); off += n
        scale.append(blob[off:off + cout]); off += cout
        bias.append(blob[off:off + cout]); off += cout
    assert off == blob.size
    # express folded scale/bias as a BatchNorm with var = 1-eps, mean = 0
    bn = [(s * np.sqrt(np.float64(1.0)), b, np.zeros_like(b), np.full_like(b, 1.0 - 1e-3)) for s, b in zip(scale[:-1], bias[:-1])]
    return {"conv": conv, "bn": bn}


def unpack_head_blob(n_in, dims, layernorm, final_act, blob):
    layers, off = [], 0
    for i in range(len(dims) - 1):
        din, dout = dims[i], dims[i + 1]
        Wm = blob[off:off + din * dout].reshape(din, dout); off += din * dout
        b = blob[off:off + dout]; off += dout
        ln = None
        if layernorm and i < len(dims) - 2:
            ln = (blob[off:off + dout], blob[off + dout:off + 2 * dout]); off += 2 * dout
        layers.append({"W": Wm, "b": b, "ln": ln})
    assert off == blob.size
    fin = {v: k for k, v in W.FINAL_CODES.items()}[final_act]
    return {"n_in": n_in, "layers": layers, "final": fin}


class FakeContext:
    features = True         # False: steps only record audio (no oracle CNN, no scores)
    n_detect_labels = 0
    audio_history = 0
    _RECORD_BYTES = 1 << 20

    def __init__(self, device=0, max_chunks=4, cnn_mode=_native.CNN_TC_INCREMENTAL, window_batch=0, fuse_step=True,
                 tc_heads=True, tc_heads_terms=3, split_from=None, group_heads=True):
        self.max_chunks = max_chunks
        self._config = (cnn_mode, split_from)
        self.heads, self.gates = [], []
        self.hbanks = []            # head banks: the bank's columns follow the heads'
        self.banks = []             # verifier banks, of ordinary heads and of head banks
        self.verifiers_on = True
        self.feature_reads = 0      # the host's get_features calls
        self.unverified = {}        # stream -> its score row of its last step before the verifier banks
        self._n = 0
        self.det = self._labels = self._ing = None

    def _ids(self, stream_ids):
        return np.arange(self._n) if stream_ids is None else np.asarray(stream_ids)

    # ---- weights, heads and gates ----
    def load_mel(self, window512=None, mel_fb=None):
        pass

    def load_embedding(self, blob):
        self.emb = unpack_embedding_blob(np.asarray(blob, np.float32))

    def add_head(self, n_in, dims, layernorm, final_act, blob):
        self.heads.append(unpack_head_blob(n_in, list(dims), layernorm, final_act, np.asarray(blob, np.float32)))
        return len(self.heads) - 1

    def add_gate(self, main_head, verifier_head, threshold=0.5):
        self.gates.append((main_head, verifier_head, float(threshold)))

    def _col0(self, hid):
        return sum(h["layers"][-1]["W"].shape[1] for h in self.heads[:hid])

    @property
    def n_outputs(self):
        return self._col0(len(self.heads)) + sum(b["n_out"] for b in self.hbanks)

    # ---- head banks: a stream on slot k gets head k's max over its chunk windows, a stream on slot -1 gets 0 ----
    def add_head_bank(self, n_in, dims, layernorm, final_act, capacity):
        if self._config[0] == _native.CNN_FP32_WINDOW:
            raise _native.NativeError("head banks run on the tensor cores: not in cnn_mode 0")
        self.hbanks.append({"shape": (n_in, list(dims), layernorm, final_act), "n_out": dims[-1], "capacity": capacity,
                            "heads": [None] * capacity, "assign": np.full(self._n, -1, np.int32), "clip": -1})
        return len(self.hbanks) - 1

    def load_bank_head(self, bank, slot, blob):
        b = self.hbanks[bank]
        assert 0 <= slot < b["capacity"]
        b["heads"][slot] = unpack_head_blob(*b["shape"], np.asarray(blob, np.float32))

    def assign_bank_head(self, bank, stream_ids, slots, stream=None):
        b = self.hbanks[bank]
        for i, s in zip(self._ids(stream_ids), np.asarray(slots)):
            assert s == -1 or b["heads"][s] is not None
            b["assign"][i] = s

    def set_head_bank_clip_slot(self, bank, slot):
        self.hbanks[bank]["clip"] = slot

    # ---- verifier banks: after the max over the chunk windows, columns of the bank's head >= threshold (fp32) become
    #      p of the stream's slot; a verifier bank of a head bank only where the stream has a bank model ----
    def _add_verifier_bank(self, col0, n_cols, n_in, capacity, threshold, head_bank=None):
        self.banks.append(dict(col0=col0, n_cols=n_cols, n_in=n_in, thr=np.float32(threshold), slots={},
                               assign=np.full(self._n, -1, np.int32), clip=-1, capacity=capacity, hbank=head_bank))
        return len(self.banks) - 1

    def add_verifier_bank(self, head_id, capacity, threshold):
        h = self.heads[head_id]
        return self._add_verifier_bank(self._col0(head_id), h["layers"][-1]["W"].shape[1], h["n_in"], capacity, threshold)

    def add_bank_verifier_bank(self, head_bank, capacity, threshold):
        hb = self.hbanks[head_bank]
        col0 = self._col0(len(self.heads)) + sum(b["n_out"] for b in self.hbanks[:head_bank])
        return self._add_verifier_bank(col0, hb["n_out"], hb["shape"][0], capacity, threshold, head_bank)

    def load_verifier(self, bank, slot, mean, weight, bias):
        assert 0 <= slot < self.banks[bank]["capacity"]
        self.banks[bank]["slots"][slot] = (np.asarray(mean, np.float32), np.asarray(weight, np.float32), np.float32(bias))

    def assign_verifier(self, bank, stream_ids, slots, stream=None):
        self.banks[bank]["assign"][self._ids(stream_ids)] = slots

    def set_verifier_clip_slot(self, bank, slot):
        self.banks[bank]["clip"] = slot

    def set_verifier_threshold(self, bank, threshold):
        self.banks[bank]["thr"] = np.float32(threshold)

    def enable_verifiers(self, enabled):
        self.verifiers_on = bool(enabled)

    def verifier_predict_host(self, bank, slot, feats):
        return kernel_order_proba(*self.banks[bank]["slots"][slot], feats)

    # ---- streams ----
    @property
    def n_streams(self):
        return self._n

    def set_streams(self, n):
        self._n = n
        self.af = [ostream.OracleAudioFeatures(self.emb) for _ in range(n)]
        for b in self.hbanks + self.banks:
            b["assign"] = np.full(n, -1, np.int32)
        self._new_detectors()
        self._alloc_ring()
        if self._ing is not None:
            self._new_ing()

    def reset(self, stream_ids=None, feature_init=None):
        for b in self._ids(stream_ids):
            self.af[b].reset(feature_init=np.zeros((41, 96), np.float32) if feature_init is None else feature_init)
            if self.det:
                self.det[b].reset()
            if self._ing is not None:
                self._ing["S"][b], self._ing["staged"][b], self._ing["res"][b] = 0, np.zeros(0, np.int16), None
            self.pos[b] = 0

    def _features(self, stream_id, n, back=0):
        fb = self.af[stream_id].feature_buffer
        end = fb.shape[0] - back
        rows = fb[max(end - n, 0):end]
        if rows.shape[0] < n:
            rows = np.vstack((np.zeros((n - rows.shape[0], 96), np.float32), rows))
        return rows.astype(np.float32)

    def get_features(self, stream_id, n, back=0):
        self.feature_reads += 1
        return self._features(stream_id, n, back)

    def get_counts(self, stream_id):
        # the oracle caps its buffers like the reference; uncapped counts are not needed by the host logic under test
        return self.af[stream_id].melspectrogram_buffer.shape[0], self.af[stream_id].feature_buffer.shape[0]

    def get_mel(self, stream_id, n_rows=76):
        return self.af[stream_id].melspectrogram_buffer[-n_rows:].astype(np.float32)

    # ---- steps ----
    def _windows(self, b, h, chunks):
        """head h on stream b's feature window of each of its last `chunks` chunks, oldest first -> [chunks, n_out]; rows
        older than the stream has (a reset with fewer feature rows than n_in) are zeros, as on the handle's ring"""
        return np.stack([oheads.forward(h, self._features(b, h["n_in"], i)[None])[0] for i in range(chunks - 1, -1, -1)])

    def _gated(self, raw):
        """the gates on the heads' [chunks, columns] window scores: per chunk, before the max over chunks (as the gated
        graph would)"""
        for m, v, thr in self.gates:
            cm, cv = self._col0(m), self._col0(v)
            raw[:, cm] = np.where(raw[:, cm] > np.float32(thr), raw[:, cv], raw[:, cm])
        return raw

    def _bank_scores(self, b, hb, chunks):
        k = hb["assign"][b]
        return np.zeros(hb["n_out"], np.float32) if k < 0 else self._windows(b, hb["heads"][k], chunks).max(axis=0)

    @staticmethod
    def _verified(cols, thr):
        return cols >= thr

    def _step(self, b, pcm, chunks, scores):
        """stream b steps the first `chunks` chunks of its samples pcm into its score row"""
        x = pcm[:chunks * CHUNK]
        self._append(b, x)
        if not self.features:
            return
        assert self.af[b](x) == chunks * CHUNK
        raw = self._gated(np.concatenate([self._windows(b, h, chunks) for h in self.heads], axis=1))
        scores[:raw.shape[1]] = raw.max(axis=0)
        col = raw.shape[1]
        for hb in self.hbanks:
            scores[col:col + hb["n_out"]] = self._bank_scores(b, hb, chunks)
            col += hb["n_out"]
        self.unverified[b] = scores.copy()          # the row before the verifier banks, for tests that judge them
        for bk in self.banks if self.verifiers_on else []:
            slot = bk["assign"][b] if bk["hbank"] is None or self.hbanks[bk["hbank"]]["assign"][b] >= 0 else -1
            cols = scores[bk["col0"]:bk["col0"] + bk["n_cols"]]
            if slot < 0 or not self._verified(cols, bk["thr"]).any():
                continue
            p = kernel_order_proba(*bk["slots"][slot], self._features(b, bk["n_in"])[None])[0]
            cols[self._verified(cols, bk["thr"])] = p

    def step_host(self, pcm, n_chunks, scores_out):
        for b in range(self._n):
            self._step(b, pcm[b], n_chunks, scores_out[b])

    def step_host_ragged(self, pcm, chunks, scores_out):
        """stream b steps chunks[b] chunks of its row, held streams are skipped"""
        for b in range(self._n):
            if chunks[b]:
                self._step(b, pcm[b], int(chunks[b]), scores_out[b])

    def new_scores(self):
        return np.zeros((self._n, self.n_outputs), np.float32)

    def step_pcm(self, pcm, n_chunks, d_scores):
        self.step_host(pcm, n_chunks, d_scores)

    def step_ragged_pcm(self, pcm, chunks, d_scores):
        self.step_host_ragged(pcm, chunks, d_scores)

    # ---- stream records: [payload bytes, configuration key, the pickled oracle state of the stream], the key at bytes
    #      8..16 as in the library's records; the rest of the library's byte layout is deliberately not modelled (only
    #      the key is read across), so a record moves between handles of one kind only ----
    def stream_state_info(self):
        h = hashlib.sha256(repr(self._config).encode())
        for c in self.emb["conv"]:
            h.update(np.ascontiguousarray(c).tobytes())
        return self._RECORD_BYTES, int.from_bytes(h.digest()[:8], "little")

    def export_records(self, stream_ids, stream=None):
        _, key = self.stream_state_info()
        out = np.zeros((len(stream_ids), self._RECORD_BYTES), np.uint8)
        for i, b in enumerate(stream_ids):
            blob = pickle.dumps({k: getattr(self.af[b], k) for k in _FIELDS})
            assert 16 + len(blob) <= self._RECORD_BYTES
            out[i, :16] = np.frombuffer(np.array([len(blob), key], np.uint64).tobytes(), np.uint8)
            out[i, 16:16 + len(blob)] = np.frombuffer(blob, np.uint8)
        return torch.from_numpy(out)

    def import_records(self, stream_ids, records, stream=None):
        _, key = self.stream_state_info()
        rec = records.cpu().numpy()
        assert len(set(int(b) for b in stream_ids)) == len(stream_ids)
        for i, b in enumerate(stream_ids):
            n, k = np.frombuffer(rec[i, :16].tobytes(), np.uint64)
            if int(k) != key:
                raise ValueError("records of another configuration")
            for f, v in pickle.loads(rec[i, 16:16 + int(n)].tobytes()).items():
                setattr(self.af[b], f, v)

    # ---- detector: one oracle StreamDetector per stream; "device" buffers are NumPy arrays ----
    def _new_detectors(self):
        self.det = [odet.StreamDetector(self._labels, self._debounce) for _ in range(self._n)] if self._labels else None

    def set_detector(self, labels, debounce_time=0.0):
        new = [odet.Label(*row) for row in labels]
        odet.check(new, debounce_time)
        old, self._labels, self._debounce = self._labels, new, debounce_time
        self.n_detect_labels = len(new)
        if old and [(a.column, a.repeats) for a in old] == [(a.column, a.repeats) for a in new] and self.det:
            for d in self.det:
                d.configure(new, debounce_time)
        else:
            self._new_detectors()

    def detect_events(self, d_scores, prepared, d_final=None, max_events=None):
        prepared = np.broadcast_to(np.asarray(prepared, np.int32), (self._n,))
        ev = []
        for b in range(self._n):
            r = self.det[b].detect(d_scores[b], int(prepared[b]))
            if r is None:
                continue
            if d_final is not None:
                d_final[b] = r[0]
            ev += [(b, j, s, i) for j, s, i in r[1]]
        cap = self._n * self.n_detect_labels if max_events is None else max_events
        return np.array(ev[:cap], _native.EVENT_DTYPE), len(ev)

    def detector_history(self, stream_ids):
        out = [self.det[b].export() for b in stream_ids]
        return (np.stack([h for h, _ in out]).reshape(len(out), self.n_detect_labels, 30),
                np.array([c for _, c in out], np.int32))

    def set_detector_history(self, stream_ids, hist, counts):
        assert len(set(int(b) for b in stream_ids)) == len(stream_ids)
        for i, b in enumerate(stream_ids):
            self.det[b].load(hist[i], counts[i])

    # ---- audio history: ring [B, H], pos [B]; every step appends what it steps ----
    def set_audio_history(self, n_samples):
        if n_samples < 0 or n_samples % 1280 or n_samples > 960000:
            raise _native.NativeError("n_samples")
        self.audio_history = n_samples
        self._alloc_ring()

    def _alloc_ring(self):
        self.ring = np.zeros((self._n, self.audio_history), np.int16)
        self.pos = np.zeros(self._n, np.int64)

    def _append(self, b, x):
        H = self.audio_history
        if not H:
            return
        p = self.pos[b] + np.arange(x.size)
        self.ring[b, p % H] = x
        self.pos[b] += x.size

    def _window(self, b, e, n):
        H, p = self.audio_history, self.pos[b]
        q = np.arange(e - n, e)
        ok = (q >= max(p - H, 0)) & (q < p)
        out = np.zeros(n, np.int16)
        out[ok] = self.ring[b, q[ok] % H]
        return out

    def _clips(self, ids, ends, n):
        """int16 [len(ids), n]: stream ids[i]'s audio up to sample ends[i]"""
        if not self.audio_history:
            raise _native.NativeError("no audio history")
        return np.array([self._window(b, e, n) for b, e in zip(ids, ends)], np.int16).reshape(len(ids), n)

    def audio_state(self, stream_ids):
        ids = np.asarray(stream_ids, np.int64)
        return self._clips(ids, self.pos[ids], self.audio_history), self.pos[ids].copy()

    def set_audio_state(self, stream_ids, audio, pos):
        ids, audio, H = np.asarray(stream_ids, np.int64), np.asarray(audio, np.int16), self.audio_history
        if not H or len(set(ids.tolist())) != ids.size:
            raise _native.NativeError("no audio history or duplicate ids")
        if audio.shape != (ids.size, H):
            raise ValueError("audio shape")
        for i, b in enumerate(ids):
            p = max(int(pos[i]), 0)
            self.ring[b, (p + np.arange(H)) % H] = audio[i]
            self.pos[b] = p

    def read_audio(self, stream_ids, n_samples, ends=None):
        ids = np.asarray(stream_ids, np.int64).ravel()
        e = [self.pos[b] if ends is None or ends[i] < 0 else ends[i] for i, b in enumerate(ids)]
        return torch.from_numpy(self._clips(ids, e, n_samples)), torch.from_numpy(self.pos[ids].copy())

    def detect_capture(self, d_scores, prepared, n_samples, max_events=None):
        if not self.audio_history:
            raise _native.NativeError("no audio history")
        events, n = self.detect_events(d_scores, prepared, None, max_events)
        s = events["stream"]
        return events, n, torch.from_numpy(self._clips(s, self.pos[s], n_samples)), self.pos[s].copy()

    # ---- ingest: resampling by the oracle (the library's fp32 taps in float64, rounded half to even), the capacity
    #      from the library's own host arithmetic, then the step core ----
    def _new_ing(self):
        n = self._n
        self._ing = dict(rate=np.full(n, 16000, np.int32), S=np.zeros(n, np.int64),
                         staged=[np.zeros(0, np.int16) for _ in range(n)], res=[None] * n)

    def set_input_rates(self, stream_ids, rates, stream=None):
        for r in np.unique(rates):
            _native.resampler_taps(int(r))
        if self._ing is None:
            self._new_ing()
        for b, r in zip(self._ids(stream_ids), rates):
            self._ing["rate"][b], self._ing["S"][b], self._ing["res"][b] = r, 0, None

    def _res(self, b):
        g = self._ing
        if g["res"][b] is None:
            h, _, _ = _native.resampler_taps(int(g["rate"][b]))
            g["res"][b] = ores.StreamResampler(int(g["rate"][b]), h=h.astype(np.float64) if h.size else None)
            g["res"][b].S = int(g["S"][b])
        return g["res"][b]

    def ingest_capacity(self):
        g = self._ing
        return np.array([_native.ingest_plan(int(g["rate"][b]), self.max_chunks, int(g["S"][b]), g["staged"][b].size, 0)[3]
                         for b in range(self._n)], np.int64)

    def ingest_pcm(self, pcm, offsets, d_scores):
        g = self._ing
        n = np.diff(offsets)
        if (n > self.ingest_capacity()).any():
            raise _native.NativeError("over capacity")
        tot = []
        for b in range(self._n):
            y = self._res(b).feed(pcm[offsets[b]:offsets[b + 1]])
            tot.append(np.concatenate((g["staged"][b], ores.to_int16(y))))
            g["S"][b] += n[b]
        chunks = np.array([t.size // CHUNK for t in tot], np.int32)
        for b in np.nonzero(chunks)[0]:
            self._step(b, tot[b], int(chunks[b]), d_scores[b])
        g["staged"] = [t[c * CHUNK:] for t, c in zip(tot, chunks)]
        return chunks, np.where(chunks > 0, chunks * CHUNK, [t.size for t in tot]).astype(np.int32)

    def ingest_state(self, stream_ids, samples=True):
        g = self._ing
        ids = list(stream_ids)
        staged = np.array([g["staged"][b].size for b in ids], np.int32)
        x = np.zeros((len(ids), max(int(staged.max(initial=0)), 1)), np.int16)
        hist = np.zeros((len(ids), 128), np.int16)
        for i, b in enumerate(ids):
            x[i, :staged[i]] = g["staged"][b]
            if g["rate"][b] != 16000 and g["S"][b]:
                hist[i] = np.asarray(self._res(b).hist[-128:], np.int16)
        return g["rate"][ids].copy(), g["S"][ids].copy(), staged, x, hist

    def set_ingest_state(self, stream_ids, rates, consumed, staged, samples, hist):
        g = self._ing
        assert len(set(int(b) for b in stream_ids)) == len(stream_ids)
        for i, b in enumerate(stream_ids):
            g["rate"][b], g["S"][b], g["res"][b] = rates[i], consumed[i], None
            g["staged"][b] = np.asarray(samples[i, :staged[i]], np.int16).copy()
            if rates[i] != 16000:
                self._res(b).hist[-128:] = hist[i]

    # ---- whole clips through the float64 clip reference on the library's fp32 taps ----
    def resample_clips(self, d_in, in_offsets, rates, pad_samples, d_out, out_offsets, stream=None):
        for i, r in enumerate(rates):
            h, _, _ = _native.resampler_taps(int(r))
            x = d_in[in_offsets[i]:in_offsets[i + 1]]
            y = cref.resample_clip(x, int(r), pad_samples, h=h.astype(np.float64) if h.size else None)
            d_out[out_offsets[i]:out_offsets[i + 1]] = ores.to_int16(y)
