"""StreamEngine: the batched, dictionary-free face of the streaming hot path.

``Model`` mirrors the reference's per-call dict API; the engine is what a serving loop (and
bench.py) drives: B streams, one ``step`` = every stream consumes n_chunks*1280 samples and yields
``float32[B, n_cols]`` raw head outputs.  ``step`` takes device-resident PCM (torch int16 tensor)
and enqueues on the current CUDA stream with no synchronisation; ``step_host`` takes a host array
and includes the H2D/D2H copies (pinned staging inside the library)."""
import numpy as np

from . import _native
from . import weights as _weights
from .utils import load_embedding_weights, _torch
from .custom_verifier_model import load_verifier, linear_verifier_params


class StreamEngine:
    def __init__(self, heads, n_streams, embedding="synthetic:0", feature_init=None, device_index=0,
                 max_chunks=1, cnn_mode=_native.CNN_TC_INCREMENTAL, window_batch=0, fuse_step=True,
                 tc_heads=True, tc_heads_terms=3, split_from=None, group_heads=True):
        """heads: list of head dicts (weights.synthetic_head / load_head; gated pairs allowed)."""
        self.ctx = _native.Context(device=device_index, max_chunks=max_chunks, cnn_mode=cnn_mode,
                                   window_batch=window_batch, fuse_step=fuse_step, tc_heads=tc_heads,
                                   tc_heads_terms=tc_heads_terms, split_from=split_from, group_heads=group_heads)
        self.ctx.load_mel()
        self.ctx.load_embedding(_weights.pack_embedding_blob(load_embedding_weights(embedding)))
        self.columns = []                       # per entry of `heads`: (first score column, n_out); a gated pair's
        col = 0                                 # verifier network occupies one further (raw) column
        self.head_ids = []                      # per entry of `heads`: its (main) head id on the handle
        for h in heads:
            parts = [h["main"], h["verifier"]] if _weights.is_gated(h) else [h]
            ids = []
            for q in parts:
                n_in, dims, ln, fin = _weights.head_desc(q)
                ids.append(self.ctx.add_head(n_in, dims, ln, fin, _weights.pack_head_blob(q)))
            if len(ids) == 2:
                self.ctx.add_gate(ids[0], ids[1], h["threshold"])
            self.head_ids.append(ids[0])
            n_out = parts[0]["layers"][-1]["W"].shape[1]
            self.columns.append((col, n_out))
            col += n_out if len(ids) == 1 else 2
        self.n_streams = n_streams
        self.n_cols = self.ctx.n_outputs
        self.device_index = device_index
        self.ctx.set_streams(n_streams)
        self.reset(feature_init)

    def reset(self, feature_init=None, stream_ids=None):
        fi = np.zeros((41, 96), np.float32) if feature_init is None else feature_init
        self.ctx.reset(stream_ids, fi)

    def reset_async(self, feature_init=None, stream_ids=None, stream=None):
        """Stream-ordered reset on the current CUDA stream (no synchronisation; for the device-resident ``step`` path).
        The reset streams re-prime at their next step while the others keep the fused kernel."""
        torch = _torch()
        fi = np.zeros((41, 96), np.float32) if feature_init is None else feature_init
        if stream is None:
            stream = torch.cuda.current_stream(torch.device("cuda", self.device_index)).cuda_stream
        self.ctx.reset_async(stream_ids, fi, stream)

    def set_streams(self, n_streams, feature_init=None):
        """Reallocate for n_streams streams: every stream starts afresh, without a verifier or bank head (export the
        streams to keep first, then import them and reassign)."""
        self.ctx.set_streams(n_streams)
        self.n_streams = n_streams
        self.reset(feature_init)

    # ---- stream records: moving live streams (include/owwb200.h, oww_export_streams) ----
    def export_streams(self, stream_ids, stream=None):
        """The state of streams stream_ids -> torch.uint8 [n, record bytes] on the engine's device, enqueued on the current
        CUDA stream (or `stream`) after the steps enqueued there and the submitted host steps."""
        return self.ctx.export_records(stream_ids, stream)

    def import_streams(self, stream_ids, records, stream=None):
        """Stream stream_ids[i] (distinct) becomes the stream record i was exported from.  records: uint8 [n, record
        bytes] on any device or the CPU.  Records of another configuration (cnn_mode, split_from, weights) raise
        ValueError before anything is enqueued.  Verifier and head-bank assignments stay as they are."""
        self.ctx.import_records(stream_ids, records, stream)

    def _check_step(self, d_pcm, n_chunks, out):
        """-> the row stride of d_pcm, after refusing what the library would read or write out of bounds: d_pcm must be
        int16 [n_streams, >= n_chunks*1280] with unit inner stride (rows may be column slices of a wider buffer), out
        float32 [n_streams, n_cols] contiguous, both on the engine's device."""
        torch = _torch()
        dev = torch.device("cuda", self.device_index)
        if not isinstance(d_pcm, torch.Tensor) or d_pcm.dtype != torch.int16 or d_pcm.dim() != 2 or d_pcm.device != dev:
            raise _native.ArgumentError(f"d_pcm must be an int16 [n_streams, samples] tensor on {dev}")
        if d_pcm.shape[0] != self.n_streams or d_pcm.shape[1] < n_chunks * 1280 or d_pcm.stride(1) != 1:
            raise _native.ArgumentError(f"d_pcm has shape {tuple(d_pcm.shape)} and strides {d_pcm.stride()}; this call "
                                        f"reads [{self.n_streams}, {n_chunks * 1280}] with unit inner stride")
        if out is not None and (not isinstance(out, torch.Tensor) or out.dtype != torch.float32 or out.device != dev
                                or tuple(out.shape) != (self.n_streams, self.n_cols) or not out.is_contiguous()):
            raise _native.ArgumentError(f"out must be a contiguous float32 [{self.n_streams}, {self.n_cols}] tensor "
                                        f"on {dev}")
        # a one-stream view may carry any stride for its single row
        return d_pcm.stride(0) if self.n_streams > 1 else max(d_pcm.stride(0), d_pcm.shape[1])

    def step(self, d_pcm, n_chunks=1, out=None):
        torch = _torch()
        stride = self._check_step(d_pcm, n_chunks, out)
        if out is None:
            out = torch.empty((self.n_streams, self.n_cols), dtype=torch.float32, device=d_pcm.device)
        self.ctx.step(d_pcm, stride, n_chunks, out, torch.cuda.current_stream(d_pcm.device).cuda_stream)
        return out

    def step_host(self, pcm, n_chunks=1, out=None):
        if out is None:
            out = np.empty((self.n_streams, self.n_cols), np.float32)
        self.ctx.step_host(pcm, n_chunks, out)
        return out

    def submit(self, pcm, n_chunks=1):
        """Pipelined host path: enqueue H2D + step + D2H and return a ticket; at most two in flight."""
        return self.ctx.step_host_submit(pcm, n_chunks)

    def collect(self, ticket, out=None):
        """Scores of a submitted step; with out None the rows a ragged ticket held come back as NaN."""
        if out is None:
            out = np.full((self.n_streams, self.n_cols), np.nan, np.float32)
        self.ctx.step_host_collect(ticket, out)
        return out

    # ---- ragged steps: every stream at its own pace (include/owwb200.h, oww_step_ragged) ----
    def step_ragged(self, d_pcm, chunks, out=None):
        """Stream b consumes chunks[b] (host ints, 0..max_chunks) chunks, the first chunks[b]*1280 samples of row b of
        d_pcm.  A stream with 0 chunks is held: its state does not change and its row of `out` is not written."""
        torch = _torch()
        # counts above max_chunks are the library's to refuse; the rows must hold the largest count it accepts
        stride = self._check_step(d_pcm, min(int(np.max(chunks, initial=0)), self.ctx.max_chunks), out)
        if out is None:
            out = torch.full((self.n_streams, self.n_cols), float("nan"), dtype=torch.float32, device=d_pcm.device)
        self.ctx.step_ragged(d_pcm, stride, chunks, out, torch.cuda.current_stream(d_pcm.device).cuda_stream)
        return out

    def step_host_ragged(self, pcm, chunks, out=None):
        """Host form of ``step_ragged``; held rows of `out` keep their values (NaN when `out` is None)."""
        if out is None:
            out = np.full((self.n_streams, self.n_cols), np.nan, np.float32)
        self.ctx.step_host_ragged(pcm, chunks, out)
        return out

    def submit_ragged(self, pcm, chunks):
        """Pipelined ragged host step; complete it with ``collect`` (held rows of its `out` are left as they were, NaN
        when `out` is None)."""
        return self.ctx.step_host_ragged_submit(pcm, chunks)

    # ---- ingest: packets at any sample rate (include/owwb200.h, oww_set_input_rates / oww_ingest) ----
    def set_input_rates(self, rates, stream_ids=None):
        """Streams stream_ids (None = all; rates then has one entry per stream) take packets at rates[i] Hz (8000, 11025,
        12000, 16000, 22050, 24000, 32000, 44100 or 48000) from the next ``ingest`` on; their resamplers restart and the
        16 kHz samples they hold are kept.  The first call allocates the ingest state (every other stream at 16000)."""
        if stream_ids is None and np.ndim(rates) == 0:
            rates = np.full(self.n_streams, int(rates), np.int32)
        elif stream_ids is not None:
            rates = np.broadcast_to(np.asarray(rates, np.int64), np.shape(np.ravel(stream_ids)))
        self.ctx.set_input_rates(stream_ids, rates, self._stream(None))

    def ingest_capacity(self):
        """-> int64 [n_streams]: the most input samples each stream's next ``ingest`` may take"""
        return self.ctx.ingest_capacity()

    def ingest(self, d_packets, offsets, out=None):
        """Every stream's new packet, at its own rate, in one packed int16 tensor on the engine's device: stream b's
        samples are d_packets[offsets[b]:offsets[b+1]] (host ints, n_streams + 1 of them; a stream may get none).  The
        device resamples them to 16 kHz, steps every stream's whole chunks as ``step_ragged`` does and keeps the rest.
        The scores go to out (float32 [n_streams, n_cols] on the device; None: ``self.ingest_scores``, a matrix the engine
        keeps), rows of streams that stepped nothing are not written.  -> (chunks, prepared): int32 [n_streams] host arrays
        filled without synchronisation; prepared is what ``detect`` takes (chunks*1280, or the samples staged when a
        stream stepped nothing).  Enqueued on the current CUDA stream.  A packet longer than ``ingest_capacity`` raises
        NativeError before anything is enqueued.
        Typical loop:  chunks, prepared = eng.ingest(packets, offsets)
                       ev, n = eng.detect(eng.ingest_scores, prepared)"""
        torch = _torch()
        dev = torch.device("cuda", self.device_index)
        if not isinstance(d_packets, torch.Tensor) or d_packets.dtype != torch.int16 or d_packets.device != dev \
                or d_packets.dim() != 1 or not d_packets.is_contiguous():
            raise _native.ArgumentError(f"d_packets must be a contiguous 1-D int16 tensor on {dev}")
        off = np.ascontiguousarray(offsets, np.int64).ravel()
        if off.size != self.n_streams + 1 or (off.size and (off[0] < 0 or off[-1] > d_packets.numel())):
            raise _native.ArgumentError(f"offsets must hold {self.n_streams + 1} sample offsets into d_packets "
                                        f"({d_packets.numel()} samples)")
        if out is None:
            if getattr(self, "ingest_scores", None) is None or tuple(self.ingest_scores.shape) != (self.n_streams,
                                                                                                 self.n_cols):
                self.ingest_scores = torch.full((self.n_streams, self.n_cols), float("nan"), dtype=torch.float32,
                                                device=dev)
            out = self.ingest_scores
        else:
            self.ctx._cuda("out", out, torch.float32, (self.n_streams, self.n_cols))
        return self.ctx.ingest(d_packets, off, out, torch.cuda.current_stream(dev).cuda_stream)

    # ---- pipelined detection from host audio (include/owwb200.h, oww_detect_host_submit) ----
    def submit_detect(self, packets, offsets, max_events=None, capture=None, final=False):
        """Every stream's new packet from host memory, ingested and detected on the device without waiting for it: what
        ``ingest`` then ``detect`` (with ``capture``: the last `capture` samples of each event's stream, as
        ``detect(capture=...)``) give, delivered to host memory.  packets: a contiguous 1-D int16 NumPy array, stream b's
        packet packets[offsets[b]:offsets[b+1]] at its own rate (set_input_rates; needs a detector, and with capture an
        audio history).  A page-locked array (e.g. torch.empty(n, dtype=torch.int16).pin_memory().numpy()) is copied
        straight from, so it must not change before the collect; any other is staged before the call returns.
        max_events None: n_streams * n_labels, which never truncates (with capture it must be given: the clips are
        buffered for max_events events).  -> a ticket; at most two are in flight.  Calls made between two submits
        (settings, resets, exports, imports) apply to the later one.
        Typical serving loop, the next call's copy overlapping the device work of the one before:
            pending = []
            for packets, offsets in source:
                pending.append(eng.submit_detect(packets, offsets, max_events=64, capture=16000))
                if len(pending) == 2:
                    events, n, chunks, prepared, clips, ends = eng.collect_detect(pending.pop(0))
            while pending:
                events, n, chunks, prepared, clips, ends = eng.collect_detect(pending.pop(0))"""
        if max_events is None:
            if capture:
                raise ValueError("submit_detect with capture needs max_events (the clip buffers hold that many events)")
            max_events = self.n_streams * self.ctx.n_detect_labels
        return self.ctx.detect_host_submit(packets, offsets, int(max_events), capture, bool(final))

    def collect_detect(self, ticket):
        """Waits for a ticket of ``submit_detect`` (collect them in submission order) -> (events, n, chunks, prepared):
        the first min(n, max_events) of the n events (_native.EVENT_DTYPE, ascending by stream then label), and the chunks
        and prepared samples of the ingest, int32 [n_streams]; with capture + (clips int16 [events, capture], ends int64
        [events]: each clip's end, its stream's position); with final + (float32 [n_streams, n_labels] predictions,)."""
        events, n, chunks, prepared, clips, ends, fin = self.ctx.detect_host_collect(ticket)
        out = (events, n, chunks, prepared)
        if clips is not None:
            out += (clips, ends)
        if fin is not None:
            out += (fin,)
        return out

    # ---- detections on the device (include/owwb200.h, oww_set_detector) ----
    def set_detector(self, labels, threshold, patience={}, debounce_time=0.0):
        """Configure the detector.  labels: one (column, repeats) per label - the score column it reads (-1: always 0.0)
        and whether it repeats its previous prediction when fewer than 1280 samples were prepared (True for the label of a
        single-output head, False for a class of a multi-output head).  threshold: one float for every label, or {label
        index: float} (a label without one never fires); patience: {label index: 1..30}; debounce_time: seconds.
        Patience needs a threshold and excludes a debounce_time (NativeError, as the reference's ValueErrors).  New
        thresholds, patience or debounce_time under the same labels keep the streams' histories; other labels clear them.
        Synchronises the device."""
        table = []
        for j, (col, rep) in enumerate(labels):
            thr = threshold.get(j) if isinstance(threshold, dict) else threshold
            table.append((col, rep, thr, patience.get(j, 0)))
        self.ctx.set_detector(table, debounce_time)

    def detect(self, scores, prepared=1280, final=None, max_events=None, capture=None):
        """The detections of the step that wrote `scores` (float32 [n_streams, n_cols] on the engine's device).
        prepared: the samples every stream prepared in that step, or host ints [n_streams] (< 0: the stream is skipped,
        as for one held in step_ragged; 0..1279: it repeats its previous prediction).  final: float32 [n_streams, n_labels]
        on the device, receives every prediction after the first-5 zeroing, patience and debounce (optional).
        -> (events, n): n = the (stream, label) pairs at or above their threshold; events = the first min(n, max_events)
        of them, ascending by stream then label, as a host NumPy array of dtype _native.EVENT_DTYPE (fields stream, label,
        score, index = which prediction of the stream since its reset).  max_events None: n_streams * n_labels.
        Runs on the current CUDA stream and synchronises it to read the count; only the count and the events are copied.
        Typical loop:  scores = eng.step_ragged(pcm, chunks);
                       ev, n = eng.detect(scores, np.where(chunks > 0, chunks * 1280, -1))
        capture: a number of samples (needs set_audio_history): the last `capture` samples of each event's stream are
        gathered on the device right after the detection, before the count is read, and the call returns (events, n,
        clips, ends): clips int16 [min(n, max_events), capture] on the device, ends int64 (host) = each clip's end, the
        stream's sample position.  `final` is not written then."""
        torch = _torch()
        self.ctx._cuda("scores", scores, torch.float32, (self.n_streams, self.n_cols))
        if capture is not None:
            return self.ctx.detect_capture(scores, prepared, int(capture), max_events)
        if final is not None:
            self.ctx._cuda("final", final, torch.float32, (self.n_streams, self.ctx.n_detect_labels))
        return self.ctx.detect_events(scores, prepared, final, max_events)

    # ---- per-stream detection settings (include/owwb200.h, oww_set_stream_detection) ----
    def set_stream_detection(self, stream_ids, threshold=None, patience=None, debounce_time=None, stream=None):
        """Streams stream_ids (distinct; None = all) detect at their own sensitivity from the next ``detect`` enqueued on
        the current CUDA stream (or `stream`) on.  threshold: one float for every label, or {label index: float, or None
        for no threshold on these streams (the label never fires there)}; patience: one int for every label, or {label
        index: 0..30}; debounce_time: seconds.  What is not given (None, a label missing from a dict, a NaN threshold)
        stays the handle's (set_detector).  The call replaces the streams' earlier settings.  Each stream's resulting
        values are checked as set_detector checks the handle's (NativeError: a patience without a threshold, patience
        together with a debounce_time).  set_detector clears every stream's settings; reset keeps them; set_streams keeps
        those of the streams below the new count."""
        n = self.n_streams if stream_ids is None else np.size(stream_ids)
        L = self.ctx.n_detect_labels
        rec = np.zeros((n, L), _native.STREAM_DETECT_DTYPE)
        rec["threshold"], rec["patience"] = np.nan, -1
        for field, val in (("threshold", threshold), ("patience", patience)):
            if val is None:
                continue
            for j, v in (val.items() if isinstance(val, dict) else ((j, val) for j in range(L))):
                if not isinstance(j, (int, np.integer)) or not 0 <= j < L:
                    raise ValueError(f"no label {j!r}: the detector has {L} labels")
                if field == "threshold" and v is None:
                    rec["flags"][:, j] = _native.DETECT_NO_THRESHOLD
                elif v is not None:
                    rec[field][:, j] = v
        deb = np.nan if debounce_time is None else float(debounce_time)
        self.ctx.set_stream_detection(stream_ids, rec, deb, self._stream(stream))

    def clear_stream_detection(self, stream_ids=None, stream=None):
        """Streams stream_ids (None = all) detect with the handle's settings again."""
        self.ctx.set_stream_detection(stream_ids, None, None, self._stream(stream))

    def stream_detection(self, stream_ids=None):
        """-> (records _native.STREAM_DETECT_DTYPE [n, n_labels], float64 [n] debounce) of streams stream_ids (None = all):
        threshold NaN / patience -1 / debounce NaN = the handle's, flags _native.DETECT_NO_THRESHOLD = no threshold.  What
        ``set_stream_detection_records`` takes, on this engine or another with the same labels, to move the settings."""
        return self.ctx.stream_detection(stream_ids)

    def set_stream_detection_records(self, stream_ids, records, debounce):
        """Streams stream_ids (distinct) take the settings ``stream_detection`` returned for other streams."""
        self.ctx.set_stream_detection(stream_ids, records, debounce, self._stream(None))

    # ---- stream audio on the device (include/owwb200.h, oww_set_audio_history) ----
    def set_audio_history(self, n_samples):
        """Keep the last n_samples (a multiple of 1280, up to 960000; 0 = off) samples every stream steps on the device.
        Synchronises the device; every stream starts with an empty history."""
        self.ctx.set_audio_history(n_samples)

    def get_audio(self, stream_ids, n_samples, end=None):
        """-> (int16 [n, n_samples] on the device, int64 [n] on the device): row i = samples [e - n_samples, e) of stream
        stream_ids[i] (ids may repeat), e = end[i] (None or < 0: the stream's position, the samples it has stepped since its
        reset), and the stream's position.  Samples the history does not hold (before it, overwritten, or not stepped yet)
        are zeros.  Enqueued on the current CUDA stream, after the steps enqueued there and the submitted host steps."""
        return self.ctx.read_audio(stream_ids, n_samples, end)

    def audio_history(self, stream_ids):
        """-> (int16 [n, H] oldest first, int64 [n] positions) host arrays of the listed streams, for moving them"""
        return self.ctx.audio_state(stream_ids)

    def set_audio_history_state(self, stream_ids, audio, pos):
        """Streams stream_ids (distinct) continue from the history `audio_history` returned, of this engine or another
        with the same history length."""
        self.ctx.set_audio_state(stream_ids, audio, pos)

    def detector_history(self, stream_ids):
        """-> (float32 [n, n_labels, 30] oldest first, int32 [n] predictions since the reset) of the listed streams"""
        return self.ctx.detector_history(stream_ids)

    def set_detector_history(self, stream_ids, hist, counts):
        """Streams stream_ids (distinct) continue from the history `detector_history` returned for other streams, of this
        engine or another with the same labels."""
        self.ctx.set_detector_history(stream_ids, hist, counts)

    # ---- custom verifier models (include/owwb200.h, oww_add_verifier_bank) ----
    def add_verifier_bank(self, head_index, capacity, threshold=0.1):
        """Slots for `capacity` verifiers of entry `head_index` of `heads`; every stream starts without one."""
        return self.ctx.add_verifier_bank(self.head_ids[head_index], capacity, threshold)

    def add_bank_verifier_bank(self, bank, capacity, threshold=0.1):
        """Slots for `capacity` verifiers of head bank `bank` (add_head_bank); a stream verifies only while it has a
        model in that bank."""
        return self.ctx.add_bank_verifier_bank(bank, capacity, threshold)

    def load_verifier(self, bank, slot, verifier):
        """verifier: a pickle path or pipeline of train_verifier_model's form, or (mean, weight, bias) arrays, on the head's
        n_in*96 features.  Synchronises the device: steps already enqueued use the slot's old contents."""
        if isinstance(verifier, tuple):
            params = verifier
        else:
            params = linear_verifier_params(load_verifier(verifier) if isinstance(verifier, str) else verifier)
            if params is None:
                raise ValueError("not a linear verifier pipeline (FunctionTransformer -> StandardScaler -> LogisticRegression)")
        self.ctx.load_verifier(bank, slot, *params)

    def assign_verifier(self, bank, slots, stream_ids=None, stream=None):
        """Stream stream_ids[i] (None = all) uses slot slots[i] (-1 = none) from the next ``step`` enqueued on the current
        CUDA stream (or `stream`) and the next ``step_host`` / ``submit``."""
        self.ctx.assign_verifier(bank, stream_ids, slots, self._stream(stream))

    def _stream(self, stream):
        if stream is None:
            torch = _torch()
            stream = torch.cuda.current_stream(torch.device("cuda", self.device_index)).cuda_stream
        return stream

    # ---- per-stream head banks (include/owwb200.h, oww_add_head_bank) ----
    def add_head_bank(self, shape, capacity):
        """Slots for `capacity` heads of the shape of head dict `shape` (one network, not a gated pair); every stream
        starts on slot -1 (zeros).  Its columns follow the current ones: returns (bank id, first column, n_out)."""
        n_in, dims, ln, fin = _weights.head_desc(shape)
        col0 = self.ctx.n_outputs
        bank = self.ctx.add_head_bank(n_in, dims, ln, fin, capacity)
        self.n_cols = self.ctx.n_outputs
        return bank, col0, dims[-1]

    def load_bank_head(self, bank, slot, head):
        """head: a head dict of the bank's shape.  Synchronises the device: steps already enqueued keep the old one."""
        self.ctx.load_bank_head(bank, slot, _weights.pack_head_blob(head))

    def assign_bank_head(self, bank, slots, stream_ids=None, stream=None):
        """Stream stream_ids[i] (None = all) runs the head of slot slots[i] (-1 = none) from the next ``step`` enqueued on
        the current CUDA stream (or `stream`) and the next ``step_host`` / ``submit``."""
        self.ctx.assign_bank_head(bank, stream_ids, slots, self._stream(stream))

    def set_head_bank_clip_slot(self, bank, slot):
        self.ctx.set_head_bank_clip_slot(bank, slot)

    def bank_head_predict(self, bank, slot, d_feats, out):
        """d_feats: CUDA float32 [n, n_in, 96] -> out [n, n_out] with the head of `slot` (stateless)."""
        self.ctx.bank_head_predict(bank, slot, d_feats, d_feats.shape[0], out, self._stream(None))
        return out
