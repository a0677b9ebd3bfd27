"""CUDA mirror of the reference's ``openwakeword.utils`` surface for the inference hot path.

``AudioFeatures`` keeps the reference's constructor / call / attribute surface
(openwakeword/utils.py:33-463) but owns a libowwb200 ``Context``: the PCM tail,
mel ring and embedding ring live in HBM and one ``__call__`` is one C-ABI step for every stream.
``bulk_predict`` keeps the reference signature (utils.py:467-539) and runs clips of any lengths through
``oww_predict_clips_ragged`` with fresh state per clip.  Host code here only moves arguments, shapes and
errors; all arithmetic is in the CUDA library.
"""
import functools
import os
import wave
from collections import deque

import numpy as np

from . import _native
from . import weights as _weights

CHUNK = 1280
_MODELS_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "resources", "models")


def re_arg(kwarg_map):
    """Rename deprecated keyword arguments (same role as the reference's ``re_arg`` shim,
    utils.py:677-688, used for ``wakeword_model_paths`` -> ``wakeword_models``)."""
    def deco(fn):
        @functools.wraps(fn)
        def wrapped(*args, **kwargs):
            renamed = {kwarg_map.get(k, k): v for k, v in kwargs.items()}
            return fn(*args, **renamed)
        return wrapped
    return deco


def _torch():
    import torch
    return torch


def load_embedding_weights(path):
    """'' -> resources/models/embedding_model.{npz,onnx} ; 'synthetic[:seed]' -> seeded synthetic weights;
    '*.npz' -> weights.load_embedding ; '*.onnx' -> onnx_io.embedding_from_onnx (SURVEY.md Appendix E)."""
    if isinstance(path, dict):
        return path
    if path.startswith("synthetic"):
        seed = int(path.split(":")[1]) if ":" in path else 0
        return _weights.synthetic_embedding(seed)
    if path == "":
        path = os.path.join(_MODELS_DIR, "embedding_model.npz")
        if not os.path.exists(path) and os.path.exists(path[:-4] + ".onnx"):
            path = path[:-4] + ".onnx"
    if ".tflite" in path:
        raise ValueError("The b200 inference framework is selected, but tflite models were provided!")
    if not os.path.exists(path):
        raise ValueError(
            f"Embedding model file '{path}' not found. The reference's released weights are download-only; "
            "convert them with openwakeword_b200.weights.save_embedding or pass embedding_model_path='synthetic:0'.")
    if path.endswith(".onnx"):
        from .onnx_io import embedding_from_onnx
        return embedding_from_onnx(path)
    return _weights.load_embedding(path)


class AudioFeatures:
    """PCM -> log-mel -> speech-embedding features, streaming and batch, on one GPU.

    Extra keywords over the reference: ``n_streams`` (independent audio streams packed on the batch
    axis; 1 behaves exactly like the reference object), ``feature_init`` ([rows,96] initial content
    of the embedding ring - the reference fills it from unseeded noise, SURVEY.md F6; default is
    the embeddings of ``np.random.randint(-1000,1000,64000)`` computed on the GPU, as the reference
    does), ``max_chunks`` (largest multiple of 1280 samples one call may carry), ``cnn_mode``, ``audio_history``
    (seconds, a multiple of 0.08; 0 = off): the last samples every stream stepped are kept on the device
    (include/owwb200.h, oww_set_audio_history) and ``raw_data_buffer`` reads them as the reference's deque.

    ``sr``, the reference's keyword ("The sample rate of the audio"): 16000 (the default) keeps the host-side chunk
    accumulation.  Any other rate of the library's table (8000, 11025, 12000, 22050, 24000, 32000, 44100, 48000), or a
    sequence of n_streams rates, turns on device ingest for every stream of the handle (include/owwb200.h, oww_ingest):
    calls take each stream's audio at its own rate, the device resamples it to 16 kHz and keeps the samples below a chunk
    there.  Features, scores and the audio history are then those of the 16 kHz samples the resampler makes final.
    """

    def __init__(self, melspec_model_path="", embedding_model_path="", sr=16000, ncpu=1,
                 inference_framework="b200", device="gpu", n_streams=1, feature_init=None,
                 max_chunks=8, cnn_mode=_native.CNN_TC_INCREMENTAL, window_batch=0, device_index=0, split_from=None,
                 audio_history=0.0):
        if inference_framework != "b200":
            raise ValueError(f"openwakeword_b200 only provides inference_framework='b200' (got '{inference_framework}')")
        self.n_streams = int(n_streams)
        self.sample_rates = input_rates(sr, self.n_streams)    # None: 16 kHz on the host-side path
        self.ingest = self.sample_rates is not None
        self.audio_history_samples = audio_history_samples(audio_history)
        self.ctx = _native.Context(device=device_index, max_chunks=max_chunks, cnn_mode=cnn_mode,
                                   window_batch=window_batch, split_from=split_from)
        if melspec_model_path.endswith(".npz"):
            z = np.load(melspec_model_path)
            self.ctx.load_mel(z["window"], z["mel_fb"])
        else:       # '' / 'builtin' / a melspectrogram.onnx path: the graph's constants are closed-form (SURVEY App. A)
            if ".tflite" in melspec_model_path:
                raise ValueError("The b200 inference framework is selected, but tflite models were provided!")
            self.ctx.load_mel()
        self.embedding_weights = load_embedding_weights(embedding_model_path)
        self.ctx.load_embedding(_weights.pack_embedding_blob(self.embedding_weights))
        if self.audio_history_samples:
            self.ctx.set_audio_history(self.audio_history_samples)
        self.cnn_mode = cnn_mode
        self.max_chunks = max_chunks
        self.device_index = device_index
        self.onnx_execution_provider = "B200ExecutionProvider"
        self.melspectrogram_max_len = 10 * 97
        self.feature_buffer_max_len = 120
        self._feature_init = None if feature_init is None else np.asarray(feature_init, np.float32)
        self._streams_ready = False
        self._pending = np.zeros((self.n_streams, 0), np.int16)
        self._rpend = None
        # per stream: the samples it holds not yet stepped are in the reference's raw_data_buffer (its last call stepped
        # nothing, accumulated_samples > 0 there); a remainder left after a step is not
        self._held_in_raw = np.zeros(self.n_streams, bool)
        self._verifier_banks = False    # set by Model once the handle has a verifier bank (split calls skip the banks)
        # the three session callables of the reference (utils.py:87,93), numpy in / numpy out
        self.melspec_model_predict = self._melspec_model_predict
        self.embedding_model_predict = self._embedding_model_predict

    # ---- lazily allocate the stream state (heads must be registered on ctx first) ----
    def _ensure_streams(self):
        if not self._streams_ready:
            self._set_streams()
            self.reset()

    def _set_streams(self):
        self.ctx.set_streams(self.n_streams)
        if self.ingest:
            self.ctx.set_input_rates(None, self.sample_rates)
        self._streams_ready = True

    def set_sample_rates(self, stream_ids, rates):
        """Streams stream_ids take audio at rates[i] (one int for all, or one per id) from the next call on; their
        resamplers restart and the 16 kHz samples they hold are kept.  Needs device ingest (``sr`` other than 16000)."""
        if not self.ingest:
            raise ValueError("set_sample_rates needs device ingest: construct with sr=<rate> or sr=[one rate per stream]")
        self._ensure_streams()
        ids = np.asarray(stream_ids, np.int64).ravel()
        if ids.size and (ids.min() < 0 or ids.max() >= self.n_streams):
            raise ValueError(f"stream ids must lie in [0, {self.n_streams})")
        r = np.broadcast_to(np.asarray(rates, np.int64), ids.shape).astype(np.int32)
        self.ctx.set_input_rates(ids.astype(np.int32), r)
        self.sample_rates[ids] = r

    def reset(self, feature_init=None, stream_ids=None):
        """Reset buffers (utils.py:172-178).  ``feature_init`` overrides the ring content."""
        if not self._streams_ready:
            self._set_streams()
        fi = feature_init if feature_init is not None else self._feature_init
        if fi is None:
            noise = np.random.randint(-1000, 1000, 16000 * 4).astype(np.int16)
            fi = self._get_embeddings(noise)
        self.ctx.reset(stream_ids, np.asarray(fi, np.float32))
        if stream_ids is None:
            self._pending = np.zeros((self.n_streams, 0), np.int16)
            self._rpend = None
            self.accumulated_samples = 0
            self._held_in_raw[:] = False
        else:
            buf, lens = self._ragged_pending()
            lens[np.asarray(stream_ids, np.int64)] = 0
            self._set_ragged_pending(buf, lens)
            self._held_in_raw[np.asarray(stream_ids, np.int64)] = False

    # ---- per-stream remainders: `_pending` [B, L] while every stream holds the same number of samples, else
    #      `_rpend` = (int16 [B, 1279], lengths [B]) ----
    def _ragged_pending(self):
        if self._rpend is not None:
            return self._rpend[0].copy(), self._rpend[1].copy()
        buf = np.zeros((self.n_streams, CHUNK - 1), np.int16)
        L = self._pending.shape[1]
        buf[:, :L] = self._pending
        return buf, np.full(self.n_streams, L, np.int64)

    def _set_ragged_pending(self, buf, lens):
        if (lens == lens[0]).all():
            self._pending = buf[:, :int(lens[0])].copy()
            self._rpend = None
        else:
            self._rpend = (buf, lens)

    @property
    def pending_ragged(self):
        """True while the streams hold different numbers of not yet stepped samples (lockstep input then runs through
        the ragged path).  Always true with device ingest, whose calls are per stream."""
        return self._rpend is not None or self.ingest

    # ---- session-shaped calls ----
    def _melspec_model_predict(self, x):
        """float32/int16 [B,n] -> [array [B,1,T,32]] raw dB (what melspectrogram.onnx returns)."""
        x = np.asarray(x)
        x = x[None] if x.ndim == 1 else x
        return [self._mel_device(x.astype(np.int16), affine=False).cpu().numpy()[:, None]]

    def _embedding_model_predict(self, x):
        """float32 [N,76,32,1] -> squeezed [N,96] ([96] for N=1), as utils.py:93."""
        torch = _torch()
        x = np.ascontiguousarray(np.asarray(x, np.float32).reshape(-1, 76, 32))
        d = torch.from_numpy(x).to(f"cuda:{self.device_index}")
        out = torch.empty((x.shape[0], 96), dtype=torch.float32, device=d.device)
        self.ctx.embed_windows(d, x.shape[0], out, torch.cuda.current_stream(d.device).cuda_stream)
        return out.cpu().numpy().squeeze()

    def _mel_device(self, x_int16, affine=True):
        torch = _torch()
        x = np.ascontiguousarray(x_int16)
        n, s = x.shape
        if s < 512:
            raise ValueError("The number of input frames must be at least 512 samples for the mel model")
        d = torch.from_numpy(x).to(f"cuda:{self.device_index}")
        T = (s - 512) // 160 + 1
        out = torch.empty((n, T, 32), dtype=torch.float32, device=d.device)
        self.ctx.melspectrogram(d, n, s, out, affine, torch.cuda.current_stream(d.device).cuda_stream)
        return out

    def _get_melspectrogram(self, x, melspec_transform=None):
        """utils.py:180-208: int16 (or list) -> mel [T,32] (or [B,T,32]) after x/10+2."""
        x = np.array(x).astype(np.int16) if isinstance(x, list) else np.asarray(x)
        if x.dtype != np.int16:
            raise ValueError("Input data must be 16-bit integers (i.e., 16-bit PCM audio)."
                             f"You provided {x.dtype} data.")
        x = x[None] if x.ndim < 2 else x
        if melspec_transform is None:
            return np.squeeze(self._mel_device(x, affine=True).cpu().numpy())
        return melspec_transform(np.squeeze(self._mel_device(x, affine=False).cpu().numpy()))

    def _get_embeddings_from_melspec(self, melspec):
        melspec = np.asarray(melspec, np.float32)
        if melspec.shape[0] != 1:
            melspec = melspec[None]
        return self._embedding_model_predict(melspec)

    def _get_embeddings(self, x, window_size=76, step_size=8, **kwargs):
        """utils.py:225-236: whole-clip mel, 76-row windows every 8 rows -> [W,96]."""
        x = np.asarray(x)
        if x.dtype != np.int16:
            raise ValueError(f"Input data must be 16-bit integers. You provided {x.dtype} data.")
        return self.embed_clips(x[None])[0]

    def get_embedding_shape(self, audio_length, sr=16000):
        n = int(audio_length * sr)
        T = (n - 512) // 160 + 1
        return ((T - 76) // 8 + 1, 96)

    def _get_melspectrogram_batch(self, x, batch_size=128, ncpu=1):
        return self._mel_device(np.asarray(x, np.int16), affine=True).cpu().numpy()

    def _get_embeddings_batch(self, x, batch_size=128, ncpu=1):
        x = np.asarray(x, np.float32)
        if x.ndim == 4:
            x = x[..., 0]
        if x.shape[1] < 76:
            raise ValueError("Embedding model requires the input melspectrograms to have at least 76 frames")
        n_w = (x.shape[1] - 76) // 8 + 1
        wins = np.stack([x[:, 8 * i:8 * i + 76] for i in range(n_w)], axis=1).reshape(-1, 76, 32)
        return np.atleast_2d(self._embedding_model_predict(wins)).reshape(x.shape[0], n_w, 96)

    def embed_clips(self, x, batch_size=128, ncpu=1, sr=16000):
        """utils.py:358-385: int16 [N,samples] -> float32 [N,(T-76)//8+1,96]; one device call.  ``sr``: the clips' rate;
        at another rate of the table they are resampled on the device first (resample_clips, no padding) and T counts
        the A(samples) 16 kHz samples."""
        torch = _torch()
        x = np.ascontiguousarray(np.asarray(x))
        if x.dtype != np.int16:
            raise ValueError(f"Input data must be 16-bit integers. You provided {x.dtype} data.")
        n, s = x.shape
        if int(sr) != 16000:
            s = _native.resample_clip_plan(int(sr), s, 0)
        T = (s - 512) // 160 + 1 if s >= 512 else 0
        if T < 76:
            raise ValueError("Embedding model requires the input melspectrograms to have at least 76 frames")
        W = (T - 76) // 8 + 1
        if int(sr) != 16000:
            d, _ = self.resample_clips(x.reshape(-1), np.arange(n + 1, dtype=np.int64) * x.shape[1], int(sr), 0)
        else:
            d = torch.from_numpy(x).to(f"cuda:{self.device_index}")
        out = torch.empty((n, W, 96), dtype=torch.float32, device=d.device)
        self.ctx.embed_clips(d, n, s, out, torch.cuda.current_stream(d.device).cuda_stream)
        return out.cpu().numpy()

    def resample_clips(self, pcm, offsets, rates, pad_samples=0):
        """Clips at any rates of the table -> 16 kHz on the device in one launch (include/owwb200.h, oww_resample_clips):
        clip i is ``pcm[offsets[i]:offsets[i+1]]`` (int16 host array or tensor) at ``rates[i]`` Hz (or one rate for all),
        padded with ``pad_samples`` 16 kHz samples each side.  Returns (int16 CUDA tensor, int64 host offsets [N+1]) of the
        resampled clips, pads included: what a fresh stream of that rate makes of the padded clip."""
        torch = _torch()
        offsets = np.ascontiguousarray(offsets, np.int64).ravel()
        n = offsets.size - 1
        rates = np.ascontiguousarray(np.broadcast_to(np.asarray(rates, np.int64).ravel(), (n,)), np.int32)
        lengths = [_native.resample_clip_plan(int(r), int(k), int(pad_samples)) for r, k in zip(rates, np.diff(offsets))]
        out_off = np.concatenate([[0], np.cumsum(lengths, dtype=np.int64)]).astype(np.int64)
        dev = f"cuda:{self.device_index}"
        if isinstance(pcm, torch.Tensor):
            d_in = pcm.to(device=dev, dtype=torch.int16, non_blocking=True).contiguous()
        else:
            d_in = torch.from_numpy(np.ascontiguousarray(pcm, np.int16)).to(dev)
        d_out = torch.empty(max(int(out_off[-1]), 1), dtype=torch.int16, device=dev)[:int(out_off[-1])]
        self.ctx.resample_clips(d_in, offsets, rates, int(pad_samples), d_out, out_off,
                                torch.cuda.current_stream(d_out.device).cuda_stream)
        return d_out, out_off

    def mix_clips(self, fg, bg, n_samples, params, rirs=None):
        """Foreground clips mixed with background clips at an SNR, reverberated with room impulse responses and levelled,
        on the device in one call (include/owwb200.h, oww_mix_clips): the noisy, reverberant positives of a false-reject
        evaluation (the reference's mix_clips_batch).  ``fg`` and ``bg`` are int16 clips, ``rirs`` float32 ones, each a
        sequence of 1-D arrays or a ``(pcm, offsets)`` pair; ``params`` holds one ``_native.MIX_DTYPE`` record per
        mixture.  Returns (int16 CUDA tensor [n_mix, n_samples], bool CUDA tensor [n_mix] valid); the tensor goes to
        ``predict_clips_array`` / ``predict_clips_ragged`` / ``detect_clips`` as it is."""
        return _mix_clips_on(self.ctx, self.device_index, fg, bg, n_samples, params, rirs)

    # ---- streaming ----
    def _coerce(self, x):
        x = np.asarray(x)
        if x.dtype != np.int16:
            x = x.astype(np.int16)          # the reference's list->int16 truncation (utils.py:194)
        if x.ndim == 1:
            x = x[None]
        if x.shape[0] != self.n_streams:
            raise ValueError(f"expected audio for {self.n_streams} stream(s), got {x.shape[0]}")
        return x

    def _streaming_features(self, x, scores_out=None, device=False):
        """Chunk accumulation of utils.py:409-452, shared by all streams (same lengths).
        Returns (n_prepared_samples, n_chunks_run).  Scores land in scores_out when a step ran.  device: scores_out is a
        device score matrix (Context.new_scores) and the steps run on the current CUDA stream without a copy back."""
        self._ensure_streams()
        x = self._coerce(x)
        step = self.ctx.step_pcm if device else self.ctx.step_host
        if scores_out is None:
            scores_out = np.empty((self.n_streams, max(self.ctx.n_outputs, 1)), np.float32)
        if self.ingest:                     # device ingest: per stream, at its rate
            n_prepared, n_chunks, _ = self._ingest_features(list(x), scores_out, device)
            self._last_scores = scores_out
            return n_prepared, n_chunks
        if self._rpend is not None:         # the streams hold different remainders: per-stream accumulation
            n_prepared, n_chunks, _ = self._streaming_features_ragged(list(x), scores_out, device)
            self._last_scores = scores_out
            return n_prepared, n_chunks
        buf = np.concatenate((self._pending, x), axis=1) if self._pending.shape[1] else x
        total = buf.shape[1]
        if total >= CHUNK:
            rem = total % CHUNK
            ready = buf[:, :total - rem]
            self._pending = buf[:, total - rem:].copy()
        else:
            self._pending = buf.copy()
            self.accumulated_samples = total
            self._held_in_raw[:] = True
            return total, 0
        n_chunks = ready.shape[1] // CHUNK
        if scores_out is None:
            scores_out = np.empty((self.n_streams, max(self.ctx.n_outputs, 1)), np.float32)
        if n_chunks <= self.max_chunks:
            step(np.ascontiguousarray(ready), n_chunks, scores_out)
        else:
            # a call longer than max_chunks*1280 samples (the reference accepts up to its 10 s raw buffer) runs as
            # several device calls of <= max_chunks chunks; per head the result is the max over all chunk windows, as in
            # model.py:287-298.  Only the scope of the mel graph's -80 dB clamp differs (per device call, not per host call).
            # Custom verifiers run after that max, on the newest window (model.py:319-328): the parts run without the
            # verifier banks and Model.predict verifies the max.
            part = self.ctx.new_scores() if device else np.empty_like(scores_out)
            every = np.ones(self.n_streams, bool)
            if self._verifier_banks:
                self.ctx.enable_verifiers(False)
            try:
                for k, c0 in enumerate(range(0, n_chunks, self.max_chunks)):
                    c1 = min(c0 + self.max_chunks, n_chunks)
                    step(np.ascontiguousarray(ready[:, c0 * CHUNK:c1 * CHUNK]), c1 - c0, scores_out if k == 0 else part)
                    if k:
                        _take_rows(scores_out, part, every, True)
            finally:
                if self._verifier_banks:
                    self.ctx.enable_verifiers(True)
        self.accumulated_samples = 0
        self._held_in_raw[:] = False
        self._last_scores = scores_out
        return ready.shape[1], n_chunks

    def _streaming_features_ragged(self, xs, scores_out, device=False):
        """Chunk accumulation of utils.py:409-452 per stream: stream b gets xs[b] (1-D int16, any length), steps the
        whole chunks of its remainder + xs[b] and keeps the rest.  One oww_step_host_ragged call per max_chunks chunks.
        Returns (n_prepared [B], n_chunks [B], split): n_prepared as the reference's AudioFeatures.__call__ returns it
        (the samples stepped, or the samples accumulated when no chunk was stepped); rows of scores_out of streams that
        stepped nothing are not written.  split: a stream stepped more than max_chunks chunks, so the calls ran without
        the verifier banks (the caller verifies the max over all chunk windows).  device: scores_out is a device score
        matrix (Context.new_scores) and the steps run on the current CUDA stream without a copy back."""
        self._ensure_streams()
        if self.ingest:
            return self._ingest_features(xs, scores_out, device)
        B = self.n_streams
        step = self.ctx.step_ragged_pcm if device else self.ctx.step_host_ragged
        buf, lens = self._ragged_pending()
        tot = lens + np.array([x.shape[0] for x in xs], np.int64)
        n_chunks = tot // CHUNK
        ready = [np.concatenate((buf[b, :lens[b]], xs[b])) if lens[b] else xs[b] for b in range(B)]
        new_buf = np.zeros_like(buf)
        new_lens = tot - n_chunks * CHUNK
        for b in range(B):
            if new_lens[b]:
                new_buf[b, :new_lens[b]] = ready[b][n_chunks[b] * CHUNK:]
        split = bool((n_chunks > self.max_chunks).any())
        part = (self.ctx.new_scores() if device else np.empty_like(scores_out)) if split else scores_out
        if split and self._verifier_banks:
            self.ctx.enable_verifiers(False)
        try:
            done = np.zeros(B, np.int64)
            while (done < n_chunks).any():
                c = np.minimum(n_chunks - done, self.max_chunks).astype(np.int32)
                pcm = np.zeros((B, int(c.max()) * CHUNK), np.int16)
                for b in np.nonzero(c)[0]:
                    pcm[b, :c[b] * CHUNK] = ready[b][done[b] * CHUNK:(done[b] + c[b]) * CHUNK]
                first = (done == 0) & (c > 0)
                step(pcm, c, part)
                if split:               # per stream the max over all its parts
                    _take_rows(scores_out, part, first, False)
                    _take_rows(scores_out, part, (done > 0) & (c > 0), True)
                done += c
        finally:
            if split and self._verifier_banks:
                self.ctx.enable_verifiers(True)
        self._set_ragged_pending(new_buf, new_lens)
        self._held_in_raw = n_chunks == 0
        n_prepared = np.where(n_chunks > 0, n_chunks * CHUNK, tot)
        return n_prepared, n_chunks, split

    def _ingest_features(self, xs, scores_out, device=False):
        """_streaming_features_ragged with device ingest: stream b's xs[b] is audio at its own rate.  One oww_ingest call
        when every stream's audio fits its capacity (oww_ingest_capacity), else as many as needed, each taking what fits;
        then, as on the host path, per stream the max over the parts and the verifier banks off for all of them (split).
        Returns (n_prepared [B], n_chunks [B], split) as _streaming_features_ragged does."""
        B = self.n_streams
        xs = [np.asarray(x).astype(np.int16, copy=False).ravel() for x in xs]
        lens = np.array([x.size for x in xs], np.int64)
        if getattr(self, "_d_ingest_scores", None) is None:
            self._d_ingest_scores = self.ctx.new_scores()
        d_scores = scores_out if device else self._d_ingest_scores
        split = bool((lens > self.ctx.ingest_capacity()).any())
        part = self.ctx.new_scores() if split else d_scores
        done = np.zeros(B, np.int64)
        prepared = np.zeros(B, np.int64)
        pos = np.zeros(B, np.int64)
        if split and self._verifier_banks:
            self.ctx.enable_verifiers(False)
        try:
            while True:
                take = np.minimum(lens - pos, self.ctx.ingest_capacity())
                offsets = np.concatenate([[0], np.cumsum(take)]).astype(np.int64)
                pcm = np.concatenate([xs[b][pos[b]:pos[b] + take[b]] for b in range(B)])
                c, p = self.ctx.ingest_pcm(pcm, offsets, part)
                if split:               # per stream the max over all its parts
                    _take_rows(d_scores, part, (done == 0) & (c > 0), False)
                    _take_rows(d_scores, part, (done > 0) & (c > 0), True)
                done += c
                prepared = p.astype(np.int64)
                pos += take
                if (pos >= lens).all():
                    break
        finally:
            if split and self._verifier_banks:
                self.ctx.enable_verifiers(True)
        if not device:
            stepped = done > 0
            if stepped.any():
                host = d_scores if isinstance(d_scores, np.ndarray) else d_scores.cpu().numpy()
                scores_out[stepped] = host[stepped]
        self._held_in_raw = done == 0
        n_prepared = np.where(done > 0, done * CHUNK, prepared)
        return n_prepared, done, split

    def _held(self, b):
        """int16 samples stream b holds not yet stepped (16 kHz)"""
        if self.ingest:
            _, _, staged, x, _ = self.ctx.ingest_state([b])
            return x[0, :staged[0]]
        buf, lens = self._ragged_pending()
        return buf[b, :lens[b]]

    def __call__(self, x):
        return self._streaming_features(x)[0]

    def get_features(self, n_feature_frames=16, start_ndx=-1, stream=0):
        """utils.py:454-460 on the device ring -> float32 [1,n,96]."""
        self._ensure_streams()
        n = int(n_feature_frames)
        if start_ndx == -1:
            return self.ctx.get_features(stream, n, 0)[None]
        # feature_buffer[start_ndx:end_ndx] of the reference: its buffer holds the last min(rows written, 120) rows
        length = self._feature_len(stream)
        end = start_ndx + n if start_ndx + n != 0 else length
        lo, hi, _ = slice(start_ndx, end).indices(length)
        if hi <= lo:
            return np.zeros((1, 0, 96), np.float32)
        return self.ctx.get_features(stream, hi - lo, length - hi)[None]

    def _feature_len(self, stream=0):
        return min(self.ctx.get_counts(stream)[1], self.feature_buffer_max_len)

    @property
    def feature_buffer(self):
        """[rows, 96]: the stream-0 buffer as the reference keeps it (at most 120 rows, utils.py:449-450)."""
        self._ensure_streams()
        return self.ctx.get_features(0, self._feature_len(0), 0)

    @property
    def melspectrogram_buffer(self):
        self._ensure_streams()
        return self.ctx.get_mel(0, 76)

    @property
    def raw_data_buffer(self):
        """What the reference's ``raw_data_buffer`` holds for stream 0 (utils.py:164,403-430), as a
        ``deque(maxlen=H)`` of ints, H = the audio history in samples: the samples the stream stepped, from the device,
        followed by the samples it holds not yet stepped when its last call stepped nothing (the reference buffers
        those at once, but not a remainder left over after a step).  Needs ``audio_history``; reads the device."""
        H = self.audio_history_samples
        if not H:
            raise AttributeError("raw_data_buffer needs the audio history on the device: construct AudioFeatures (or "
                                 "Model) with audio_history=<seconds>, e.g. audio_history=10 as the reference keeps")
        self._ensure_streams()
        audio, pos = self.ctx.audio_state([0])
        x = audio[0, H - int(min(pos[0], H)):]
        if self._held_in_raw[0]:
            x = np.concatenate((x, self._held(0)))[-H:]
        return deque(x.tolist(), maxlen=H)


def input_rates(sr, n_streams):
    """sr (an int, or a sequence of n_streams ints) -> int32 [n_streams] input rates for device ingest, or None for the
    default int 16000 (the host-side path).  ValueError for a rate the library does not take (oww_resampler_taps)."""
    if np.ndim(sr) == 0:
        if int(sr) == 16000:
            return None
        rates = np.full(n_streams, int(sr), np.int32)
    else:
        rates = np.asarray(sr, np.int64).ravel()
        if rates.size != n_streams:
            raise ValueError(f"sr has {rates.size} rates for {n_streams} streams")
        rates = rates.astype(np.int32)
    for r in np.unique(rates):
        _native.resampler_taps(int(r))
    return rates


def audio_history_samples(seconds):
    """audio_history in seconds -> samples (a multiple of 1280, up to 60 s); ValueError otherwise"""
    n = int(round(float(seconds) * 16000))
    if n < 0 or n % CHUNK or n > 60 * 16000 or abs(n - float(seconds) * 16000) > 1e-6 * max(n, 1):
        raise ValueError(f"audio_history={seconds}: seconds in whole 80 ms chunks (a multiple of 0.08), at most 60")
    return n


def _packed_clips(clips, dtype, dev):
    """A sequence of 1-D arrays or a (pcm, offsets) pair, told apart by the int64 offsets -> (CUDA tensor of `dtype`,
    int64 host offsets)"""
    torch = _torch()
    if isinstance(clips, tuple) and len(clips) == 2 and np.asarray(clips[1]).dtype == np.int64:
        pcm, off = clips
        off = np.ascontiguousarray(off, np.int64).ravel()
    else:
        parts = [np.asarray(c).ravel() for c in clips]
        off = np.concatenate([[0], np.cumsum([p.size for p in parts], dtype=np.int64)]).astype(np.int64)
        pcm = np.concatenate(parts) if parts else np.zeros(0, dtype)
    if isinstance(pcm, torch.Tensor):
        if pcm.dtype != getattr(torch, np.dtype(dtype).name):
            raise ValueError(f"clips must be {np.dtype(dtype).name}, got {pcm.dtype}")
        d = pcm.to(dev).contiguous().reshape(-1)
    else:
        pcm = np.asarray(pcm)
        if pcm.dtype != dtype:
            raise ValueError(f"clips must be {np.dtype(dtype).name}, got {pcm.dtype}")
        d = torch.from_numpy(np.ascontiguousarray(pcm).reshape(-1)).to(dev)
    return d, off


def _mix_clips_on(ctx, device_index, fg, bg, n_samples, params, rirs=None):
    """AudioFeatures.mix_clips on a bare Context (data.mix_clips_batch needs no model weights)"""
    torch = _torch()
    dev = f"cuda:{device_index}"
    params = np.ascontiguousarray(params, _native.MIX_DTYPE).ravel()
    d_fg, fg_off = _packed_clips(fg, np.int16, dev)
    d_bg, bg_off = _packed_clips(bg, np.int16, dev)
    d_rir, rir_off = _packed_clips([] if rirs is None else rirs, np.float32, dev)
    n = params.size
    out = torch.empty((n, int(n_samples)), dtype=torch.int16, device=dev)
    valid = torch.empty(n, dtype=torch.uint8, device=dev)
    ctx.mix_clips(d_fg, fg_off, d_bg, bg_off, d_rir, rir_off, params, int(n_samples), out, valid,
                  torch.cuda.current_stream(out.device).cuda_stream)
    return out, valid.bool()


def _take_rows(dst, src, rows, maximum):
    """dst[rows] = src[rows], or the element-wise max of the two; host arrays or device tensors, rows: bool [B]"""
    if not isinstance(dst, np.ndarray):
        torch = _torch()
        rows = torch.from_numpy(rows).to(dst.device)
        dst[rows] = torch.maximum(dst[rows], src[rows]) if maximum else src[rows]
    else:
        dst[rows] = np.maximum(dst[rows], src[rows]) if maximum else src[rows]


def _read_wav_rate(path):
    """16-bit single-channel WAV at any rate of the resampler's table -> (int16 samples, rate); ValueError naming the
    file otherwise"""
    with wave.open(path, mode="rb") as f:
        rate = f.getframerate()
        if f.getnchannels() != 1 or f.getsampwidth() != 2:
            raise ValueError(f"{path}: expected a 16-bit, single-channel WAV")
        if rate != 16000:
            try:
                _native.resampler_taps(rate)
            except ValueError as e:
                raise ValueError(f"{path}: {e}") from None
        return np.frombuffer(f.readframes(f.getnframes()), dtype=np.int16), rate


def _read_wav(path):
    pcm, rate = _read_wav_rate(path)
    if rate != 16000:
        raise ValueError(f"{path}: expected 16-bit, 16 khz, single-channel WAV")
    return pcm


def _read_wavs(paths, n_threads=1, reader=_read_wav):
    """RIFF parsing is I/O bound: read the files on ``n_threads`` host threads, keep the order."""
    if n_threads <= 1 or len(paths) < 2:
        return [reader(p) for p in paths]
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=int(n_threads)) as pool:
        return list(pool.map(reader, paths))


def compute_features_from_generator(generator, n_total, clip_duration, output_file, device="gpu", ncpu=1,
                                    audio_features=None, sr=16000):
    """Reference signature (utils.py:542-601): pull int16 batches ``[batch, clip_duration]`` from ``generator``,
    embed them (``AudioFeatures.embed_clips``, one device call per batch) and write float32
    ``[n, (T-76)//8+1, 96]`` to the ``.npy`` file ``output_file`` through a memmap, so the result may exceed host
    memory.  ``n_total`` may over-estimate the number of clips: the file is cut to the rows actually written (the
    reference trims trailing all-zero rows with ``data.trim_mmap`` - same result unless a clip embeds to exactly
    zero).  ``device``/``ncpu`` are accepted for signature compatibility; the work runs on the GPU.
    ``audio_features`` lets a caller reuse an existing ``AudioFeatures`` (weights already on the device).  ``sr``: the
    generator's rate; ``clip_duration`` counts its samples, and T those of the clip resampled to 16 kHz on the device."""
    from numpy.lib.format import open_memmap
    F = audio_features if audio_features is not None else AudioFeatures(device=device)
    n16 = clip_duration if int(sr) == 16000 else _native.resample_clip_plan(int(sr), int(clip_duration), 0)
    n_windows, dim = F.get_embedding_shape(n16 / 16000)
    if n_windows < 1:
        raise ValueError("clip_duration is too short for one 76-frame embedding window")
    n_total = int(n_total)
    fp = open_memmap(output_file, mode="w+", dtype=np.float32, shape=(n_total, n_windows, dim))
    rows = 0
    for k, audio in enumerate(generator):
        audio = np.asarray(audio)
        if k == 0 and audio.shape[0] > n_total:
            del fp
            os.remove(output_file)
            raise ValueError(f"The value of 'n_total' ({n_total}) is less than the batch size ({audio.shape[0]})."
                             " Please increase 'n_total' to be >= batch size.")
        if rows >= n_total:
            break
        kw = {} if int(sr) == 16000 else {"sr": int(sr)}
        feats = F.embed_clips(audio, batch_size=audio.shape[0], ncpu=ncpu, **kw)[: n_total - rows]
        fp[rows:rows + feats.shape[0]] = feats
        rows += feats.shape[0]
        fp.flush()
    del fp
    if rows < n_total:                                         # cut the file to what was produced
        tmp = output_file + ".trim.npy"
        src = np.load(output_file, mmap_mode="r")
        dst = open_memmap(tmp, mode="w+", dtype=np.float32, shape=(rows, n_windows, dim))
        for i in range(0, rows, 4096):
            dst[i:i + 4096] = src[i:min(rows, i + 4096)]
        dst.flush()
        del src, dst
        os.replace(tmp, output_file)


# pinned host staging per device call of bulk_predict: the files of one batch, int16 (a corpus larger than host memory
# streams through in batches of about this size)
BULK_STAGING_BYTES = 256 << 20


def _wav_batches(paths, budget):
    """consecutive groups of paths whose files total at most `budget` bytes (a larger file forms a group of its own)"""
    batch, size = [], 0
    for p in paths:
        b = os.path.getsize(p)
        if batch and size + b > budget:
            yield batch
            batch, size = [], 0
        batch.append(p)
        size += b
    if batch:
        yield batch


def bulk_predict(file_paths, wakeword_models, prediction_function="predict_clip", ncpu=1,
                 inference_framework="b200", **kwargs):
    """Reference signature (utils.py:467-539).  Clips are batched on the GPU instead of forked across ``ncpu``
    processes; ``ncpu`` is the number of host threads that read the WAV files.  Each clip starts from a fresh state (the
    reference bleeds state across the clips of one worker, SURVEY.md F9).  Files of any lengths go through one device call
    per batch of about BULK_STAGING_BYTES of audio (Model.predict_clips_ragged).  As in the reference, keyword arguments
    go to the Model constructor and to the prediction function where they name one of its parameters, and are dropped
    otherwise.  ``prediction_function``: "predict_clip" (``padding``, ``chunk_size``) or
    "_get_positive_prediction_frames" (``threshold``, ``return_type``).  Returns {path: result of the function}.
    Files are 16-bit single-channel WAVs at any rate of the resampler's table, mixed freely; each is read at its
    header's rate and resampled to 16 kHz on the device (one launch per batch; none for a batch of 16 kHz files).  An
    ``sr`` keyword is checked against every header and is not passed to the Model."""
    from .model import Model, _rows_to_dicts
    if prediction_function not in ("predict_clip", "_get_positive_prediction_frames"):
        raise ValueError("the b200 bulk path implements prediction_function='predict_clip' and "
                         "'_get_positive_prediction_frames'")
    import inspect
    init_names = set(inspect.signature(Model.__init__).parameters) | set(inspect.signature(AudioFeatures.__init__).parameters)
    init_kw = {k: v for k, v in kwargs.items() if k in init_names and k != "sr"}
    fn_names = set(inspect.signature(getattr(Model, prediction_function)).parameters) - {"self", "kwargs"}
    fn_kw = {k: v for k, v in kwargs.items() if k in fn_names}
    sr = kwargs.get("sr")
    mdl = Model(wakeword_models=wakeword_models, inference_framework=inference_framework, **init_kw)
    torch = _torch()
    out = {}
    for paths in _wav_batches(list(file_paths), BULK_STAGING_BYTES):
        read = _read_wavs(paths, ncpu, _read_wav_rate)        # RIFF parsing on ncpu host threads, order kept
        clips = [c for c, _ in read]
        rates = np.array([r for _, r in read], np.int32)
        if sr is not None:
            for p, r in zip(paths, rates):
                if r != int(sr):
                    raise ValueError(f"{p}: the header says {r} Hz, sr={sr}")
        rates = None if (rates == 16000).all() else rates      # 16 kHz batches run exactly as before
        if prediction_function == "_get_positive_prediction_frames":
            res = mdl._positive_frames_bulk(clips, threshold=fn_kw.get("threshold", 0.5),
                                            return_type=fn_kw.get("return_type", "features"), sr=rates)
            out.update(zip(paths, res))
            continue
        # the batch is gathered in page-locked memory so the H2D copy is a single asynchronous DMA (the reference forks
        # one process per ncpu instead, utils.py:505-536)
        offsets = np.concatenate([[0], np.cumsum([c.shape[0] for c in clips])]).astype(np.int64)
        stage = torch.empty(int(offsets[-1]), dtype=torch.int16, pin_memory=True)
        view = stage.numpy()
        for c, o in zip(clips, offsets):
            view[o:o + c.shape[0]] = c
        scores, row_off, labels = mdl.predict_clips_ragged(stage, offsets, padding=fn_kw.get("padding", 1),
                                                           chunk_size=fn_kw.get("chunk_size", CHUNK), sr=rates)
        out.update(zip(paths, _rows_to_dicts(scores, row_off, labels)))
    return out
