"""CUDA mirror of the reference's ``openwakeword.utils`` surface for the inference hot path.

``AudioFeatures`` keeps the reference's constructor / call / attribute surface
(openwakeword/utils.py:33-463) but owns a libowwb200 ``Context``: the PCM tail,
mel ring and embedding ring live in HBM and one ``__call__`` is one C-ABI step for every stream.
``bulk_predict`` keeps the reference signature (utils.py:467-539) and runs clips through
``oww_predict_clips`` with fresh state per clip.  Host code here only moves arguments, shapes and
errors; all arithmetic is in the CUDA library.
"""
import functools
import os
import wave

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
    does), ``max_chunks`` (largest multiple of 1280 samples one call may carry), ``cnn_mode``.
    """

    def __init__(self, melspec_model_path="", embedding_model_path="", sr=16000, ncpu=1,
                 inference_framework="b200", device="gpu", n_streams=1, feature_init=None,
                 max_chunks=8, cnn_mode=_native.CNN_TC_INCREMENTAL, window_batch=0, device_index=0, split_from=None):
        if inference_framework != "b200":
            raise ValueError(f"openwakeword_b200 only provides inference_framework='b200' (got '{inference_framework}')")
        if sr != 16000:
            raise ValueError("only 16 kHz audio is supported")
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
        self.n_streams = int(n_streams)
        self.cnn_mode = cnn_mode
        self.max_chunks = max_chunks
        self.device_index = device_index
        self.onnx_execution_provider = "B200ExecutionProvider"
        self.melspectrogram_max_len = 10 * 97
        self.feature_buffer_max_len = 120
        self._feature_init = None if feature_init is None else np.asarray(feature_init, np.float32)
        self._streams_ready = False
        # the three session callables of the reference (utils.py:87,93), numpy in / numpy out
        self.melspec_model_predict = self._melspec_model_predict
        self.embedding_model_predict = self._embedding_model_predict

    # ---- lazily allocate the stream state (heads must be registered on ctx first) ----
    def _ensure_streams(self):
        if not self._streams_ready:
            self.ctx.set_streams(self.n_streams)
            self._streams_ready = True
            self.reset()

    def reset(self, feature_init=None, stream_ids=None):
        """Reset buffers (utils.py:172-178).  ``feature_init`` overrides the ring content."""
        if not self._streams_ready:
            self.ctx.set_streams(self.n_streams)
            self._streams_ready = True
        fi = feature_init if feature_init is not None else self._feature_init
        if fi is None:
            noise = np.random.randint(-1000, 1000, 16000 * 4).astype(np.int16)
            fi = self._get_embeddings(noise)
        self.ctx.reset(stream_ids, np.asarray(fi, np.float32))
        if stream_ids is None:
            self._pending = np.zeros((self.n_streams, 0), np.int16)
            self.accumulated_samples = 0

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

    def embed_clips(self, x, batch_size=128, ncpu=1):
        """utils.py:358-385: int16 [N,samples] -> float32 [N,(T-76)//8+1,96]; one device call."""
        torch = _torch()
        x = np.ascontiguousarray(np.asarray(x))
        if x.dtype != np.int16:
            raise ValueError(f"Input data must be 16-bit integers. You provided {x.dtype} data.")
        n, s = x.shape
        T = (s - 512) // 160 + 1 if s >= 512 else 0
        if T < 76:
            raise ValueError("Embedding model requires the input melspectrograms to have at least 76 frames")
        W = (T - 76) // 8 + 1
        d = torch.from_numpy(x).to(f"cuda:{self.device_index}")
        out = torch.empty((n, W, 96), dtype=torch.float32, device=d.device)
        self.ctx.embed_clips(d, n, s, out, torch.cuda.current_stream(d.device).cuda_stream)
        return out.cpu().numpy()

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

    def _streaming_features(self, x, scores_out=None):
        """Chunk accumulation of utils.py:409-452, shared by all streams (same lengths).
        Returns (n_prepared_samples, n_chunks_run).  Scores land in scores_out when a step ran."""
        self._ensure_streams()
        x = self._coerce(x)
        buf = np.concatenate((self._pending, x), axis=1) if self._pending.shape[1] else x
        total = buf.shape[1]
        if total >= CHUNK:
            rem = total % CHUNK
            ready = buf[:, :total - rem]
            self._pending = buf[:, total - rem:].copy()
        else:
            self._pending = buf.copy()
            self.accumulated_samples = total
            return total, 0
        n_chunks = ready.shape[1] // CHUNK
        if scores_out is None:
            scores_out = np.empty((self.n_streams, max(self.ctx.n_outputs, 1)), np.float32)
        if n_chunks <= self.max_chunks:
            self.ctx.step_host(np.ascontiguousarray(ready), n_chunks, scores_out)
        else:
            # a call longer than max_chunks*1280 samples (the reference accepts up to its 10 s raw buffer) runs as
            # several device calls of <= max_chunks chunks; per head the result is the max over all chunk windows, as in
            # model.py:287-298.  Only the scope of the mel graph's -80 dB clamp differs (per device call, not per host call).
            part = np.empty_like(scores_out)
            for k, c0 in enumerate(range(0, n_chunks, self.max_chunks)):
                c1 = min(c0 + self.max_chunks, n_chunks)
                self.ctx.step_host(np.ascontiguousarray(ready[:, c0 * CHUNK:c1 * CHUNK]), c1 - c0, scores_out if k == 0 else part)
                if k:
                    np.maximum(scores_out, part, out=scores_out)
        self.accumulated_samples = 0
        self._last_scores = scores_out
        return ready.shape[1], n_chunks

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


def _read_wav(path):
    with wave.open(path, mode="rb") as f:
        if f.getframerate() != 16000 or f.getnchannels() != 1 or f.getsampwidth() != 2:
            raise ValueError(f"{path}: expected 16-bit, 16 khz, single-channel WAV")
        return np.frombuffer(f.readframes(f.getnframes()), dtype=np.int16)


def _read_wavs(paths, n_threads=1):
    """RIFF parsing is I/O bound: read the files on ``n_threads`` host threads, keep the order."""
    if n_threads <= 1 or len(paths) < 2:
        return [_read_wav(p) for p in paths]
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=int(n_threads)) as pool:
        return list(pool.map(_read_wav, paths))


def compute_features_from_generator(generator, n_total, clip_duration, output_file, device="gpu", ncpu=1,
                                    audio_features=None):
    """Reference signature (utils.py:542-601): pull int16 batches ``[batch, clip_duration]`` from ``generator``,
    embed them (``AudioFeatures.embed_clips``, one device call per batch) and write float32
    ``[n, (T-76)//8+1, 96]`` to the ``.npy`` file ``output_file`` through a memmap, so the result may exceed host
    memory.  ``n_total`` may over-estimate the number of clips: the file is cut to the rows actually written (the
    reference trims trailing all-zero rows with ``data.trim_mmap`` - same result unless a clip embeds to exactly
    zero).  ``device``/``ncpu`` are accepted for signature compatibility; the work runs on the GPU.
    ``audio_features`` lets a caller reuse an existing ``AudioFeatures`` (weights already on the device)."""
    from numpy.lib.format import open_memmap
    F = audio_features if audio_features is not None else AudioFeatures(device=device)
    n_windows, dim = F.get_embedding_shape(clip_duration / 16000)
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
        feats = F.embed_clips(audio, batch_size=audio.shape[0], ncpu=ncpu)[: n_total - rows]
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


def bulk_predict(file_paths, wakeword_models, prediction_function="predict_clip", ncpu=1,
                 inference_framework="b200", **kwargs):
    """Reference signature (utils.py:467-539).  Clips are batched on the GPU instead of forked across ``ncpu``
    processes; ``ncpu`` is the number of host threads that read the WAV files.  Each clip starts from a fresh state (the
    reference bleeds state across the clips of one worker, SURVEY.md F9).  Returns {path: list of dicts}."""
    from .model import Model
    if prediction_function != "predict_clip":
        raise ValueError("the b200 bulk path implements prediction_function='predict_clip'")
    import inspect
    init_names = set(inspect.signature(Model.__init__).parameters) | set(inspect.signature(AudioFeatures.__init__).parameters)
    init_kw = {k: v for k, v in kwargs.items() if k in init_names}
    clip_kw = {k: v for k, v in kwargs.items() if k not in init_names}
    mdl = Model(wakeword_models=wakeword_models, inference_framework=inference_framework, **init_kw)
    clips = _read_wavs(file_paths, ncpu)                       # RIFF parsing on ncpu host threads, order kept
    out = {}
    by_len = {}
    for p, c in zip(file_paths, clips):
        by_len.setdefault(c.shape[0], []).append(p)
    lookup = dict(zip(file_paths, clips))
    torch = _torch()
    for length, paths in by_len.items():
        # equal-length clips form one device batch; they are gathered in page-locked memory so the H2D copy is a single
        # asynchronous DMA (the reference forks one process per ncpu instead, utils.py:505-536)
        stage = torch.empty((len(paths), length), dtype=torch.int16, pin_memory=True)
        view = stage.numpy()
        for i, p in enumerate(paths):
            view[i] = lookup[p]
        res = mdl.predict_clips(stage, **clip_kw)
        for p, r in zip(paths, res):
            out[p] = r
    return out
