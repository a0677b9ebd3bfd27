"""ctypes binding of libowwb200.so (the C ABI in include/owwb200.h).

The library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is no CPU
fallback: if the shared object is missing, or no H100-class (sm_90) GPU is present, constructing a
``Context`` raises - the product path never routes through the NumPy oracle.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libowwb200.so")
MAX_HEAD_LAYERS = 8

CNN_FP32_WINDOW = 0
CNN_FP32_INCREMENTAL = 1
CNN_TC_WINDOW = 2
CNN_TC_INCREMENTAL = 3


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("max_chunks", C.c_int32), ("cnn_mode", C.c_int32),
                ("window_batch", C.c_int32), ("reserved", C.c_int32 * 4)]


class HeadDesc(C.Structure):
    _fields_ = [("n_in", C.c_int32), ("n_layers", C.c_int32), ("dims", C.c_int32 * (MAX_HEAD_LAYERS + 1)),
                ("layernorm", C.c_int32), ("final_act", C.c_int32)]


# name -> (restype, argtypes): every symbol include/owwb200.h declares
_P = C.c_void_p
_SIGNATURES = {
    "oww_create": (C.c_int, [C.POINTER(Config), C.POINTER(_P)]),
    "oww_destroy": (None, [_P]),
    "oww_last_error": (C.c_char_p, [_P]),
    "oww_version": (C.c_char_p, []),
    "oww_load_mel": (C.c_int, [_P, _P, _P]),
    "oww_load_embedding": (C.c_int, [_P, _P, C.c_size_t]),
    "oww_add_head": (C.c_int, [_P, C.POINTER(HeadDesc), _P, C.c_size_t, C.POINTER(C.c_int)]),
    "oww_add_gate": (C.c_int, [_P, C.c_int, C.c_int, C.c_float]),
    "oww_n_heads": (C.c_int, [_P]),
    "oww_n_outputs": (C.c_int, [_P]),
    "oww_melspectrogram": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, C.c_int, _P]),
    "oww_embed_windows": (C.c_int, [_P, _P, C.c_int, _P, _P]),
    "oww_head_predict": (C.c_int, [_P, C.c_int, _P, C.c_int, _P, _P]),
    "oww_set_streams": (C.c_int, [_P, C.c_int]),
    "oww_n_streams": (C.c_int, [_P]),
    "oww_reset": (C.c_int, [_P, _P, C.c_int, _P, C.c_int]),
    "oww_reset_async": (C.c_int, [_P, _P, C.c_int, _P, C.c_int, _P]),
    "oww_step": (C.c_int, [_P, _P, C.c_int64, C.c_int, _P, _P]),
    "oww_step_host": (C.c_int, [_P, _P, C.c_int64, C.c_int, _P]),
    "oww_step_host_submit": (C.c_int, [_P, _P, C.c_int64, C.c_int, C.POINTER(C.c_int)]),
    "oww_step_host_collect": (C.c_int, [_P, C.c_int, _P]),
    "oww_get_features": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P]),
    "oww_get_mel": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "oww_get_counts": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "oww_embed_clips": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P]),
    "oww_predict_clips": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, _P]),
    "oww_debug_layer": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P]),
    "oww_debug_inc_plan": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int]),
    "oww_debug_inc_clocks": (C.c_int, [_P, _P]),
    "oww_debug_inc_clocks_read": (C.c_int, [_P, _P]),
    "oww_debug_heads_clocks": (C.c_int, [_P, _P]),
    "oww_peer_alloc": (C.c_int, [_P, C.c_size_t, C.POINTER(C.c_void_p), C.c_char_p]),
    "oww_peer_free": (C.c_int, [_P, _P]),
    "oww_peer_open": (C.c_int, [_P, C.c_char_p, C.POINTER(C.c_void_p)]),
    "oww_peer_close": (C.c_int, [_P, _P]),
    "oww_peer_copy": (C.c_int, [_P, _P, _P, C.c_size_t, _P]),
    "oww_peer_signal": (C.c_int, [_P, _P, C.c_uint64, _P]),
    "oww_peer_wait": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_uint64, C.c_double, _P]),
    "oww_peer_status": (C.c_int, [_P, C.POINTER(C.c_int)]),
    "oww_metrics_false_positives": (C.c_int, [_P, _P, C.c_int64, C.c_int, C.c_int, _P, C.c_int, C.c_int, _P, _P]),
    "oww_metrics_count_ge": (C.c_int, [_P, _P, C.c_int64, _P, C.c_int, _P, _P]),
    "oww_launch_count": (C.c_uint64, [_P]),
    "oww_enable_stage_timing": (C.c_int, [_P, C.c_int]),
    "oww_stage_ms": (C.c_int, [_P, _P]),
}
EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib = None


def load_library():
    """dlopen the in-tree library and bind every exported symbol (no GPU needed for this)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: the CUDA extension has not been built. Run "
            "`python -c 'import __graft_entry__ as g; g.build()'` at the repo root (nvcc, sm_90a). "
            "There is no CPU fallback for the b200 backend.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError here = header/library mismatch
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class NativeError(RuntimeError):
    pass


def _ptr(a):
    """Device/host address of a numpy array, torch tensor, int or None."""
    if a is None:
        return None
    if isinstance(a, int):
        return a
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return a.data_ptr()      # torch.Tensor


class Context:
    """One handle = one GPU's weights + stream state (include/owwb200.h conventions)."""

    def __init__(self, device=0, max_chunks=4, cnn_mode=CNN_TC_INCREMENTAL, window_batch=0, fuse_step=True,
                 tc_heads=True, tc_heads_terms=3, split_from=None, group_heads=True, late_blocked=True):
        """split_from: first conv layer that takes fp16 hi/lo split operands in the tensor-core modes (fp32-grade products;
        11 = default: scores within ~2e-4 of the fp32 graph; 20 = plain fp16 everywhere: the whole step as ONE fused
        launch, ~9e-4)."""
        self.lib = load_library()
        cfg = Config(device=device, max_chunks=max_chunks, cnn_mode=cnn_mode, window_batch=window_batch)
        cfg.reserved[0] = ((0 if fuse_step else 1) | (0 if tc_heads else 2) | (4 if tc_heads_terms == 1 else 0)
                           | (0 if group_heads else 8) | (0 if late_blocked else 16)
                           | int(os.environ.get("OWW_FLAGS", "0"), 0))      # extra reserved[0] bits for A/B runs (include/owwb200.h)
        if split_from is None:                      # library default (0), or OWW_SPLIT_FROM for experiments
            split_from = int(os.environ.get("OWW_SPLIT_FROM", "0"))
        cfg.reserved[1] = int(split_from)
        h = _P()
        rc = self.lib.oww_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise NativeError(f"oww_create failed ({rc}): {self.lib.oww_last_error(None).decode()}")
        self.h = h
        self.device = device
        self.max_chunks = max_chunks

    def close(self):
        if getattr(self, "h", None):
            self.lib.oww_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise NativeError(f"libowwb200 error {rc}: {self.lib.oww_last_error(self.h).decode()}")

    # ---- weights ----
    def load_mel(self, window512=None, mel_fb=None):
        w = None if window512 is None else np.ascontiguousarray(window512, np.float32)
        f = None if mel_fb is None else np.ascontiguousarray(mel_fb, np.float32)
        self._check(self.lib.oww_load_mel(self.h, _ptr(w), _ptr(f)))

    def load_embedding(self, blob):
        blob = np.ascontiguousarray(blob, np.float32)
        self._check(self.lib.oww_load_embedding(self.h, _ptr(blob), blob.size))

    def add_head(self, n_in, dims, layernorm, final_act, blob):
        d = HeadDesc(n_in=n_in, n_layers=len(dims) - 1, layernorm=int(layernorm), final_act=int(final_act))
        if len(dims) - 1 > MAX_HEAD_LAYERS:
            raise NativeError("too many head layers")
        for i, v in enumerate(dims):
            d.dims[i] = int(v)
        blob = np.ascontiguousarray(blob, np.float32)
        hid = C.c_int(-1)
        self._check(self.lib.oww_add_head(self.h, C.byref(d), _ptr(blob), blob.size, C.byref(hid)))
        return hid.value

    def add_gate(self, main_head, verifier_head, threshold=0.5):
        self._check(self.lib.oww_add_gate(self.h, int(main_head), int(verifier_head), float(threshold)))

    @property
    def n_outputs(self):
        return self.lib.oww_n_outputs(self.h)

    @property
    def n_streams(self):
        return self.lib.oww_n_streams(self.h)

    @property
    def launch_count(self):
        return int(self.lib.oww_launch_count(self.h))

    # ---- stateless graph calls (device pointers) ----
    def melspectrogram(self, d_pcm, n_clips, n_samples, d_mel, affine=True, stream=None):
        self._check(self.lib.oww_melspectrogram(self.h, _ptr(d_pcm), n_clips, n_samples, _ptr(d_mel), int(affine), stream))

    def embed_windows(self, d_windows, n, d_emb, stream=None):
        self._check(self.lib.oww_embed_windows(self.h, _ptr(d_windows), n, _ptr(d_emb), stream))

    def head_predict(self, head_id, d_feats, n, d_out, stream=None):
        self._check(self.lib.oww_head_predict(self.h, head_id, _ptr(d_feats), n, _ptr(d_out), stream))

    # ---- streaming ----
    def set_streams(self, n):
        self._check(self.lib.oww_set_streams(self.h, int(n)))

    def reset(self, stream_ids=None, feature_init=None):
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, np.int32)
        fi = None if feature_init is None else np.ascontiguousarray(feature_init, np.float32)
        n_rows = 41 if fi is None else fi.shape[0]
        self._check(self.lib.oww_reset(self.h, _ptr(ids), 0 if ids is None else ids.size, _ptr(fi), n_rows))

    def reset_async(self, stream_ids=None, feature_init=None, stream=None):
        """Stream-ordered reset (no synchronisation): enqueue on the stream the steps run on."""
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, np.int32)
        fi = None if feature_init is None else np.ascontiguousarray(feature_init, np.float32)
        n_rows = 41 if fi is None else fi.shape[0]
        self._check(self.lib.oww_reset_async(self.h, _ptr(ids), 0 if ids is None else ids.size, _ptr(fi), n_rows, stream))

    def step(self, d_pcm, pcm_stride, n_chunks, d_scores, stream=None):
        self._check(self.lib.oww_step(self.h, _ptr(d_pcm), pcm_stride, n_chunks, _ptr(d_scores), stream))

    def step_host(self, pcm, n_chunks, scores_out):
        """pcm: C-contiguous int16 [B, n_chunks*1280]; scores_out: float32 [B, n_outputs]."""
        assert pcm.dtype == np.int16 and pcm.flags.c_contiguous
        assert scores_out.dtype == np.float32 and scores_out.flags.c_contiguous
        self._check(self.lib.oww_step_host(self.h, _ptr(pcm), pcm.shape[1], n_chunks, _ptr(scores_out)))

    def step_host_submit(self, pcm, n_chunks):
        assert pcm.dtype == np.int16 and pcm.flags.c_contiguous
        t = C.c_int(-1)
        self._check(self.lib.oww_step_host_submit(self.h, _ptr(pcm), pcm.shape[1], n_chunks, C.byref(t)))
        return t.value

    def step_host_collect(self, ticket, scores_out):
        assert scores_out.dtype == np.float32 and scores_out.flags.c_contiguous
        self._check(self.lib.oww_step_host_collect(self.h, ticket, _ptr(scores_out)))

    def get_features(self, stream_id, n, back=0):
        out = np.empty((n, 96), np.float32)
        self._check(self.lib.oww_get_features(self.h, stream_id, n, back, _ptr(out)))
        return out

    def get_counts(self, stream_id):
        """(mel rows, feature rows) written since the stream's last reset, initial rows included."""
        m, f = C.c_int(0), C.c_int(0)
        self._check(self.lib.oww_get_counts(self.h, stream_id, C.byref(m), C.byref(f)))
        return m.value, f.value

    def get_mel(self, stream_id, n_rows=76):
        out = np.empty((n_rows, 32), np.float32)
        self._check(self.lib.oww_get_mel(self.h, stream_id, n_rows, _ptr(out)))
        return out

    # ---- batch ----
    def embed_clips(self, d_pcm, n_clips, n_samples, d_emb, stream=None):
        self._check(self.lib.oww_embed_clips(self.h, _ptr(d_pcm), n_clips, n_samples, _ptr(d_emb), stream))

    def predict_clips(self, d_pcm, n_clips, n_samples, pad_samples, feature_init, d_scores, stream=None):
        fi = None if feature_init is None else np.ascontiguousarray(feature_init, np.float32)
        self._check(self.lib.oww_predict_clips(self.h, _ptr(d_pcm), n_clips, n_samples, pad_samples, _ptr(fi),
                                               41 if fi is None else fi.shape[0], _ptr(d_scores), stream))

    def debug_layer(self, d_windows, n, layer, d_out, stream=None):
        self._check(self.lib.oww_debug_layer(self.h, _ptr(d_windows), n, layer, _ptr(d_out), stream))

    def debug_inc_clocks_arm(self):
        out = np.zeros(104, np.int64)
        self._check(self.lib.oww_debug_inc_clocks(self.h, _ptr(out)))

    def debug_inc_clocks_read(self):
        out = np.zeros(104, np.int64)
        self._check(self.lib.oww_debug_inc_clocks_read(self.h, _ptr(out)))
        return out

    def debug_heads_clocks(self):
        """First call arms; later calls -> int64[8, 8] clock stamps per head group (include/owwb200.h)."""
        out = np.zeros(256, np.int64)
        self._check(self.lib.oww_debug_heads_clocks(self.h, _ptr(out)))
        return out

    # ---- peer memory (multi-GPU gather without a collective; include/owwb200.h) ----
    def peer_alloc(self, n_bytes):
        """-> (device address, 64-byte IPC handle) of a zero-filled buffer other ranks can open."""
        p = C.c_void_p()
        h = C.create_string_buffer(64)
        self._check(self.lib.oww_peer_alloc(self.h, int(n_bytes), C.byref(p), h))
        return int(p.value), bytes(h.raw)

    def peer_free(self, addr):
        self._check(self.lib.oww_peer_free(self.h, int(addr)))

    def peer_open(self, handle):
        p = C.c_void_p()
        self._check(self.lib.oww_peer_open(self.h, C.create_string_buffer(bytes(handle), 64), C.byref(p)))
        return int(p.value)

    def peer_close(self, addr):
        self._check(self.lib.oww_peer_close(self.h, int(addr)))

    def peer_copy(self, dst_addr, src, n_bytes, stream=None):
        """Stream-ordered block copy; src / dst: device addresses (int) or tensors."""
        self._check(self.lib.oww_peer_copy(self.h, dst_addr if isinstance(dst_addr, int) else _ptr(dst_addr),
                                           src if isinstance(src, int) else _ptr(src), int(n_bytes), stream))

    def peer_signal(self, flag_addr, value, stream=None):
        self._check(self.lib.oww_peer_signal(self.h, int(flag_addr), int(value), stream))

    def peer_wait(self, flags_addr, n, stride, value, timeout_s=10.0, stream=None):
        self._check(self.lib.oww_peer_wait(self.h, int(flags_addr), int(n), int(stride), int(value), float(timeout_s), stream))

    def peer_timed_out(self):
        """True if a peer_wait since the last call ran into its timeout (synchronises the device; clears the flag)."""
        v = C.c_int(0)
        self._check(self.lib.oww_peer_status(self.h, C.byref(v)))
        return bool(v.value)

    # ---- metrics (device-resident scores) ----
    def metrics_false_positives(self, d_scores, series_stride, n_series, n_frames, thresholds, grouping_window=50, stream=None):
        thr = np.ascontiguousarray(thresholds, np.float64)
        out = np.zeros((n_series, thr.size), np.int32)
        self._check(self.lib.oww_metrics_false_positives(self.h, _ptr(d_scores), int(series_stride), int(n_series), int(n_frames),
                                                         _ptr(thr), thr.size, int(grouping_window), _ptr(out), stream))
        return out

    def metrics_count_ge(self, d_scores, n, thresholds, stream=None):
        thr = np.ascontiguousarray(thresholds, np.float64)
        out = np.zeros(thr.size, np.uint64)
        for j0 in range(0, thr.size, 64):
            t = np.ascontiguousarray(thr[j0:j0 + 64])
            o = np.zeros(t.size, np.uint64)
            self._check(self.lib.oww_metrics_count_ge(self.h, _ptr(d_scores), int(n), _ptr(t), t.size, _ptr(o), stream))
            out[j0:j0 + 64] = o
        return out

    # ---- introspection ----
    def enable_stage_timing(self, n_slots=1):
        self._check(self.lib.oww_enable_stage_timing(self.h, int(n_slots)))

    def stage_ms(self):
        out = (C.c_float * 3)()
        self._check(self.lib.oww_stage_ms(self.h, out))
        return {"mel": out[0], "cnn": out[1], "heads": out[2]}
