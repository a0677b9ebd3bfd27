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
MAX_CHUNKS = 131062          # OWW_MAX_CHUNKS: the largest max_chunks a handle takes

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


class DetectLabel(C.Structure):
    _fields_ = [("column", C.c_int32), ("repeats", C.c_int32), ("threshold", C.c_float), ("patience", C.c_int32)]


# one record of oww_detect's event list (oww_event): 16 bytes
EVENT_DTYPE = np.dtype([("stream", "<i4"), ("label", "<i4"), ("score", "<f4"), ("index", "<i4")])

# one (stream, label) record of oww_set_stream_detection (oww_stream_detect): 12 bytes.  threshold NaN: the handle's;
# patience -1: the handle's; flags DETECT_NO_THRESHOLD: the label has no threshold on the stream
STREAM_DETECT_DTYPE = np.dtype([("threshold", "<f4"), ("patience", "<i4"), ("flags", "<i4")])
DETECT_NO_THRESHOLD = 1

# one mixture of oww_mix_clips (oww_mix_params): 64 bytes.  rir = -1: no reverb; volume < 0: no volume
MIX_DTYPE = np.dtype([("fg", "<i4"), ("bg", "<i4"), ("rir", "<i4"), ("reserved", "<i4"), ("fg_start", "<i8"),
                      ("fg_len", "<i8"), ("bg_offset", "<i8"), ("start", "<i8"), ("snr_db", "<f8"), ("volume", "<f8")])


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
    "oww_add_verifier_bank": (C.c_int, [_P, C.c_int, C.c_int, C.c_float, C.POINTER(C.c_int)]),
    "oww_add_bank_verifier_bank": (C.c_int, [_P, C.c_int, C.c_int, C.c_float, C.POINTER(C.c_int)]),
    "oww_load_verifier": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, C.c_float]),
    "oww_assign_verifier": (C.c_int, [_P, C.c_int, _P, C.c_int, _P, _P]),
    "oww_set_verifier_clip_slot": (C.c_int, [_P, C.c_int, C.c_int]),
    "oww_set_verifier_threshold": (C.c_int, [_P, C.c_int, C.c_float]),
    "oww_enable_verifiers": (C.c_int, [_P, C.c_int]),
    "oww_verifier_predict": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int, _P, _P]),
    "oww_fit_verifiers": (C.c_int, [_P, _P, C.c_int64, C.c_int, _P, _P, _P, C.c_int, C.c_double, C.c_int, C.c_double,
                                    _P, _P, _P, _P, _P, _P, _P]),
    "oww_load_verifiers": (C.c_int, [_P, C.c_int, _P, C.c_int, _P, _P, _P, _P]),
    "oww_add_head_bank": (C.c_int, [_P, C.POINTER(HeadDesc), C.c_int, C.POINTER(C.c_int)]),
    "oww_load_bank_head": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_size_t]),
    "oww_assign_bank_head": (C.c_int, [_P, C.c_int, _P, C.c_int, _P, _P]),
    "oww_set_head_bank_clip_slot": (C.c_int, [_P, C.c_int, C.c_int]),
    "oww_bank_head_predict": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int, _P, _P]),
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
    "oww_step_ragged": (C.c_int, [_P, _P, C.c_int64, _P, _P, _P]),
    "oww_step_host_ragged": (C.c_int, [_P, _P, C.c_int64, _P, _P]),
    "oww_step_host_ragged_submit": (C.c_int, [_P, _P, C.c_int64, _P, C.POINTER(C.c_int)]),
    "oww_get_features": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P]),
    "oww_get_mel": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "oww_get_counts": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "oww_stream_state_info": (C.c_int, [_P, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)]),
    "oww_export_streams": (C.c_int, [_P, _P, C.c_int, _P, _P]),
    "oww_import_streams": (C.c_int, [_P, _P, C.c_int, _P, _P]),
    "oww_stream_state_status": (C.c_int, [_P, C.POINTER(C.c_int)]),
    "oww_set_detector": (C.c_int, [_P, C.POINTER(DetectLabel), C.c_int, C.c_double]),
    "oww_detect": (C.c_int, [_P, _P, C.c_int, _P, _P, _P, C.c_int, _P, _P]),
    "oww_detect_clips": (C.c_int, [_P, C.POINTER(DetectLabel), C.c_int, C.c_double, _P, _P, C.c_float, _P, C.c_int, C.c_int,
                                   _P, _P, C.c_int, _P, _P]),
    "oww_detector_export": (C.c_int, [_P, _P, C.c_int, _P, _P, _P]),
    "oww_detector_import": (C.c_int, [_P, _P, C.c_int, _P, _P, _P]),
    "oww_set_stream_detection": (C.c_int, [_P, _P, C.c_int, _P, _P, _P]),
    "oww_get_stream_detection": (C.c_int, [_P, _P, C.c_int, _P, _P]),
    "oww_set_audio_history": (C.c_int, [_P, C.c_int]),
    "oww_get_audio": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "oww_capture_events": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "oww_audio_export": (C.c_int, [_P, _P, C.c_int, _P, _P, _P]),
    "oww_audio_import": (C.c_int, [_P, _P, C.c_int, _P, _P, _P]),
    "oww_set_input_rates": (C.c_int, [_P, _P, C.c_int, _P, _P]),
    "oww_ingest": (C.c_int, [_P, _P, _P, _P, _P, _P, _P]),
    "oww_ingest_capacity": (C.c_int, [_P, _P]),
    "oww_ingest_plan": (C.c_int, [C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int64, C.POINTER(C.c_int64),
                                  C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "oww_resampler_taps": (C.c_int, [C.c_int, _P, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "oww_ingest_export": (C.c_int, [_P, _P, C.c_int, _P, _P, _P, _P, C.c_int64, _P, _P]),
    "oww_ingest_import": (C.c_int, [_P, _P, C.c_int, _P, _P, _P, _P, C.c_int64, _P, _P]),
    "oww_detect_host_submit": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "oww_detect_host_collect": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P, _P, _P]),
    "oww_embed_clips": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P]),
    "oww_predict_clips": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, _P]),
    "oww_clip_schedule": (C.c_int, [C.c_int, C.c_int64, _P, C.c_int]),
    "oww_predict_clips_ragged": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, _P, _P, _P]),
    "oww_predict_clips_streams": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, _P, _P, _P, _P]),
    "oww_clip_slab_plan": (C.c_int, [_P, _P, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "oww_resample_clip_plan": (C.c_int, [C.c_int, C.c_int64, C.c_int, C.POINTER(C.c_int64)]),
    "oww_resample_clips": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "oww_mix_clips": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, C.c_int, _P, _P, C.c_int, _P, C.c_int, C.c_int64, _P, _P, _P]),
    "oww_debug_layer": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P]),
    "oww_debug_inc_plan": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int]),
    "oww_debug_inc_cut_plan": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P, C.c_int]),
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
    "oww_metrics_false_positives_f64": (C.c_int, [_P, _P, C.c_int64, C.c_int, C.c_int, _P, C.c_int, C.c_int, _P, _P]),
    "oww_metrics_count_ge": (C.c_int, [_P, _P, C.c_int64, _P, C.c_int, _P, _P]),
    "oww_metrics_count_ge_f64": (C.c_int, [_P, _P, C.c_int64, _P, C.c_int, _P, _P]),
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


class ArgumentError(NativeError, ValueError):
    """A buffer the library would read or write out of bounds, refused in Python before the call.  A ValueError, and a
    NativeError like the library's own refusal of a short stride, so callers that catch either keep working."""


def clip_schedule(chunk_size, n_padded_samples):
    """Chunks each predict call of predict_clip(chunk_size) steps on n_padded_samples samples -> int32 [calls]
    (oww_clip_schedule: pure host code, no GPU needed)."""
    lib = load_library()
    n = lib.oww_clip_schedule(int(chunk_size), int(n_padded_samples), None, 0)
    if n < 0:
        raise NativeError(f"oww_clip_schedule failed ({n}): {lib.oww_last_error(None).decode()}")
    out = np.zeros(n, np.int32)
    if n:
        lib.oww_clip_schedule(int(chunk_size), int(n_padded_samples), _ptr(out), n)
    return out


def clip_slab_plan(steps, ctx=None):
    """Slabs the ragged bulk path runs for clips of `steps` chunks -> (slabs, steps computed, steps needed); pure host."""
    lib = load_library()
    st = np.ascontiguousarray(steps, np.int32)
    done, need = C.c_int64(0), C.c_int64(0)
    n = lib.oww_clip_slab_plan(ctx, _ptr(st), st.size, C.byref(done), C.byref(need))
    if n < 0:
        raise NativeError(f"oww_clip_slab_plan failed ({n})")
    return n, done.value, need.value


def resampler_taps(rate):
    """-> (float32 taps, up, down) the library resamples input at `rate` Hz with (no taps at 16000: a copy); ValueError
    for a rate outside its table (oww_resampler_taps: pure host code, no GPU needed)."""
    lib = load_library()
    up, down = C.c_int(0), C.c_int(0)
    n = lib.oww_resampler_taps(int(rate), None, 0, C.byref(up), C.byref(down))
    if n < 0:
        raise ValueError(f"sample rate {rate} Hz is not supported: the input rates are 8000, 11025, 12000, 16000, 22050, "
                         "24000, 32000, 44100 and 48000 Hz")
    taps = np.zeros(n, np.float32)
    if n:
        lib.oww_resampler_taps(int(rate), _ptr(taps), n, None, None)
    return taps, up.value, down.value


def ingest_plan(rate, max_chunks, n_before, staged, n_in):
    """What one oww_ingest call does to a stream (oww_ingest_plan: pure host, no GPU) -> (new final samples, chunks
    stepped, samples left staged, capacity); the first three are None when n_in is over the capacity."""
    lib = load_library()
    n_out, chunks, after, max_in = C.c_int64(0), C.c_int32(0), C.c_int32(0), C.c_int64(0)
    rc = lib.oww_ingest_plan(int(rate), int(max_chunks), int(n_before), int(staged), int(n_in), C.byref(n_out),
                             C.byref(chunks), C.byref(after), C.byref(max_in))
    if rc and n_in <= max_in.value:
        raise ValueError(f"oww_ingest_plan refused rate {rate}")
    if rc:
        return None, None, None, max_in.value
    return n_out.value, chunks.value, after.value, max_in.value


def resample_clip_plan(rate, n_in, pad_samples):
    """16 kHz samples a clip of n_in samples at `rate` becomes with pad_samples of padding each side (oww_resample_clip_plan:
    pure host, no GPU); ValueError for a rate outside the table, negative arguments, or a pad the rate cannot take."""
    lib = load_library()
    n = C.c_int64(0)
    if lib.oww_resample_clip_plan(int(rate), int(n_in), int(pad_samples), C.byref(n)):
        raise ValueError(f"oww_resample_clip_plan refused rate {rate}, {n_in} samples, pad {pad_samples}: the rates are "
                         "8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100 and 48000 Hz, and the padding a multiple "
                         "of 640 samples (40 ms)")
    return n.value


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
                 tc_heads=True, tc_heads_terms=3, split_from=None, group_heads=True):
        """split_from: first conv layer that takes fp16 hi/lo split operands in the tensor-core modes (fp32-grade products;
        11 = default: scores within ~2e-4 of the fp32 graph; 20 = plain fp16 everywhere: the whole step as ONE fused
        launch, ~9e-4)."""
        self.lib = load_library()
        cfg = Config(device=device, max_chunks=max_chunks, cnn_mode=cnn_mode, window_batch=window_batch)
        cfg.reserved[0] = ((0 if fuse_step else 1) | (0 if tc_heads else 2) | (4 if tc_heads_terms == 1 else 0)
                           | (0 if group_heads else 8)
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
        self._head_n_in = []                # per head id: n_in (verifier banks take n_in*96 floats per slot)
        self._bank_d = []                   # per verifier bank: D
        self._head_bank_n_in = []           # per head bank: n_in
        self.n_detect_labels = 0            # labels of the detector (set_detector)
        self._det_buf = None                # device event list and count of detect_events
        self.audio_history = 0              # samples of audio history per stream (set_audio_history; 0 = off)
        self._det_tickets = {}              # detect ticket -> (packets kept alive, the output arrays of its collect)

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

    @staticmethod
    def _desc(n_in, dims, layernorm, final_act):
        d = HeadDesc(n_in=n_in, n_layers=len(dims) - 1, layernorm=int(layernorm), final_act=int(final_act))
        if len(dims) - 1 > MAX_HEAD_LAYERS:
            raise NativeError("too many head layers")
        for i, v in enumerate(dims):
            d.dims[i] = int(v)
        return d

    def add_head(self, n_in, dims, layernorm, final_act, blob):
        d = self._desc(n_in, dims, layernorm, final_act)
        blob = np.ascontiguousarray(blob, np.float32)
        hid = C.c_int(-1)
        self._check(self.lib.oww_add_head(self.h, C.byref(d), _ptr(blob), blob.size, C.byref(hid)))
        self._head_n_in.append(int(n_in))
        return hid.value

    # ---- per-stream head banks (include/owwb200.h, oww_add_head_bank) ----
    def add_head_bank(self, n_in, dims, layernorm, final_act, capacity):
        """`capacity` slots of one head shape; its n_out columns are appended to the score row."""
        d = self._desc(n_in, dims, layernorm, final_act)
        bid = C.c_int(-1)
        self._check(self.lib.oww_add_head_bank(self.h, C.byref(d), int(capacity), C.byref(bid)))
        self._head_bank_n_in.append(int(n_in))
        return bid.value

    def load_bank_head(self, bank, slot, blob):
        """blob: weights.pack_head_blob of a head of the bank's shape (synchronises the device)."""
        blob = np.ascontiguousarray(blob, np.float32)
        self._check(self.lib.oww_load_bank_head(self.h, int(bank), int(slot), _ptr(blob), blob.size))

    def assign_bank_head(self, bank, stream_ids, slots, stream=None):
        """Stream-ordered like assign_verifier: stream_ids None = all streams; slot -1 = none (zeros)."""
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, np.int32)
        sl = np.ascontiguousarray(slots, np.int32)
        n = sl.size if ids is None else ids.size
        if sl.size != n:
            raise ValueError(f"{sl.size} slots for {n} streams")
        self._check(self.lib.oww_assign_bank_head(self.h, int(bank), _ptr(ids), n, _ptr(sl), stream))

    def set_head_bank_clip_slot(self, bank, slot):
        self._check(self.lib.oww_set_head_bank_clip_slot(self.h, int(bank), int(slot)))

    def bank_head_predict(self, bank, slot, d_feats, n, d_out, stream=None):
        self._check(self.lib.oww_bank_head_predict(self.h, int(bank), int(slot), _ptr(d_feats), int(n), _ptr(d_out), stream))

    def add_gate(self, main_head, verifier_head, threshold=0.5):
        self._check(self.lib.oww_add_gate(self.h, int(main_head), int(verifier_head), float(threshold)))

    # ---- custom verifier banks (include/owwb200.h) ----
    def add_verifier_bank(self, head_id, capacity, threshold):
        bid = C.c_int(-1)
        self._check(self.lib.oww_add_verifier_bank(self.h, int(head_id), int(capacity), float(threshold), C.byref(bid)))
        self._bank_d.append(self._head_n_in[int(head_id)] * 96)
        return bid.value

    def add_bank_verifier_bank(self, head_bank, capacity, threshold):
        """A verifier bank whose parent is head bank `head_bank` (its other calls are those of add_verifier_bank's)."""
        bid = C.c_int(-1)
        self._check(self.lib.oww_add_bank_verifier_bank(self.h, int(head_bank), int(capacity), float(threshold),
                                                        C.byref(bid)))
        self._bank_d.append(self._head_bank_n_in[int(head_bank)] * 96)
        return bid.value

    def load_verifier(self, bank, slot, mean, weight, bias):
        """mean, weight: the bank's D = n_in*96 floats each (synchronises the device)."""
        mean = np.ascontiguousarray(mean, np.float32).ravel()
        weight = np.ascontiguousarray(weight, np.float32).ravel()
        if not 0 <= int(bank) < len(self._bank_d):
            raise NativeError(f"bad verifier bank {bank}")
        D = self._bank_d[int(bank)]
        if mean.size != D or weight.size != D:
            raise ValueError(f"verifier bank {bank} takes {D} means and weights, got {mean.size} and {weight.size}")
        self._check(self.lib.oww_load_verifier(self.h, int(bank), int(slot), _ptr(mean), _ptr(weight), float(bias)))

    def assign_verifier(self, bank, stream_ids, slots, stream=None):
        """Stream-ordered on `stream` and on the handle's own stream of step_host / submit: stream_ids None = all streams
        (slots then has one entry per stream); slot -1 = none."""
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, np.int32)
        sl = np.ascontiguousarray(slots, np.int32)
        n = sl.size if ids is None else ids.size
        if sl.size != n:
            raise ValueError(f"{sl.size} slots for {n} streams")
        self._check(self.lib.oww_assign_verifier(self.h, int(bank), _ptr(ids), n, _ptr(sl), stream))

    def set_verifier_clip_slot(self, bank, slot):
        self._check(self.lib.oww_set_verifier_clip_slot(self.h, int(bank), int(slot)))

    def set_verifier_threshold(self, bank, threshold):
        self._check(self.lib.oww_set_verifier_threshold(self.h, int(bank), float(threshold)))

    def enable_verifiers(self, enabled):
        self._check(self.lib.oww_enable_verifiers(self.h, int(bool(enabled))))

    def verifier_predict(self, bank, slot, d_feats, n, d_out, stream=None):
        self._check(self.lib.oww_verifier_predict(self.h, int(bank), int(slot), _ptr(d_feats), int(n), _ptr(d_out), stream))

    def verifier_predict_host(self, bank, slot, feats):
        """float32 [n, n_in, 96] host windows -> float32 [n] (synchronises)."""
        import torch
        x = torch.from_numpy(np.ascontiguousarray(feats, np.float32)).to(f"cuda:{self.device}")
        out = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
        self.verifier_predict(bank, slot, x, x.shape[0], out, torch.cuda.current_stream(x.device).cuda_stream)
        return out.cpu().numpy()

    def _cuda(self, name, t, dtype, shape=None):
        """Refuse a tensor the library would misread: not a contiguous `dtype` tensor on this handle's device, or (with
        `shape`, -1 = any extent) of another shape."""
        import torch
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or t.device != torch.device("cuda", self.device):
            raise ArgumentError(f"{name} must be a {dtype} tensor on cuda:{self.device}")
        if not t.is_contiguous():
            raise ArgumentError(f"{name} must be contiguous")
        if shape is not None and (t.dim() != len(shape) or any(s >= 0 and s != e for s, e in zip(shape, t.shape))):
            raise ArgumentError(f"{name} has shape {tuple(t.shape)}, expected {tuple(shape)} (-1: any)")
        return t

    def fit_verifiers(self, rows, n_in, first_row, sample_offsets, labels, C=0.001, max_iter=100, tol=1e-10, stream=None):
        """Train one verifier per user on the device (include/owwb200.h, oww_fit_verifiers).  rows: float32 [R, 96];
        first_row: int64 [N] (sample i = rows[first_row[i] : first_row[i] + n_in]); labels: uint8 [N]; sample_offsets:
        host int64 [U + 1], user u owns samples offsets[u] .. offsets[u+1].  -> dict of new tensors mean, var, coef
        (float64 [U, n_in*96]), intercept (float64 [U]), iters, status (int32 [U]); enqueued on `stream` (None: the
        device's current stream)."""
        import torch
        self._cuda("rows", rows, torch.float32, (-1, 96))
        if rows.data_ptr() % 16:
            raise ArgumentError("rows must start on a 16-byte boundary")
        off = np.ascontiguousarray(sample_offsets, np.int64).ravel()
        if off.size < 1 or off[0] != 0 or (np.diff(off) < 0).any():
            raise ArgumentError("sample_offsets must start at 0 and not decrease")
        N, U = int(off[-1]), off.size - 1
        self._cuda("first_row", first_row, torch.int64, (N,))
        self._cuda("labels", labels, torch.uint8, (N,))
        if not 1 <= int(n_in) <= 120:
            raise ArgumentError(f"n_in={n_in} outside [1, 120]")
        dev = torch.device("cuda", self.device)
        D = int(n_in) * 96
        f64 = dict(dtype=torch.float64, device=dev)
        out = {"mean": torch.empty((U, D), **f64), "var": torch.empty((U, D), **f64), "coef": torch.empty((U, D), **f64),
               "intercept": torch.empty(U, **f64), "iters": torch.empty(U, dtype=torch.int32, device=dev),
               "status": torch.empty(U, dtype=torch.int32, device=dev)}
        s = torch.cuda.current_stream(dev).cuda_stream if stream is None else stream
        self._check(self.lib.oww_fit_verifiers(self.h, _ptr(rows), rows.shape[0], int(n_in), _ptr(first_row), _ptr(off),
                                               _ptr(labels), U, float(C), int(max_iter), float(tol), _ptr(out["mean"]),
                                               _ptr(out["var"]), _ptr(out["coef"]), _ptr(out["intercept"]),
                                               _ptr(out["iters"]), _ptr(out["status"]), s))
        return out

    def load_verifiers(self, bank, slots, mean, weight, bias, stream=None):
        """Slots `slots` (distinct) of verifier bank `bank` <- float32 device tensors mean, weight [n, D] and bias [n];
        stream-ordered (include/owwb200.h, oww_load_verifiers; stream None: the device's current stream)."""
        import torch
        if not 0 <= int(bank) < len(self._bank_d):
            raise ArgumentError(f"bad verifier bank {bank}")
        sl = np.ascontiguousarray(slots, np.int32).ravel()
        D = self._bank_d[int(bank)]
        self._cuda("mean", mean, torch.float32, (sl.size, D))
        self._cuda("weight", weight, torch.float32, (sl.size, D))
        self._cuda("bias", bias, torch.float32, (sl.size,))
        s = torch.cuda.current_stream(torch.device("cuda", self.device)).cuda_stream if stream is None else stream
        self._check(self.lib.oww_load_verifiers(self.h, int(bank), _ptr(sl), sl.size, _ptr(mean), _ptr(weight),
                                                _ptr(bias), s))

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
        """pcm: C-contiguous int16 [B, >= n_chunks*1280]; scores_out: float32 [B, n_outputs]."""
        self._host_pcm(pcm, n_chunks)
        self._host_scores(scores_out)
        self._check(self.lib.oww_step_host(self.h, _ptr(pcm), pcm.shape[1], n_chunks, _ptr(scores_out)))

    def step_host_submit(self, pcm, n_chunks):
        self._host_pcm(pcm, n_chunks)
        t = C.c_int(-1)
        self._check(self.lib.oww_step_host_submit(self.h, _ptr(pcm), pcm.shape[1], n_chunks, C.byref(t)))
        return t.value

    def step_host_collect(self, ticket, scores_out):
        self._host_scores(scores_out)
        self._check(self.lib.oww_step_host_collect(self.h, ticket, _ptr(scores_out)))

    def _host_pcm(self, pcm, n_chunks):
        """The library reads n_chunks*1280 samples of each of the n_streams rows of a host buffer: refuse a shorter one."""
        if not isinstance(pcm, np.ndarray) or pcm.dtype != np.int16 or pcm.ndim != 2 or not pcm.flags.c_contiguous:
            raise ArgumentError("pcm must be a C-contiguous int16 numpy array [n_streams, samples]")
        if pcm.shape[0] != self.n_streams or pcm.shape[1] < int(n_chunks) * 1280:
            raise ArgumentError(f"pcm has shape {pcm.shape}; this call reads [{self.n_streams}, {int(n_chunks) * 1280}]")

    def _host_scores(self, scores_out):
        """The collect writes n_streams rows of n_outputs floats (nothing when there are no outputs)."""
        if not isinstance(scores_out, np.ndarray) or scores_out.dtype != np.float32 or not scores_out.flags.c_contiguous:
            raise ArgumentError("scores_out must be a C-contiguous float32 numpy array")
        B, n_out = self.n_streams, self.n_outputs
        if scores_out.ndim != 2 or scores_out.shape[0] != B or (n_out and scores_out.shape[1] != n_out):
            raise ArgumentError(f"scores_out has shape {scores_out.shape}, the handle writes [{B}, {n_out}]")

    def _chunks(self, chunks):
        c = np.ascontiguousarray(chunks, np.int32)
        if c.shape != (self.n_streams,):
            raise ValueError(f"chunks has shape {c.shape}, the handle has {self.n_streams} streams")
        return c

    def step_ragged(self, d_pcm, pcm_stride, chunks, d_scores, stream=None):
        """Stream b steps chunks[b] (host int32 [B], 0..max_chunks) chunks: the first chunks[b]*1280 samples of row b.
        Rows of d_scores of streams with 0 chunks are not written (include/owwb200.h, oww_step_ragged)."""
        c = self._chunks(chunks)
        self._check(self.lib.oww_step_ragged(self.h, _ptr(d_pcm), int(pcm_stride), _ptr(c), _ptr(d_scores), stream))

    def step_host_ragged(self, pcm, chunks, scores_out):
        """pcm: C-contiguous int16 [B, >= max(chunks)*1280]; rows of scores_out of held streams are left as they were."""
        c = self._chunks(chunks)
        self._host_pcm(pcm, c.max(initial=0))
        self._host_scores(scores_out)
        self._check(self.lib.oww_step_host_ragged(self.h, _ptr(pcm), pcm.shape[1], _ptr(c), _ptr(scores_out)))

    def step_host_ragged_submit(self, pcm, chunks):
        c = self._chunks(chunks)
        self._host_pcm(pcm, c.max(initial=0))
        t = C.c_int(-1)
        self._check(self.lib.oww_step_host_ragged_submit(self.h, _ptr(pcm), pcm.shape[1], _ptr(c), C.byref(t)))
        return t.value

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

    # ---- stream records: moving live streams (include/owwb200.h, oww_export_streams) ----
    def stream_state_info(self):
        """-> (record bytes, configuration key) of this handle's stream records."""
        n, key = C.c_size_t(0), C.c_uint64(0)
        self._check(self.lib.oww_stream_state_info(self.h, C.byref(n), C.byref(key)))
        return n.value, key.value

    def export_streams(self, stream_ids, d_records, stream=None):
        """Stream stream_ids[i] -> record i of d_records (device, [n][record bytes]); stream-ordered."""
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        self._check(self.lib.oww_export_streams(self.h, _ptr(ids), ids.size, _ptr(d_records), stream))

    def import_streams(self, stream_ids, d_records, stream=None):
        """Record i of d_records -> stream stream_ids[i] (distinct ids); stream-ordered.  Records of another
        configuration are skipped on the device and counted (stream_state_rejected)."""
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        self._check(self.lib.oww_import_streams(self.h, _ptr(ids), ids.size, _ptr(d_records), stream))

    def stream_state_rejected(self):
        """Records the imports since the last call skipped (synchronises the device; clears the count)."""
        v = C.c_int(0)
        self._check(self.lib.oww_stream_state_status(self.h, C.byref(v)))
        return v.value

    def export_records(self, stream_ids, stream=None):
        """export_streams into a new torch.uint8 [n, record bytes] on the handle's device; stream None: the current CUDA
        stream of that device."""
        import torch
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        n_bytes, _ = self.stream_state_info()
        dev = torch.device("cuda", self.device)
        out = torch.empty((ids.size, n_bytes), dtype=torch.uint8, device=dev)
        self.export_streams(ids, out, torch.cuda.current_stream(dev).cuda_stream if stream is None else stream)
        return out

    def import_records(self, stream_ids, records, stream=None):
        """import_streams from a torch.uint8 [n, record bytes] on any device or the CPU (moved with .to()).  Records of
        another configuration raise ValueError before anything is enqueued."""
        import torch
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        n_bytes, key = self.stream_state_info()
        if records.dtype != torch.uint8 or records.dim() != 2 or records.shape[0] != ids.size:
            raise ValueError(f"records must be uint8 [{ids.size}, {n_bytes}], got {records.dtype} {tuple(records.shape)}")
        if records.shape[1] != n_bytes:
            raise ValueError(f"records of {records.shape[1]} bytes; this configuration's have {n_bytes}")
        if ids.size:
            keys = np.ascontiguousarray(records[:, 8:16].cpu().numpy()).view(np.uint64).ravel()
            if (keys != np.uint64(key)).any():
                raise ValueError("records of another configuration (cnn_mode, split_from or weights)")
        dev = torch.device("cuda", self.device)
        d = records.to(dev).contiguous()                   # on the current CUDA stream of the device
        if stream is None:
            self.import_streams(ids, d, torch.cuda.current_stream(dev).cuda_stream)
        else:                                              # after that copy, whose memory must outlive the import
            ext = torch.cuda.ExternalStream(stream, device=dev)
            ext.wait_stream(torch.cuda.current_stream(dev))
            self.import_streams(ids, d, stream)
            d.record_stream(ext)

    # ---- detections on the device (include/owwb200.h, oww_set_detector) ----
    @staticmethod
    def _label_table(labels):
        arr = (DetectLabel * max(len(labels), 1))()
        for i, (col, rep, thr, pat) in enumerate(labels):
            arr[i] = DetectLabel(int(col), int(bool(rep)), float("nan") if thr is None else float(thr), int(pat))
        return arr

    def set_detector(self, labels, debounce_time=0.0):
        """labels: [(column, repeats, threshold or None / NaN, patience)], one per label; [] removes the detector.
        Synchronises the device.  The same columns and repeats as before keep the histories."""
        self._check(self.lib.oww_set_detector(self.h, self._label_table(labels), len(labels), float(debounce_time)))
        self.n_detect_labels = len(labels)
        self._det_buf = None

    def detect(self, d_scores, prepared, d_final, d_events, max_events, d_n_events, stream=None):
        """oww_detect: prepared is one int for every stream or host int32 [n_streams] (< 0: the stream is skipped)."""
        if np.ndim(prepared) == 0:
            all_, per = int(prepared), None
        else:
            all_, per = 0, np.ascontiguousarray(prepared, np.int32)
            if per.shape != (self.n_streams,):
                raise ValueError(f"prepared has shape {per.shape}, the handle has {self.n_streams} streams")
        self._check(self.lib.oww_detect(self.h, _ptr(d_scores), all_, _ptr(per), _ptr(d_final), _ptr(d_events),
                                        int(max_events), _ptr(d_n_events), stream))

    def detect_clips(self, labels, debounce_time, d_scores, d_verified, verifier_threshold, row_offsets, chunk_size,
                     d_final, d_events, max_events, d_n_events, stream=None):
        """oww_detect_clips: labels as set_detector; row_offsets host int64 [n_clips + 1]; d_verified [rows][n_labels]
        or None."""
        off = np.ascontiguousarray(row_offsets, np.int64).ravel()
        self._check(self.lib.oww_detect_clips(self.h, self._label_table(labels), len(labels), float(debounce_time),
                                              _ptr(d_scores), _ptr(d_verified), float(verifier_threshold), _ptr(off),
                                              off.size - 1, int(chunk_size), _ptr(d_final), _ptr(d_events),
                                              int(max_events), _ptr(d_n_events), stream))

    def detector_export(self, stream_ids, d_hist, d_counts, stream=None):
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        self._check(self.lib.oww_detector_export(self.h, _ptr(ids), ids.size, _ptr(d_hist), _ptr(d_counts), stream))

    def detector_import(self, stream_ids, d_hist, d_counts, stream=None):
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        self._check(self.lib.oww_detector_import(self.h, _ptr(ids), ids.size, _ptr(d_hist), _ptr(d_counts), stream))

    def set_stream_detection(self, stream_ids, records, debounce=None, stream=None):
        """oww_set_stream_detection: streams stream_ids (distinct; None = all) take records (STREAM_DETECT_DTYPE [n,
        n_labels]; None: back to the handle's settings) and debounce (float64 [n], NaN: the handle's; None: all NaN), on
        the current CUDA stream (or `stream`)."""
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, np.int32).ravel()
        n = self.n_streams if ids is None else ids.size
        rec = deb = None
        if records is not None:
            rec = np.ascontiguousarray(records, STREAM_DETECT_DTYPE)
            if rec.shape != (n, self.n_detect_labels):
                raise ValueError(f"records have shape {rec.shape}, expected {(n, self.n_detect_labels)}")
            if debounce is not None:
                deb = np.ascontiguousarray(np.broadcast_to(np.asarray(debounce, np.float64), (n,)))
        if stream is None:
            stream = self._current_stream()
        self._check(self.lib.oww_set_stream_detection(self.h, _ptr(ids), n, _ptr(rec), _ptr(deb), stream))

    def stream_detection(self, stream_ids=None):
        """-> (STREAM_DETECT_DTYPE [n, n_labels], float64 [n] debounce) of streams stream_ids (None = all); host only"""
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, np.int32).ravel()
        n = self.n_streams if ids is None else ids.size
        rec = np.zeros((n, self.n_detect_labels), STREAM_DETECT_DTYPE)
        deb = np.zeros(n, np.float64)
        self._check(self.lib.oww_get_stream_detection(self.h, _ptr(ids), n, _ptr(rec), _ptr(deb)))
        return rec, deb

    def _current_stream(self):
        import torch
        return torch.cuda.current_stream(torch.device("cuda", self.device)).cuda_stream

    def new_scores(self):
        """a device score matrix [n_streams, n_outputs] for step_ragged_pcm / detect_events"""
        import torch
        return torch.zeros((self.n_streams, self.n_outputs), dtype=torch.float32, device=torch.device("cuda", self.device))

    def step_pcm(self, pcm, n_chunks, d_scores):
        """step on a host int16 [n_streams, >= n_chunks*1280] array, uploaded and stepped on the current CUDA stream; the
        scores stay on the device."""
        import torch
        self._host_pcm(pcm, n_chunks)
        d = torch.from_numpy(pcm).to(d_scores.device)
        self.step(d, pcm.shape[1], int(n_chunks), d_scores, self._current_stream())

    def step_ragged_pcm(self, pcm, chunks, d_scores):
        """step_ragged on a host int16 [n_streams, >= max(chunks)*1280] array: uploaded and stepped on the current CUDA
        stream; the scores stay on the device."""
        import torch
        c = self._chunks(chunks)
        self._host_pcm(pcm, c.max(initial=0))
        d = torch.from_numpy(pcm).to(d_scores.device)
        self.step_ragged(d, pcm.shape[1], c, d_scores, self._current_stream())

    def detect_events(self, d_scores, prepared, d_final=None, max_events=None):
        """oww_detect on the current CUDA stream, then the event count and that many events to the host (synchronises):
        -> (EVENT_DTYPE array of min(n, max_events) events in ascending (stream, label) order, n).  max_events None:
        n_streams * n_labels, which never truncates."""
        import torch
        cap = self.n_streams * self.n_detect_labels if max_events is None else int(max_events)
        if self._det_buf is None or self._det_buf[0].shape[0] < cap:
            dev = torch.device("cuda", self.device)
            self._det_buf = (torch.empty((cap, 4), dtype=torch.int32, device=dev),
                             torch.zeros(1, dtype=torch.int32, device=dev))
        ev, n_ev = self._det_buf
        self.detect(d_scores, prepared, d_final, ev if cap else None, cap, n_ev, self._current_stream())
        n = int(n_ev.item())
        return ev[:min(n, cap)].cpu().numpy().view(EVENT_DTYPE).reshape(-1), n

    def detector_history(self, stream_ids):
        """-> (float32 [n, n_labels, 30] oldest first, int32 [n] counts) of the listed streams (synchronises)"""
        import torch
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        dev = torch.device("cuda", self.device)
        hist = torch.empty((ids.size, self.n_detect_labels, 30), dtype=torch.float32, device=dev)
        cnt = torch.empty(ids.size, dtype=torch.int32, device=dev)
        self.detector_export(ids, hist, cnt, self._current_stream())
        return hist.cpu().numpy(), cnt.cpu().numpy()

    def set_detector_history(self, stream_ids, hist, counts):
        """the reverse of detector_history (distinct ids), on the current CUDA stream"""
        import torch
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        dev = torch.device("cuda", self.device)
        h = torch.from_numpy(np.ascontiguousarray(hist, np.float32).reshape(ids.size, self.n_detect_labels, 30)).to(dev)
        c = torch.from_numpy(np.ascontiguousarray(counts, np.int32).reshape(ids.size)).to(dev)
        self.detector_import(ids, h, c, self._current_stream())

    # ---- stream audio on the device (include/owwb200.h, oww_set_audio_history) ----
    def set_audio_history(self, n_samples):
        """n_samples: 0 (off) or a multiple of 1280 up to 960000.  Synchronises the device; every history starts empty."""
        self.audio_history = 0
        self._check(self.lib.oww_set_audio_history(self.h, int(n_samples)))
        self.audio_history = int(n_samples)

    def get_audio(self, stream_ids, ends, n_samples, d_out, d_pos, stream=None):
        """oww_get_audio: ends None or host int64 [n] (< 0: the stream's pos)."""
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        e = None if ends is None else np.ascontiguousarray(ends, np.int64).ravel()
        if e is not None and e.size != ids.size:
            raise ValueError(f"{e.size} ends for {ids.size} streams")
        self._check(self.lib.oww_get_audio(self.h, _ptr(ids), _ptr(e), ids.size, int(n_samples), _ptr(d_out), _ptr(d_pos),
                                           stream))

    def capture_events(self, d_events, d_n_events, max_events, n_samples, d_out, d_pos, stream=None):
        self._check(self.lib.oww_capture_events(self.h, _ptr(d_events), _ptr(d_n_events), int(max_events), int(n_samples),
                                                _ptr(d_out), _ptr(d_pos), stream))

    def audio_export(self, stream_ids, d_audio, d_pos, stream=None):
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        self._check(self.lib.oww_audio_export(self.h, _ptr(ids), ids.size, _ptr(d_audio), _ptr(d_pos), stream))

    def audio_import(self, stream_ids, d_audio, d_pos, stream=None):
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        self._check(self.lib.oww_audio_import(self.h, _ptr(ids), ids.size, _ptr(d_audio), _ptr(d_pos), stream))

    def read_audio(self, stream_ids, n_samples, ends=None):
        """oww_get_audio on the current CUDA stream into new tensors -> (int16 [n, n_samples] on the device, int64 [n]
        pos on the device)"""
        import torch
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        dev = torch.device("cuda", self.device)
        out = torch.empty((ids.size, int(n_samples)), dtype=torch.int16, device=dev)
        pos = torch.empty(ids.size, dtype=torch.int64, device=dev)
        self.get_audio(ids, ends, n_samples, out, pos, self._current_stream())
        return out, pos

    def detect_capture(self, d_scores, prepared, n_samples, max_events=None):
        """detect_events with oww_capture_events enqueued right after oww_detect -> (events, n, clips int16 [min(n,
        max_events), n_samples] on the device, ends int64 [same] on the host).  max_events None: the clips are gathered
        once the count is known (n_streams * n_labels rows of clips could be gigabytes), with nothing enqueued between."""
        import torch
        dev = torch.device("cuda", self.device)
        if max_events is None:
            events, n = self.detect_events(d_scores, prepared)
            clips = torch.empty((n, int(n_samples)), dtype=torch.int16, device=dev)
            ends = torch.empty(n, dtype=torch.int64, device=dev)
            if n:
                self.capture_events(self._det_buf[0], self._det_buf[1], n, n_samples, clips, ends, self._current_stream())
            return events, n, clips, ends.cpu().numpy()
        cap = int(max_events)
        if self._det_buf is None or self._det_buf[0].shape[0] < cap:
            self._det_buf = (torch.empty((cap, 4), dtype=torch.int32, device=dev),
                             torch.zeros(1, dtype=torch.int32, device=dev))
        ev, n_ev = self._det_buf
        clips = torch.empty((cap, int(n_samples)), dtype=torch.int16, device=dev)
        ends = torch.empty(cap, dtype=torch.int64, device=dev)
        s = self._current_stream()
        self.detect(d_scores, prepared, None, ev if cap else None, cap, n_ev, s)
        self.capture_events(ev, n_ev, cap, n_samples, clips, ends, s)
        n = int(n_ev.item())
        k = min(n, cap)
        return ev[:k].cpu().numpy().view(EVENT_DTYPE).reshape(-1), n, clips[:k], ends[:k].cpu().numpy()

    def audio_state(self, stream_ids):
        """-> (int16 [n, H] oldest first, int64 [n] pos) host arrays of the listed streams (synchronises)"""
        import torch
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        dev = torch.device("cuda", self.device)
        audio = torch.empty((ids.size, self.audio_history), dtype=torch.int16, device=dev)
        pos = torch.empty(ids.size, dtype=torch.int64, device=dev)
        self.audio_export(ids, audio, pos, self._current_stream())
        return audio.cpu().numpy(), pos.cpu().numpy()

    def set_audio_state(self, stream_ids, audio, pos):
        """the reverse of audio_state (distinct ids, records of this handle's H), on the current CUDA stream"""
        import torch
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        a = np.ascontiguousarray(audio, np.int16)
        if a.shape != (ids.size, self.audio_history):
            raise ValueError(f"audio has shape {a.shape}; this handle keeps [{ids.size}, {self.audio_history}]")
        dev = torch.device("cuda", self.device)
        d = torch.from_numpy(a).to(dev)
        p = torch.from_numpy(np.ascontiguousarray(pos, np.int64).reshape(ids.size)).to(dev)
        self.audio_import(ids, d, p, self._current_stream())

    # ---- ingest: packets at any rate (include/owwb200.h, oww_set_input_rates) ----
    def set_input_rates(self, stream_ids, rates, stream=None):
        """stream_ids None = all streams (rates then has one entry per stream); their resamplers restart."""
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, np.int32).ravel()
        r = np.ascontiguousarray(rates, np.int32).ravel()
        n = r.size if ids is None else ids.size
        if r.size != n:
            raise ValueError(f"{r.size} rates for {n} streams")
        for v in np.unique(r):
            resampler_taps(int(v))                        # ValueError outside the table
        self._check(self.lib.oww_set_input_rates(self.h, _ptr(ids), n, _ptr(r), stream))

    def ingest(self, d_in, offsets, d_scores, stream=None):
        """oww_ingest: stream b's samples are d_in[offsets[b]:offsets[b+1]] (host int64 offsets) -> (chunks, prepared)
        int32 [n_streams] host arrays."""
        off = np.ascontiguousarray(offsets, np.int64).ravel()
        if off.size != self.n_streams + 1:
            raise ValueError(f"offsets has {off.size} entries, the handle takes {self.n_streams + 1}")
        chunks = np.zeros(self.n_streams, np.int32)
        prepared = np.zeros(self.n_streams, np.int32)
        self._check(self.lib.oww_ingest(self.h, _ptr(d_in), _ptr(off), _ptr(chunks), _ptr(prepared), _ptr(d_scores),
                                        stream))
        return chunks, prepared

    def ingest_pcm(self, pcm, offsets, d_scores):
        """ingest on a host int16 array of packed packets, uploaded and ingested on the current CUDA stream"""
        import torch
        x = np.ascontiguousarray(pcm, np.int16).ravel()
        d = torch.from_numpy(x if x.size else np.zeros(1, np.int16)).to(torch.device("cuda", self.device))
        return self.ingest(d, offsets, d_scores, self._current_stream())

    def ingest_capacity(self):
        """-> int64 [n_streams]: the most input samples each stream's next ingest call may take"""
        out = np.zeros(self.n_streams, np.int64)
        self._check(self.lib.oww_ingest_capacity(self.h, _ptr(out)))
        return out

    def ingest_state(self, stream_ids, samples=True):
        """-> (rates int32 [n], input counts int64 [n], staged counts int32 [n], staged int16 [n, max staged] or None,
        history int16 [n, 128] or None) of the listed streams; host arrays (synchronises when samples)"""
        import torch
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        rates, S, staged = np.zeros(ids.size, np.int32), np.zeros(ids.size, np.int64), np.zeros(ids.size, np.int32)
        self._check(self.lib.oww_ingest_export(self.h, _ptr(ids), ids.size, _ptr(rates), _ptr(S), _ptr(staged), None, 0,
                                               None, None))
        if not samples:
            return rates, S, staged, None, None
        dev = torch.device("cuda", self.device)
        width = max(int(staged.max(initial=0)), 1)
        d = torch.empty((ids.size, width), dtype=torch.int16, device=dev)
        hist = torch.empty((ids.size, 128), dtype=torch.int16, device=dev)
        if ids.size:
            self._check(self.lib.oww_ingest_export(self.h, _ptr(ids), ids.size, None, None, None, _ptr(d), width,
                                                   _ptr(hist), self._current_stream()))
        return rates, S, staged, d.cpu().numpy(), hist.cpu().numpy()

    def set_ingest_state(self, stream_ids, rates, consumed, staged, samples, hist):
        """the reverse of ingest_state (distinct ids), on the current CUDA stream"""
        import torch
        ids = np.ascontiguousarray(stream_ids, np.int32).ravel()
        r = np.ascontiguousarray(rates, np.int32).ravel()
        S = np.ascontiguousarray(consumed, np.int64).ravel()
        st = np.ascontiguousarray(staged, np.int32).ravel()
        x = np.ascontiguousarray(samples, np.int16).reshape(ids.size, -1)
        dev = torch.device("cuda", self.device)
        d = torch.from_numpy(x).to(dev)
        h = torch.from_numpy(np.ascontiguousarray(hist, np.int16).reshape(ids.size, 128)).to(dev)
        self._check(self.lib.oww_ingest_import(self.h, _ptr(ids), ids.size, _ptr(r), _ptr(S), _ptr(st), _ptr(d),
                                               x.shape[1], _ptr(h), self._current_stream()))

    # ---- pipelined detection from host audio (include/owwb200.h, oww_detect_host_submit) ----
    def detect_host_submit(self, packets, offsets, max_events, capture=None, final=False):
        """oww_detect_host_submit: ingest + detect (+ capture of `capture` samples per event) of host int16 packets
        (stream b's: packets[offsets[b]:offsets[b+1]]) -> ticket.  The output arrays of the ticket are allocated here; the
        packets array is kept until the collect (a page-locked one is read by the copy engine until then)."""
        if not isinstance(packets, np.ndarray) or packets.dtype != np.int16 or packets.ndim != 1 \
                or not packets.flags.c_contiguous:
            raise ArgumentError("packets must be a contiguous 1-D int16 numpy array")
        off = np.ascontiguousarray(offsets, np.int64).ravel()
        B, L = self.n_streams, self.n_detect_labels
        if off.size != B + 1 or off[0] < 0 or off[-1] > packets.size:
            raise ArgumentError(f"offsets must hold {B + 1} sample offsets into packets ({packets.size} samples)")
        m, cs = int(max_events), 0 if capture is None else int(capture)
        rows = max(m, 0) if cs > 0 else 0
        out = (np.empty(max(m, 0), EVENT_DTYPE), np.zeros(1, np.int32), np.empty((rows, max(cs, 0)), np.int16),
               np.empty(rows, np.int64), np.zeros(B, np.int32), np.zeros(B, np.int32),
               np.empty((B, L), np.float32) if final else None)
        t = C.c_int(-1)
        self._check(self.lib.oww_detect_host_submit(self.h, _ptr(packets), _ptr(off), m, cs, int(bool(final)), C.byref(t)))
        self._det_tickets[t.value] = (packets, cs, out)
        return t.value

    def detect_host_collect(self, ticket):
        """oww_detect_host_collect -> (events EVENT_DTYPE [k], n, chunks int32 [B], prepared int32 [B], clips int16 [k,
        capture] or None, ends int64 [k] or None, final float32 [B, n_labels] or None), k = min(n, max_events)."""
        entry = self._det_tickets.get(ticket)
        if entry is None:                                  # the library's refusal (not in flight)
            self._check(self.lib.oww_detect_host_collect(self.h, int(ticket), None, None, None, None, None, None, None))
            raise NativeError(f"detect ticket {ticket} is not in flight")
        _, cs, (ev, n, clips, ends, chunks, prepared, fin) = entry
        self._check(self.lib.oww_detect_host_collect(self.h, int(ticket), _ptr(ev), _ptr(n), _ptr(clips), _ptr(ends),
                                                     _ptr(chunks), _ptr(prepared), _ptr(fin)))
        del self._det_tickets[ticket]
        k = min(int(n[0]), ev.size)
        return (ev[:k], int(n[0]), chunks, prepared, clips[:k] if cs > 0 else None, ends[:k] if cs > 0 else None, fin)

    # ---- batch ----
    def embed_clips(self, d_pcm, n_clips, n_samples, d_emb, stream=None):
        self._check(self.lib.oww_embed_clips(self.h, _ptr(d_pcm), n_clips, n_samples, _ptr(d_emb), stream))

    def predict_clips(self, d_pcm, n_clips, n_samples, pad_samples, feature_init, d_scores, stream=None):
        fi = None if feature_init is None else np.ascontiguousarray(feature_init, np.float32)
        self._check(self.lib.oww_predict_clips(self.h, _ptr(d_pcm), n_clips, n_samples, pad_samples, _ptr(fi),
                                               41 if fi is None else fi.shape[0], _ptr(d_scores), stream))

    def predict_clips_ragged(self, d_pcm, offsets, pad_samples, chunk_size, feature_init, d_scores, d_stepped, d_emb=None,
                             stream=None, clip_streams=None):
        """offsets: host int64 [n_clips + 1] sample offsets into d_pcm; d_scores [rows][n_outputs], d_stepped uint8 [rows],
        d_emb [steps][96] or None (include/owwb200.h, oww_predict_clips_ragged).  clip_streams: host int32 [n_clips],
        clip i scored with the models and verifiers of stream clip_streams[i] (oww_predict_clips_streams)."""
        off = np.ascontiguousarray(offsets, np.int64)
        fi = None if feature_init is None else np.ascontiguousarray(feature_init, np.float32)
        args = (self.h, _ptr(d_pcm), _ptr(off), off.size - 1, int(pad_samples), int(chunk_size), _ptr(fi),
                41 if fi is None else fi.shape[0], _ptr(d_scores), _ptr(d_stepped), _ptr(d_emb))
        if clip_streams is None:
            self._check(self.lib.oww_predict_clips_ragged(*args, stream))
            return
        cs = np.ascontiguousarray(clip_streams, np.int32)
        if cs.size != off.size - 1:
            raise ValueError(f"{cs.size} clip streams for {off.size - 1} clips")
        self._check(self.lib.oww_predict_clips_streams(*args, _ptr(cs), stream))

    def resample_clips(self, d_in, in_offsets, rates, pad_samples, d_out, out_offsets, stream=None):
        """oww_resample_clips: clip i is d_in[in_offsets[i]:in_offsets[i+1]] at rates[i] Hz -> d_out[out_offsets[i]:
        out_offsets[i+1]] at 16 kHz with pad_samples of padding each side (host int64 offsets, host int32 rates)."""
        off = np.ascontiguousarray(in_offsets, np.int64).ravel()
        out = np.ascontiguousarray(out_offsets, np.int64).ravel()
        r = np.ascontiguousarray(rates, np.int32).ravel()
        if r.size != off.size - 1 or out.size != off.size:
            raise ValueError(f"{off.size} input offsets, {out.size} output offsets and {r.size} rates")
        self._check(self.lib.oww_resample_clips(self.h, _ptr(d_in), _ptr(off), _ptr(r), r.size, int(pad_samples),
                                                _ptr(d_out), _ptr(out), stream))

    def mix_clips(self, d_fg, fg_offsets, d_bg, bg_offsets, d_rir, rir_offsets, params, n_samples, d_out, d_valid,
                  stream=None):
        """oww_mix_clips: mixture i of the MIX_DTYPE records `params` -> d_out[i] (int16 [n_mix][n_samples]) and d_valid[i]
        (uint8); clips packed on the device with host int64 offsets (int16 foregrounds and backgrounds, float32 RIRs)."""
        p = np.ascontiguousarray(params, MIX_DTYPE).ravel()
        offs = [np.ascontiguousarray(o if len(o) else [0], np.int64).ravel() for o in (fg_offsets, bg_offsets, rir_offsets)]
        n = [o.size - 1 for o in offs]
        self._check(self.lib.oww_mix_clips(self.h, _ptr(d_fg), _ptr(offs[0]), n[0], _ptr(d_bg), _ptr(offs[1]), n[1],
                                           _ptr(d_rir), _ptr(offs[2]), n[2], _ptr(p), p.size,
                                           int(n_samples), _ptr(d_out), _ptr(d_valid), stream))

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
    @staticmethod
    def _metrics_f64(d_scores):
        """True for float64 scores (the _f64 entry points), False for float32; any other dtype is refused."""
        name = str(d_scores.dtype)
        if name not in ("torch.float32", "torch.float64"):
            raise ValueError(f"metrics take float32 or float64 scores, got {name}")
        return name == "torch.float64"

    def metrics_false_positives(self, d_scores, series_stride, n_series, n_frames, thresholds, grouping_window=50, stream=None):
        """Thresholds are compared as the float64 values given (round them to the comparison dtype first: metrics.py)."""
        fn = self.lib.oww_metrics_false_positives_f64 if self._metrics_f64(d_scores) else self.lib.oww_metrics_false_positives
        thr = np.ascontiguousarray(thresholds, np.float64)
        out = np.zeros((n_series, thr.size), np.int32)
        self._check(fn(self.h, _ptr(d_scores), int(series_stride), int(n_series), int(n_frames), _ptr(thr), thr.size,
                       int(grouping_window), _ptr(out), stream))
        return out

    def metrics_count_ge(self, d_scores, n, thresholds, stream=None):
        fn = self.lib.oww_metrics_count_ge_f64 if self._metrics_f64(d_scores) else self.lib.oww_metrics_count_ge
        thr = np.ascontiguousarray(thresholds, np.float64)
        out = np.zeros(thr.size, np.uint64)
        for j0 in range(0, thr.size, 64):
            t = np.ascontiguousarray(thr[j0:j0 + 64])
            o = np.zeros(t.size, np.uint64)
            self._check(fn(self.h, _ptr(d_scores), int(n), _ptr(t), t.size, _ptr(o), stream))
            out[j0:j0 + 64] = o
        return out

    # ---- introspection ----
    def enable_stage_timing(self, n_slots=1):
        self._check(self.lib.oww_enable_stage_timing(self.h, int(n_slots)))

    def stage_ms(self):
        out = (C.c_float * 3)()
        self._check(self.lib.oww_stage_ms(self.h, out))
        return {"mel": out[0], "cnn": out[1], "heads": out[2]}
