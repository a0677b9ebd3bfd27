"""CUDA mirror of ``openwakeword.metrics`` (openwakeword/metrics.py:24-100): false positives per hour
and ROC points from score sequences - evaluated on the device, so the ``[clips, steps]`` score tensors that
``Model.predict_clips_array`` / bulk prediction leave in HBM never have to come back as Python lists.

Same function names, arguments and results as the reference (``get_false_positives`` including its grouping rule,
``generate_roc_curve_fprs``, ``generate_roc_curve_tprs``); scores may be a list, a NumPy array or a CUDA torch tensor.
``false_positives_batch`` is the batched form: one launch for ``[n_series, n_frames]`` x ``[n_thresholds]``.
There is no CPU fallback: the counts come from libowwb200 (csrc/metrics.cu)."""
import numpy as np

from . import _native

_ctx = {}


def _context(device_index=0):
    if device_index not in _ctx:
        _ctx[device_index] = _native.Context(device=device_index, max_chunks=1)
    return _ctx[device_index]


def _to_device(scores, device_index):
    import torch
    if isinstance(scores, torch.Tensor):
        t = scores.to(device=f"cuda:{device_index}", dtype=torch.float32)
    else:
        t = torch.from_numpy(np.ascontiguousarray(np.asarray(scores), np.float32)).to(f"cuda:{device_index}")
    return t.contiguous()


def false_positives_batch(scores, thresholds, grouping_window=50, device_index=0):
    """scores [n_series, n_frames] (or [n_frames]) -> int32 [n_series, n_thresholds]."""
    import torch
    t = _to_device(scores, device_index)
    if t.dim() == 1:
        t = t[None]
    n_series, n_frames = t.shape
    stream = torch.cuda.current_stream(t.device).cuda_stream
    return _context(device_index).metrics_false_positives(t, t.stride(0), n_series, n_frames, np.atleast_1d(thresholds),
                                                          grouping_window, stream)


def get_false_positives(scores, threshold, grouping_window=50, device_index=0):
    """metrics.py:24-45."""
    return int(false_positives_batch(scores, [threshold], grouping_window, device_index)[0, 0])


def generate_roc_curve_fprs(scores, n_points=25, time_per_prediction=.08, device_index=0, **kwargs):
    """metrics.py:48-78: false positives per hour at np.linspace(0.01, 0.99, n_points)."""
    n = len(scores)
    total_hours = time_per_prediction * n / 3600
    thr = np.linspace(0.01, 0.99, num=n_points)
    fp = false_positives_batch(scores, thr, kwargs.get("grouping_window", 50), device_index)[0]
    return [float(c) / total_hours for c in fp]


def generate_roc_curve_tprs(scores, n_points=25, device_index=0):
    """metrics.py:81-100: fraction of scores >= threshold at np.linspace(0.01, 0.99, n_points)."""
    import torch
    t = _to_device(scores, device_index).reshape(-1)
    thr = np.linspace(0.01, 0.99, num=n_points)
    cnt = _context(device_index).metrics_count_ge(t, t.numel(), thr, torch.cuda.current_stream(t.device).cuda_stream)
    return [float(c) / t.numel() for c in cnt]
