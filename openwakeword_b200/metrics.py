"""CUDA mirror of ``openwakeword.metrics`` (openwakeword/metrics.py:24-100): false positives per hour
and ROC points from score sequences - evaluated on the device, so the ``[clips, steps]`` score tensors that
``Model.predict_clips_array`` / bulk prediction leave in HBM never have to come back as Python lists.

Same function names, arguments and results as the reference (``get_false_positives`` including its grouping rule,
``generate_roc_curve_fprs``, ``generate_roc_curve_tprs``); scores may be a list, a NumPy array or a torch tensor.
``false_positives_batch`` is the batched form: one launch for ``[n_series, n_frames]`` x ``[n_thresholds]``.
Each score is compared with each threshold in the dtype the reference's ``np.array(scores) >= threshold`` compares
in (``comparison_dtype``), so the counts are the reference's exactly, at every precision.
There is no CPU fallback: the counts come from libowwb200 (csrc/metrics.cu)."""
import numpy as np

from . import _native

MAX_FP_THRESHOLDS = 4096            # thresholds per oww_metrics_false_positives call

_ctx = {}


def _context(device_index=0):
    if device_index not in _ctx:
        _ctx[device_index] = _native.Context(device=device_index, max_chunks=1)
    return _ctx[device_index]


def comparison_dtype(scores_dtype, threshold):
    """The dtype in which NumPy (>= 2, NEP 50 promotion) evaluates ``scores >= threshold`` for an array of
    ``scores_dtype``: a Python float or int threshold is weak and takes the scores' dtype (float32 scores against
    ``0.7`` compare with ``float32(0.7)``); a NumPy scalar promotes normally (float32 scores against
    ``np.float64(0.7)`` compare in float64)."""
    return np.result_type(scores_dtype, threshold)


def _rounded_thresholds(scores_dtype, thresholds):
    """Each threshold rounded to its comparison dtype, as float64: ``double(score) >= that`` is exactly NumPy's
    comparison, since widening float16/32/64 scores and a threshold already rounded to that dtype to double is exact.
    A list keeps each element's own type (Python floats stay weak); an array's elements are NumPy scalars."""
    items = [thresholds] if np.ndim(thresholds) == 0 else list(thresholds)
    out = np.empty(len(items), np.float64)
    with np.errstate(over="ignore"):                # a threshold beyond the dtype's range rounds to +-inf, as in NumPy
        for j, t in enumerate(items):
            d = comparison_dtype(scores_dtype, t)
            out[j] = np.asarray(t).astype(d) if d.kind == "f" else float(t)
    return out


def _to_device(scores, device_index):
    """-> (contiguous float32 or float64 CUDA tensor, the NumPy dtype the reference would see the scores as).
    float64 stays float64 and float32 stays float32; float16 and bfloat16 widen to float32 (exact); integer and bool
    scores become float64.  A bfloat16 tensor compares as float32 scores would (NumPy has no bfloat16)."""
    import torch
    if isinstance(scores, torch.Tensor):
        sdt = np.dtype(np.float32 if scores.dtype == torch.bfloat16 else str(scores.dtype).removeprefix("torch."))
    else:
        scores = np.asarray(scores)
        sdt = scores.dtype
    wide = not (sdt.kind == "f" and sdt.itemsize <= 4)
    if isinstance(scores, torch.Tensor):
        t = scores.to(device=f"cuda:{device_index}", dtype=torch.float64 if wide else torch.float32)
    else:
        t = torch.from_numpy(np.ascontiguousarray(scores, np.float64 if wide else np.float32)).to(f"cuda:{device_index}")
    return t.contiguous(), sdt


def false_positives_batch(scores, thresholds, grouping_window=50, device_index=0):
    """scores [n_series, n_frames] (or [n_frames]) -> int32 [n_series, n_thresholds]; column j is
    ``get_false_positives(series, thresholds[j], grouping_window)``."""
    import torch
    t, sdt = _to_device(scores, device_index)
    if t.dim() == 1:
        t = t[None]
    n_series, n_frames = t.shape
    thr = _rounded_thresholds(sdt, thresholds)
    out = np.zeros((n_series, thr.size), np.int32)
    if n_series == 0 or n_frames == 0:              # nothing to count (and no device buffer to point at)
        return out
    stream = torch.cuda.current_stream(t.device).cuda_stream
    ctx = _context(device_index)
    for j0 in range(0, thr.size, MAX_FP_THRESHOLDS):
        out[:, j0:j0 + MAX_FP_THRESHOLDS] = ctx.metrics_false_positives(t, t.stride(0), n_series, n_frames,
                                                                        thr[j0:j0 + MAX_FP_THRESHOLDS], grouping_window,
                                                                        stream)
    return out


def get_false_positives(scores, threshold, grouping_window=50, device_index=0):
    """metrics.py:24-45."""
    return int(false_positives_batch(scores, [threshold], grouping_window, device_index)[0, 0])


def generate_roc_curve_fprs(scores, n_points=25, time_per_prediction=.08, device_index=0, **kwargs):
    """metrics.py:48-78: false positives per hour at np.linspace(0.01, 0.99, n_points); ``kwargs`` go to the
    false-positive count as the reference passes them to ``get_false_positives`` (an unknown one raises TypeError)."""
    n = len(scores)
    total_hours = time_per_prediction * n / 3600
    thr = np.linspace(0.01, 0.99, num=n_points)
    fp = false_positives_batch(scores, thr, device_index=device_index, **kwargs)[0]
    return [float(c) / total_hours for c in fp]


def generate_roc_curve_tprs(scores, n_points=25, device_index=0):
    """metrics.py:81-100: fraction of scores >= threshold at np.linspace(0.01, 0.99, n_points)."""
    import torch
    t, sdt = _to_device(scores, device_index)
    t = t.reshape(-1)
    thr = _rounded_thresholds(sdt, np.linspace(0.01, 0.99, num=n_points))
    cnt = _context(device_index).metrics_count_ge(t, t.numel(), thr, torch.cuda.current_stream(t.device).cuda_stream)
    return [float(c) / t.numel() for c in cnt]
