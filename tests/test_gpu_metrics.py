"""-m gpu: the score metrics kernels (csrc/metrics.cu) and their wrappers (openwakeword_b200/metrics.py), exactly.

* tests/golden/metrics_edges.npz (the reference's own counts at the precision edges of ``np.array(scores) >=
  threshold`` and at the start-of-series edges of its grouping rule) through get_false_positives,
  false_positives_batch and the ROC helpers, with every series given as a NumPy array, a list and a CUDA tensor of the
  dtype the reference saw (float16, float32, float64).
* The false-positive kernel's layout against the oracle: 1..4097 thresholds (a warp per 32, idle lanes past
  n_thresholds, the 4096-per-call chunking), 1..1000 series (4 series per CTA at 32 thresholds, so 3 and 5 leave the
  last CTA part full), 0..100 000 frames, windows 0..10^6, series that end on a rise, NaN and +-inf in scores and
  thresholds, scores equal to thresholds, and rows of a wider buffer (series_stride > n_frames).
* count_ge against np.count_nonzero around the block and grid boundaries (G = sm_count * 8 blocks of 256), with 64
  and 65 thresholds.
* predict_clips_array scores, one label's column as a non-contiguous CUDA view, through the ROC helpers.
* Refusals at the ABI (nothing launched) for the float32 and float64 entry points."""
import numpy as np
import pytest

from oracle import metrics as om
from test_metrics import edge_golden, edge_threshold

pytestmark = pytest.mark.gpu
EINVAL = -1


@pytest.fixture(scope="module")
def torch_cuda(built_library):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


@pytest.fixture(scope="module")
def M(torch_cuda):
    from openwakeword_b200 import metrics
    return metrics


def _forms(torch, s):
    """The ways a user hands the reference the same float16 / float32 / float64 series: the array, a list of its
    NumPy scalars, a list of Python floats (float64 only: np.array of it is float64) and a CUDA tensor."""
    out = [s, list(s), torch.from_numpy(s).cuda()]
    if s.dtype == np.float64:
        out.append(s.tolist())
    return out


def test_edge_goldens_through_every_entry_point(torch_cuda, M):
    torch = torch_cuda
    z = edge_golden()
    thr = [edge_threshold(t, k) for t in z["base"] for k in z["kinds"]]     # a list: each keeps its own type
    windows = [int(w) for w in z["windows"]]
    for i in range(int(z["n_series"])):
        s = z[f"s{i}"]
        want = z["fp"][i].reshape(len(thr), len(windows))
        for form in _forms(torch, s):
            for wi, w in enumerate(windows):
                got = M.false_positives_batch(form, thr, w)
                assert got.shape == (1, len(thr)) and list(got[0]) == list(want[:, wi]), (i, s.dtype, type(form), w)
        assert [M.get_false_positives(list(s), t) for t in thr] == list(want[:, windows.index(50)]), i
    for j in range(2):
        s, w = z[f"roc_s{j}"], int(z[f"roc_window{j}"])
        for form in _forms(torch, s):
            assert M.generate_roc_curve_fprs(form, 25, 0.08, grouping_window=w) == list(z[f"roc_fprs{j}"]), (j, type(form))
            assert M.generate_roc_curve_tprs(form, 25) == list(z[f"roc_tprs{j}"]), (j, type(form))


def test_comparison_precision_cases(torch_cuda, M):
    """float32 scores against a Python float compare in float32 (the reference counts float32(0.7) >= 0.7); a list of
    Python floats is float64 (0.5 - 1e-10 < 0.5, though it rounds to 0.5 in float32)."""
    torch = torch_cuda
    a = np.array([0, np.float32(0.7), 0, 0], np.float32)
    for form in (a, list(a), torch.from_numpy(a).cuda()):
        assert M.get_false_positives(form, 0.7) == 1
        assert M.get_false_positives(form, np.float64(0.7)) == 0
    b = [0, 0.5 - 1e-10, 0, 0]
    for form in (b, np.array(b), torch.tensor(b, dtype=torch.float64, device="cuda")):
        assert M.get_false_positives(form, 0.5) == 0
    assert M.get_false_positives(torch.tensor(b, dtype=torch.float32, device="cuda"), 0.5) == 1
    assert M.get_false_positives([], 0.5) == 0
    assert M.get_false_positives([0.1, 0.9], 0.5) == 1            # ends on a rise: the reference raises, here a no-op


def test_half_precision_inputs(torch_cuda, M):
    """float16 arrays and tensors compare as float16 against a Python float; bfloat16 tensors as float32 scores
    of the same values."""
    torch = torch_cuda
    rng = np.random.default_rng(5)
    h = rng.choice(np.float16([0, 0.7, 0.6997, 0.7004, 0.1, 0.5, 1]), 300)
    h[-1] = 0
    for t in (0.7, np.float64(0.7), np.float32(0.7), 0.1, 0.5):
        want = om.get_false_positives(h, t, 5)
        assert M.get_false_positives(h, t, 5) == want
        assert M.get_false_positives(torch.from_numpy(h).cuda(), t, 5) == want
    bf = torch.from_numpy(rng.uniform(0, 1, 500).astype(np.float32)).to(torch.bfloat16)
    host = bf.float().numpy()
    host[-1] = 0
    bf[-1] = 0
    for t in (0.7, np.float64(0.3), float(host[7])):
        assert M.get_false_positives(bf.cuda(), t, 50) == om.get_false_positives(host, t, 50)
    assert M.generate_roc_curve_tprs(bf.cuda(), 25) == om.generate_roc_curve_tprs(host, 25)


def _thresholds(rng, n, dtype):
    """n thresholds: NaN, +-inf, 0 and 1 first, the rest uniform, all exactly representable in the score dtype."""
    t = np.concatenate([[np.nan, np.inf, -np.inf, 0.0, 1.0], rng.uniform(0, 1, max(n - 5, 0))])[:n]
    return t.astype(dtype).astype(np.float64)


def _scores(rng, n_series, n_frames, thr, dtype):
    """Uniform scores with 30 % drawn from the thresholds themselves, NaN and +-inf; a low/high alternating start so the
    grouping rule acts; every other series ends on a rise for most thresholds."""
    pool = np.concatenate([thr[np.isfinite(thr)], [np.nan, np.inf, -np.inf, 0.0, 1.0]])
    S = rng.uniform(0, 1, (n_series, n_frames))
    pick = rng.random(S.shape) < 0.3
    S[pick] = rng.choice(pool, int(pick.sum()))
    k = min(n_frames, 80)
    S[:, 0:k:2] = -1.0
    if n_frames >= 2:
        S[::2, -2:] = [-2.0, 2.0]
    return S.astype(dtype)


def _oracle_fp(S, thr, w):
    return np.array([[om.get_false_positives(s, np.float64(t), w) for t in thr] for s in S], np.int64).reshape(len(S), len(thr))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_false_positive_kernel_layout(torch_cuda, M, dtype):
    torch = torch_cuda
    rng = np.random.default_rng(11)
    cases = [(ns, 64, nt, 7) for nt in (1, 31, 32, 33, 63, 64, 65, 4096, 4097) for ns in (1, 3, 5)]
    cases += [(1000, 40, nt, 50) for nt in (1, 33)]
    for ns, nf, nt, w in cases:
        thr = _thresholds(rng, nt, dtype)
        S = _scores(rng, ns, nf, thr, dtype)
        got = M.false_positives_batch(torch.from_numpy(S).cuda(), thr, w)          # an array: np.float64 thresholds
        assert np.array_equal(got, _oracle_fp(S, thr, w)), (ns, nf, nt, w)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_false_positive_kernel_frames_windows_and_stride(torch_cuda, M, dtype):
    """Rows of a wider buffer whose tail is +inf (>= every threshold but NaN), so a read past n_frames shows."""
    torch = torch_cuda
    rng = np.random.default_rng(12)
    ctx = M._context(0)
    stream = torch.cuda.current_stream().cuda_stream
    for nf in (0, 1, 2, 3, 5000, 100000):
        thr = _thresholds(rng, 33, dtype)
        S = _scores(rng, 3, nf, thr, dtype)
        stride = nf + 37
        buf = np.full((3, stride), np.inf, dtype)
        buf[:, :nf] = S
        d = torch.from_numpy(buf).cuda()
        for w in (0, 1, 7, 50, 10 ** 6):
            got = ctx.metrics_false_positives(d, stride, 3, nf, thr, w, stream)
            assert np.array_equal(got, _oracle_fp(S, thr, w)), (nf, w)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_count_ge_block_and_grid_boundaries(torch_cuda, M, dtype):
    torch = torch_cuda
    rng = np.random.default_rng(13)
    ctx = M._context(0)
    stream = torch.cuda.current_stream().cuda_stream
    G = torch.cuda.get_device_properties(0).multi_processor_count * 8
    sizes = [0, 1, 255, 256, 257, G * 256 - 1, G * 256, G * 256 + 1]
    if dtype == np.float32:
        sizes.append(10 ** 7)                                            # 40 MB
    for nt in (64, 65):
        thr = _thresholds(rng, nt, dtype)
        pool = np.concatenate([thr[np.isfinite(thr)], [np.nan, np.inf, -np.inf]])
        host = rng.uniform(0, 1, max(sizes) + 1)
        pick = rng.random(host.size) < 0.5
        host[pick] = rng.choice(pool, int(pick.sum()))                   # many scores exactly on a threshold
        host = host.astype(dtype)
        d = torch.from_numpy(host).cuda()
        for n in sizes:
            got = ctx.metrics_count_ge(d, n, thr, stream)
            want = [np.count_nonzero(host[:n] >= np.float64(t)) for t in thr]
            assert list(got) == want, (nt, n)
        del d


def test_roc_on_predict_clips_array_columns(torch_cuda, M):
    torch = torch_cuda
    from helpers import emb_weights, head
    from openwakeword_b200 import Model
    m = Model(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")},
                               {"name": "mycroft", "head": head("hey_mycroft_v0.1")}], embedding_model_path=emb_weights())
    rng = np.random.default_rng(21)
    clips = np.clip(rng.normal(0, 4000, (3, 48000)), -32768, 32767).astype(np.int16)
    scores, labels = m.predict_clips_array(clips, padding=1)
    d = scores if isinstance(scores, torch.Tensor) else torch.from_numpy(np.asarray(scores))
    d = d.cuda()
    host = d.cpu().numpy()
    assert d.dtype == torch.float32 and d.dim() == 3 and d.shape[2] == len(labels) >= 2
    for j in range(len(labels)):
        for i in range(d.shape[0]):
            col = d[i, :, j]
            assert not col.is_contiguous()
            assert M.generate_roc_curve_fprs(col, 25) == om.generate_roc_curve_fprs(host[i, :, j], 25)
            assert M.generate_roc_curve_tprs(col, 25) == om.generate_roc_curve_tprs(host[i, :, j], 25)
        cols = d[:, :, j]
        got = M.false_positives_batch(cols, np.linspace(0.01, 0.99, 25), 50)
        assert np.array_equal(got, _oracle_fp(host[:, :, j], np.linspace(0.01, 0.99, 25), 50))
        assert M.generate_roc_curve_tprs(cols, 9) == om.generate_roc_curve_tprs(host[:, :, j].reshape(-1), 9)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_refusals_launch_nothing(torch_cuda, M, dtype):
    torch = torch_cuda
    ctx = M._context(0)
    lib, h = ctx.lib, ctx.h
    fp = lib.oww_metrics_false_positives if dtype == "float32" else lib.oww_metrics_false_positives_f64
    ge = lib.oww_metrics_count_ge if dtype == "float32" else lib.oww_metrics_count_ge_f64
    d = torch.zeros(64, dtype=getattr(torch, dtype), device="cuda")
    p = d.data_ptr()
    thr = np.zeros(4097)
    cnt32 = np.zeros((4, 4097), np.int32)
    cnt64 = np.zeros(65, np.uint64)
    t, c32, c64 = thr.ctypes.data, cnt32.ctypes.data, cnt64.ctypes.data
    before = ctx.launch_count
    assert fp(h, p, 16, 4, 16, t, 0, 50, c32, None) == EINVAL
    assert fp(h, p, 16, 4, 16, t, 4097, 50, c32, None) == EINVAL
    assert fp(h, p, 16, 0, 16, t, 8, 50, c32, None) == EINVAL
    assert fp(h, p, 16, 4, -1, t, 8, 50, c32, None) == EINVAL
    assert fp(h, None, 16, 4, 16, t, 8, 50, c32, None) == EINVAL
    assert fp(h, p, 16, 4, 16, None, 8, 50, c32, None) == EINVAL
    assert fp(h, p, 16, 4, 16, t, 8, 50, None, None) == EINVAL
    assert fp(None, p, 16, 4, 16, t, 8, 50, c32, None) == EINVAL
    assert ge(h, p, 64, t, 0, c64, None) == EINVAL
    assert ge(h, p, 64, t, 65, c64, None) == EINVAL
    assert ge(h, p, -1, t, 8, c64, None) == EINVAL
    assert ge(h, None, 64, t, 8, c64, None) == EINVAL
    assert ge(h, p, 64, None, 8, c64, None) == EINVAL
    assert ge(h, p, 64, t, 8, None, None) == EINVAL
    assert ge(None, p, 64, t, 8, c64, None) == EINVAL
    assert ctx.launch_count == before
    assert not cnt32.any() and not cnt64.any()
    with pytest.raises(ValueError):
        ctx.metrics_count_ge(d.half(), 64, [0.5])
