"""Custom verifier models (openwakeword/custom_verifier_model.py, docs/custom_verifier_models.md of the original
project): training them on the GPU, loading the pickles ``train_verifier_model`` writes without the reference package,
and the reduction of the recognised pipeline to the form the device evaluates (include/owwb200.h, ``oww_load_verifier``).

``train_verifier_model``, ``get_reference_clip_features`` and ``train_custom_verifier`` keep the reference's signatures.
The fit (StandardScaler -> LogisticRegression(C=0.001), scikit-learn's lbfgs in the reference) runs as a float64 Newton
solve on the device (``oww_fit_verifiers``, csrc/verifier_fit.cu) and comes back as the scikit-learn pipeline the
reference pickles, with the fitted attributes scikit-learn's own fit sets.  These three need scikit-learn, as in the
reference; loading and running verifiers does not."""
import io
import os
import pickle
import types
import warnings

import numpy as np

_REF_FLATTEN = ("openwakeword.custom_verifier_model", "flatten_features")


def flatten_features(x):
    """custom_verifier_model.py:91-92: [N, n_in, 96] -> N rows of n_in*96."""
    return [i.flatten() for i in x]


class _Unpickler(pickle.Unpickler):
    def find_class(self, module, name):
        if (module, name) == _REF_FLATTEN:
            return flatten_features
        return super().find_class(module, name)


def load_verifier(path):
    """Unpickle a verifier.  The reference pipeline's FunctionTransformer stores its function as
    ``openwakeword.custom_verifier_model.flatten_features``; that one global resolves to this module's function, so
    loading needs neither the reference package nor onnxruntime.  Everything else resolves normally."""
    with open(path, "rb") as fh:
        return _Unpickler(fh).load()


def _is_flatten(func):
    return func is flatten_features or (getattr(func, "__module__", None), getattr(func, "__qualname__", None)) == _REF_FLATTEN


def linear_verifier_params(obj):
    """(mean float32[D], weight float32[D], bias float) of the reference's pipeline
    FunctionTransformer(flatten_features) -> StandardScaler -> binary LogisticRegression, such that
    ``predict_proba(x)[:, -1] = 1 / (1 + exp(-(bias + sum((x - mean) * weight))))`` with weight = coef_ / scale_
    (float64 on the host, then fp32).  None for anything else: other estimators, multi-class models, extra steps,
    objects that only have ``predict_proba``."""
    try:
        from sklearn.pipeline import Pipeline
        from sklearn.preprocessing import FunctionTransformer, StandardScaler
        from sklearn.linear_model import LogisticRegression
    except ImportError:
        return None
    if not isinstance(obj, Pipeline) or len(obj.steps) != 3:
        return None
    ft, sc, lr = (s[1] for s in obj.steps)
    if type(ft) is not FunctionTransformer or not _is_flatten(ft.func) or ft.kw_args:
        return None
    if type(sc) is not StandardScaler or type(lr) is not LogisticRegression:
        return None
    classes = getattr(lr, "classes_", None)
    coef = getattr(lr, "coef_", None)
    if classes is None or len(classes) != 2 or coef is None or coef.shape[0] != 1:
        return None
    D = coef.shape[1]
    if D % 96:
        return None
    mean = np.asarray(sc.mean_, np.float64) if sc.with_mean else np.zeros(D)
    scale = np.asarray(sc.scale_, np.float64) if sc.with_std else np.ones(D)
    if mean.shape != (D,) or scale.shape != (D,):
        return None
    w = np.asarray(coef[0], np.float64) / scale
    return mean.astype(np.float32), w.astype(np.float32), float(lr.intercept_[0])


# ---- training --------------------------------------------------------------------------------------------------------

C_DEFAULT = 0.001        # LogisticRegression(random_state=0, max_iter=2000, C=0.001) of train_verifier_model
FIT_TOL = 1e-10          # max |gradient| <= FIT_TOL * C * n: below scikit-learn's lbfgs stopping error by orders of magnitude
FIT_MAX_ITER = 100       # Newton iterations (4-5 at C = 0.001)
_contexts = {}


def _fit_context(device):
    from . import _native
    if device not in _contexts:
        _contexts[device] = _native.Context(device=device, cnn_mode=_native.CNN_FP32_WINDOW, max_chunks=1)
    return _contexts[device]


def _as_windows(features):
    """[N, n_in, 96] (or [N, n_in*96]) -> float32 [N, n_in, 96]"""
    x = np.asarray(features, np.float32)
    if x.ndim == 2 and x.shape[1] % 96 == 0:
        x = x.reshape(x.shape[0], -1, 96)
    if x.ndim != 3 or x.shape[2] != 96 or x.shape[1] < 1:
        raise ValueError(f"features must be windows [N, n_in, 96], got shape {x.shape}")
    return np.ascontiguousarray(x)


def fit_windows(rows, n_in, first_row, sample_offsets, labels, C=C_DEFAULT, max_iter=FIT_MAX_ITER, tol=FIT_TOL,
                device=None):
    """Fit one verifier per user on the device.  rows: float32 [R, 96] (numpy or a CUDA tensor); first_row: int64 [N]
    (sample i is rows[first_row[i] : first_row[i] + n_in]); labels: [N] (nonzero = positive); sample_offsets: int64
    [U + 1].  -> dict of host arrays mean, var, coef [U, n_in*96] and intercept [U] (float64), iters and status [U]
    (include/owwb200.h, oww_fit_verifiers: 0 converged, 1 stopped at max_iter, 2 one class or no samples, 3 non-finite
    input or a window outside rows).  The fit runs on `device` (a CUDA ordinal), else on the device of a tensor `rows`,
    else on the current CUDA device."""
    import torch
    if device is not None:
        dev = torch.device("cuda", int(device))
    elif isinstance(rows, torch.Tensor):
        dev = rows.device
    else:
        dev = torch.device("cuda", torch.cuda.current_device())
    ctx = _fit_context(dev.index)

    def to(x, dtype):
        t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))
        return t.to(device=dev, dtype=dtype).contiguous()
    lab = labels if isinstance(labels, torch.Tensor) else torch.from_numpy(np.asarray(labels) != 0)
    out = ctx.fit_verifiers(to(rows, torch.float32), int(n_in), to(first_row, torch.int64), sample_offsets,
                            to(lab != 0, torch.uint8), C, max_iter, tol)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _pipeline(n, n_in, classes, fit, u=0):
    """The fitted reference pipeline FunctionTransformer(flatten_features) -> StandardScaler -> LogisticRegression of
    user u of `fit`, with the attributes scikit-learn's fit on that user's n windows [n, n_in, 96] sets."""
    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import FunctionTransformer, StandardScaler
    ft = FunctionTransformer(flatten_features).fit(np.zeros((1, n_in, 96), np.float32))   # sets n_features_in_ = n_in
    D = fit["coef"].shape[1]
    sc = StandardScaler()
    sc.n_features_in_ = D
    sc.n_samples_seen_ = np.float64(n)
    sc.mean_ = fit["mean"][u].copy()
    sc.var_ = fit["var"][u].copy()
    eps = np.finfo(np.float64).eps
    n = float(n)
    const = sc.var_ <= n * eps * sc.var_ + (n * sc.mean_ * eps) ** 2      # scikit-learn's _is_constant_feature
    sc.scale_ = np.where(const, 1.0, np.sqrt(sc.var_))
    lr = LogisticRegression(random_state=0, max_iter=2000, C=C_DEFAULT)
    lr.n_features_in_ = D
    lr.classes_ = np.asarray(classes)
    lr.coef_ = fit["coef"][u][None].copy()
    lr.intercept_ = np.array([fit["intercept"][u]])
    lr.n_iter_ = np.array([fit["iters"][u]], np.int32)
    return make_pipeline(ft, sc, lr)


def train_verifier_model(features, labels):
    """custom_verifier_model.py:95-113: fit FunctionTransformer(flatten_features) -> StandardScaler ->
    LogisticRegression(random_state=0, max_iter=2000, C=0.001) on windows ``features`` [N, n_in, 96] and binary
    ``labels`` [N], on the GPU.  Returns the fitted scikit-learn pipeline."""
    x = _as_windows(features)
    y = np.asarray(labels).ravel()
    if y.shape[0] != x.shape[0]:
        raise ValueError(f"{x.shape[0]} windows but {y.shape[0]} labels")
    classes = np.unique(y)
    if classes.size != 2:
        raise ValueError(f"a verifier needs samples of exactly 2 classes; the data has {classes.size}")
    N, n_in = x.shape[:2]
    fit = fit_windows(x.reshape(-1, 96), n_in, np.arange(N, dtype=np.int64) * n_in, np.array([0, N], np.int64),
                      y == classes[1])
    status = int(fit["status"][0])
    if status == 3:
        raise ValueError("features contain NaN or infinity")
    if status == 1:
        from sklearn.exceptions import ConvergenceWarning
        warnings.warn(f"the verifier fit stopped after {int(fit['iters'][0])} Newton iterations without converging",
                      ConvergenceWarning, stacklevel=2)
    return _pipeline(N, n_in, classes, fit)


class _RefPickler(pickle._Pickler):
    """Writes this module's ``flatten_features`` under the reference's global name, so the pickle loads with the
    reference package as well as with ``load_verifier``."""
    dispatch = dict(pickle._Pickler.dispatch)

    def _save_function(self, obj, name=None):
        if obj is flatten_features:
            self.save(_REF_FLATTEN[0])
            self.save(_REF_FLATTEN[1])
            self.write(pickle.STACK_GLOBAL)
            self.memoize(obj)
        else:
            pickle._Pickler.save_global(self, obj, name)
    dispatch[types.FunctionType] = _save_function


def dumps_verifier(pipeline):
    """Pickle a verifier pipeline the way the reference's train_custom_verifier writes it (pickle protocol 4+)."""
    buf = io.BytesIO()
    _RefPickler(buf, protocol=max(4, pickle.DEFAULT_PROTOCOL)).dump(pipeline)
    return buf.getvalue()


def get_reference_clip_features(reference_clip, oww_model, model_name, threshold=0.5, N=3, **kwargs):
    """custom_verifier_model.py:32-88: run `reference_clip` (WAV path or int16 array) N times through
    ``oww_model.predict`` in 1280-sample steps (each pass after N != 1 first drops np.random.randint(0, 1280) samples),
    and stack the n_in newest feature rows of every step whose prediction for `model_name` is >= threshold ->
    [n, n_in, 96].  The model is not reset, as in the reference."""
    from .utils import _read_wav
    n_in = oww_model.model_inputs[model_name]
    hits = []
    for _ in range(N):
        dat = _read_wav(reference_clip) if isinstance(reference_clip, (str, os.PathLike)) else reference_clip
        if N != 1:
            dat = dat[np.random.randint(0, 1280):]
        for i in range(0, dat.shape[0] - 1280, 1280):
            if oww_model.predict(dat[i:i + 1280], **kwargs)[model_name] >= threshold:
                hits.append(oww_model.preprocessor.get_features(n_in))       # [1, n_in, 96]
    return np.vstack(hits) if hits else np.empty((0, n_in, 96))


def enrollment_passes(lengths_pos, lengths_neg):
    """The passes train_custom_verifier makes over the clips, in order: positives N = 5 (an offset drawn with
    np.random.randint(0, 1280) per pass), negatives N = 1 (offset 0).  -> list of (positive, clip index, offset,
    steps), steps = len(range(0, length - offset - 1280, 1280)).  Consumes the NumPy global RNG as the reference does."""
    out = []
    for pos, lengths, n in ((True, lengths_pos, 5), (False, lengths_neg, 1)):
        for c, L in enumerate(lengths):
            for _ in range(n):
                o = np.random.randint(0, 1280) if n != 1 else 0
                out.append((pos, c, o, len(range(0, int(L) - o - 1280, 1280))))
    return out


def enrollment_clip(pos, neg, passes):
    """One clip whose 1280-sample steps are the steps of every pass in order: each pass's stepped prefix, concatenated,
    plus one chunk of zeros so that a bulk run with padding 0 (len(range(0, L - 1280, 1280)) steps) steps them all.
    -> (int16 pcm, per-step label 1/0)"""
    parts, lab = [], []
    for p, c, o, k in passes:
        parts.append(np.asarray((pos if p else neg)[c], np.int16)[o:o + k * 1280])
        lab.append(np.full(k, 1 if p else 0, np.int8))
    parts.append(np.zeros(1280, np.int16))
    return np.concatenate(parts), (np.concatenate(lab) if lab else np.zeros(0, np.int8))


def enroll(oww, model_name, users, feature_init=None, streams=None):
    """Capture and fit the verifiers of several users on one Model, without touching its streams or banks.

    users: list of (positive clips, negative clips), each clip an int16 array.  For every user in turn, the NumPy
    global RNG draws that user's pass offsets (``enrollment_passes``); the user's passes become one clip
    (``enrollment_clip``).  All users' clips then run in one bulk call (padding 0, 1280-sample calls) from the Model's
    fresh state, and every captured window becomes a first-row index into [feature_init | that user's embedding rows]
    for one ``oww_fit_verifiers`` call.  streams (stream models): user u's clip is scored by stream streams[u]'s own
    model (``Model.predict_clips(..., streams=)``).  Returns per user a dict: pipeline (None unless status 0 or 1), status, passes,
    counts (windows captured per pass), and the device parameters mean, weight (float32 [D]) and bias (float32)."""
    n_in = oww.model_inputs[model_name]
    passes = [enrollment_passes([len(c) for c in pos], [len(c) for c in neg]) for pos, neg in users]
    clips = [enrollment_clip(pos, neg, ps) for (pos, neg), ps in zip(users, passes)]
    pcm = np.concatenate([c for c, _ in clips])
    offsets = np.concatenate([[0], np.cumsum([c.size for c, _ in clips])]).astype(np.int64)
    scores, row_off, labels, emb, step_off, fi = oww._predict_ragged(pcm, offsets, 0, 1280, feature_init,
                                                                     want_features=True, streams=streams)
    if model_name not in labels:          # a multi-output model has no label of its own name
        raise KeyError(model_name)
    if n_in > len(fi):
        raise ValueError(f"model '{model_name}' reads {n_in} feature rows; the initial feature ring has {len(fi)}")
    s = scores[:, labels.index(model_name)]
    blocks, first, lab, counts, base = [], [], [], [], 0
    for u, (_, step_label) in enumerate(clips):
        su = s[row_off[u]:row_off[u + 1]]
        take = np.where(step_label == 1, su >= 0.5, su >= 0.0)
        k = np.nonzero(take)[0]
        first.append(base + len(fi) + k + 1 - n_in)
        lab.append(step_label[k])
        ends = np.cumsum([p[3] for p in passes[u]])
        counts.append(np.diff(np.concatenate([[0], np.searchsorted(k, ends)])))
        blocks += [fi, emb[step_off[u]:step_off[u + 1]]]
        base += len(fi) + int(step_off[u + 1] - step_off[u])
    sample_off = np.concatenate([[0], np.cumsum([len(f) for f in first])]).astype(np.int64)
    fit = fit_windows(np.concatenate(blocks), n_in, np.concatenate(first), sample_off, np.concatenate(lab),
                      device=oww.preprocessor.device_index)
    out = []
    for u in range(len(users)):
        st = int(fit["status"][u])
        n = int(sample_off[u + 1] - sample_off[u])
        pipe = _pipeline(n, n_in, np.array([0, 1]), fit, u) if st in (0, 1) else None
        scale = pipe.steps[1][1].scale_ if pipe is not None else np.ones(n_in * 96)
        out.append({"pipeline": pipe, "status": st, "passes": passes[u], "counts": counts[u],
                    "mean": fit["mean"][u].astype(np.float32), "weight": (fit["coef"][u] / scale).astype(np.float32),
                    "bias": np.float32(fit["intercept"][u])})
    return out


def train_custom_verifier(positive_reference_clips, negative_reference_clips, output_path, model_name, **kwargs):
    """custom_verifier_model.py:116-177: train a speaker's verifier for `model_name` (a model file path, or the name
    of a model the Model built from ``**kwargs`` has) and pickle it to `output_path`.

    As in the reference, one Model runs every pass without a reset: positives 5 times each from a random offset,
    capturing windows that score >= 0.5, then negatives once each, capturing every step.  Here all passes run as one
    clip on the bulk path (their stepped prefixes are whole chunks), and the fit runs on the Model's GPU."""
    from .model import Model
    from .utils import _read_wav
    if os.path.exists(model_name):
        oww = Model(wakeword_models=[model_name], **kwargs)
        model_name = os.path.splitext(model_name)[0].split(os.path.sep)[-1]
    else:
        oww = Model(**kwargs)
    pre = oww.preprocessor
    if pre._feature_init is None:         # the reference draws the initial feature ring at construction, before the offsets
        pre._feature_init = pre._get_embeddings(np.random.randint(-1000, 1000, 16000 * 4).astype(np.int16))
    if model_name not in oww.model_inputs:
        raise KeyError(model_name)
    read = lambda c: _read_wav(c) if isinstance(c, (str, os.PathLike)) else np.asarray(c, np.int16)   # noqa: E731
    r = enroll(oww, model_name, [([read(c) for c in positive_reference_clips],
                                  [read(c) for c in negative_reference_clips])])[0]
    if not sum(c for (pos, _, _, _), c in zip(r["passes"], r["counts"]) if pos):
        raise ValueError("The positive features were not created! Make sure that the positive reference clips contain the "
                         "appropriate audio for the desired model.")
    if r["status"] == 3:
        raise ValueError("features contain NaN or infinity")
    if r["status"] == 2:
        raise ValueError("a verifier needs both positive and negative windows; no negative window was captured")
    with open(output_path, "wb") as fh:
        fh.write(dumps_verifier(r["pipeline"]))
    return r["pipeline"]
