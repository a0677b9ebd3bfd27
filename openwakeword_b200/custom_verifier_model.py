"""Custom verifier models (openwakeword/custom_verifier_model.py:91-113, docs/custom_verifier_models.md of the
original project): loading the pickles ``train_verifier_model`` writes without the reference package, and the
reduction of the recognised pipeline to the form the device evaluates (include/owwb200.h, ``oww_load_verifier``).
Training stays with the reference (SURVEY.md section 2 #9)."""
import pickle

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
