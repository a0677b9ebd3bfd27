"""Custom verifier models restated in float64 (openwakeword/custom_verifier_model.py:91-113 and the score replacement
of openwakeword/model.py:319-328 in the original project).

``verifier_proba`` evaluates the reference's pipeline FunctionTransformer(flatten_features) -> StandardScaler ->
binary LogisticRegression from its fitted attributes, without calling scikit-learn.  ``VerifiedOracleModel`` is an
``OracleModel`` of one stream with its own verifiers: where a label of a verified parent reaches the threshold
(compared in float32, as NumPy compares a float32 score with a Python float), the verifier's probability on the
parent's newest n_in feature rows replaces the score, before the first-five zeroing.  Each label is verified once,
with its own parent's n_in (DESIGN.md, K3 verifiers).
"""
import numpy as np

from .streaming import OracleModel, _n_out


def verifier_proba(pipeline, feats):
    """P(positive) = predict_proba(feats)[:, -1] of a fitted pipeline; feats [n, n_in, 96] -> float64 [n]."""
    _, scaler, lr = (s[1] for s in pipeline.steps)
    x = np.asarray(feats, np.float64).reshape(len(feats), -1)
    if scaler.with_mean:
        x = x - np.asarray(scaler.mean_, np.float64)
    if scaler.with_std:
        x = x / np.asarray(scaler.scale_, np.float64)
    z = x @ np.asarray(lr.coef_[0], np.float64) + float(lr.intercept_[0])
    return 1.0 / (1.0 + np.exp(-z))


class VerifiedOracleModel(OracleModel):
    """OracleModel with ``verifiers`` {parent name: fitted pipeline or None}; ``verifiers`` may be changed between
    calls (a reassignment takes effect at the next call).  patience / debounce_time are not restated here."""

    def __init__(self, emb_weights, heads, verifiers=None, threshold=0.1, **kw):
        super().__init__(emb_weights, heads, **kw)
        self.verifiers = dict(verifiers or {})
        self.verifier_threshold = threshold

    def predict(self, x, patience=None, threshold=None, debounce_time=0.0):
        if patience or debounce_time > 0:
            raise NotImplementedError("VerifiedOracleModel restates predict without patience / debounce")
        before = {lab: len(b) for lab, b in self.prediction_buffer.items()}
        out = super().predict(x)
        thr = np.float32(self.verifier_threshold)
        for name, v in self.verifiers.items():
            if v is None:
                continue
            labs = [name] if _n_out(self.heads[name]) == 1 else list(self.class_mapping[name].values())
            p = None
            for lab in labs:
                if before.get(lab, 0) < 5:             # zeroed after the replacement anyway (model.py:330-333)
                    continue
                if np.float32(out[lab]) >= thr:
                    if p is None:
                        p = float(verifier_proba(v, self.preprocessor.get_features(self.heads[name]["n_in"]))[0])
                    out[lab] = p
                    self.prediction_buffer[lab][-1] = p
        return out

