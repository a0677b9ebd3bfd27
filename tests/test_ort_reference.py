"""Auto-upgrade of the parity harness to the GENUINE reference (SURVEY.md section 7.3c / 8c, last row).

When ``onnxruntime`` is importable AND the released model files (melspectrogram.onnx, embedding_model.onnx, <head>.onnx)
are found (oracle/probe.py), this test drives the unmodified ``openwakeword.Model(inference_framework="onnx")``
(openwakeword/model.py:149-159, utils.py:79-93) and this repository's CUDA path on the same int16 frames
with the same injected ``feature_buffer`` (SURVEY.md F6) and holds every per-frame, per-label score to the 1e-3 gate of
BASELINE.json.  Neither exists in this image or on the GPU box (SURVEY.md F2/F3), so today the test SKIPS - it is the
hook that turns "parity vs the NumPy restatement on synthetic weights" into "parity vs ONNX" the moment the assets appear.
"""
import glob
import importlib
import os
import sys

import numpy as np
import pytest

from oracle import probe

_OK, _WHERE = probe.ort_reference_available()
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not _OK, reason=f"genuine reference unavailable: {_WHERE}")]


def _import_reference():
    """the unmodified reference package: installed, or from baseline/_ref"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for extra in (None, os.path.join(root, "baseline", "_ref")):
        if extra and os.path.isdir(extra) and extra not in sys.path:
            sys.path.insert(0, extra)
        try:
            return importlib.import_module("openwakeword")
        except Exception:          # noqa: BLE001
            continue
    pytest.skip("the reference package cannot be imported")


def test_probe_reports_consistently():
    ok, where = probe.ort_reference_available()
    assert ok and os.path.isdir(where)
    assert "onnxruntime reference" in probe.parity_label()


def test_scores_match_genuine_onnx_reference_within_1e3(built_library):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import openwakeword_b200 as owb
    ow = _import_reference()
    heads = sorted(p for p in glob.glob(os.path.join(_WHERE, "*.onnx"))
                   if os.path.basename(p) not in ("melspectrogram.onnx", "embedding_model.onnx", "silero_vad.onnx"))
    assert heads, "no wake-word head files next to the feature models"
    mel_p, emb_p = os.path.join(_WHERE, "melspectrogram.onnx"), os.path.join(_WHERE, "embedding_model.onnx")
    rng = np.random.default_rng(0)
    fi = None
    worst = 0.0
    for cnn_mode in (0, 3):
        ref = ow.Model(wakeword_models=heads, inference_framework="onnx", melspec_model_path=mel_p, embedding_model_path=emb_p)
        if fi is None:
            fi = np.asarray(ref.preprocessor.feature_buffer, np.float32).copy()      # unseeded noise embeddings (F6): share them
        ref.preprocessor.feature_buffer = fi.copy()
        ours = owb.Model(wakeword_models=heads, melspec_model_path=mel_p, embedding_model_path=emb_p, feature_init=fi, cnn_mode=cnn_mode)
        pcm = np.concatenate([rng.integers(-1000, 1000, 40 * 1280), (rng.uniform(-1, 1, 40 * 1280) * 32767).astype(np.int64),
                              np.zeros(10 * 1280, np.int64), rng.normal(0, 8000, 40 * 1280).astype(np.int64)])
        pcm = np.clip(pcm, -32768, 32767).astype(np.int16)
        for i in range(0, pcm.shape[0], 1280):
            a = ref.predict(pcm[i:i + 1280])
            b = ours.predict(pcm[i:i + 1280])
            assert set(a) == set(b)
            worst = max(worst, max(abs(float(a[k]) - float(b[k])) for k in a))
        print(f"cnn_mode {cnn_mode}: max |score - onnxruntime reference| = {worst:.3e}")
        assert worst <= 1e-3
