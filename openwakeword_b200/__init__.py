"""openwakeword_b200 - CUDA-native (H100, sm_90a) drop-in for openWakeWord's streaming inference hot path.

Mirrors the public names of openwakeword/__init__.py for the path in scope
(SURVEY.md section 8): ``Model``, ``MODELS``, ``FEATURE_MODELS``, ``model_class_mappings``,
``get_pretrained_model_paths``, ``train_custom_verifier``; ``utils.AudioFeatures`` and ``utils.bulk_predict``.
Importing the package needs neither a GPU nor the built library; constructing a ``Model`` /
``AudioFeatures`` does (and fails loudly otherwise - there is no CPU fallback).
"""
from .registry import MODELS, FEATURE_MODELS, model_class_mappings, get_pretrained_model_paths  # noqa: F401
from .model import Model  # noqa: F401
from .utils import AudioFeatures, bulk_predict, compute_features_from_generator  # noqa: F401
from .custom_verifier_model import train_custom_verifier  # noqa: F401

__all__ = ["Model", "AudioFeatures", "bulk_predict", "compute_features_from_generator", "MODELS", "FEATURE_MODELS",
           "model_class_mappings", "get_pretrained_model_paths", "train_custom_verifier"]
__version__ = "0.1.0"
