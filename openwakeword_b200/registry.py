"""Model registry mirroring openwakeword/__init__.py:8-69 (names, file names, timer
class mapping).  Paths point at ``resources/models/<name>_v0.1.npz`` - the b200 container written by
``weights.save_head`` (the reference's .tflite/.onnx assets are download-only and absent here)."""
import os

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "resources", "models")

FEATURE_MODELS = {
    "embedding": {"model_path": os.path.join(_DIR, "embedding_model.npz")},
    "melspectrogram": {"model_path": "builtin"},
}
MODELS = {name: {"model_path": os.path.join(_DIR, f"{name}_v0.1.npz")}
          for name in ("alexa", "hey_mycroft", "hey_jarvis", "hey_rhasspy", "timer", "weather")}

model_class_mappings = {
    "timer": {"1": "1_minute_timer", "2": "5_minute_timer", "3": "10_minute_timer",
              "4": "20_minute_timer", "5": "30_minute_timer", "6": "1_hour_timer"}
}


def get_pretrained_model_paths(inference_framework="b200"):
    """Paths of the six pretrained heads: the .npz container if present, else a same-named .onnx (the reference's
    release asset dropped into resources/models/), else the .npz path (construction then reports the missing file)."""
    out = []
    for k in MODELS:
        p = MODELS[k]["model_path"]
        if not os.path.exists(p) and os.path.exists(p[:-4] + ".onnx"):
            p = p[:-4] + ".onnx"
        out.append(p)
    return out
