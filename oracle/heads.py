"""Wake-word classifier head restatement (the graphs inside ``<head>.onnx``).

Family from openwakeword/train.py:56-83 (``Net``/``FCNBlock``:
Flatten -> Linear -> LayerNorm -> ReLU -> n x [Linear -> LayerNorm -> ReLU] ->
Linear -> Sigmoid | ReLU(+softmax at export, train.py:144-165)) and the model
cards docs/models/alexa.md:11-36 (1536-64-64-1, LayerNorm) and
docs/models/timers.md:9-34 (3264-128-128-7, no LayerNorm, softmax).
A head is {"n_in": frames, "layers": [{"W":[in,out], "b":[out], "ln":(g,b)|None}],
"final": "sigmoid"|"relu_softmax"|"softmax"|"none"}.
"""
import numpy as np

LN_EPS = 1e-5


def forward(head, feats, dtype=np.float32):
    """feats [N, n_in, 96] -> [N, n_out].  A gated pair {"main", "verifier", "threshold"} (the released hey_jarvis graph,
    docs/models/hey_jarvis.md:9,38: the verifier "only predict[s] on audio frames that have a score > 0.5 from the first
    model", the routing being part of the exported graph) evaluates both networks and takes the verifier's score where
    the main score exceeds the threshold."""
    if "verifier" in head:
        p1 = forward(head["main"], feats, dtype)
        p2 = forward(head["verifier"], feats, dtype)
        return np.where(p1 > np.float32(head["threshold"]), p2, p1).astype(np.float32)
    x = np.asarray(feats, dtype=np.float32).reshape(feats.shape[0], -1).astype(dtype)
    L = head["layers"]
    for i, lay in enumerate(L):
        x = x @ lay["W"].astype(dtype) + lay["b"].astype(dtype)
        last = i == len(L) - 1
        if not last:
            if lay.get("ln") is not None:
                g, b = lay["ln"]
                mu = x.mean(axis=1, keepdims=True)
                var = ((x - mu) ** 2).mean(axis=1, keepdims=True)
                x = (x - mu) / np.sqrt(var + dtype(LN_EPS)) * g.astype(dtype) + b.astype(dtype)
            x = np.maximum(x, 0)
    fin = head["final"]
    if fin == "relu":
        x = np.maximum(x, 0)
    elif fin == "sigmoid":
        x = 1.0 / (1.0 + np.exp(-x))
    elif fin in ("relu_softmax", "softmax"):
        if fin == "relu_softmax":
            x = np.maximum(x, 0)
        x = x - x.max(axis=1, keepdims=True)
        e = np.exp(x)
        x = e / e.sum(axis=1, keepdims=True)
    return x.astype(np.float32)
