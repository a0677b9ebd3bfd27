"""A stand-in ``onnxruntime`` whose sessions evaluate this oracle's graphs.

Used ONLY in the build container by tests/golden/make_golden.py: it lets the
*unmodified reference plumbing* (openwakeword/model.py,
utils.py) run end to end although neither onnxruntime nor the released .onnx
files exist here (SURVEY.md F2-F4).  The ORT surface emulated is exactly what
the reference touches (utils.py:79-93; model.py:149-157): SessionOptions,
InferenceSession(path, sess_options, providers).run/get_inputs/get_outputs/
get_providers.  Sessions are chosen by file basename: ``melspectrogram*`` ->
oracle.mel, ``embedding_model*`` -> oracle.embedding, anything else -> a head
registered in ``HEADS[basename-without-extension]``.
"""
import os
import sys
import types
import numpy as np
from . import mel as _mel, embedding as _emb, heads as _heads

EMBEDDING_WEIGHTS = {}
HEADS = {}
CALLS = []


class _IO:
    def __init__(self, name, shape):
        self.name, self.shape = name, shape


class SessionOptions:
    inter_op_num_threads = 1
    intra_op_num_threads = 1


class InferenceSession:
    def __init__(self, path, sess_options=None, providers=None):
        base = os.path.splitext(os.path.basename(path))[0]
        self.kind = "mel" if base.startswith("melspectrogram") else \
            "emb" if base.startswith("embedding_model") else "head"
        self.base = base
        if self.kind == "head":
            self.head = HEADS[base]

    def get_providers(self):
        return ["CPUExecutionProvider"]

    def get_inputs(self):
        if self.kind == "mel":
            return [_IO("input", ["batch", "samples"])]
        if self.kind == "emb":
            return [_IO("input_1", ["batch", 76, 32, 1])]
        return [_IO("onnx::Flatten_0", [1, self.head["n_in"], 96])]

    def get_outputs(self):
        if self.kind == "head":
            net = self.head["main"] if "verifier" in self.head else self.head
            return [_IO("out", [1, net["layers"][-1]["W"].shape[1]])]
        return [_IO("output", [])]

    def run(self, _names, feed):
        (x,) = feed.values()
        x = np.asarray(x)
        CALLS.append((self.kind, x.shape))
        if self.kind == "mel":
            if x.dtype != np.float32:
                raise TypeError("melspectrogram.onnx takes float32")
            raws = []
            for row in x:      # global max over the whole output tensor, as the graph does
                T = _mel.n_frames(row.shape[0])
                cr, ci, mw = _mel._consts(np.float32)
                idx = np.arange(T)[:, None] * _mel.HOP + np.arange(_mel.N_FFT)[None, :]
                fr = row[idx]
                p = (fr @ cr) ** 2 + (fr @ ci) ** 2
                raws.append(np.float32(10.0) * np.log(np.maximum(p @ mw, np.float32(1e-10))) / np.log(np.float32(10.0)))
            ls = np.stack(raws)
            ls = np.maximum(ls, ls.max() - np.float32(80.0))
            return [ls[:, None].astype(np.float32)]
        if self.kind == "emb":
            if x.dtype != np.float32 or x.shape[1:] != (76, 32, 1):
                raise TypeError("embedding_model.onnx takes float32 [N,76,32,1]")
            return [_emb.embed_windows(EMBEDDING_WEIGHTS["w"], x[..., 0])[:, None, None, :]]
        if x.dtype != np.float32:
            raise TypeError("head takes float32")
        return [_heads.forward(self.head, x)]


def install(emb_weights, heads):
    """Register weights and put this module in sys.modules as ``onnxruntime``."""
    EMBEDDING_WEIGHTS["w"] = emb_weights
    HEADS.clear()
    HEADS.update(heads)
    mod = types.ModuleType("onnxruntime")
    mod.SessionOptions = SessionOptions
    mod.InferenceSession = InferenceSession
    sys.modules["onnxruntime"] = mod
    return mod
