"""CPU oracle for the openWakeWord streaming-inference hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``openwakeword_b200/`` imports this
package; only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` may.  It is a NumPy restatement of the
three graphs the reference executes through onnxruntime (melspectrogram.onnx,
embedding_model.onnx, <head>.onnx) plus the pure-Python streaming state machine
of ``openwakeword/model.py`` and ``openwakeword/utils.py``.

PARITY STATUS
  * state machine  : PINNED - driven against the reference's own plumbing
    (``openwakeword`` (the original project) imported with a stub ``onnxruntime`` whose
    sessions call this oracle's graph functions; ``tests/golden/make_golden.py``)
    and frozen in ``tests/golden/*.npz``.
  * graph arithmetic: PARITY UNPINNED at the onnxruntime boundary - neither
    onnxruntime nor the released ``*.onnx`` files exist in this image
    (SURVEY.md F2/F3), and the reference's tests hold no golden vectors
    (SURVEY.md section 4).  The restatement follows the export notebooks
    (file:line cited per function) and is cross-checked against independent
    implementations (torch.stft + torchaudio filterbank; torch conv2d).
"""
from . import mel, embedding, heads, streaming, probe  # noqa: F401
