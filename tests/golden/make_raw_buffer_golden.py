"""Generate tests/golden/raw_buffer.npz by running the UNMODIFIED reference ``AudioFeatures``.

Needs a checkout of the original openWakeWord project (OWW_REFERENCE = its root directory):
    OWW_REFERENCE=/path/to/openWakeWord python tests/golden/make_raw_buffer_golden.py
Its ``openwakeword.utils.AudioFeatures`` is imported with ``oracle.ref_stub_ort`` standing in for onnxruntime (as in
make_golden.py) and fed one seeded int16 signal in a fixed sequence of call lengths: sub-chunk calls, non-multiples of
1280, multi-chunk calls, calls longer than 8 chunks (AudioFeatures' default max_chunks), a ``reset()``, and enough audio
after it for the 10 s ``raw_data_buffer`` (deque(maxlen=160000)) to wrap.  After every call the buffer is checked to be
one contiguous slice of the signal, and the slice bounds are stored with the call's return value:
    signal   int16 [S]        the audio, consumed in order
    calls    int64 [C]        samples of each call, -1 = reset()
    ret      int64 [C]        what the call returned (-1 for a reset)
    raw_lo, raw_hi  int64 [C] raw_data_buffer after the call == signal[raw_lo:raw_hi]
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from openwakeword_b200 import weights as W          # noqa: E402
from oracle import ref_stub_ort                     # noqa: E402

EMB_SEED = 0
SIGNAL_SEED = 11
CALLS = ([5, 400, 1000, 2559, 3000, 1280, 5120, 3840, 12800, 700, 0, 1275, 5]
         + [-1]                                                   # reset()
         + [3000, 100, 1180, 2559, 20000] + [10000] * 13 + [5, 1275, 2560, 1279, 1, 640, 9000, 777])


def main():
    ref_stub_ort.install(W.synthetic_embedding(EMB_SEED), {})
    sys.path.insert(0, os.environ["OWW_REFERENCE"])
    from openwakeword.utils import AudioFeatures     # the reference, unmodified

    tmp = tempfile.mkdtemp()
    paths = {k: os.path.join(tmp, k + ".onnx") for k in ("melspectrogram", "embedding_model")}
    for p in paths.values():
        open(p, "w").close()
    np.random.seed(0)
    af = AudioFeatures(melspec_model_path=paths["melspectrogram"], embedding_model_path=paths["embedding_model"],
                       inference_framework="onnx")
    S = sum(c for c in CALLS if c > 0)
    signal = np.random.default_rng(SIGNAL_SEED).integers(-2000, 2000, S).astype(np.int16)
    off = 0
    ret, lo, hi = [], [], []
    for c in CALLS:
        if c < 0:
            af.reset()
            ret.append(-1)
        else:
            ret.append(int(af(signal[off:off + c])))
            off += c
        buf = np.array(list(af.raw_data_buffer), np.int16)
        # the buffer ends at some position e <= off of the signal: find it (the samples held back are not in it)
        for e in range(off, off - 1280, -1):
            if e >= buf.size and np.array_equal(signal[e - buf.size:e], buf):
                break
        else:
            raise AssertionError(f"raw_data_buffer after call {len(ret) - 1} is not a slice of the signal")
        lo.append(e - buf.size)
        hi.append(e)
    assert max(h - l for l, h in zip(lo, hi)) == 160000, "the deque must wrap"
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "raw_buffer.npz")
    np.savez_compressed(out, signal=signal, calls=np.array(CALLS, np.int64), ret=np.array(ret, np.int64),
                        raw_lo=np.array(lo, np.int64), raw_hi=np.array(hi, np.int64))
    print("wrote", out, "calls", len(CALLS), "samples", S)


if __name__ == "__main__":
    main()
