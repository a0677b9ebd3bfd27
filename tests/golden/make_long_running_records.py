"""Make long_running_records.npz (needs the GPU): a twin pair of stream records from one cnn_mode 0 handle.

Stream 0 steps 6 calls; its record is imported into stream 1 with the mel count set to 2^30 - 3; both step one more
chunk of the same samples, so the twin's mel count crosses 2^30 and is rebased.  Saved: both records after that step,
the twin's counts before it and after it."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main(out):
    import torch
    from helpers import emb_weights, head, mixes
    from openwakeword_b200.engine import StreamEngine
    rng = np.random.default_rng(0)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    eng = StreamEngine([head("alexa_v0.1")], 2, embedding=emb_weights(), feature_init=fi, max_chunks=1, cnn_mode=0)
    for _ in range(6):
        eng.step(torch.from_numpy(mixes(rng, 2, 1280)).cuda(), 1)
    rec = eng.export_streams([0]).cpu().numpy()
    w = rec.view(np.int32)
    w[0, 5] = (1 << 30) - 3
    before = (int(w[0, 5]), int(w[0, 6]))
    eng.import_streams([1], torch.from_numpy(rec))
    assert eng.ctx.stream_state_rejected() == 0
    x = mixes(rng, 2, 1280)
    x[1] = x[0]
    eng.step(torch.from_numpy(x).cuda(), 1)
    r = eng.export_streams([0, 1]).cpu().numpy()
    np.savez_compressed(out, ctrl=r[0], twin=r[1], twin_before=np.array(before, np.int64),
                        twin_counts=np.array(eng.ctx.get_counts(1), np.int64))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                            "long_running_records.npz"))
