"""Cost of training verifiers on the GPU (oww_fit_verifiers, csrc/verifier_fit.cu) and of a whole batched enrollment.

    python scripts/verifier_fit_cost.py [--out result.json]

- fit: U in {1, 64, 1024, 8192} users x ~700 windows at n_in 16 (D = 1536), and at U = 1024 a sweep of n_u; device time
  by CUDA events around the call, median of 5 after 2 warm-up calls; the bytes of ONE pass over the users' windows
  (n_u * D * 4) and of the fixed work (statistics: 2 passes), and the Newton iterations, from the shapes and outputs;
- enrollment: Model.train_custom_verifiers for 1024 streams (bulk capture + fit + load), host clock around the call
  after one warm-up call;
- scikit-learn's LogisticRegression(C=0.001) pipeline fit per user on the host cores (a CPU number), 3 users of 700;
- the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def fit_case(ctx, torch, U, n_mean, n_in=16, seed=0):
    rng = np.random.default_rng(seed)
    R = max(4096, U * 64)
    rows = torch.from_numpy(rng.normal(0, 1, (R, 96)).astype(np.float32)).cuda()
    n_u = np.clip(rng.normal(n_mean, n_mean * 0.2, U).astype(np.int64), 2, None)
    off = np.concatenate([[0], np.cumsum(n_u)]).astype(np.int64)
    first = torch.from_numpy(rng.integers(0, R - n_in + 1, int(off[-1])).astype(np.int64)).cuda()
    lab = (rng.uniform(0, 1, int(off[-1])) < 0.3).astype(np.uint8)
    lab[off[:-1]] = 1
    lab[off[:-1] + 1] = 0
    lab = torch.from_numpy(lab).cuda()
    for _ in range(2):
        out = ctx.fit_verifiers(rows, n_in, first, off, lab)
    ms = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = ctx.fit_verifiers(rows, n_in, first, off, lab)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    D = n_in * 96
    return {"users": U, "windows": int(off[-1]), "mean_n_u": float(n_u.mean()), "ms": float(np.median(ms)),
            "bytes_one_pass": int(off[-1]) * D * 4, "newton_iters_mean": float(out["iters"].float().mean()),
            "status_counts": np.unique(out["status"].cpu().numpy(), return_counts=True)[1].tolist()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    from openwakeword_b200 import _native, Model, weights as W
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    ctx = _native.Context(device=0, cnn_mode=_native.CNN_FP32_WINDOW, max_chunks=1)
    res = {"gpu": gpu, "fit": [fit_case(ctx, torch, U, 700) for U in (1, 64, 1024, 8192)],
           "fit_sweep_n_u": [fit_case(ctx, torch, 1024, n) for n in (100, 300, 1500, 3000)]}

    rng = np.random.default_rng(1)
    B = 1024
    h = W.synthetic_head(seed=1)
    h["layers"][-1]["b"] = h["layers"][-1]["b"] + np.float32(4.0)     # scores above 0.5: positives are captured
    m = Model(wakeword_models=[{"name": "alexa", "head": h}], embedding_model_path=W.synthetic_embedding(0),
              n_streams=B, feature_init=rng.normal(0, 1, (41, 96)).astype(np.float32))
    clip = lambda n: np.clip(rng.normal(0, 3000, n), -32768, 32767).astype(np.int16)   # noqa: E731
    users = {b: ([clip(32000)], [clip(48000)]) for b in range(B)}
    m.train_custom_verifiers("alexa", dict(list(users.items())[:8]))
    torch.cuda.synchronize()
    t = time.perf_counter()
    st = m.train_custom_verifiers("alexa", users)
    torch.cuda.synchronize()
    res["enroll_1024"] = {"s": time.perf_counter() - t, "positive_s_per_user": 2.0, "negative_s_per_user": 3.0,
                          "status_counts": np.unique([s for _, s in st.values()], return_counts=True)[1].tolist()}

    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import FunctionTransformer, StandardScaler
    from openwakeword_b200.custom_verifier_model import flatten_features
    cpu = []
    for _ in range(3):
        x = rng.normal(0, 1, (700, 16, 96)).astype(np.float32)
        y = (rng.uniform(0, 1, 700) < 0.3).astype(int)
        t = time.perf_counter()
        make_pipeline(FunctionTransformer(flatten_features), StandardScaler(),
                      LogisticRegression(random_state=0, max_iter=2000, C=0.001)).fit(x, y)
        cpu.append(time.perf_counter() - t)
    res["sklearn_cpu_s_per_user"] = {"median": float(np.median(cpu)), "cores": os.cpu_count(), "kind": "CPU"}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
