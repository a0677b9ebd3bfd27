"""Device cost of custom verifier banks on the bench headline workload (8192 streams x 7 head networks, cnn_mode 3,
one chunk per step), in device milliseconds per step (CUDA events around `--steps` steps after `--warmup`):

  - no bank (what bench.py measures);
  - a bank on the first head with one distinct verifier per stream at threshold 0: every stream is verified;
  - the same at threshold 0.5, with the fraction of streams verified;
  - the host path it replaces (per verified stream oww_get_features + scikit-learn predict_proba) for a few steps, at
    the same threshold 0.5, as wall-clock ms per step.

Prints the card name and power limit with the numbers.  python scripts/verifier_cost.py [--streams 8192]"""
import argparse
import importlib.util
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--host-steps", type=int, default=3)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    from openwakeword_b200.engine import StreamEngine
    from openwakeword_b200.custom_verifier_model import flatten_features
    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import FunctionTransformer, StandardScaler
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card: {smi[0] if smi else torch.cuda.get_device_name(0)}")

    B = args.streams
    heads = list(bench.bench_heads("c3").values())
    rng = np.random.default_rng(0)
    pcm = torch.from_numpy(np.clip(rng.normal(0, 3000, (B, 1280 * 8)), -32768, 32767).astype(np.int16)).cuda()
    n_in = heads[0]["n_in"] if "n_in" in heads[0] else 16
    D = n_in * 96

    def engine(thr):
        eng = StreamEngine(heads, B, embedding="synthetic:0", max_chunks=1, cnn_mode=3)
        if thr is not None:
            bank = eng.add_verifier_bank(0, B, thr)
            for s in range(B):           # distinct verifiers: every verified stream reads its own mean and weight rows
                eng.load_verifier(bank, s, (rng.normal(0, 1, D).astype(np.float32), rng.normal(0, 0.01, D).astype(np.float32),
                                            float(rng.normal())))
            eng.assign_verifier(bank, np.arange(B, dtype=np.int32))
            torch.cuda.synchronize()
        return eng

    def timed(eng):
        for i in range(args.warmup):
            eng.step(pcm[:, (i % 8) * 1280:(i % 8 + 1) * 1280])
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for i in range(args.steps):
            out = eng.step(pcm[:, (i % 8) * 1280:(i % 8 + 1) * 1280])
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps, out.cpu().numpy()

    res = {}
    plain = engine(None)
    res["no bank"], raw = timed(plain)
    frac = float((raw[:, 0] >= np.float32(0.5)).mean())
    del plain
    for thr in (0.0, 0.5):
        eng = engine(thr)
        res[f"threshold {thr}"], _ = timed(eng)
        del eng
        torch.cuda.empty_cache()
    for k, v in res.items():
        print(f"{k:>16}: {v:.3f} ms/step (device, {B} streams)")
    print(f"fraction of streams verified at threshold 0.5: {frac:.3f} (last timed step, first head)")

    # host path: the step, then one get_features + predict_proba per stream at or above the threshold
    x = rng.normal(0, 1, (60, n_in, 96)).astype(np.float32)
    pipe = make_pipeline(FunctionTransformer(flatten_features), StandardScaler(),
                         LogisticRegression(C=0.001, max_iter=2000)).fit(x, np.arange(60) % 2)
    eng = StreamEngine(heads, B, embedding="synthetic:0", max_chunks=1, cnn_mode=3)
    for i in range(args.warmup):
        eng.step(pcm[:, (i % 8) * 1280:(i % 8 + 1) * 1280])
    torch.cuda.synchronize()
    t, n_ver = [], 0
    for i in range(args.host_steps):
        t0 = time.perf_counter()
        out = eng.step(pcm[:, (i % 8) * 1280:(i % 8 + 1) * 1280]).cpu().numpy()
        for b in np.nonzero(out[:, 0] >= np.float32(0.5))[0]:
            out[b, 0] = pipe.predict_proba(eng.ctx.get_features(int(b), n_in)[None])[0, -1]
            n_ver += 1
        t.append(time.perf_counter() - t0)
    print(f"host path, threshold 0.5: {1e3 * np.mean(t):.1f} ms/step wall clock ({n_ver / args.host_steps:.0f} verified "
          f"streams per step, {args.host_steps} steps)")


if __name__ == "__main__":
    main()
