#!/usr/bin/env python
"""Mixed-length bulk prediction on one GPU: one ragged device call (oww_predict_clips_ragged) against the strategy
bulk_predict used before it, one predict_clips call per distinct clip length.

Workload: 20 000 seeded clips with lengths uniform over 0.5-4 s, 1 s padding, 1280-sample calls, the six-head set of
scripts/bench_configs.py (C5).  Both ways start from clips resident on the device and leave the scores there; times are
CUDA events around the device calls after a warm-up run.  Nearly every length is distinct, so the per-length strategy is
timed on the first --per-length-clips clips and reported as a rate.

--parent DIR: also time the equal-length device-only C5 share (bench_configs.c5's last part: 25 000 x 2 s clips, one
oww_predict_clips call) with this tree's library and with the library of the tree at DIR (the parent commit, built),
alternating the two in subprocesses, and report every run.  Prints one JSON object."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

EQUAL_SNIPPET = r"""
import json, sys
import numpy as np, torch
sys.path.insert(0, '.')
from openwakeword_b200 import Model
from scripts.bench_configs import heads6
m = Model(wakeword_models=[{"name": f"h{i}", "head": h} for i, h in enumerate(heads6())], embedding_model_path="synthetic:0",
          feature_init=np.zeros((41, 96), np.float32), cnn_mode=3)
N, S = 25000, 32000
d = torch.from_numpy(np.random.default_rng(2).integers(-2000, 2000, (N, S)).astype(np.int16)).cuda()
steps = len(range(0, S + 32000 - 1280, 1280))
raw = torch.zeros((N, steps, m._n_cols), dtype=torch.float32, device="cuda")
fi = np.zeros((41, 96), np.float32)
st = torch.cuda.current_stream().cuda_stream
m.preprocessor.ctx.predict_clips(d, N, S, 16000, fi, raw, st)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
ts = []
for _ in range(3):
    torch.cuda.synchronize(); e0.record()
    m.preprocessor.ctx.predict_clips(d, N, S, 16000, fi, raw, st)
    e1.record(); torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1) * 1e-3)
print(json.dumps({"seconds": ts, "clips_per_s": N / min(ts), "checksum": float(raw.double().sum())}))
"""


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                                    # the query is informational
        return {"gpu": "unknown", "error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=20000)
    ap.add_argument("--per-length-clips", type=int, default=1000)
    ap.add_argument("--parent", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch
    from openwakeword_b200 import Model, _native
    from scripts.bench_configs import heads6

    out = gpu_info()
    m = Model(wakeword_models=[{"name": f"h{i}", "head": h} for i, h in enumerate(heads6())],
              embedding_model_path="synthetic:0", feature_init=np.zeros((41, 96), np.float32), cnn_mode=3)
    ctx, fi, pad = m.preprocessor.ctx, np.zeros((41, 96), np.float32), 16000
    rng = np.random.default_rng(0)
    lens = rng.integers(8000, 64001, args.clips)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    pcm = torch.from_numpy(rng.integers(-2000, 2000, int(off[-1])).astype(np.int16)).cuda()
    calls = np.array([len(range(0, int(n) + 2 * pad - 1280, 1280)) for n in lens])
    rows = int(calls.sum())
    n_slabs, computed, needed = _native.clip_slab_plan(calls.astype(np.int32))
    out["slab_plan"] = {"slabs": n_slabs, "steps_computed": computed, "steps_needed": needed,
                        "padded_step_fraction": computed / needed - 1}
    st = torch.cuda.current_stream().cuda_stream
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    # one ragged call over every clip
    raw = torch.zeros((rows, m._n_cols), dtype=torch.float32, device="cuda")
    stepped = torch.zeros(rows, dtype=torch.uint8, device="cuda")
    ctx.predict_clips_ragged(pcm, off, pad, 1280, fi, raw, stepped, None, st)       # warm-up
    ts = []
    for _ in range(args.rounds):
        torch.cuda.synchronize(); e0.record()
        ctx.predict_clips_ragged(pcm, off, pad, 1280, fi, raw, stepped, None, st)
        e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3)
    t = min(ts)
    out["ragged"] = {"clips": args.clips, "seconds": ts, "clips_per_s": args.clips / t, "frames_per_s": rows / t}

    # one predict_clips call per distinct length (what bulk_predict grouped by before)
    k = min(args.per_length_clips, args.clips)
    by_len = {}
    for i in range(k):
        by_len.setdefault(int(lens[i]), []).append(i)
    groups = []
    for n, idx in by_len.items():
        d = torch.stack([pcm[off[i]:off[i + 1]] for i in idx]).contiguous()
        steps = len(range(0, n + 2 * pad - 1280, 1280))
        groups.append((d, len(idx), n, torch.zeros((len(idx), steps, m._n_cols), dtype=torch.float32, device="cuda")))
    for d, c, n, r in groups[:8]:
        ctx.predict_clips(d, c, n, pad, fi, r, st)                                    # warm-up
    torch.cuda.synchronize(); e0.record()
    for d, c, n, r in groups:
        ctx.predict_clips(d, c, n, pad, fi, r, st)
    e1.record(); torch.cuda.synchronize()
    t1 = e0.elapsed_time(e1) * 1e-3
    out["per_length"] = {"clips": k, "device_calls": len(groups), "seconds": t1, "clips_per_s": k / t1,
                         "frames_per_s": int(calls[:k].sum()) / t1}
    out["speedup_clips_per_s"] = out["ragged"]["clips_per_s"] / out["per_length"]["clips_per_s"]

    if args.parent:
        del raw, pcm, groups
        torch.cuda.empty_cache()
        runs = {"this": [], "parent": []}
        for _ in range(args.rounds):
            for tag, tree in (("parent", os.path.abspath(args.parent)), ("this", ROOT)):
                r = subprocess.run([sys.executable, "-c", EQUAL_SNIPPET], cwd=tree, capture_output=True, text=True)
                if r.returncode:
                    raise SystemExit(f"{tag} run failed:\n{r.stderr[-3000:]}")
                runs[tag].append(json.loads(r.stdout.strip().splitlines()[-1]))
        out["equal_length_c5_device"] = {
            tag: {"clips_per_s": [x["clips_per_s"] for x in v], "checksum": v[0]["checksum"]} for tag, v in runs.items()}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
