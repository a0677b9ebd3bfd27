"""Fused step kernel, several trees side by side on one GPU: python scripts/compare_fused.py OUT_DIR REPS TREE [TREE ...]

1. bench.py --gpus 1 in each tree, the trees alternated REPS times, with --dump-outputs so that the scores of the last
   timed step of every tree can be compared with the first tree's (same seeded inputs);
2. torch.profiler (CUDA activities, a run of its own per tree): device time per step of each kernel at 8192 streams x 7
   networks, the fused kernel tc_inc_kernel<11> among them;
3. phase clocks (scripts/clocks_tree.py) at 8192 and 1024 streams, split_from 11.
Each tree must have been built (python __graft_entry__.py) beforehand.  The card's name, power limit and maximum SM
clock come first in the output; everything is also written under OUT_DIR."""
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))

PROFILE = r'''
import os, sys, json
tree = os.path.abspath(sys.argv[1]); sys.path.insert(0, tree)
import numpy as np, torch
from torch.profiler import profile, ProfilerActivity
from openwakeword_b200.engine import StreamEngine
from openwakeword_b200 import weights as W
B, steps = 8192, 20
eng = StreamEngine([W.synthetic_head(seed=s) for s in range(7)], B, cnn_mode=3)
rng = np.random.default_rng(0)
pcm = [rng.integers(-1000, 1000, (B, 1280)).astype(np.int16) for _ in range(4)]
for i in range(10):
    eng.step_host(pcm[i % 4], 1)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for i in range(steps):
        eng.step_host(pcm[i % 4], 1)
    torch.cuda.synchronize()
rows = sorted(((e.key, e.self_device_time_total / steps) for e in prof.key_averages()), key=lambda kv: -kv[1])
print(json.dumps({k[:60]: round(v, 1) for k, v in rows[:8]}))
'''


def run(cmd, cwd=None, stdout_only=False):
    r = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True)
    return r.stdout if stdout_only and r.stdout.strip() else r.stdout + r.stderr


def main():
    out, reps, trees = os.path.abspath(sys.argv[1]), int(sys.argv[2]), [os.path.abspath(p) for p in sys.argv[3:]]
    tags = [os.path.basename(t) or t for t in trees]
    os.makedirs(out, exist_ok=True)
    print(run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]).strip(), flush=True)
    with open(os.path.join(out, "bench.jsonl"), "w") as f:
        for rep in range(reps):
            for tag, tree in zip(tags, trees):
                txt = run([sys.executable, "bench.py", "--gpus", "1", "--dump-outputs", os.path.join(out, f"dump_{tag}_{rep}")], cwd=tree)
                res = [l for l in txt.splitlines() if l.startswith("{")]
                r = json.loads(res[-1]) if res else None
                f.write(json.dumps({"tree": tag, "rep": rep, "result": r if r else txt[-2000:]}) + "\n")
                if r:
                    c2, v = r["secondary"]["c2"], {x["split_from"]: x["value"] for x in r.get("variants", [])}
                    print(f"bench {tag} rep {rep}: value {r['value'] / 1e6:.3f} M  cnn {r['roofline']['stage_ms']['cnn']:.4f} ms  "
                          f"c2 {c2['value'] / 1e6:.3f} M  split15 {v.get(15, 0) / 1e6:.3f} M  split20 {v.get(20, 0) / 1e6:.3f} M", flush=True)
                else:
                    print(f"bench {tag} rep {rep}: no result line\n{txt[-2000:]}", flush=True)
    # scores of the last timed step: every tree against the first, every workload and run
    import numpy as np
    for rep in range(reps):
        d0 = os.path.join(out, f"dump_{tags[0]}_{rep}")
        for tag in tags[1:]:
            d1 = os.path.join(out, f"dump_{tag}_{rep}")
            for fn in sorted(os.listdir(d0)) if os.path.isdir(d0) else []:
                a, b = np.load(os.path.join(d0, fn)), np.load(os.path.join(d1, fn))
                print(f"outputs rep {rep} {tag} vs {tags[0]} {fn}: identical={np.array_equal(a, b)} "
                      f"max|diff|={float(np.abs(a - b).max()):.3e}", flush=True)
    for tag, tree in zip(tags, trees):
        print("profile", tag, "us/step:", run([sys.executable, "-c", PROFILE, tree], stdout_only=True).strip().splitlines()[-1], flush=True)
    for tag, tree in zip(tags, trees):
        for b in (8192, 1024):
            print(run([sys.executable, os.path.join(HERE, "clocks_tree.py"), tree, str(b), "11"]), flush=True)


if __name__ == "__main__":
    main()
