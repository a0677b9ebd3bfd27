"""Device cost of a per-stream head bank on the C3 workload (8192 streams x 7 head networks, cnn_mode 3, one chunk per
step, device-resident PCM, StreamEngine without Model), in device milliseconds per step (CUDA events around `--steps`
steps after `--warmup`):

  - no bank, and a bank of 8 slots against the same 8 heads added as ordinary heads (7 + 8 <= 16), alternated;
  - one bank of 16x96 -> 64 -> 64 -> 1 and one of 16x96 -> 128 -> 128 -> 1, each with D in {1, 16, 128, 1024, 8192}
    slots on a seeded uniform assignment of the streams;
  - per configuration the bytes of the slot weights a step reads (computed from the shapes: every used slot once), and
    those bytes over the step time added to the no-bank step, as a share of the H100 SXM data-sheet 3.35 TB/s;
  - --profile (a separate run): torch.profiler device time per kernel and step for the bank configurations.

Prints the card name, power limit and SM clock read in the same run, then every result as one JSON line; --json PATH
also writes that record to PATH.
python scripts/head_bank_cost.py [--streams 8192] [--profile] [--json PATH]"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_TBS = 3.35


def slot_bytes(n_in, hidden, n_blocks=1, n_out=1):
    """bytes of one slot a step reads: fp16 hi/lo packing of every layer (128-byte blocks) + fp32 biases / LayerNorm"""
    np_ = lambda d: (d + 15) & ~15
    r = lambda b: (b + 127) & ~127
    w = r(n_in * 96 * np_(hidden) * 4)
    for _ in range(n_blocks):
        w += r(np_(hidden) * np_(hidden) * 4)
    w += r(np_(hidden) * np_(n_out) * 4)
    p = (1 + n_blocks) * 3 * ((hidden + 3) & ~3) + ((n_out + 3) & ~3)
    return w + 4 * p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--ds", default="1,16,128,1024,8192")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    from openwakeword_b200 import weights as W
    from openwakeword_b200.engine import StreamEngine
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"card (name, power limit, SM clock, max SM clock): {smi or torch.cuda.get_device_name(0)}", flush=True)

    B = args.streams
    heads = list(bench.bench_heads("c3").values())
    rng = np.random.default_rng(0)
    pcm = torch.from_numpy(np.clip(rng.normal(0, 3000, (B, 1280 * 8)), -32768, 32767).astype(np.int16)).cuda()
    pool = {h: [W.synthetic_head(hidden=h, seed=300 + i) for i in range(32)] for h in (64, 128)}

    def engine(extra=(), hidden=None, D=0):
        eng = StreamEngine(list(heads) + list(extra), B, embedding="synthetic:0", max_chunks=1, cnn_mode=3)
        used = 0
        if D:
            bank, _, _ = eng.add_head_bank(pool[hidden][0], D)
            for k in range(D):             # D distinct slots (contents cycle through the pool)
                eng.load_bank_head(bank, k, pool[hidden][k % len(pool[hidden])])
            slots = np.random.default_rng(D).integers(0, D, B).astype(np.int32)
            used = int(np.unique(slots).size)
            eng.assign_bank_head(bank, slots)
        torch.cuda.synchronize()
        return eng, used

    def time_ms(eng, steps):
        out = torch.empty((B, eng.n_cols), dtype=torch.float32, device="cuda")
        for i in range(args.warmup):
            eng.step(pcm[:, (i % 8) * 1280:(i % 8 + 1) * 1280], out=out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            eng.step(pcm[:, (i % 8) * 1280:(i % 8 + 1) * 1280], out=out)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    res = {"card": smi, "streams": B, "steps": args.steps, "rows": []}
    if args.profile:
        from torch.profiler import profile, ProfilerActivity
        for hidden, D in ((64, 1024), (64, 8192), (128, 8192)):
            eng, used = engine(hidden=hidden, D=D)
            time_ms(eng, 5)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for i in range(20):
                    eng.step(pcm[:, (i % 8) * 1280:(i % 8 + 1) * 1280])
                torch.cuda.synchronize()
            rows = {}
            for ev in prof.key_averages():
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                if t > 0:
                    rows[ev.key[:90]] = t / 20
            print(f"--- profile hidden {hidden} D {D} ({used} slots used): device us per step")
            for k, v in sorted(rows.items(), key=lambda kv: -kv[1])[:8]:
                print(f"  {v:9.1f}  {k}")
            res["rows"].append({"profile": f"hidden {hidden} D {D}", "us_per_step": rows})
            del eng
            torch.cuda.empty_cache()
    else:
        # baselines, alternated in one process: no bank | bank of 8 slots | the same 8 heads as ordinary heads
        eights = pool[64][:8]
        base = {"no bank": engine()[0], "bank D=8": engine(hidden=64, D=8)[0], "8 ordinary heads": engine(extra=eights)[0]}
        times = {k: [] for k in base}
        for rnd in range(3):
            for k, eng in base.items():
                times[k].append(time_ms(eng, args.steps))
        for k, v in times.items():
            print(f"{k:18s} ms/step: " + " ".join(f"{t:.4f}" for t in v), flush=True)
            res["rows"].append({"config": k, "ms_per_step": v})
        t0 = min(times["no bank"])
        del base
        torch.cuda.empty_cache()
        for hidden in (64, 128):
            for D in [int(x) for x in args.ds.split(",")]:
                eng, used = engine(hidden=hidden, D=D)
                t = min(time_ms(eng, args.steps) for _ in range(2))
                nbytes = used * slot_bytes(16, hidden)
                extra = t - t0
                share = nbytes / (extra * 1e-3) / (HBM_TBS * 1e12) if extra > 0 else float("nan")
                print(f"hidden {hidden:3d} D {D:5d} ({used:5d} used): {t:.4f} ms/step (+{extra:.4f}), "
                      f"{nbytes / 1e6:8.1f} MB of slot weights, {100 * share:5.1f} % of 3.35 TB/s over the added time",
                      flush=True)
                res["rows"].append({"hidden": hidden, "D": D, "used": used, "ms_per_step": t, "added_ms": extra,
                                    "slot_mb": nbytes / 1e6, "share_of_hbm": share})
                del eng
                torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
