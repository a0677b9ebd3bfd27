"""Cost of ragged steps (oww_step_ragged) on the bench headline workload: 8192 streams x the bench's 7 head networks,
cnn_mode 3 at its default split, max_chunks 2.  Device milliseconds per step (CUDA events around `--steps` steps after
`--warmup`, every shape warmed up) and wall-clock milliseconds per step (host clock around the same steps, ending in a
synchronise: includes the host's per-call count staging) for

  - lockstep one-chunk (oww_step(1): what bench.py measures) and lockstep two-chunk;
  - ragged all ones (dispatches to oww_step(1));
  - 10 / 50 / 90 % of the streams held (0/1 counts), and the manual alternative: a lockstep step of a handle that holds
    only the stepping streams;
  - 1 % of the streams at 2 chunks and the rest at 1, and the manual alternative: one lockstep step per distinct count
    on two handles (99 % of the streams at 1 chunk, 1 % at 2).

SM clocks and throttle reasons are sampled over the timed regions as bench.py does; the card name and power limit are
printed with the numbers.  python scripts/ragged_step_cost.py [--streams 8192]"""
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
    ap.add_argument("--profile", action="store_true",
                    help="instead: per-kernel device time (torch.profiler) of a lockstep step and of a 10 %%-held step")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    from openwakeword_b200.engine import StreamEngine
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card: {smi[0] if smi else torch.cuda.get_device_name(0)}")

    B = args.streams
    heads = list(bench.bench_heads("c3").values())
    rng = np.random.default_rng(0)
    pcm = torch.from_numpy(bench.synth_pcm_fast(B, 16, 0)).cuda()        # [B, 16*1280]
    engines = {}

    def engine(n):
        if n not in engines:
            engines[n] = StreamEngine(heads, n, embedding="synthetic:0", max_chunks=2, cnn_mode=3)
        return engines[n]

    sampler = bench.ClockSampler(0)
    sampler.start()
    windows = []

    def timed(calls):
        """calls: list of (engine, fn(engine, i)) run in order each step."""
        for i in range(args.warmup):
            for eng, fn in calls:
                fn(eng, i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        for i in range(args.steps):
            for eng, fn in calls:
                fn(eng, i)
        e1.record()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        windows.append((t0, t1))
        return e0.elapsed_time(e1) / args.steps, 1e3 * (t1 - t0) / args.steps

    def x(i, n, src=None):
        """the i-th call's n chunks of every row of src (default: all streams); sub-batches are gathered once, untimed"""
        s = (i % (16 // n)) * n * 1280
        return (pcm if src is None else src)[:, s:s + n * 1280]

    outs = {}

    def out(eng):
        """one preallocated score buffer per handle: no allocation or fill inside the timed steps"""
        if id(eng) not in outs:
            outs[id(eng)] = torch.empty((eng.n_streams, eng.n_cols), dtype=torch.float32, device="cuda")
        return outs[id(eng)]

    def lock(n):
        return lambda eng, i: eng.step(x(i, n), n, out=out(eng))

    def ragged(counts):
        return lambda eng, i: eng.step_ragged(x(i, 2), counts, out=out(eng))

    full = engine(B)
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        c = (rng.random(B) >= 0.1).astype(np.int32)
        for name, fn in (("lockstep 1 chunk", lock(1)), ("ragged, 10 % held", ragged(c))):
            for i in range(args.warmup):
                fn(full, i)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for i in range(20):
                    fn(full, i)
                torch.cuda.synchronize()
            print(f"{name}: per-kernel device time over 20 steps (programmatic dependent launches overlap a kernel's "
                  "prologue with its predecessor, so the times of the small kernels include waiting)")
            print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=16, max_name_column_width=48))
        return
    res = {}
    res["lockstep 1 chunk"] = timed([(full, lock(1))])
    res["lockstep 2 chunks"] = timed([(full, lock(2))])
    res["ragged, all 1"] = timed([(full, ragged(np.ones(B, np.int32)))])
    for frac in (0.1, 0.5, 0.9):
        held = rng.random(B) < frac
        c = (~held).astype(np.int32)
        res[f"ragged, {int(frac * 100)} % held"] = timed([(full, ragged(c))])
        m = int(c.sum())
        sub = engine(m)
        src = pcm[torch.from_numpy(np.nonzero(c)[0]).cuda()]
        res[f"manual, {int(frac * 100)} % held: lockstep step of the {m} stepping streams"] = \
            timed([(sub, lambda eng, i, p=src: eng.step(x(i, 1, p), 1, out=out(eng)))])
        outs.pop(id(engines.pop(m)), None)
        torch.cuda.empty_cache()
    two = rng.random(B) < 0.01
    c = np.where(two, 2, 1).astype(np.int32)
    res["ragged, 1 % at 2 chunks, rest 1"] = timed([(full, ragged(c))])
    n2 = int(two.sum())
    p1, p2 = (pcm[torch.from_numpy(np.nonzero(v)[0]).cuda()] for v in (~two, two))
    e1, e2 = engine(B - n2), engine(n2)
    res[f"manual, 1 % at 2 chunks: lockstep steps of {B - n2} x 1 and {n2} x 2 chunks"] = \
        timed([(e1, lambda eng, i: eng.step(x(i, 1, p1), 1, out=out(eng))), (e2, lambda eng, i: eng.step(x(i, 2, p2), 2, out=out(eng)))])
    clocks = sampler.stop(windows)
    for k, (dev, wall) in res.items():
        print(f"{k:>72}: {dev:.3f} ms/step device, {wall:.3f} ms/step wall ({B} streams)")
    print(f"clocks: {clocks}")


if __name__ == "__main__":
    main()
