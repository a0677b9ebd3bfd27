"""What device ingest (oww_set_input_rates / oww_ingest, csrc/ingest.cu) costs, on the bench headline configuration C3:
8192 streams x the bench's 7 head networks, cnn_mode 3, max_chunks 2, 80 ms packets.

Engine arms, alternated `--rounds` times, `--steps` calls after `--warmup`, CUDA events around the calls:
  16 kHz step_ragged:  device PCM, one chunk per stream (what a server that resamples elsewhere would run);
  ingest at 48000, 44100 and 8000 Hz:  one packed device buffer of every stream's 80 ms packet per call.
Then a separate torch.profiler pass that records resample_kernel's device time per rate, with the bytes it has to move
(input and output int16) set against the data sheet's 3.35 TB/s for an H100 SXM (a figure for a 700 W card, not a
measured peak).
Model arms (`--model-steps` calls each, wall clock, alternated): Model(sr=48000).predict_ragged on host 48 kHz packets,
against scipy.signal.resample_poly on each packet on the host followed by a 16 kHz Model.predict_ragged - what the
reference's server example does.  Card name, power limit and SM clock are printed with the numbers.  No GPU: it fails.

python scripts/ingest_cost.py [--streams 8192]"""
import argparse
import importlib.util
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
DATA_SHEET_BYTES_PER_S = 3.35e12
CHUNK = 1280


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--model-steps", type=int, default=5)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    from openwakeword_b200 import Model
    from openwakeword_b200.engine import StreamEngine
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)

    def card():
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name(0)

    print(f"card, power limit, SM clock now, SM clock max: {card()}")
    B = args.streams
    heads = bench.bench_heads("c3")
    eng = StreamEngine(list(heads.values()), B, embedding="synthetic:0", max_chunks=2, cnn_mode=3)
    pcm = torch.from_numpy(bench.synth_pcm_fast(B, 16, 0)).cuda()              # int16 [B, 16*1280] on the device
    out = torch.empty((B, eng.n_cols), dtype=torch.float32, device="cuda")
    ones = np.ones(B, np.int32)
    rng = np.random.default_rng(0)
    packets = {}
    for r in (48000, 44100, 8000):
        n = r * 8 // 100
        packets[r] = [torch.from_numpy(rng.integers(-8000, 8000, B * n).astype(np.int16)).cuda() for _ in range(4)]
    offsets = {r: np.arange(B + 1, dtype=np.int64) * (r * 8 // 100) for r in packets}
    eng.set_input_rates(16000)                                              # allocates the ingest state once

    def ragged16(i):
        eng.step_ragged(pcm[:, (i % 16) * CHUNK:], ones, out)

    def ingest(rate):
        def fn(i):
            eng.ingest(packets[rate][i % 4], offsets[rate], out)
        return fn

    work = [("16 kHz step_ragged, 1 chunk", ragged16, None)] + \
           [(f"ingest {r} Hz, 80 ms packets", ingest(r), r) for r in packets]
    sampler = bench.ClockSampler(0)
    sampler.start()
    windows, res = [], {w: [] for w, _, _ in work}
    for _ in range(args.rounds):
        for name, fn, rate in work:
            if rate:
                eng.set_input_rates(rate)
            for i in range(args.warmup):
                fn(i)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record()
            for i in range(args.steps):
                fn(i)
            e1.record()
            torch.cuda.synchronize()
            windows.append((t0, time.perf_counter()))
            res[name].append(e0.elapsed_time(e1) / args.steps)
    base = min(res[work[0][0]])
    print(f"engine: CUDA events around {args.steps} calls after {args.warmup} warm-up, {args.rounds} rounds alternating; "
          f"ms/call best (all rounds)")
    for name, _, _ in work:
        v = res[name]
        print(f"{name:>32}: {min(v):.4f} ({', '.join(f'{x:.4f}' for x in v)}), {100 * (min(v) - base) / base:+.2f} % "
              f"against 16 kHz step_ragged")
    print(f"clocks during the timed windows: {sampler.stop(windows)}")

    from torch.profiler import ProfilerActivity, profile
    print("resample_kernel (torch.profiler):")
    for name, fn, rate in work[1:]:
        eng.set_input_rates(rate)
        for i in range(args.warmup):
            fn(i)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(args.steps):
                fn(i)
            torch.cuda.synchronize()
        ka = [e for e in prof.key_averages() if "resample_kernel" in e.key]
        tot = [e for e in prof.key_averages() if e.device_type.name == "CUDA"]
        if not ka:
            print(f"{name:>32}: resample_kernel not found in the profile")
            continue
        attr = "device_time" if hasattr(ka[0], "device_time") else "cuda_time"
        us = getattr(ka[0], attr)
        total_us = sum(getattr(e, attr + "_total") for e in tot) / args.steps
        nbytes = 2 * B * (rate * 8 // 100) + 2 * B * CHUNK
        print(f"{name:>32}: {us:.1f} us per launch ({ka[0].count} launches), {100 * us / total_us:.2f} % of the call's "
              f"kernel time ({total_us:.0f} us); {nbytes / 1e6:.1f} MB -> {nbytes / (us * 1e-6) / 1e9:.0f} GB/s, "
              f"{100 * nbytes / (us * 1e-6) / DATA_SHEET_BYTES_PER_S:.1f} % of 3.35 TB/s "
              f"(the bound: {1e6 * nbytes / DATA_SHEET_BYTES_PER_S:.1f} us)")

    # Model level: device ingest against host resample_poly per packet (the reference's server example)
    from scipy.signal import resample_poly
    del eng, pcm, packets
    torch.cuda.empty_cache()
    specs = [{"name": k, "head": v} for k, v in heads.items()]
    fi = np.zeros((41, 96), np.float32)
    m48 = Model(wakeword_models=specs, embedding_model_path="synthetic:0", n_streams=B, feature_init=fi, max_chunks=2,
                sr=48000)
    m16 = Model(wakeword_models=specs, embedding_model_path="synthetic:0", n_streams=B, feature_init=fi, max_chunks=2)
    host = [list(rng.integers(-8000, 8000, (B, 3840)).astype(np.int16)) for _ in range(2)]

    def dev_arm(i):
        m48.predict_ragged(host[i % 2])

    def host_arm(i):
        m16.predict_ragged([resample_poly(x, 1, 3).astype(np.int16) for x in host[i % 2]])

    mres = {"Model(sr=48000).predict_ragged": [], "host resample_poly + 16 kHz predict_ragged": []}
    for _ in range(args.rounds):
        for (name, fn) in zip(mres, (dev_arm, host_arm)):
            fn(0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(args.model_steps):
                fn(i)
            torch.cuda.synchronize()
            mres[name].append(1e3 * (time.perf_counter() - t0) / args.model_steps)
    print(f"Model: wall clock per call over {args.model_steps} calls of {B} streams x 80 ms at 48 kHz, {args.rounds} rounds "
          "alternating; ms/call best (all rounds)")
    for name, v in mres.items():
        print(f"{name:>44}: {min(v):.1f} ({', '.join(f'{x:.1f}' for x in v)})")
    print(f"card after the run: {card()}")


if __name__ == "__main__":
    main()
