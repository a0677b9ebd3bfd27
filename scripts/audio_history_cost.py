"""What the stream audio history (oww_set_audio_history, csrc/audio.cu) costs a streaming step, and what capturing the
clips of detections costs, on the bench headline configuration C3: 8192 streams x the bench's 7 head networks,
cnn_mode 3, device PCM in.

One engine (max_chunks 2) runs three workloads with history off and with 10 s of history, the two alternating,
`--rounds` times each, `--steps` steps after `--warmup`, timed with CUDA events around the steps:
  lockstep:  oww_step, 1 chunk per stream (the fused single-launch path);
  2 chunks:  oww_step, 2 chunks per stream (the general path);
  ragged:    oww_step_ragged, 1 chunk for 90 % of the streams, the other 10 % held.
Then oww_capture_events for 1, 64 and 1024 events of 5 s clips (CUDA events over `--launches` launches), and a
separate torch.profiler run that records audio_append_kernel's device time in each workload.  The bytes each kernel has
to move are computed from the shapes and set against the data sheet's 3.35 TB/s for an H100 SXM (a figure for a 700 W
card, not a measured peak).  Card name, power limit and SM clock are printed with the numbers.  No GPU: it fails.

python scripts/audio_history_cost.py [--streams 8192] [--seconds 10]"""
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
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--seconds", type=float, default=10.0)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    from openwakeword_b200.engine import StreamEngine
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)

    def card():
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name(0)

    print(f"card, power limit, SM clock now, SM clock max: {card()}")
    B, H = args.streams, int(round(args.seconds * 16000))
    heads = bench.bench_heads("c3")
    eng = StreamEngine(list(heads.values()), B, embedding="synthetic:0", max_chunks=2, cnn_mode=3)
    pcm = torch.from_numpy(bench.synth_pcm_fast(B, 16, 0)).cuda()              # int16 [B, 16*1280] on the device
    out = torch.empty((B, eng.n_cols), dtype=torch.float32, device="cuda")
    held = np.ones(B, np.int32)
    held[np.random.default_rng(0).permutation(B)[:B // 10]] = 0

    def lockstep(i):
        eng.step(pcm[:, (i % 16) * CHUNK:], 1, out)

    def two(i):
        eng.step(pcm[:, (i % 8) * 2 * CHUNK:], 2, out)

    def ragged(i):
        eng.step_ragged(pcm[:, (i % 16) * CHUNK:], held, out)

    work = [("lockstep, 1 chunk", lockstep, B * CHUNK), ("max_chunks 2, 2 chunks", two, 2 * B * CHUNK),
            ("ragged, 1 chunk, 10 % held", ragged, int(held.sum()) * CHUNK)]
    sampler = bench.ClockSampler(0)
    sampler.start()
    windows, res = [], {(w, h): [] for w, _, _ in work for h in (0, H)}
    for _ in range(args.rounds):
        for hist in (0, H):
            eng.set_audio_history(hist)
            for name, fn, _ in work:
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
                res[(name, hist)].append(e0.elapsed_time(e1) / args.steps)
    print(f"steps: CUDA events around {args.steps} steps after {args.warmup} warm-up, {args.rounds} rounds alternating "
          f"history off / {H} samples; ms/step best (all rounds)")
    for name, _, samples in work:
        off, on = res[(name, 0)], res[(name, H)]
        d = min(on) - min(off)
        print(f"{name:>28}: off {min(off):.4f} ({', '.join(f'{v:.4f}' for v in off)}), "
              f"on {min(on):.4f} ({', '.join(f'{v:.4f}' for v in on)}), difference {1e3 * d:+.1f} us = "
              f"{100 * d / min(off):+.2f} % of the step; append moves {2 * 2 * samples / 1e6:.1f} MB")

    # capture: E events of 5 s clips
    eng.set_audio_history(H)
    for i in range(H // CHUNK + 2):                                        # fill every ring
        lockstep(i)
    ctx = eng.ctx
    stream = torch.cuda.current_stream().cuda_stream
    n_clip = 5 * 16000
    print(f"capture: oww_capture_events of {n_clip}-sample clips, CUDA events over {args.launches} launches")
    for E in (1, 64, 1024):
        ev = torch.zeros((E, 4), dtype=torch.int32, device="cuda")
        ev[:, 0] = torch.from_numpy(np.random.default_rng(E).permutation(B)[:E].astype(np.int32)).cuda()
        n_ev = torch.tensor([E], dtype=torch.int32, device="cuda")
        clips = torch.empty((E, n_clip), dtype=torch.int16, device="cuda")
        ends = torch.empty(E, dtype=torch.int64, device="cuda")
        for _ in range(5):
            ctx.capture_events(ev, n_ev, E, n_clip, clips, ends, stream)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        for _ in range(args.launches):
            ctx.capture_events(ev, n_ev, E, n_clip, clips, ends, stream)
        e1.record()
        torch.cuda.synchronize()
        windows.append((t0, time.perf_counter()))
        us = 1e3 * e0.elapsed_time(e1) / args.launches
        nbytes = 2 * 2 * E * n_clip
        print(f"{E:>6} events: {us:.1f} us/call; {nbytes / 1e6:.1f} MB moved -> {nbytes / (us * 1e-6) / 1e9:.0f} GB/s, "
              f"{100 * nbytes / (us * 1e-6) / DATA_SHEET_BYTES_PER_S:.1f} % of the data-sheet 3.35 TB/s")
    print(f"clocks during the timed windows: {sampler.stop(windows)}")

    # the append kernel alone, from a profile of its own
    from torch.profiler import ProfilerActivity, profile
    print("append kernel (torch.profiler, history on):")
    for name, fn, samples in work:
        for i in range(args.warmup):
            fn(i)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(args.steps):
                fn(i)
            torch.cuda.synchronize()
        ka = [e for e in prof.key_averages() if "audio_append_kernel" in e.key]
        tot = [e for e in prof.key_averages() if e.device_type.name == "CUDA"]
        if not ka:
            print(f"{name:>28}: audio_append_kernel not found in the profile")
            continue
        attr = "device_time" if hasattr(ka[0], "device_time") else "cuda_time"
        us = getattr(ka[0], attr)                                           # average per launch, microseconds
        cnt = ka[0].count
        total_us = sum(getattr(e, attr + "_total") for e in tot) / args.steps
        nbytes = 2 * 2 * samples
        print(f"{name:>28}: {us:.1f} us per launch ({cnt} launches), {100 * us / total_us:.2f} % of the step's kernel "
              f"time ({total_us:.0f} us); {nbytes / 1e6:.1f} MB -> {nbytes / (us * 1e-6) / 1e9:.0f} GB/s, "
              f"{100 * nbytes / (us * 1e-6) / DATA_SHEET_BYTES_PER_S:.1f} % of 3.35 TB/s")
    print(f"memory: {B} streams x {H} samples: {(2 * H + 8) * B / 1e9:.2f} GB; card after the run: {card()}")


if __name__ == "__main__":
    main()
