"""What a serving loop pays for detections from host audio, on the bench headline configuration C3: 8192 streams x the
bench's 7 head networks, cnn_mode 3, one 80 ms packet per stream per call, at 16 kHz and at 48 kHz, threshold 0.5 plain
and with a 0.5 s debounce.

Arms, alternated `--rounds` times in one process, wall clock over `--calls` calls after `--warmup` (the pipelined arms
include collecting their last two tickets):
  (a) sync:      the synchronous loop from pageable host memory - H2D of the packets, ingest, detect (it waits for the
                 count, then copies the events);
  (b) submit:    submit_detect / collect_detect with two tickets in flight, packets in pageable host memory (staged
                 through the handle's pinned slots);
  (b) pinned:    the same with a page-locked packet buffer, DMA'd straight from it;
  (c) scores:    scores only through submit / collect (oww_step_host_submit) of 1280 16 kHz samples per stream, two in
                 flight - the floor: no resampling, no detection, and the whole score matrix comes back;
  (c) pinned:    the same from a page-locked buffer.
Then a separate torch.profiler pass over arm (b): detect_deliver_kernel's device time per launch and the bytes it writes
to host memory (count, events, and with capture the ends and clip rows) over that time, at threshold 0.5 and at
threshold 0 with max_events 1024 and 1 s clips (every pair fires: 1024 clips of 32 KB per call).  Card name, power
limit and SM clocks are printed with the numbers.  No GPU: it fails.

python scripts/serve_cost.py [--streams 8192] [--calls 200] [--warmup 20] [--rounds 3]"""
import argparse
import importlib.util
import os
import subprocess
import sys
import time
from collections import deque

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CLIP = 16000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8192)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    from openwakeword_b200.engine import StreamEngine
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)

    def card():
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name(0)

    print(f"card, power limit, SM clock now, SM clock max: {card()}")
    B = args.streams
    eng = StreamEngine(list(bench.bench_heads("c3").values()), B, embedding="synthetic:0", max_chunks=1, cnn_mode=3)
    eng.set_audio_history(2 * CLIP)
    # one label per network: alexa 0, hey_mycroft 1, hey_jarvis 2 (its verifier's raw score 3), hey_rhasspy 4,
    # weather 5, the timer's first class 7
    labels = [(0, True), (1, True), (2, True), (4, True), (5, True), (7, False)]
    pcm16 = [bench.synth_pcm_fast(B, 1, s) for s in range(4)]                  # int16 [B, 1280]
    pcm16_pinned = []
    for p in pcm16:
        t = torch.empty(p.shape, dtype=torch.int16).pin_memory()
        t.numpy()[:] = p
        pcm16_pinned.append(t)
    scores = np.empty((B, eng.n_cols), np.float32)

    def packets(rate):
        n = rate * 8 // 100
        pk = [np.ascontiguousarray(np.repeat(p, 3, axis=1)[:, :n]).ravel() if rate == 48000 else p.ravel()
              for p in pcm16]
        pinned = []
        for p in pk:
            t = torch.empty(p.size, dtype=torch.int16).pin_memory()
            t.numpy()[:] = p
            pinned.append(t)
        return pk, pinned, np.arange(B + 1, dtype=np.int64) * n

    def sync_arm(pk, off):
        def fn(i):
            chunks, prepared = eng.ingest(torch.from_numpy(pk[i % 4]).cuda(), off)
            eng.detect(eng.ingest_scores, prepared)
        return fn, None

    def submit_arm(src, off):
        q = deque()

        def fn(i):
            q.append(eng.submit_detect(src[i % 4], off))
            if len(q) == 2:
                eng.collect_detect(q.popleft())

        def drain():
            while q:
                eng.collect_detect(q.popleft())
        return fn, drain

    def scores_arm(src):
        q = deque()

        def fn(i):
            q.append(eng.submit(src[i % 4]))
            if len(q) == 2:
                eng.collect(q.popleft(), scores)

        def drain():
            while q:
                eng.collect(q.popleft(), scores)
        return fn, drain

    sampler = bench.ClockSampler(0)
    sampler.start()
    windows = []
    print(f"wall clock per call over {args.calls} calls after {args.warmup} warm-up, {args.rounds} rounds alternating; "
          "ms/call best (all rounds)")
    for rate in (16000, 48000):
        pk, pinned, off = packets(rate)
        pinned_np = [t.numpy() for t in pinned]
        eng.set_input_rates(rate)
        for debounce in (0.0, 0.5):
            eng.set_detector(labels, 0.5, debounce_time=debounce)
            arms = {"(a) sync": sync_arm(pk, off), "(b) submit": submit_arm(pk, off),
                    "(b) pinned": submit_arm(pinned_np, off), "(c) scores": scores_arm(pcm16),
                    "(c) pinned": scores_arm([t.numpy() for t in pcm16_pinned])}
            res = {k: [] for k in arms}
            for _ in range(args.rounds):
                for name, (fn, drain) in arms.items():
                    for i in range(args.warmup):
                        fn(i)
                    if drain:
                        drain()
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for i in range(args.calls):
                        fn(i)
                    if drain:
                        drain()
                    torch.cuda.synchronize()
                    t1 = time.perf_counter()
                    windows.append((t0, t1))
                    res[name].append(1e3 * (t1 - t0) / args.calls)
            what = f"{rate} Hz, threshold 0.5" + (f", debounce {debounce} s" if debounce else " plain")
            for name, v in res.items():
                floor = min(res["(c) pinned" if "pinned" in name else "(c) scores"])
                print(f"{what:>36} {name:>11}: {min(v):.3f} ({', '.join(f'{x:.3f}' for x in v)})  "
                      f"{B / (min(v) * 1e-3) / 1e6:.2f} M frames/s, {min(v) / floor:.2f} x (c) from the same kind of buffer")
    print(f"clocks during the timed windows: {sampler.stop(windows)}")

    from torch.profiler import ProfilerActivity, profile
    print("detect_deliver_kernel (torch.profiler, arm (b) pageable, 48 kHz):")
    pk, _, off = packets(48000)
    eng.set_input_rates(48000)
    for thr, M, cs in ((0.5, None, None), (0.0, 1024, CLIP)):
        eng.set_detector(labels, thr)
        got = []
        q = deque()
        for i in range(args.warmup):
            q.append(eng.submit_detect(pk[i % 4], off, max_events=M, capture=cs))
            if len(q) == 2:
                eng.collect_detect(q.popleft())
        while q:
            eng.collect_detect(q.popleft())
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(args.warmup):
                q.append(eng.submit_detect(pk[i % 4], off, max_events=M, capture=cs))
                if len(q) == 2:
                    got.append(eng.collect_detect(q.popleft()))
            while q:
                got.append(eng.collect_detect(q.popleft()))
            torch.cuda.synchronize()
        ka = [e for e in prof.key_averages() if "detect_deliver_kernel" in e.key]
        if not ka:
            print("  detect_deliver_kernel not found in the profile")
            continue
        attr = "device_time" if hasattr(ka[0], "device_time") else "cuda_time"
        us = getattr(ka[0], attr)
        k = np.mean([len(r[0]) for r in got])
        nbytes = 4 + k * 16 + (k * (8 + 2 * cs) if cs else 0)
        print(f"  threshold {thr}, max_events {M or 'n_streams x n_labels'}, capture {cs or 0}: {us:.1f} us per launch "
              f"({ka[0].count} launches), {k:.1f} events per call (count mean {np.mean([r[1] for r in got]):.1f}), "
              f"{nbytes / 1e6:.3f} MB to host memory per call -> {nbytes / (us * 1e-6) / 1e9:.2f} GB/s over the kernel")
    print(f"card after the run: {card()}")


if __name__ == "__main__":
    main()
