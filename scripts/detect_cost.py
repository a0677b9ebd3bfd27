"""What the host-side post-processing of Model.predict costs, and what the device detector (oww_detect) costs instead, on
the bench headline workload C3: 8192 streams x the bench's 7 head networks (11 labels), cnn_mode 3, one 1280-sample
chunk per call, host PCM in.  Three arms alternate in one process, `--rounds` times, `--steps` calls after `--warmup`:

  (a) step + D2H of the whole score matrix (StreamEngine.step_host): what an engine caller pays to post-process itself;
  (b) Model.predict: (a) + the history rules in NumPy on the host (Model._finish);
  (c) step + detect + D2H of the event count and the events, through the engine (H2D, oww_step, oww_detect) and through
      Model.detect;

(b) and (c) also with debounce on and with patience on.  Wall-clock milliseconds per call: a host clock around calls
that each end synchronised.  Then the detect call alone: CUDA events around `--launches` back-to-back launches, for
detect_kernel by itself (d_final only) and with the event compaction (detect_events_kernel), and the bytes the call has
to move, computed from the shapes, over that time against the data sheet's 3.35 TB/s of an H100 SXM (a figure for a
700 W card; not a measured peak).  Card name, power limit and SM clock are printed with the numbers.  No GPU: it fails.

python scripts/detect_cost.py [--streams 8192]"""
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


def detect_bytes(B, n_out, L, window, final):
    """bytes one oww_detect call at prepared >= 1280 needs: the scores and counts in, one history slot, the fired score
    and the counts out, `window` history entries per label read where patience or debounce is on, d_final if asked"""
    return 4 * (B * n_out + B + 2 * B * L + B + window * B * L + (B * L if final else 0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=2000)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    import openwakeword_b200 as owb
    from openwakeword_b200.engine import StreamEngine
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card, power limit, SM clock now, SM clock max: {smi[0] if smi else torch.cuda.get_device_name(0)}")

    B = args.streams
    heads = bench.bench_heads("c3")
    pcm = bench.synth_pcm_fast(B, 16, 0)                                 # host int16 [B, 16*1280]
    chunks = [np.ascontiguousarray(pcm[:, i * 1280:(i + 1) * 1280]) for i in range(16)]
    eng = StreamEngine(list(heads.values()), B, embedding="synthetic:0", max_chunks=1, cnn_mode=3)
    model = owb.Model(wakeword_models=[{"name": k, "head": v} for k, v in heads.items()], embedding_model_path="synthetic:0",
                      n_streams=B, max_chunks=1, feature_init=np.zeros((41, 96), np.float32))
    names = list(heads)
    labels = []                                                          # the engine's detector: the Model's label table
    for (col0, n_out) in eng.columns:
        labels += [(col0, True)] if n_out == 1 else [(col0 + k, False) for k in range(n_out)]
    L = len(labels)
    thr = {n: 0.5 for n in names}
    modes = {"plain": {}, "debounce": dict(debounce_time=0.5), "patience": dict(patience={n: 3 for n in names})}
    eng_modes = {"plain": {}, "debounce": dict(debounce_time=0.5), "patience": dict(patience={j: 3 for j in range(L)})}
    h_scores = np.empty((B, eng.n_cols), np.float32)
    d_scores = torch.empty((B, eng.n_cols), dtype=torch.float32, device="cuda")

    def arm_a(i):
        eng.step_host(chunks[i % 16], 1, h_scores)

    def arm_c_engine(i):
        d = torch.from_numpy(chunks[i % 16]).cuda()
        eng.detect(eng.step(d, 1, out=d_scores), 1280)

    arms = [("(a) step_host: step + D2H of the scores", arm_a, None)]
    for mode in modes:
        arms.append((f"(b) Model.predict, {mode}", lambda i, kw=modes[mode]: model.predict(chunks[i % 16], threshold=thr, **kw), None))
        arms.append((f"(c) engine: H2D + step + detect + events, {mode}", arm_c_engine, eng_modes[mode]))
        arms.append((f"(c) Model.detect, {mode}", lambda i, kw=modes[mode]: model.detect(chunks[i % 16], thr, **kw), None))

    sampler = bench.ClockSampler(0)
    sampler.start()
    windows, res = [], {name: [] for name, _, _ in arms}
    for _ in range(args.rounds):
        for name, fn, det in arms:
            if det is not None:
                eng.set_detector(labels, 0.5, **det)
            for i in range(args.warmup):
                fn(i)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(args.steps):
                fn(i)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            windows.append((t0, t1))
            res[name].append(1e3 * (t1 - t0) / args.steps)
    for name, ms in res.items():
        best = min(ms)
        print(f"{name:>56}: {best:.3f} ms/call wall (rounds: {', '.join(f'{v:.3f}' for v in ms)}), "
              f"{B / best * 1e-3:.2f} M frames/s")

    # the detect call alone, on the scores of the last step
    ctx = eng.ctx
    stream = torch.cuda.current_stream().cuda_stream
    final = torch.empty((B, L), dtype=torch.float32, device="cuda")
    ev = torch.empty((B * L, 4), dtype=torch.int32, device="cuda")
    n_ev = torch.zeros(1, dtype=torch.int32, device="cuda")
    for mode, det in eng_modes.items():
        eng.set_detector(labels, 0.5, **det)
        window = {"plain": 0, "debounce": 7, "patience": 3}[mode]
        for what, call, with_final in (("detect_kernel (d_final)", lambda: ctx.detect(d_scores, 1280, final, None, 0, None, stream), True),
                                       ("detect_kernel + detect_events_kernel", lambda: ctx.detect(d_scores, 1280, None, ev, B * L, n_ev, stream), False)):
            for _ in range(50):
                call()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record()
            for _ in range(args.launches):
                call()
            e1.record()
            torch.cuda.synchronize()
            windows.append((t0, time.perf_counter()))
            us = 1e3 * e0.elapsed_time(e1) / args.launches
            nbytes = detect_bytes(B, eng.n_cols, L, window, with_final)
            print(f"{what + ', ' + mode:>56}: {us:.2f} us/call over {args.launches} launches (includes the launch gaps); "
                  f"{nbytes / 1e6:.2f} MB needed at most -> {nbytes / (us * 1e-6) / 1e9:.0f} GB/s, "
                  f"{100 * nbytes / (us * 1e-6) / DATA_SHEET_BYTES_PER_S:.1f} % of the data-sheet 3.35 TB/s")
    print(f"history state: {30 * B * L * 4 / 1e6:.1f} MB; clocks: {sampler.stop(windows)}")


if __name__ == "__main__":
    main()
