"""What per-stream detection settings (oww_set_stream_detection) cost oww_detect, on the bench headline workload C3: 8192
streams x the bench's 7 head networks (11 labels), threshold 0.5, one 1280-sample chunk's scores per call.  Three arms
on one engine, alternated `--rounds` times in one process:

  none: no stream has settings of its own (the kernel reads no record: the path of a handle that never had any);
  1 %:  every 100th stream has its own thresholds and debounce (the kernel reads the records of every stream);
  100 %: every stream has them.

Per arm, CUDA events around `--launches` back-to-back oww_detect calls on the scores of the last step, for detect_kernel
alone (d_final only) and with the event compaction (detect_events_kernel); launch gaps included.  The best round is the
figure, every round is printed.  The card name, power limit and SM clocks are printed with the numbers.  No GPU: it
fails.  `--package-root DIR` imports openwakeword_b200 from another tree (a build without the settings call runs the
"none" arm only), to compare builds in separate processes of one command.

python scripts/stream_detect_cost.py [--streams 8192] [--launches 2000] [--rounds 3]"""
import argparse
import importlib.util
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8192)
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--package-root", default=ROOT)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.package_root))
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    from openwakeword_b200.engine import StreamEngine
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card, power limit, SM clock now, SM clock max: {smi[0] if smi else torch.cuda.get_device_name(0)}")
    print(f"package: {os.path.abspath(args.package_root)}")

    B = args.streams
    heads = bench.bench_heads("c3")
    eng = StreamEngine(list(heads.values()), B, embedding="synthetic:0", max_chunks=1, cnn_mode=3)
    labels = []
    for (col0, n_out) in eng.columns:
        labels += [(col0, True)] if n_out == 1 else [(col0 + k, False) for k in range(n_out)]
    L = len(labels)
    eng.set_detector(labels, 0.5, debounce_time=0.5)
    pcm = torch.from_numpy(bench.synth_pcm_fast(B, 1, 0)).cuda()
    d_scores = eng.step(pcm, 1)
    for _ in range(6):                                   # past the first-5 zeroing: the rules run on real scores
        eng.detect(d_scores, 1280)
    torch.cuda.synchronize()
    has_settings = hasattr(eng, "set_stream_detection")
    arms = {"none": None, "1 %": np.arange(0, B, 100), "100 %": np.arange(B)} if has_settings else {"none": None}

    def configure(ids):
        if not has_settings:
            return
        eng.clear_stream_detection()
        if ids is not None:
            eng.set_stream_detection(ids, threshold={j: 0.4 + 0.01 * (j % 5) for j in range(L)}, debounce_time=1.0)

    ctx = eng.ctx
    stream = torch.cuda.current_stream().cuda_stream
    final = torch.empty((B, L), dtype=torch.float32, device="cuda")
    ev = torch.empty((B * L, 4), dtype=torch.int32, device="cuda")
    n_ev = torch.zeros(1, dtype=torch.int32, device="cuda")
    calls = {"detect_kernel (d_final)": lambda: ctx.detect(d_scores, 1280, final, None, 0, None, stream),
             "detect_kernel + detect_events_kernel": lambda: ctx.detect(d_scores, 1280, None, ev, B * L, n_ev, stream)}
    res = {(a, c): [] for a in arms for c in calls}
    for _ in range(args.rounds):
        for arm, ids in arms.items():
            configure(ids)
            for what, call in calls.items():
                for _ in range(50):
                    call()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.launches):
                    call()
                e1.record()
                torch.cuda.synchronize()
                res[(arm, what)].append(1e3 * e0.elapsed_time(e1) / args.launches)
    for (arm, what), us in res.items():
        print(f"{what + ', ' + arm:>50}: {min(us):.2f} us/call (rounds: {', '.join(f'{v:.2f}' for v in us)}) over "
              f"{args.launches} launches")
    if has_settings:
        print(f"settings table: {B * L * 12 / 1e6:.2f} MB records + {B * 8 / 1e6:.3f} MB debounce")


if __name__ == "__main__":
    main()
