"""Device cost of moving live streams on the C3 workload (8192 streams x 7 head networks, cnn_mode 3, split_from 11,
StreamEngine without Model): device milliseconds of oww_export_streams and oww_import_streams of n = 1, 64, 1024 and 8192
streams (scattered ids), from CUDA events around `--reps` calls after `--warmup`, and the bytes each call moves over that
time as a share of the H100 SXM data-sheet 3.35 TB/s.

Bytes moved per stream (from the record size): an export reads the stream's state and writes its record (the state is
the record's content, so 2 x record bytes; the rings it reads in 16-byte units are the newest rows only).  An import
reads the record and writes the whole mel and feature rings of the stream (older slots are cleared) plus the record's
other sections, and rebuilds the stream's fp16 feature mirror; counted as record bytes + ring bytes.

Prints the card name, power limit and SM clock read in the same run, then the results as one JSON line; --json PATH
also writes that record to PATH.
python scripts/stream_state_cost.py [--streams 8192] [--reps 50] [--json PATH]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ns", default="1,64,1024,8192")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    from openwakeword_b200.engine import StreamEngine
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"card (name, power limit, SM clock, max SM clock): {smi or torch.cuda.get_device_name(0)}", flush=True)

    B = args.streams
    eng = StreamEngine(list(bench.bench_heads("c3").values()), B, embedding="synthetic:0", max_chunks=1, cnn_mode=3,
                       split_from=11)
    rng = np.random.default_rng(0)
    pcm = torch.from_numpy(np.clip(rng.normal(0, 3000, (B, 1280)), -32768, 32767).astype(np.int16)).cuda()
    for _ in range(3):
        eng.step(pcm)
    rec_bytes, _ = eng.ctx.stream_state_info()
    mel_rows = 1 << (76 + 8 - 1).bit_length()        # the handle's ring sizes at max_chunks 1 (oww_set_streams)
    feat_rows = 1 << (120 + 1 - 1).bit_length()
    ring_bytes = (mel_rows * 32 + feat_rows * 96) * 4
    s = torch.cuda.current_stream()
    results = {"card": smi, "streams": B, "record_bytes": rec_bytes, "export": {}, "import": {}}
    for n in [int(v) for v in args.ns.split(",")]:
        ids = np.sort(rng.choice(B, n, replace=False)).astype(np.int32)
        recs = eng.export_streams(ids)
        for kind in ("export", "import"):
            call = (lambda: eng.ctx.export_streams(ids, recs, s.cuda_stream)) if kind == "export" else \
                (lambda: eng.ctx.import_streams(ids, recs, s.cuda_stream))
            for _ in range(args.warmup):
                call()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(s)
            for _ in range(args.reps):
                call()
            t1.record(s)
            t1.synchronize()
            ms = t0.elapsed_time(t1) / args.reps
            moved = n * (2 * rec_bytes if kind == "export" else rec_bytes + ring_bytes)
            tbs = moved / (ms * 1e-3) / 1e12
            results[kind][n] = {"ms": round(ms, 5), "bytes": moved, "TB/s": round(tbs, 3),
                                "share_of_3.35TB/s": round(tbs / HBM_TBS, 3)}
            print(f"{kind} n={n}: {ms * 1e3:.1f} us, {moved / 1e6:.2f} MB, {tbs:.2f} TB/s "
                  f"({100 * tbs / HBM_TBS:.0f} % of {HBM_TBS} TB/s)", flush=True)
    assert eng.ctx.stream_state_rejected() == 0
    line = json.dumps(results)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
