"""Device cost of custom verifiers on a per-stream head bank (oww_add_bank_verifier_bank) on the C3 workload (8192
streams x 7 head networks, cnn_mode 3, one chunk per step, device-resident PCM, StreamEngine without Model):

  - streaming: a bank of 16x96 -> 64 -> 64 -> 1 with D in {1, 1024, 8192} slots on a seeded uniform assignment, run
    three ways, alternated: no stream verifiers | a distinct verifier on every stream at threshold 0 (every stream with
    a model verified) | the same at threshold 0.5.  Device milliseconds per step (CUDA events around `--steps` steps
    after `--warmup`), and the verifier bytes a verified stream reads (mean + weight, D = 16*96 floats each);
  - bulk: `--clips` clips of 2 s through oww_predict_clips_ragged with every clip on one clip slot, against
    oww_predict_clips_streams with clip i on stream i % streams (the bank's D slots, each stream's own verifier),
    alternated; milliseconds per call (CUDA events around the call, host table building included).

Verifier parameters are random (the cost does not depend on their values).  Prints the card name, power limit and SM
clock read in the same run, then every result as one JSON line; --json PATH also writes that record to PATH.
python scripts/stream_verifier_cost.py [--streams 8192] [--clips 10000] [--json PATH]"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--ds", default="1,1024,8192")
    ap.add_argument("--clips", type=int, default=10000)
    ap.add_argument("--bulk-d", type=int, default=1024)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    from openwakeword_b200 import _native
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
    pool = [W.synthetic_head(hidden=64, seed=300 + i) for i in range(32)]
    D_in = 16 * 96

    def engine(D, verifiers):
        eng = StreamEngine(list(heads), B, embedding="synthetic:0", max_chunks=1, cnn_mode=3)
        bank, _, _ = eng.add_head_bank(pool[0], D)
        for k in range(D):
            eng.load_bank_head(bank, k, pool[k % len(pool)])
        eng.assign_bank_head(bank, np.random.default_rng(D).integers(0, D, B).astype(np.int32))
        vb = None
        if verifiers:
            vb = eng.add_bank_verifier_bank(bank, B, 0.0)
            g = torch.Generator(device="cuda").manual_seed(1)
            mean = torch.randn((B, D_in), device="cuda", generator=g)
            weight = torch.randn((B, D_in), device="cuda", generator=g) * 0.02
            bias = torch.zeros(B, device="cuda")
            slots = np.arange(B, dtype=np.int32)
            eng.ctx.load_verifiers(vb, slots, mean, weight, bias)
            eng.assign_verifier(vb, slots)
        torch.cuda.synchronize()
        return eng, bank, vb

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

    res = {"card": smi, "streams": B, "steps": args.steps, "verifier_bytes_per_stream": 2 * D_in * 4, "rows": []}
    for D in [int(x) for x in args.ds.split(",")]:
        plain, _, _ = engine(D, False)
        ver, _, vb = engine(D, True)
        times = {"no stream verifiers": [], "threshold 0": [], "threshold 0.5": []}
        for _ in range(2):
            times["no stream verifiers"].append(time_ms(plain, args.steps))
            ver.ctx.set_verifier_threshold(vb, 0.0)
            times["threshold 0"].append(time_ms(ver, args.steps))
            ver.ctx.set_verifier_threshold(vb, 0.5)
            times["threshold 0.5"].append(time_ms(ver, args.steps))
        for k, v in times.items():
            print(f"D {D:5d} {k:20s} ms/step: " + " ".join(f"{t:.4f}" for t in v), flush=True)
            res["rows"].append({"D": D, "config": k, "ms_per_step": v})
        del plain, ver
        torch.cuda.empty_cache()

    # bulk: one clip slot against per-clip streams
    D = args.bulk_d
    eng, bank, vb = engine(D, True)
    ctx = eng.ctx
    ctx.set_head_bank_clip_slot(bank, 0)
    ctx.set_verifier_clip_slot(vb, 0)
    ctx.set_verifier_threshold(vb, 0.0)
    n, L = args.clips, 32000
    clips = torch.from_numpy(np.clip(rng.normal(0, 3000, n * L), -32768, 32767).astype(np.int16)).cuda()
    off = np.arange(n + 1, dtype=np.int64) * L
    rows = n * _native.clip_schedule(1280, L + 32000).size
    raw = torch.zeros((rows, ctx.n_outputs), dtype=torch.float32, device="cuda")
    stepped = torch.zeros(rows, dtype=torch.uint8, device="cuda")
    cs = (np.arange(n) % B).astype(np.int32)

    def call_ms(clip_streams):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ctx.predict_clips_ragged(clips, off, 16000, 1280, None, raw, stepped, None,
                                 torch.cuda.current_stream().cuda_stream, clip_streams=clip_streams)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)
    call_ms(None), call_ms(cs)
    bulk = {"one clip slot": [], "per-clip streams": []}
    for _ in range(3):
        bulk["one clip slot"].append(call_ms(None))
        bulk["per-clip streams"].append(call_ms(cs))
    for k, v in bulk.items():
        print(f"bulk {n} clips of 2 s, D {D}: {k:16s} ms/call: " + " ".join(f"{t:.2f}" for t in v), flush=True)
        res["rows"].append({"bulk_clips": n, "D": D, "config": k, "ms_per_call": v})
    print(json.dumps(res), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
