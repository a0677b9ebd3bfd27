"""What the detector of the bulk clip path (oww_detect_clips, csrc/detect.cu) costs.

Workload: 10 000 noise clips of 2 s (padding 1 s), the heads of bench.py's C3 workload (six models, 11 labels), chunk
sizes 1280 and 1024.
1. Plain predict_clips / predict_clips_ragged (no patience, threshold or debounce) in this tree and in `--parent` (a
   built checkout of the parent commit), each in its own process, the trees alternated `--rounds` times: wall clock
   per call, and the rows of both trees compared.
2. predict_clips and detect_clips with debounce_time=1.25 and threshold=0.5, and the host loop predict_clip(**kw)
   after reset on `--host-clips` clips, scaled to 10 000 clips (printed as scaled).
3. The two kernels alone: CUDA events around `--iters` oww_detect_clips calls on the raw rows of the clip call, final
   rows only and events only.  Bytes the kernels must move (each label's score column of every row read once, the
   final rows written once) over the time, against the data sheet's 3.35 TB/s of an H100 SXM (a 700 W figure, not a
   measured peak).
4. `--bench`: bench.py --gpus 1 in the parent tree and in this one, alternated; the value and the parity of each run.
Card name, power limit and SM clocks are read in the same process.  No GPU: it fails.

python scripts/clip_detect_cost.py --parent DIR [--rounds 2] [--bench] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA_SHEET_BYTES_PER_S = 3.35e12
N_CLIPS, SECONDS = 10000, 2.0
CHUNKS = (1280, 1024)
TIMER_MAP = {"1": "1_minute_timer", "2": "5_minute_timer", "3": "10_minute_timer",
             "4": "20_minute_timer", "5": "30_minute_timer", "6": "1_hour_timer"}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def model(tree):
    sys.path.insert(0, tree)
    import openwakeword_b200 as owb
    from openwakeword_b200 import weights as W
    hs = {}
    for i, nm in enumerate(["alexa", "hey_mycroft", "hey_jarvis", "hey_rhasspy", "weather"]):     # bench.py's C3 heads
        hs[nm] = (W.synthetic_gated_head(seed_main=10 + i, seed_verifier=40 + i, threshold=0.5) if nm == "hey_jarvis"
                  else W.synthetic_head(seed=10 + i))
    hs["timer"] = W.synthetic_head(n_in=34, hidden=128, n_out=7, layernorm=False, final="relu_softmax", seed=20)
    fi = np.random.default_rng(1).normal(0, 1, (41, 96)).astype(np.float32)
    specs = [{"name": k, "head": v, "class_mapping": TIMER_MAP if k == "timer" else None} for k, v in hs.items()]
    return owb.Model(wakeword_models=specs, embedding_model_path=W.synthetic_embedding(0), feature_init=fi, max_chunks=2)


def clips():
    rng = np.random.default_rng(7)
    return np.clip(rng.normal(0, 3000, (N_CLIPS, int(SECONDS * 16000))), -32768, 32767).astype(np.int16)


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return min(ts), out


def plain_arm(tree, out):
    """one process per tree: plain predict_clips_ragged (arrays) and predict_clips (dicts) at each chunk size"""
    m = model(tree)
    x = clips()
    pcm, off = x.reshape(-1), np.arange(N_CLIPS + 1, dtype=np.int64) * x.shape[1]
    res = {}
    for c in CHUNKS:
        t_arr, (scores, _, _) = timed(lambda: m.predict_clips_ragged(pcm, off, 1, c), 3)
        t_dict, _ = timed(lambda: m.predict_clips(x, padding=1, chunk_size=c), 1)
        np.save(os.path.join(out, f"rows_{os.path.basename(os.path.normpath(tree))}_{c}.npy"), scores)
        res[c] = {"ragged_s": t_arr, "predict_clips_s": t_dict, "rows": int(scores.shape[0])}
    print(json.dumps(res), flush=True)


def run_arm(tree, out):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--arm", tree, "--out", out], cwd=tree,
                       capture_output=True, text=True)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode or not lines:
        raise RuntimeError(f"{tree}: {r.stderr[-2000:]}")
    return {int(k): v for k, v in json.loads(lines[-1]).items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", help="a built checkout of the parent commit")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--host-clips", type=int, default=10)
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--out", help="directory for the rows the two trees are compared on (default: a new temporary one)")
    ap.add_argument("--arm", help=argparse.SUPPRESS)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    args.out = os.path.abspath(args.out) if args.out else tempfile.mkdtemp(prefix="clip_detect_cost_")
    args.parent = args.parent and os.path.abspath(args.parent)
    os.makedirs(args.out, exist_ok=True)
    if args.arm:
        return plain_arm(args.arm, args.out)
    print(f"card, power limit, SM clock now, SM clock max: {card()}", flush=True)
    print(f"workload: {N_CLIPS} clips of {SECONDS} s, padding 1 s, bench C3 heads (6 models, 11 labels)", flush=True)

    # 1. plain calls, parent and this tree alternated
    if args.parent:
        for rnd in range(args.rounds):
            for tag, tree in (("parent", args.parent), ("new", ROOT)):
                r = run_arm(tree, args.out)
                for c in CHUNKS:
                    print(f"round {rnd} {tag:6s} chunk {c}: predict_clips_ragged {r[c]['ragged_s'] * 1e3:8.1f} ms, "
                          f"predict_clips {r[c]['predict_clips_s']:6.2f} s ({r[c]['rows']} rows)", flush=True)
        for c in CHUNKS:
            a = np.load(os.path.join(args.out, f"rows_{os.path.basename(os.path.normpath(args.parent))}_{c}.npy"))
            b = np.load(os.path.join(args.out, f"rows_{os.path.basename(os.path.normpath(ROOT))}_{c}.npy"))
            print(f"chunk {c}: rows of parent and new {'bit-identical' if np.array_equal(a, b) else 'DIFFER'} "
                  f"(max |diff| {np.abs(a - b).max() if a.size else 0.0:.3g})", flush=True)

    # 2. with the new arguments
    m = model(ROOT)
    x = clips()
    kw = dict(threshold=0.5, debounce_time=1.25)
    thr = {k: 0.5 for k in m.models}
    for c in CHUNKS:
        t_pc, _ = timed(lambda: m.predict_clips(x, padding=1, chunk_size=c, threshold=thr, debounce_time=1.25), 1)
        t_dc, ev = timed(lambda: m.detect_clips(x, **kw, padding=1, chunk_size=c), 3)
        h = args.host_clips
        t0 = time.perf_counter()
        for i in range(h):
            m.reset()
            m.predict_clip(x[i], padding=1, chunk_size=c, threshold=thr, debounce_time=1.25)
        t_host = (time.perf_counter() - t0) * N_CLIPS / h
        print(f"chunk {c}, threshold 0.5, debounce 1.25 s: predict_clips {t_pc:6.2f} s, detect_clips {t_dc * 1e3:8.1f} ms "
              f"({len(ev)} events), host loop predict_clip {t_host:8.1f} s (scaled from {h} clips)", flush=True)

    # 3. the kernels alone
    ctx = m.preprocessor.ctx
    table = m._clip_table({}, thr, 1.25)
    L = len(table)
    for c in CHUNKS:
        pcm, off = x.reshape(-1), np.arange(N_CLIPS + 1, dtype=np.int64) * x.shape[1]
        raw, row_off = m._clip_call(pcm, off, 1, c, None, None, True)[:2]
        rows = int(row_off[-1])
        final = torch.empty((rows, L), dtype=torch.float32, device="cuda")
        n_ev = torch.zeros(1, dtype=torch.int32, device="cuda")
        cap = 1 << 20
        ev = torch.empty((cap, 4), dtype=torch.int32, device="cuda")
        arms = {"final rows": lambda: ctx.detect_clips(table, 1.25, raw, None, 0.5, row_off, c, final, None, 0, None),
                "events": lambda: ctx.detect_clips(table, 1.25, raw, None, 0.5, row_off, c, None, ev, cap, n_ev)}
        for name, fn in arms.items():
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            t = e0.elapsed_time(e1) / args.iters / 1e3
            passes = 1 if name == "final rows" else 2
            nbytes = passes * rows * L * 4 + (rows * L * 4 if name == "final rows" else 0)
            print(f"chunk {c} kernel ({name}): {t * 1e3:7.3f} ms for {rows} rows x {L} labels, {nbytes / 1e6:7.1f} MB, "
                  f"{nbytes / t / 1e9:7.1f} GB/s = {nbytes / t / DATA_SHEET_BYTES_PER_S:6.1%} of 3.35 TB/s", flush=True)

    # 4. bench.py, parent and this tree alternated
    if args.bench and args.parent:
        for rnd in range(args.rounds):
            for tag, tree in (("parent", args.parent), ("new", ROOT)):
                r = subprocess.run([sys.executable, "bench.py", "--gpus", "1"], cwd=tree, capture_output=True, text=True)
                lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
                if not lines:
                    print(f"bench {tag}: failed: {r.stderr[-1500:]}", flush=True)
                    continue
                b = json.loads(lines[-1])
                print(f"bench round {rnd} {tag:6s}: {b['value'] / 1e6:.3f} M {b['unit']}, parity {json.dumps(b.get('parity'))}",
                      flush=True)


if __name__ == "__main__":
    main()
