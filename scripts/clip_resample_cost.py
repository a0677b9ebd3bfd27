"""What whole-clip resampling (oww_resample_clips, csrc/ingest.cu) costs.

Kernel arm: per rate of the table, two batches of noise clips, 10 000 clips of 2 s and 64 clips of 60 s, padding 0.
CUDA events around `--iters` launches after a warm-up; the bytes the kernel has to move (input and output int16) and the
FMAs it has to issue (K per output) are set against the data sheet's 3.35 TB/s and 67 TFLOP/s FP32 (33.5 T FMA/s) of an
H100 SXM (figures for a 700 W card, not measured peaks), and the larger of the two shares names the bound.  A separate
torch.profiler pass records resample_clips_kernel's device time at 48000 and 44100 Hz.
End-to-end arm: bulk_predict wall clock over `--files` WAV files of 2 s, written to a temporary directory at 48000 Hz and
at 44100 Hz, against (a) scipy.signal.resample_poly on each file on the host, then a 16 kHz bulk_predict, and (b) the
same audio already at 16 kHz.  Card name, power limit and SM clocks are read in the same process.  No GPU: it fails.

python scripts/clip_resample_cost.py [--iters 20] [--files 2000]"""
import argparse
import os
import subprocess
import sys
import tempfile
import time
import wave

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
DATA_SHEET_BYTES_PER_S = 3.35e12
DATA_SHEET_FMA_PER_S = 67e12 / 2
RATES = (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000)


def card():
    import torch
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else torch.cuda.get_device_name(0)


def _write(path, pcm, rate):
    with wave.open(path, "wb") as f:
        f.setnchannels(1); f.setsampwidth(2); f.setframerate(rate)
        f.writeframes(pcm.tobytes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--files", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    from openwakeword_b200 import _native, weights as W
    from openwakeword_b200.utils import bulk_predict
    print(f"card, power limit, SM clock now, SM clock max: {card()}", flush=True)
    ctx = _native.Context()
    rng = np.random.default_rng(0)
    print("rate  batch            ms/launch  out Msamples  GB/s   share HBM  GFMA/s  share FP32  bound")
    for n_clips, seconds in ((10000, 2.0), (64, 60.0)):
        for r in RATES:
            taps, up, down = _native.resampler_taps(r)
            K = -(-taps.size // up) if taps.size else 0
            S = int(r * seconds)
            n_out = _native.resample_clip_plan(r, S, 0)
            d_in = torch.randint(-8000, 8000, (n_clips * S,), dtype=torch.int16, device="cuda")
            d_out = torch.empty(n_clips * n_out, dtype=torch.int16, device="cuda")
            in_off = np.arange(n_clips + 1, dtype=np.int64) * S
            out_off = np.arange(n_clips + 1, dtype=np.int64) * n_out
            rates = np.full(n_clips, r, np.int32)
            call = lambda: ctx.resample_clips(d_in, in_off, rates, 0, d_out, out_off)   # noqa: E731
            for _ in range(3):
                call()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                call()
            e1.record()
            torch.cuda.synchronize()
            t = e0.elapsed_time(e1) / args.iters / 1e3
            outs = n_clips * n_out
            nbytes = 2 * (n_clips * S + outs)
            fmas = outs * K
            hbm, fp = nbytes / t / DATA_SHEET_BYTES_PER_S, fmas / t / DATA_SHEET_FMA_PER_S
            print(f"{r:5d} {n_clips:5d} x {seconds:4.0f} s  {t * 1e3:9.3f}  {outs / 1e6:12.1f}  {nbytes / t / 1e9:6.0f}  "
                  f"{hbm:9.1%}  {fmas / t / 1e9:6.0f}  {fp:10.1%}  {'HBM' if hbm >= fp else 'FP32'}", flush=True)
            del d_in, d_out, call
            torch.cuda.empty_cache()
    # profiler pass: the kernel's own device time
    from torch.profiler import ProfilerActivity, profile
    for r in (48000, 44100):
        for n_clips in (10000, 64):
            S = int(r * (2.0 if n_clips == 10000 else 60.0))
            n_out = _native.resample_clip_plan(r, S, 0)
            d_in = torch.zeros(n_clips * S, dtype=torch.int16, device="cuda")
            d_out = torch.empty(n_clips * n_out, dtype=torch.int16, device="cuda")
            in_off = np.arange(n_clips + 1, dtype=np.int64) * S
            out_off = np.arange(n_clips + 1, dtype=np.int64) * n_out
            rates = np.full(n_clips, r, np.int32)
            ctx.resample_clips(d_in, in_off, rates, 0, d_out, out_off)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    ctx.resample_clips(d_in, in_off, rates, 0, d_out, out_off)
                torch.cuda.synchronize()
            ev = [e for e in prof.key_averages() if "resample_clips_kernel" in e.key]
            us = ev[0].device_time_total / 5 if ev else float("nan")
            print(f"profiler: resample_clips_kernel at {r} Hz, {n_clips} clips: {us / 1e3:.3f} ms per launch", flush=True)
            del d_in, d_out
    torch.cuda.empty_cache()
    # end to end
    import scipy.signal as ss
    spec = [{"name": "alexa", "head": W.synthetic_head(seed=1)},
            {"name": "timer", "head": W.synthetic_head(n_in=34, hidden=128, n_out=7, layernorm=False,
                                                      final="relu_softmax", seed=9)}]
    kw = dict(embedding_model_path="synthetic:0", feature_init=np.zeros((41, 96), np.float32), ncpu=8)
    with tempfile.TemporaryDirectory() as tmp:
        base = [np.clip(rng.normal(0, 3000, 2 * 48000), -32768, 32767).astype(np.int16) for _ in range(args.files)]
        sets = {}
        for r in (48000, 44100):
            clips = base if r == 48000 else [ss.resample_poly(c, 147, 160).astype(np.int16) for c in base]
            paths = []
            for i, c in enumerate(clips):
                p = os.path.join(tmp, f"r{r}_{i}.wav")
                _write(p, c, r)
                paths.append(p)
            p16 = []
            for i, c in enumerate(clips):
                p = os.path.join(tmp, f"s{r}_{i}.wav")
                g = np.gcd(16000, r)
                _write(p, np.clip(np.rint(ss.resample_poly(c, 16000 // g, r // g)), -32768, 32767).astype(np.int16), 16000)
                p16.append(p)
            sets[r] = (paths, p16, clips)
        bulk_predict(sets[48000][1][:16], spec, **kw)                      # warm-up: module load, first launches
        bulk_predict(sets[48000][0][:16], spec, **kw)
        audio_s = args.files * 2.0
        for rnd in range(args.rounds):
            for r, (paths, p16, clips) in sets.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                bulk_predict(paths, spec, **kw)
                t_dev = time.perf_counter() - t0
                t0 = time.perf_counter()
                g = np.gcd(16000, r)
                for p in paths:                                            # (a): host resampling, then 16 kHz
                    with wave.open(p, "rb") as f:
                        x = np.frombuffer(f.readframes(f.getnframes()), np.int16)
                    ss.resample_poly(x, 16000 // g, r // g)
                t_host = time.perf_counter() - t0
                t0 = time.perf_counter()
                bulk_predict(p16, spec, **kw)                              # (b): the audio already at 16 kHz
                t16 = time.perf_counter() - t0
                print(f"round {rnd} {r} Hz, {args.files} files x 2 s: device resampling {t_dev:.2f} s "
                      f"({audio_s / t_dev:.0f} x real time); (a) host resample_poly {t_host:.2f} s + 16 kHz "
                      f"bulk_predict {t16:.2f} s = {t_host + t16:.2f} s; (b) 16 kHz {t16:.2f} s", flush=True)
    print(f"card, power limit, SM clock now, SM clock max: {card()}")


if __name__ == "__main__":
    main()
