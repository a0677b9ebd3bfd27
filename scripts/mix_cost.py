"""Cost of clip mixing on the device (oww_mix_clips, csrc/mix.cu), printed as JSON lines (and written to the path given
as the first argument, if any).

* 10 000 mixtures of 2 s (N = 32 000) with RIRs of 0.25 / 0.5 / 1 s, over 1 / 16 / 10 000 distinct RIRs, and without
  reverb: CUDA events around each call (20 calls after 3 warm-up), then torch.profiler device time per kernel in a
  separate pass.  Each kernel against its bound: bytes / 3.35 TB/s for mix_kernel and finish_kernel, 3 N L MAC at the
  dense FP16 rate (989 TFLOP/s = 494.5 T MAC/s) for reverb_kernel.
* The same reverb on the host: NumPy FFT circular convolution of 200 of the mixtures, per mixture.
* Recall of a synthetic model over an SNR x RIR sweep (detect_clips on seeded mixtures): a pipeline figure, not a model
  quality figure.
The card's name and power limit are read in the same process."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
FP16_MAC = 989e12 / 2


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    import torch
    assert torch.cuda.is_available(), "mix_cost.py measures on a GPU"
    import __graft_entry__ as g
    g.build()
    from openwakeword_b200 import Model, _native
    from openwakeword_b200.utils import AudioFeatures
    from openwakeword_b200 import weights as W
    emb = W.synthetic_embedding(0)
    af = AudioFeatures(embedding_model_path=emb)
    rng = np.random.default_rng(0)
    N, n = 32000, 10000
    fg = [np.clip(rng.normal(0, 6000, 16000), -32768, 32767).astype(np.int16) for _ in range(100)]
    bg = [np.clip(rng.normal(0, 2000, 48000), -32768, 32767).astype(np.int16) for _ in range(100)]
    res = {"card": card(), "N": N, "n_mix": n, "runs": []}
    print(res["card"], flush=True)

    def params(n_rirs, reverb=True):
        p = np.zeros(n, _native.MIX_DTYPE)
        p["fg"] = rng.integers(0, 100, n); p["bg"] = rng.integers(0, 100, n); p["fg_len"] = 16000
        p["bg_offset"] = rng.integers(0, 48000, n); p["start"] = 8000; p["snr_db"] = rng.uniform(0, 20, n)
        p["rir"] = rng.integers(0, n_rirs, n) if reverb else -1
        p["volume"] = rng.uniform(0.02, 1.0, n)
        return p

    d_fg = (torch.from_numpy(np.concatenate(fg)).cuda(), np.arange(101, dtype=np.int64) * 16000)
    d_bg = (torch.from_numpy(np.concatenate(bg)).cuda(), np.arange(101, dtype=np.int64) * 48000)
    cases = [(0, 1, False)] + [(L, k, True) for L in (4000, 8000, 16000) for k in (1, 16, 10000)]
    for L, k, rev in cases:
        rirs = torch.from_numpy((rng.normal(0, 1, (k, max(L, 1))) * np.exp(-np.arange(max(L, 1)) / (L / 6 + 1))).astype(np.float32)).cuda()
        d_rir = (rirs.reshape(-1), np.arange(k + 1, dtype=np.int64) * max(L, 1))
        p = params(k, rev)
        for _ in range(3):
            af.mix_clips(d_fg, d_bg, N, p, d_rir)
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        times = []
        for _ in range(20):
            ev[0].record()
            af.mix_clips(d_fg, d_bg, N, p, d_rir)
            ev[1].record()
            ev[1].synchronize()
            times.append(ev[0].elapsed_time(ev[1]))
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                af.mix_clips(d_fg, d_bg, N, p, d_rir)
            torch.cuda.synchronize()
        kt = {}
        for e in prof.key_averages():
            for name in ("mix_kernel", "reverb_kernel", "finish_kernel"):
                if name in e.key:
                    kt[name] = e.device_time_total / e.count / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / e.count / 1e3
        mix_bytes = n * N * (2 * 2 + 4) + n * 16000 * 2
        fin_bytes = n * N * (4 * 2 + 2)
        r = {"L": L if rev else 0, "distinct_rirs": k if rev else 0, "ms_per_call_median": float(np.median(times)),
             "ms_per_call_min": float(np.min(times)), "kernel_ms": kt,
             "mix_bound_ms": mix_bytes / HBM * 1e3, "finish_bound_ms": fin_bytes / HBM * 1e3}
        if rev:
            r["reverb_bound_ms"] = 3 * n * N * L / FP16_MAC * 1e3
            if "reverb_kernel" in kt:
                r["reverb_share"] = r["reverb_bound_ms"] / kt["reverb_kernel"]
                r["reverb_TMACs"] = 3 * n * N * L / kt["reverb_kernel"] / 1e9
        for name, b in (("mix_kernel", "mix_bound_ms"), ("finish_kernel", "finish_bound_ms")):
            if name in kt:
                r[name + "_share"] = r[b] / kt[name]
        res["runs"].append(r)
        print(json.dumps(r), flush=True)
        del rirs
    # host FFT reverb of 200 mixtures of 2 s with a 0.5 s RIR
    h = rng.normal(0, 1, 8000)
    x = rng.normal(0, 0.1, (200, N))
    t0 = time.perf_counter()
    H = np.fft.rfft(np.concatenate([h, np.zeros(N - h.size)]))
    y = np.fft.irfft(np.fft.rfft(x, axis=1) * H, N, axis=1)
    y *= (np.abs(x).mean(1) / (np.abs(y).mean(1) + 1e-14))[:, None]
    res["host_fft_ms_per_mixture"] = (time.perf_counter() - t0) / 200 * 1e3
    print("host FFT reverb, ms per mixture:", res["host_fft_ms_per_mixture"], flush=True)
    # recall over SNR x RIR with a synthetic model
    m = Model(wakeword_models=[{"name": "alexa", "head": W.synthetic_head(seed=1)}], embedding_model_path=emb,
              feature_init=np.zeros((41, 96), np.float32))
    pos = [np.clip(rng.normal(0, 8000, 16000), -32768, 32767).astype(np.int16) for _ in range(50)]
    rirs = [(rng.normal(0, 1, 8000) * np.exp(-np.arange(8000) / 1200)).astype(np.float32) for _ in range(10)]
    clean = m.predict_clips_array(np.stack([np.concatenate([np.zeros(8000, np.int16), c, np.zeros(8000, np.int16)])
                                            for c in pos]))[0]
    thr = float(np.quantile(clean[..., 0].max(1), 0.5))
    table = {}
    for snr in (0, 5, 10, 20):
        for use_rir in (False, True):
            p = np.zeros(500, _native.MIX_DTYPE)
            p["fg"] = np.arange(500) % 50; p["bg"] = rng.integers(0, 100, 500); p["fg_len"] = 16000
            p["bg_offset"] = rng.integers(0, 48000, 500); p["start"] = 8000; p["snr_db"] = snr
            p["rir"] = (np.arange(500) // 50) if use_rir else -1
            p["volume"] = rng.uniform(0.02, 1.0, 500)
            t0 = time.perf_counter()
            out, valid = af.mix_clips(pos, bg, N, p, rirs)
            det = m.detect_clips(out, thr)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            hit = np.zeros(500, bool)
            for e in det:
                hit[e[0]] = True
            table[f"snr{snr}_{'rir' if use_rir else 'dry'}"] = {"recall": float(hit.mean()), "seconds": dt}
    res["recall_table"] = table
    res["recall_threshold"] = thr
    print(json.dumps(table), flush=True)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
