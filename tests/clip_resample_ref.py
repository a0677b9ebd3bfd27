"""Float64 restatement of whole-clip resampling (include/owwb200.h, oww_resample_clips), written from its definition and
independent of the library: a clip x of S samples at `rate` with `pad` 16 kHz samples of padding becomes the first
A(S) + 2*pad outputs of upfirdn(h, zeros(pad*down/up) ++ x ++ zeros(pad*down/up), up, down), each output the polyphase
sum over its phase's taps."""
import numpy as np

from oracle import resample as ores


def plan(rate, n_in, pad):
    """A(n_in) + 2*pad, or None where the library refuses (rate outside the table, negative arguments, up not dividing
    pad)"""
    if rate not in ores.RATES or n_in < 0 or pad < 0:
        return None
    up, down = ores.up_down(rate)
    if pad % up:
        return None
    return ores.final_outputs(n_in, up, down) + 2 * pad


def resample_clip(x, rate, pad, h=None, abs_sum=False):
    """-> float64 outputs (and with abs_sum, sum_t |h_t * x_t| of each, the round-off scale).  `h` (default:
    oracle.resample.taps(rate)) may be the library's fp32 taps, to evaluate its sums in float64."""
    up, down = ores.up_down(rate)
    assert pad % up == 0 and pad >= 0
    x = np.asarray(x, np.float64).ravel()
    if up == down:
        y = np.concatenate((np.zeros(pad), x, np.zeros(pad)))
        return (y, np.abs(y)) if abs_sum else y
    h = ores.taps(rate) if h is None else np.asarray(h, np.float64)
    P = pad * down // up
    z = np.concatenate((np.zeros(P), x, np.zeros(P)))
    L = ores.final_outputs(x.size, up, down) + 2 * pad
    K = -(-h.size // up)
    hp = np.zeros((up, K))
    for p in range(up):
        hp[p, :h[p::up].size] = h[p::up]
    y, s = np.zeros(L), np.zeros(L)
    for a in range(0, L, 8192):                              # blocks of outputs, to bound the [outputs, K] temporaries
        i = np.arange(a, min(L, a + 8192), dtype=np.int64)
        q0, p = np.divmod(i * down, up)
        idx = q0[:, None] - np.arange(K)[None, :]
        v = np.where((idx >= 0) & (idx < z.size), z[np.clip(idx, 0, max(z.size - 1, 0))] if z.size else 0.0, 0.0)
        prod = hp[p] * v
        y[a:a + i.size] = prod.sum(axis=1)
        s[a:a + i.size] = np.abs(prod).sum(axis=1)
    return (y, s) if abs_sum else y
