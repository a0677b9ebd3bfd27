"""Float64 restatement of oww_mix_clips (include/owwb200.h), written from its definition, with the round-off bound the
device's result is held to.

``mix_ref`` returns, per mixture, the int16 row, the valid flag, v = 32767 y (the value truncated) and tau, a bound on
|v_device - v| before truncation: the device stores the mixture as float32, reverberates with fp16 hi/lo split
operands and fp32 accumulation, and levels in float64.  Where trunc(v - tau) == trunc(v + tau) the device must give
exactly the int16 here; elsewhere it may differ by one.
"""
import numpy as np

U = 2.0 ** -24
SPLIT_OP = 3.0 * 2.0 ** -22              # dropped lo*lo product and the lo parts' own rounding, per product
SUB16 = 2.0 ** -25                       # half the fp16 subnormal spacing, per operand


def _circ(a, h, d, N):
    """y[n] = sum_k h[k] a[(n - k + d) mod N], float64"""
    H = np.fft.rfft(np.concatenate([h, np.zeros(N - h.size)]))
    return np.roll(np.fft.irfft(np.fft.rfft(a) * H, N), -d)


def mixture(fg, bg, N, p):
    """Stages 1-3: (m float64 [N], invalid) for the record p"""
    f = np.asarray(fg, np.float64)[p["fg_start"]:p["fg_start"] + p["fg_len"]] / 32768.0
    b = np.asarray(bg, np.float64)[(p["bg_offset"] + np.arange(N)) % len(bg)] / 32768.0
    nf, nb = np.linalg.norm(f), np.linalg.norm(b)
    if nf == 0 or nb == 0:
        return np.zeros(N), True
    g = 10.0 ** (p["snr_db"] / 20.0) * nb / nf
    m = b.copy()
    m[p["start"]:p["start"] + f.size] += g * f
    return m / 2.0, False


def check_record(p, fg_lens, bg_lens, rir_lens, N):
    """The refusals of oww_mix_clips for one record (ValueError)"""
    if not 0 <= p["fg"] < len(fg_lens) or not 0 <= p["bg"] < len(bg_lens) or not -1 <= p["rir"] < len(rir_lens):
        raise ValueError("index out of range")
    if p["fg_start"] < 0 or p["fg_len"] < 0 or p["fg_start"] + p["fg_len"] > fg_lens[p["fg"]]:
        raise ValueError("foreground window outside its clip")
    if bg_lens[p["bg"]] <= 0 or not 0 <= p["bg_offset"] < bg_lens[p["bg"]]:
        raise ValueError("background offset")
    if p["start"] < 0 or p["start"] + p["fg_len"] > N:
        raise ValueError("start + fg_len > N")
    if p["rir"] >= 0 and not 0 < rir_lens[p["rir"]] <= N:
        raise ValueError("rir length")
    if not (np.isfinite(p["snr_db"]) and np.isfinite(p["volume"])):
        raise ValueError("non-finite")


def mix_ref(fg_clips, bg_clips, rirs, params, N):
    """(int16 [n, N], valid bool [n], v float64 [n, N], tau float64 [n, N])"""
    if N <= 0:
        raise ValueError("N <= 0")
    rirs = [] if rirs is None else rirs
    for p in params:
        check_record(p, [len(c) for c in fg_clips], [len(c) for c in bg_clips], [len(h) for h in rirs], N)
    n = len(params)
    out, valid = np.zeros((n, N), np.int16), np.zeros(n, bool)
    V, T = np.zeros((n, N)), np.zeros((n, N))
    for i, p in enumerate(params):
        m, bad = mixture(fg_clips[p["fg"]], bg_clips[p["bg"]], N, p)
        if bad:
            continue
        am = np.abs(m)
        err = U * am                                     # m stored as float32
        if p["rir"] >= 0:
            h = np.asarray(rirs[p["rir"]], np.float64)
            L = h.size
            d = int(np.argmax(np.abs(h)))
            y = _circ(m, h, d, N)
            S = _circ(am, np.abs(h), d, N)
            W = _circ(am, np.ones(L), d, N)
            hs = 2.0 ** int(np.frexp(np.abs(h).max())[1]) if np.abs(h).max() > 0 else 1.0
            adds = 3 * 4 * ((L - 1) // 64 + 2) + 16
            err = (U * adds + SPLIT_OP + U) * S + SUB16 * (np.abs(h).sum() + hs * W) + _circ(err, np.abs(h), d, N)
            a0 = am.mean()
            my = np.abs(y).mean()
            s = a0 / (my + 1e-14)
            rel = err.mean() / max(my, 1e-300)           # the rescale's own error
            err = (err + np.abs(y) * rel) * s
            y = y * s
        else:
            y = m
        if p["volume"] >= 0:
            mx = y.max()
            if not mx > 0:
                continue
            F = p["volume"] / mx
            k = np.argmax(y)
            err = F * (err + np.abs(y) * err[k] / mx)
        else:
            F = 1.0 / max(np.abs(y).max(), 1.0)
            k = np.argmax(np.abs(y))
            err = F * (err + (np.abs(y) * err[k] / np.abs(y[k]) if np.abs(y).max() > 1 else 0))
        v = y * F * 32767.0
        q = np.clip(np.trunc(v), -32768, 32767).astype(np.int16)
        out[i], V[i], T[i] = q, v, 32767.0 * err + 1e-9 * np.abs(v) + 1e-9
        valid[i] = q.max() != 0
    return out, valid, V, T


def assert_int16_match(dev, q, v, tau, what=""):
    """dev == q except where v lies within tau of a truncation boundary; there |dev - q| <= 1"""
    dev = np.asarray(dev, np.int64)
    q = np.asarray(q, np.int64)
    lo = np.clip(np.trunc(v - tau), -32768, 32767)
    hi = np.clip(np.trunc(v + tau), -32768, 32767)
    near = lo != hi
    diff = np.abs(dev - q)
    bad = (diff > 1) | ((diff == 1) & ~near)
    assert not bad.any(), (f"{what}: {int(bad.sum())} samples off, first at {np.argwhere(bad)[0].tolist()}: "
                           f"device {dev[bad][0]}, reference {q[bad][0]}, v {v[bad][0]:.6f}, tau {tau[bad][0]:.3g}")
    return int(near.sum())
