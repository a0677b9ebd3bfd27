"""Float64 restatement of the device resampler (include/owwb200.h, oww_set_input_rates / oww_ingest), written from its
definition and independent of the library: scipy's resample_poly filter design, a streaming polyphase FIR that keeps a
history of input samples, and A(S) = ceil(S*up/down) final outputs after S input samples."""
from math import gcd

import numpy as np

RATES = (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000)


def up_down(rate):
    if rate not in RATES:
        raise ValueError(f"rate {rate} is not in the table")
    g = gcd(16000, rate)
    return 16000 // g, rate // g


def taps(rate):
    """float64 h of the definition: sinc((k - half)/mr) * kaiser(N, 5), sum 1, times up (empty at 16000)"""
    up, down = up_down(rate)
    if up == down:
        return np.zeros(0)
    mr = max(up, down)
    half = 10 * mr
    k = np.arange(2 * half + 1)
    h = np.sinc((k - half) / mr) * np.kaiser(2 * half + 1, 5.0)
    return h / h.sum() * up


def final_outputs(S, up, down):
    """A(S): outputs that no longer depend on later input after S input samples"""
    return -(-S * up // down)


class StreamResampler:
    """One stream: feed packets, get the outputs each packet made final (float64), as y = upfirdn(h, x, up, down) of
    everything fed.  `h` (default: taps(rate)) may be the library's fp32 taps, to evaluate its sums in float64."""

    def __init__(self, rate, h=None):
        self.rate = rate
        self.up, self.down = up_down(rate)
        self.h = taps(rate) if h is None else np.asarray(h, np.float64)
        self.S = 0
        # the input samples before the packet, newest last (at least the 128 the device keeps)
        self.hist = np.zeros(max(len(self.h), 128), np.float64)

    def feed(self, x, abs_sum=False):
        """-> float64 outputs made final by x (and with abs_sum, sum_t |h_t * x_t| of each, the round-off scale)"""
        x = np.asarray(x, np.float64)
        if self.up == self.down:
            self.S += x.size
            return (x.copy(), np.abs(x)) if abs_sum else x.copy()
        a0, a1 = final_outputs(self.S, self.up, self.down), final_outputs(self.S + x.size, self.up, self.down)
        buf = np.concatenate((self.hist, x))                # buf[len(hist) + q - S] = input sample q
        base = len(self.hist) - self.S
        y = np.zeros(a1 - a0)
        s = np.zeros(a1 - a0)
        for j, i in enumerate(range(a0, a1)):
            n = i * self.down
            q0, p = divmod(n, self.up)
            hp = self.h[p::self.up]
            idx = base + q0 - np.arange(hp.size)
            v = np.where(idx >= 0, buf[np.maximum(idx, 0)], 0.0)
            y[j] = np.dot(hp, v)
            s[j] = np.abs(hp * v).sum()
        self.S += x.size
        self.hist = buf[-len(self.hist):] if len(self.hist) else self.hist
        return (y, s) if abs_sum else y


def to_int16(y):
    """round half to even, saturating"""
    return np.clip(np.rint(y), -32768, 32767).astype(np.int16)
