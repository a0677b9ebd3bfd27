"""-m gpu: the log-mel frontend against float64, its three kernels pinned to each other bit for bit, and the PCM layouts
the step calls take.

* The stateless kernel (oww_melspectrogram, affine 0) against oracle.mel.mel_power_f64 under the round-off bound of
  tests/test_frontend_bound.py, over the signal zoo at odd and even lengths and 1, 3, the zoo's size and 1000 clips per
  call; affine 1 is the raw output's x/10+2 in float32, bit for bit.
* Custom constants through oww_load_mel: filters on bin 0, 128, 255 and the Nyquist bin, one of the full 32-tap support
  with interior zeros, one all zero, and a window that is not Hann.  A 33-tap filter is refused and changes nothing.
* The bound has teeth on the device: four small perturbations of the constants, loaded through oww_load_mel, fail it
  by at least 2x against the unperturbed reference.
* Streaming rows equal stateless rows bit for bit: after every call a stream's new mel rows are the stateless call's
  rows of that call's own span (the previous 480 samples and its chunks; after a reset its chunks only).  This pins the
  fused step kernel's frontend and the general streaming path to the float64-checked stateless kernel.
* PCM layouts: odd strides, gaps full of full-scale poison, a base pointer on an odd sample and column slices of a wider
  buffer give the bits of dense buffers in every step call.
* Argument checks: short strides, wrong shapes, dtypes and devices are refused before anything is enqueued."""
import ctypes as C

import numpy as np
import pytest

from helpers import emb_weights, head
from oracle import mel as M
from test_frontend_bound import (C_ROUNDOFF, GUARD_MARGIN, bin_sweep, bound_ratio, default_constants, perturbations,
                                 zoo)

pytestmark = pytest.mark.gpu

LENGTHS = (512, 513, 671, 672, 1280, 1761, 16000, 160001)
CHUNK = 1280
EUNSUPPORTED = -4
EINVAL = -1


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _stream(torch):
    return torch.cuda.current_stream().cuda_stream


def _mel_ctx(window=None, fb=None):
    from openwakeword_b200 import _native
    ctx = _native.Context(device=0, max_chunks=1)
    ctx.load_mel(window, fb)
    return ctx


def _stateless(torch, ctx, x, affine):
    """oww_melspectrogram of the clips x int16 [n, L] in one call -> float32 [n, T, 32]."""
    x = np.ascontiguousarray(x, np.int16)
    n, L = x.shape
    out = torch.empty((n, M.n_frames(L), 32), dtype=torch.float32, device="cuda")
    ctx.melspectrogram(torch.from_numpy(x).cuda(), n, L, out, affine=affine, stream=_stream(torch))
    return out.cpu().numpy()


def _calls(L):
    """(group, clip) lists of the calls run at length L: the whole zoo in one call, 1 clip, 3 clips, and 1000 clips at
    three lengths."""
    z = zoo(L, seed=L)
    calls = [z, z[L % len(z):][:1], [z[i % len(z)] for i in (3, 11, 20)]]
    if L in (513, 1761, 16000):
        big = [c for s in range(1, 40) for c in zoo(L, seed=1000 * s + L)]
        calls.append(big[:1000])
    return calls


def _check_calls(torch, ctx, calls, window, fb, per=None, affine_check=True):
    """Runs each call raw (and with affine 1) against the float64 reference of (window, fb) -> the worst bound ratio at
    C_ROUNDOFF; per: dict that receives the worst ratio at C = 1 of each signal group."""
    worst = 0.0
    for call in calls:
        x = np.stack([c[1] for c in call])
        raw = _stateless(torch, ctx, x, 0)
        if affine_check:
            aff = _stateless(torch, ctx, x, 1)
            assert np.array_equal(aff, raw / np.float32(10.0) + np.float32(2.0)), "affine 1 is not raw/10 + 2 in float32"
        for (g, xi), di in zip(call, raw):
            m, E = M.mel_power_f64(xi, window, fb)
            worst = max(worst, bound_ratio(di, m, E, C_ROUNDOFF))
            if per is not None:
                per[g] = max(per.get(g, 0.0), bound_ratio(di, m, E, 1.0))
    return worst


def _sweep_calls():
    calls = []
    for L in (513, 1761):
        g, x = bin_sweep(L, seed=L)
        calls.append(list(zip(g, x)))
    return calls


def test_stateless_against_float64(torch_cuda, built_library):
    torch = torch_cuda
    win, fb = default_constants()
    ctx = _mel_ctx()
    per = {}
    at_c = max(_check_calls(torch, ctx, _calls(L), win, fb, per) for L in LENGTHS)
    at_c = max(at_c, _check_calls(torch, ctx, _sweep_calls(), win, fb, per))
    worst = max(per.values())
    print(f"\nCUDA frontend, worst ratio at C = 1 per group: { {g: round(v, 4) for g, v in sorted(per.items())} }")
    print(f"worst {worst:.4f} at C = 1, {at_c:.4f} at C = {C_ROUNDOFF:g} "
          f"(smallest power of two >= 4x the C = 1 ratio: {2.0 ** np.ceil(np.log2(4 * worst)):g})")
    assert at_c <= 1.0
    assert 4 * worst <= C_ROUNDOFF, "C_ROUNDOFF no longer leaves 4x headroom over the kernel's round-off"
    ctx.close()


def _custom_constants():
    """A filterbank that reaches the spectrum's edges and the kernels' support limit, and a full-width Hamming window."""
    _, base = default_constants()
    fb = base.copy()
    fb[:, :8] = 0.0
    fb[0:6, 0] = np.linspace(1.0, 0.2, 6)                   # bin 0 (DC)
    fb[120:137, 1] = np.hanning(19)[1:-1]                  # around bin 128
    fb[250:256, 2] = 0.3                                   # up to bin 255
    fb[240:257, 3] = np.linspace(0.1, 1.0, 17)              # up to the Nyquist bin
    taps = np.linspace(0.5, 1.5, 32)
    taps[[5, 6, 17, 30]] = 0.0                             # interior zeros: the support stays 32 bins
    fb[60:92, 4] = taps
    # fb[:, 5] stays all zero: -100 dB before the clamp
    fb[256, 6] = 2.0                                       # the Nyquist bin alone
    fb[7:39, 7] = 1.0 / 32                                 # 32 taps, flat
    n = np.arange(M.N_FFT)
    win = (0.54 - 0.46 * np.cos(2 * np.pi * n / M.N_FFT)).astype(np.float32)
    return win, fb.astype(np.float32)


def test_custom_constants(torch_cuda, built_library):
    torch = torch_cuda
    win, fb = _custom_constants()
    ctx = _mel_ctx(win, fb)
    worst = 0.0
    for L in (512, 1761, 16000, 160001):
        worst = max(worst, _check_calls(torch, ctx, _calls(L)[:3], win, fb))
    worst = max(worst, _check_calls(torch, ctx, _sweep_calls(), win, fb))
    print(f"\ncustom constants, worst ratio at C = {C_ROUNDOFF:g}: {worst:.4f}")
    assert worst <= 1.0
    # the all-zero filter: -100 dB, or the call's floor where that is higher
    sil = _stateless(torch, ctx, np.zeros((1, 4000), np.int16), 0)[0]
    np.testing.assert_allclose(sil, -100.0, rtol=0, atol=1e-4)
    loud = np.random.default_rng(1).integers(-32768, 32768, (1, 4000)).astype(np.int16)
    raw = _stateless(torch, ctx, loud, 0)[0]
    assert (raw[:, 5] == raw.max() - np.float32(80.0)).all()

    # a 33-tap filter is refused and leaves the handle as it was
    before = _stateless(torch, ctx, loud, 1)
    bad = fb.copy()
    bad[:, 9] = 0.0
    bad[100:133, 9] = 0.5
    w_ = np.ascontiguousarray(win)
    rc = ctx.lib.oww_load_mel(ctx.h, w_.ctypes.data, np.ascontiguousarray(bad).ctypes.data)
    assert rc == EUNSUPPORTED, rc
    assert np.array_equal(_stateless(torch, ctx, loud, 1), before)
    bad[100:132, 9] = 0.5
    bad[132, 9] = 0.0                                      # 32 taps: accepted
    ctx.load_mel(win, bad)
    ctx.close()


def test_constants_change_the_configuration_key(torch_cuda, built_library):
    from openwakeword_b200 import _native
    from openwakeword_b200.engine import StreamEngine
    eng = StreamEngine([head("alexa_v0.1")], 3, embedding=emb_weights())
    _, k0 = eng.ctx.stream_state_info()
    win, fb = _custom_constants()
    eng.ctx.load_mel(win, fb)
    _, k1 = eng.ctx.stream_state_info()
    assert k1 != k0
    bad = fb.copy()
    bad[:, 9] = 0.0
    bad[100:133, 9] = 0.5
    with pytest.raises(_native.NativeError, match="spans 33"):
        eng.ctx.load_mel(win, bad)
    assert eng.ctx.stream_state_info()[1] == k1            # a refused load changes nothing
    eng.ctx.load_mel(win, None)
    assert eng.ctx.stream_state_info()[1] not in (k0, k1)
    eng.ctx.load_mel()
    assert eng.ctx.stream_state_info()[1] == k0
    eng.ctx.close()


def test_guards_fail_the_bound_on_the_device(torch_cuda, built_library):
    torch = torch_cuda
    win, fb = default_constants()
    calls = _calls(1761)[:1] + _calls(16000)[:1] + _sweep_calls()
    margins = {}
    for name, (pw, pfb) in sorted(perturbations().items()):
        ctx = _mel_ctx(pw, pfb)
        margins[name] = _check_calls(torch, ctx, calls, win, fb, affine_check=False)
        ctx.close()
    print(f"\nguard margins at C = {C_ROUNDOFF:g}: { {k: round(v, 2) for k, v in margins.items()} }")
    assert min(margins.values()) >= GUARD_MARGIN, margins


# ---- streaming rows against stateless rows ------------------------------------------------------------------------

KINDS = ("noise", "early_burst", "burst_chunk2", "tail_only", "tone", "silence", "full_scale", "lsb")


def _call_pcm(rng, kind, k, t):
    """One call's k*1280 samples of a stream of `kind` at call index t."""
    L = k * CHUNK
    lsb = rng.integers(-1, 2, L)
    if kind == "noise":
        x = rng.integers(-3000, 3000, L)
    elif kind == "early_burst":                      # body samples 0..40 only: a fresh stream's kept frames never see it
        x = lsb
        x[:41] = rng.integers(-32768, 32768, 41)
    elif kind == "burst_chunk2":                     # chunk 2 of a multi-chunk call (every other call of one chunk)
        x = lsb
        if k >= 2:
            x[CHUNK + 200:CHUNK + 900] = rng.integers(-32768, 32768, 700)
        elif t % 2:
            x[200:900] = rng.integers(-32768, 32768, 700)
    elif kind == "tail_only":                        # content in the last 480 samples, then a silent call
        x = np.zeros(L)
        if t % 2 == 0:
            x[-480:] = rng.integers(-32768, 32768, 480)
    elif kind == "tone":
        x = 20000 * np.cos(2 * np.pi * rng.uniform(50, 7900) * np.arange(L) / M.SR)
    elif kind == "silence":
        x = np.zeros(L)
    elif kind == "full_scale":
        x = rng.integers(-32768, 32768, L)
    else:
        x = lsb
    return np.clip(x, -32768, 32767).astype(np.int16)


def _rows_match_stateless(torch, eng, counts, resets, seed):
    """Drives eng with per-call counts [calls][B] (ragged when a call's counts differ; 0 = held) and stream resets
    {call index: ids}; after every call each stepping stream's newest mel rows must be the stateless rows of its span."""
    rng = np.random.default_rng(seed)
    B = eng.n_streams
    mc = eng.ctx.max_chunks
    prev = [None] * B                                # last 480 samples of the stream's last call; None = fresh
    n_cmp = 0
    for t, c in enumerate(counts):
        c = np.asarray(c, np.int32)
        if t in resets:
            eng.reset_async(stream_ids=resets[t])
            for b in resets[t]:
                prev[b] = None
        body = [_call_pcm(rng, KINDS[b % len(KINDS)], int(c[b]), t) if c[b] else None for b in range(B)]
        x = np.zeros((B, mc * CHUNK), np.int16)
        for b in range(B):
            if c[b]:
                x[b, :c[b] * CHUNK] = body[b]
        d = torch.from_numpy(x).cuda()
        if c.max() == 0:
            continue
        if (c == c[0]).all():
            eng.step(d[:, :int(c[0]) * CHUNK] if t % 2 else d, int(c[0]))
        else:
            eng.step_ragged(d, c)
        groups = {}
        for b in range(B):
            if c[b]:
                span = body[b] if prev[b] is None else np.concatenate([prev[b], body[b]])
                groups.setdefault(span.size, []).append((b, span))
                prev[b] = body[b][-480:]
        for L, items in groups.items():
            ref = _stateless(torch, eng.ctx, np.stack([s for _, s in items]), 1)
            for (b, _), r in zip(items, ref):
                got = eng.ctx.get_mel(b, r.shape[0])
                assert np.array_equal(got, r), (f"call {t} stream {b} ({KINDS[b % len(KINDS)]}, {c[b]} chunks, "
                                                f"span {L}): max |diff| {np.abs(got - r).max():.3e}")
                n_cmp += 1
    return n_cmp


def _engine(B, max_chunks, mel=None, **kw):
    from openwakeword_b200.engine import StreamEngine
    eng = StreamEngine([head("alexa_v0.1"), head("timer_v0.1")], B, embedding=emb_weights(), max_chunks=max_chunks, **kw)
    if mel is not None:
        eng.ctx.load_mel(*mel)
    return eng


STREAM_CONFIGS = {
    "fused_b1": dict(B=1, mc=1),
    "fused_b7": dict(B=7, mc=1),
    "fused_b300": dict(B=300, mc=1),
    "fused_b7_custom": dict(B=7, mc=1, custom=True),
    "no_fuse": dict(B=7, mc=1, kw=dict(fuse_step=False)),
    "mode3_mc4": dict(B=9, mc=4),
    "mode3_mc4_custom": dict(B=9, mc=4, custom=True),
    "mode0_mc4": dict(B=9, mc=4, kw=dict(cnn_mode=0)),
    "mode2_mc4": dict(B=9, mc=4, kw=dict(cnn_mode=2)),
    "ragged_mode3": dict(B=23, mc=4, ragged=True),
    "ragged_mode0": dict(B=23, mc=4, ragged=True, kw=dict(cnn_mode=0)),
}


@pytest.mark.parametrize("name", list(STREAM_CONFIGS))
def test_streaming_rows_equal_stateless_rows(torch_cuda, built_library, name):
    torch = torch_cuda
    cfg = STREAM_CONFIGS[name]
    B, mc, n_calls = cfg["B"], cfg["mc"], 26
    eng = _engine(B, mc, _custom_constants() if cfg.get("custom") else None, **cfg.get("kw", {}))
    rng = np.random.default_rng(len(name))
    sub_a = sorted(set(rng.choice(B, max(1, B // 3), replace=False).tolist()))
    sub_b = sorted(set(rng.choice(B, max(1, B // 4), replace=False).tolist()))
    if cfg.get("ragged"):
        counts = rng.integers(0, mc + 1, (n_calls, B))
        counts[0] = np.arange(B) % (mc + 1)
        resets = {9: sub_a, 17: sub_b}
    else:
        ks = [1] * n_calls if mc == 1 else [1 + (t * 5 + t // 4) % mc for t in range(n_calls)]
        if mc > 1:
            ks[9], ks[17] = 1, 3                          # first calls after the resets: 1 chunk and 3 chunks
        counts = [[k] * B for k in ks]
        resets = {9: sub_a, 17: sub_b}
    n = _rows_match_stateless(torch, eng, counts, resets, seed=7)
    print(f"\n{name}: {n} stream-calls bit-identical to the stateless kernel")
    assert n > 0
    eng.ctx.close()


# ---- PCM layouts ---------------------------------------------------------------------------------------------------

POISON = np.array([32767, -32768], np.int16)


def _laid_out(torch, x, layout, device=True):
    """x int16 [B, row] dense -> (buffer that must stay alive, base address, stride) of the layout; poison elsewhere."""
    B, row = x.shape
    off, stride = {"odd_stride": (0, row + 1), "gap_poison": (0, row + 640), "odd_base": (1, row + 3)}[layout]
    flat = np.resize(POISON, off + B * stride + 8).astype(np.int16)
    for b in range(B):
        flat[off + b * stride:off + b * stride + row] = x[b]
    if device:
        buf = torch.from_numpy(flat).cuda()
        return buf, buf.data_ptr() + 2 * off, stride
    return flat, flat.ctypes.data + 2 * off, stride


def _slice(torch, x, t):
    """x as a column slice of a wider [B, 8*1280] tensor full of poison, starting at an odd column on odd t."""
    B, row = x.shape
    wide = torch.from_numpy(np.resize(POISON, (B, 8 * CHUNK)).astype(np.int16)).cuda()
    c0 = (t % 3) * 1000 + (t % 2)
    wide[:, c0:c0 + row] = torch.from_numpy(x).cuda()
    return wide[:, c0:c0 + row]


def _same_state(a, b, B):
    for s in range(B):
        assert a.ctx.get_counts(s) == b.ctx.get_counts(s), s
        assert np.array_equal(a.ctx.get_mel(s, 76), b.ctx.get_mel(s, 76)), s
        assert np.array_equal(a.ctx.get_features(s, 120), b.ctx.get_features(s, 120)), s


LAYOUTS = ("odd_stride", "gap_poison", "odd_base", "column_slice")


@pytest.mark.parametrize("mode", [3, 0])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_pcm_layouts_device_steps(torch_cuda, built_library, mode, layout):
    """oww_step (fused one-chunk and two-chunk calls in mode 3, mode 0) and oww_step_ragged (the fused n = 1 path and
    the general path) on the layout against a twin fed dense buffers."""
    torch = torch_cuda
    B = 9
    rng = np.random.default_rng(5)
    dense, lay = _engine(B, 2, cnn_mode=mode), _engine(B, 2, cnn_mode=mode)
    schedule = [1, 1, 2, 1, "r01", 2, "r012", 1, "r01", "r012", 2, 1]
    for t, s in enumerate(schedule):
        if isinstance(s, str):
            c = rng.integers(0 if "0" in s else 1, 3 if "2" in s else 2, B).astype(np.int32)
            c[0], c[1] = 0, (2 if "2" in s else 1)                # ragged for sure
            n = int(c.max())
        else:
            c, n = None, s
        x = rng.integers(-32768, 32768, (B, n * CHUNK)).astype(np.int16)
        if c is not None:
            x[c == 0] = 0
        ref = torch.full((B, dense.n_cols), float("nan"), device="cuda")
        got = torch.full((B, lay.n_cols), float("nan"), device="cuda")
        xd = torch.from_numpy(x).cuda()
        if c is None:
            dense.step(xd, n, ref)
        else:
            dense.step_ragged(xd, c, ref)
        if layout == "column_slice":
            v = _slice(torch, x, t)
            if c is None:
                lay.step(v, n, got)
            else:
                lay.step_ragged(v, c, got)
        else:
            buf, addr, stride = _laid_out(torch, x, layout)
            if c is None:
                lay.ctx.step(addr, stride, n, got, _stream(torch))
            else:
                lay.ctx.step_ragged(addr, stride, c, got, _stream(torch))
            torch.cuda.synchronize()
            del buf
        assert np.array_equal(got.cpu().numpy(), ref.cpu().numpy(), equal_nan=True), (layout, t, s)
    _same_state(dense, lay, B)
    dense.ctx.close()
    lay.ctx.close()


@pytest.mark.parametrize("layout", ["odd_stride", "gap_poison", "odd_base"])
def test_pcm_layouts_host_steps(torch_cuda, built_library, layout):
    """oww_step_host and oww_step_host_ragged with stride != row (the library stages row by row) against dense calls."""
    B = 7
    rng = np.random.default_rng(6)
    dense, lay = _engine(B, 2), _engine(B, 2)
    for t in range(8):
        ragged = t % 2 == 1
        c = rng.integers(0, 3, B).astype(np.int32) if ragged else None
        if ragged:
            c[0], c[1] = 0, 2
        n = int(c.max()) if ragged else 1 + t % 3 // 2
        x = rng.integers(-32768, 32768, (B, n * CHUNK)).astype(np.int16)
        ref = np.full((B, dense.n_cols), 7.0, np.float32)
        got = ref.copy()
        buf, addr, stride = _laid_out(None, x, layout, device=False)
        if ragged:
            dense.step_host_ragged(x, c, ref)
            rc = lay.ctx.lib.oww_step_host_ragged(lay.ctx.h, addr, stride, c.ctypes.data, got.ctypes.data)
        else:
            dense.step_host(x, n, ref)
            rc = lay.ctx.lib.oww_step_host(lay.ctx.h, addr, stride, n, got.ctypes.data)
        assert rc == 0, lay.ctx.lib.oww_last_error(lay.ctx.h)
        assert np.array_equal(got, ref), (layout, t)
    _same_state(dense, lay, B)
    dense.ctx.close()
    lay.ctx.close()


# ---- argument checks --------------------------------------------------------------------------------------------------

def test_short_strides_are_refused(torch_cuda, built_library):
    """oww_step and oww_step_host(_submit) refuse a stride shorter than the call's rows before anything is enqueued
    (the buffers are large enough either way)."""
    torch = torch_cuda
    B = 5
    eng = _engine(B, 2)
    lib, h = eng.ctx.lib, eng.ctx.h
    d = torch.zeros((B, 2 * CHUNK), dtype=torch.int16, device="cuda")
    out = torch.empty((B, eng.n_cols), dtype=torch.float32, device="cuda")
    x = np.zeros((B, 2 * CHUNK), np.int16)
    sc = np.zeros((B, eng.n_cols), np.float32)
    n0 = eng.ctx.launch_count
    for n, stride in ((1, CHUNK - 1), (2, 2 * CHUNK - 1), (2, CHUNK), (1, 0)):
        assert lib.oww_step(h, d.data_ptr(), stride, n, out.data_ptr(), C.c_void_p(_stream(torch))) == EINVAL
        assert lib.oww_step_host(h, x.ctypes.data, stride, n, sc.ctypes.data) == EINVAL
        t = C.c_int(-1)
        assert lib.oww_step_host_submit(h, x.ctypes.data, stride, n, C.byref(t)) == EINVAL
        assert b"pcm_stride" in lib.oww_last_error(h)
    torch.cuda.synchronize()
    assert eng.ctx.launch_count == n0
    # the smallest valid stride still steps
    assert lib.oww_step(h, d.data_ptr(), CHUNK, 1, out.data_ptr(), C.c_void_p(_stream(torch))) == 0
    torch.cuda.synchronize()
    assert eng.ctx.launch_count > n0
    eng.ctx.close()


def test_host_wrappers_validate(torch_cuda, built_library):
    B = 5
    eng = _engine(B, 2)
    ctx = eng.ctx
    x = np.zeros((B, 2 * CHUNK), np.int16)
    sc = np.zeros((B, eng.n_cols), np.float32)
    n0 = ctx.launch_count
    bad_pcm = [x.astype(np.int32), np.asfortranarray(x), x[:, ::2], x[:-1], np.zeros((B + 1, 2 * CHUNK), np.int16),
               x[:, :CHUNK].copy(), x.ravel()]
    for p in bad_pcm:
        with pytest.raises(ValueError):
            ctx.step_host(p, 2, sc)
        with pytest.raises(ValueError):
            ctx.step_host_submit(p, 2)
        with pytest.raises(ValueError):
            ctx.step_host_ragged(p, np.full(B, 2, np.int32), sc)
        with pytest.raises(ValueError):
            ctx.step_host_ragged_submit(p, np.r_[np.ones(B - 1), 2].astype(np.int32))
    for s in (np.zeros((B, eng.n_cols + 1), np.float32), np.zeros((B - 1, eng.n_cols), np.float32),
              sc.astype(np.float64), np.zeros((eng.n_cols, B), np.float32).T, sc.ravel()):
        with pytest.raises(ValueError):
            ctx.step_host(x, 1, s)
        with pytest.raises(ValueError):
            ctx.step_host_ragged(x, np.ones(B, np.int32), s)
    assert ctx.launch_count == n0
    t = ctx.step_host_submit(x, 1)
    with pytest.raises(ValueError):
        ctx.step_host_collect(t, np.zeros((B, eng.n_cols + 1), np.float32))
    ctx.step_host_collect(t, sc)                                # the ticket is still there to collect
    ctx.step_host(x[:, :CHUNK + 7].copy(), 1, sc)              # longer rows than the call reads are fine
    ctx.close()


def test_engine_steps_validate(torch_cuda, built_library):
    torch = torch_cuda
    B = 5
    eng = _engine(B, 2)
    d = torch.zeros((B, 2 * CHUNK), dtype=torch.int16, device="cuda")
    out = torch.empty((B, eng.n_cols), dtype=torch.float32, device="cuda")
    n0 = eng.ctx.launch_count
    bad_pcm = [d.to(torch.int32), d[0], d[:-1], torch.zeros((B + 1, 2 * CHUNK), dtype=torch.int16, device="cuda"),
               d[:, ::2], d.t().contiguous().t(), d[:, :CHUNK], d.cpu()]
    for p in bad_pcm:
        with pytest.raises(ValueError):
            eng.step(p, 2)
        with pytest.raises(ValueError):
            eng.step_ragged(p, np.r_[np.ones(B - 1), 2].astype(np.int32))
    bad_out = [out[:-1], torch.empty((B, eng.n_cols + 1), device="cuda"), out.double(), out.cpu(),
               torch.empty((eng.n_cols, B), device="cuda").t(), torch.empty((B, 2 * eng.n_cols), device="cuda")[:, ::2]]
    for o in bad_out:
        with pytest.raises(ValueError):
            eng.step(d, 1, o)
        with pytest.raises(ValueError):
            eng.step_ragged(d, np.ones(B, np.int32), o)
    # short rows are refused as the library refuses a short stride too: callers that catch NativeError keep working
    from openwakeword_b200._native import NativeError
    with pytest.raises(NativeError):
        eng.step_ragged(d[:, :CHUNK], np.r_[np.ones(B - 1), 2].astype(np.int32))
    with pytest.raises(NativeError):
        eng.ctx.step_host(np.zeros((B, CHUNK), np.int16), 2, np.zeros((B, eng.n_cols), np.float32))
    torch.cuda.synchronize()
    assert eng.ctx.launch_count == n0
    # views with unit inner stride are fine: a column slice at an odd column, and a one-stream transposed column
    eng.step(d[:, 1:CHUNK + 1], 1, out)
    one = _engine(1, 1)
    col = torch.zeros((CHUNK, 1), dtype=torch.int16, device="cuda")
    one.step(col.t(), 1)
    torch.cuda.synchronize()
    assert eng.ctx.launch_count > n0
    eng.ctx.close()
    one.ctx.close()
