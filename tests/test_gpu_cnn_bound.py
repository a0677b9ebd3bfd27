"""-m gpu: every embedding-CNN layer and the heads' Linear layers against float64 with the per-element round-off bounds
of tests/test_cnn_bound.py.

CNN: oww_debug_layer (layers 0-18) and oww_embed_windows (layer 19) on 130 windows (the last 128-row tile of every
layer is ragged): the frontend zoo's signals, silence, the all-ones reset window, windows half at the -80 dB floor and
noise at three levels.  Each layer's reference is computed from the device's output of the layer before.  cnn_mode 2 at
split points 2, 11 and 20 runs every tc_conv_kernel<CGP, NP, TERMS> instance, the hi/lo (out_split) epilogues, the split
and plain pools and tc_conv0_kernel; cnn_mode 0 runs cnn_fp32.cu.  Four weight sets: two seeds, and the first with every
layer's weights x 2^-14 and x 2^17 (BatchNorm compensating, the same network): the engine's precision must not depend on
the scale of a layer's weights.

Heads: Linear layers with final 'none' (raw GEMM outputs) on heads_tc.cu at 3 terms and at 1 term, heads.cu, the grouped
streaming heads (heads_grp.cu, on features read back with oww_get_features) and the heads inside the fused step kernel.

Streaming at split points 3 and 7: feature rows bit for bit against oww_predict_clips_ragged's embeddings."""
import contextlib

import numpy as np
import pytest

from helpers import emb_weights
from test_cnn_bound import (C_ROUNDOFF, N_CONV, bound_head, bound_windows, c_needed, head_bound_parts, head_features,
                            layer_bound_parts, layer_modes, layer_params, scaled_weights)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


_WINDOWS = {}


def _windows():
    if not _WINDOWS:
        g, w = bound_windows(98)
        assert w.shape == (130, 76, 32)
        _WINDOWS.update(groups=np.array(g), wins=w)
    return _WINDOWS["groups"], _WINDOWS["wins"]


WEIGHT_SETS = {"seed0": (0, 0), "seed1": (1, 0), "seed0_x2^-14": (0, -14), "seed0_x2^17": (0, 17)}
CNN_CONFIGS = {"mode2_split2": (2, 2), "mode2_split11": (2, 11), "mode2_split20": (2, 20), "mode0_fp32": (0, 20)}


def _weights(name):
    seed, k = WEIGHT_SETS[name]
    w = emb_weights(seed)
    return w if k == 0 else scaled_weights(w, k)


def _per_window(a):
    return a.reshape(a.shape[0], -1).max(1)


@pytest.mark.parametrize("wset", list(WEIGHT_SETS))
@pytest.mark.parametrize("config", list(CNN_CONFIGS))
def test_cnn_layers_within_the_bound(torch_cuda, built_library, config, wset):
    torch = torch_cuda
    from openwakeword_b200 import _native, weights as W
    mode, split_from = CNN_CONFIGS[config]
    groups, wins = _windows()
    n = len(wins)
    weights = _weights(wset)
    params = layer_params(weights)
    ctx = _native.Context(cnn_mode=mode, split_from=split_from if mode else None)
    with contextlib.closing(ctx):
        ctx.load_mel()
        ctx.load_embedding(W.pack_embedding_blob(weights))
        d = torch.from_numpy(wins).cuda()
        x, worst, worst_c, report = wins, 0.0, 0.0, []
        for li in range(N_CONV):
            ops, store = layer_modes(li, mode, split_from)
            w, s, b = params[li]
            y, A, B = layer_bound_parts(li, x, w, s, b, ops, store)
            if li < N_CONV - 1:
                out = torch.full(y.shape, np.nan, dtype=torch.float32, device="cuda")
                ctx.debug_layer(d, n, li, out)
            else:
                out = torch.full((n, 96), np.nan, dtype=torch.float32, device="cuda")
                ctx.embed_windows(d, n, out)
            torch.cuda.synchronize()
            dev = out.cpu().numpy().reshape(y.shape)
            r = np.abs(dev.astype(np.float64) - y) / (C_ROUNDOFF * A + B)
            r = np.where(np.isfinite(dev), r, np.inf)
            per = _per_window(r)
            by_group = {g: float(per[groups == g].max()) for g in dict.fromkeys(groups)}
            cn = c_needed(dev, y, A, B)
            report.append((li, float(per.max()), cn, by_group))
            print(f"{config} {wset} layer {li:2d} ({ops}, store {store}): worst ratio {per.max():.3g} at C = {C_ROUNDOFF:g} "
                  f"(C needed {cn:.3g}); by input group " + " ".join(f"{g} {v:.3g}" for g, v in by_group.items()))
            worst, worst_c = max(worst, float(per.max())), max(worst_c, cn)
            x = dev
    print(f"{config} {wset}: worst ratio {worst:.3g} at C = {C_ROUNDOFF:g}, worst C needed {worst_c:.3g}")
    bad = [(li, r) for li, r, _, _ in report if not r <= 1.0]
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------- streaming
@pytest.mark.parametrize("split", [3, 7])
def test_streaming_feature_rows_equal_the_clip_pass(torch_cuda, built_library, split):
    """The fused step kernel and the block-major late chain at split points 3 and 7 against oww_predict_clips_ragged's
    embedding rows (tc_conv_kernel in the window layout): feature rows bit for bit."""
    torch = torch_cuda
    from openwakeword_b200.engine import StreamEngine
    from helpers import head
    from test_gpu_bulk_edges import _padded, _steps
    from test_gpu_cnn_configs import _signals
    LEN, PAD, CHUNK, n = 12800, 2560, 1280, 37
    rng = np.random.default_rng(300 + split)
    clips = _signals(rng, n, LEN)
    hs = [head("alexa_v0.1"), head("timer_v0.1")]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    S = _steps(LEN + 2 * PAD)
    eng = StreamEngine(hs, n, embedding=emb_weights(), feature_init=fi, cnn_mode=3, split_from=split)
    padded = _padded(clips, PAD)
    with contextlib.closing(eng.ctx):
        for s in range(S):
            eng.step_host(np.ascontiguousarray(padded[:, s * CHUNK:(s + 1) * CHUNK]), 1)
        feats = np.stack([eng.ctx.get_features(b, S) for b in range(n)])
    ref = StreamEngine(hs, 1, embedding=emb_weights(), cnn_mode=3, split_from=split)
    d = torch.from_numpy(np.ascontiguousarray(clips).reshape(-1)).cuda()
    off = np.arange(n + 1, dtype=np.int64) * LEN
    scores = torch.full((n * S, ref.n_cols), np.nan, dtype=torch.float32, device="cuda")
    emb = torch.full((n * S, 96), np.nan, dtype=torch.float32, device="cuda")
    with contextlib.closing(ref.ctx):
        ref.ctx.predict_clips_ragged(d, off, PAD, CHUNK, fi, scores, None, emb)
        torch.cuda.synchronize()
    bulk_f = emb.cpu().numpy().reshape(n, S, 96)
    print(f"split_from={split}: max |bulk - streaming| feature rows {np.abs(bulk_f - feats).max():.3e}")
    assert np.isfinite(bulk_f).all()
    assert np.array_equal(bulk_f, feats)


# ---------------------------------------------------------------------------------------------------- heads
def _bound_heads():
    """Single-Linear heads (n_in 3 / 16 / 34, widths 1 .. 128) and two-Linear heads without LayerNorm (ReLU between),
    all with final 'none'."""
    from openwakeword_b200 import weights as W
    hs = [bound_head(3, 1, 1), bound_head(16, 64, 2), bound_head(34, 128, 3), bound_head(16, 7, 4), bound_head(34, 33, 5)]
    for n_in, hidden, n_out, seed in ((16, 30, 5, 6), (3, 128, 2, 7), (34, 64, 128, 8)):
        hs.append(W.synthetic_head(n_in=n_in, hidden=hidden, n_blocks=0, n_out=n_out, layernorm=False, final="none", seed=seed))
    return hs


def _head_ratio(h, feats, got, terms):
    y, A, B = head_bound_parts(h, feats, terms)
    got = np.asarray(got, np.float64)
    r = np.where(np.isfinite(got), np.abs(got - y) / (C_ROUNDOFF * A + B), np.inf)
    return float(r.max()), c_needed(got, y, A, B)


@pytest.mark.parametrize("kind", ["tc3", "tc1", "cuda_core"])
def test_head_gemms_within_the_bound(torch_cuda, built_library, kind):
    """oww_head_predict on heads_tc.cu (3 terms: hi/lo bound; 1 term: fp16 bound) and heads.cu (fp32 bound), 1 / 130 /
    700 rows (ragged 128-row tiles)."""
    torch = torch_cuda
    from openwakeword_b200 import _native, weights as W
    terms = {"tc3": 3, "tc1": 1, "cuda_core": 0}[kind]
    ctx = _native.Context(cnn_mode=3, tc_heads=terms > 0, tc_heads_terms=max(terms, 1))
    with contextlib.closing(ctx):
        ctx.load_mel()
        ctx.load_embedding(W.pack_embedding_blob(emb_weights()))
        hs = _bound_heads()
        ids = [ctx.add_head(*W.head_desc(h), W.pack_head_blob(h)) for h in hs]
        rng = np.random.default_rng(40 + terms)
        worst, worst_c = 0.0, 0.0
        for n in (1, 130, 700):
            for hid, h in zip(ids, hs):
                f = head_features(rng, n, h["n_in"])
                n_out = h["layers"][-1]["W"].shape[1]
                out = torch.full((n, n_out), np.nan, dtype=torch.float32, device="cuda")
                ctx.head_predict(hid, torch.from_numpy(f).cuda(), n, out)
                torch.cuda.synchronize()
                r, cn = _head_ratio(h, f, out.cpu().numpy(), terms)
                print(f"{kind} n={n} head n_in {h['n_in']} dims {W.head_desc(h)[1]}: worst ratio {r:.3g} at C = {C_ROUNDOFF:g} "
                      f"(C needed {cn:.3g})")
                worst, worst_c = max(worst, r), max(worst_c, cn)
    print(f"{kind}: worst ratio {worst:.3g}, worst C needed {worst_c:.3g}")
    assert worst <= 1.0


@pytest.mark.parametrize("kind", ["grouped", "in_kernel"])
def test_streaming_heads_within_the_bound(torch_cuda, built_library, kind):
    """The grouped heads (heads_grp.cu, default split) and the heads inside the fused step kernel (split 20, fp32 FMA
    chains) on 130 streams, one chunk per call: each step's scores against the bound on the features the stream's ring
    holds after that step (oww_get_features).  The in-kernel case takes the heads of n_in <= 16 (the first-layer
    matrices that every group re-streams stay within oww_fused_heads_supported's limits) and requires every step after
    the first to be ONE launch, i.e. the heads ran inside the fused kernel and not as their own launch."""
    from openwakeword_b200.engine import StreamEngine
    from test_gpu_cnn_configs import _signals
    hs = _bound_heads()
    if kind == "in_kernel":
        hs = [h for h in hs if h["n_in"] <= 16]
    B, steps = 130, 4
    rng = np.random.default_rng(55)
    fi = rng.normal(0.3, 1.5, (41, 96)).astype(np.float32)
    fi[::5] *= 4.0
    pcm = _signals(rng, B, steps * 1280)
    kw = dict(split_from=20) if kind == "in_kernel" else {}
    eng = StreamEngine(hs, B, embedding=emb_weights(), feature_init=fi, cnn_mode=3, **kw)
    terms = 0 if kind == "in_kernel" else 3
    worst, worst_c, launches = 0.0, 0.0, []
    with contextlib.closing(eng.ctx):
        for s in range(steps):
            n0 = eng.ctx.launch_count
            got = eng.step_host(np.ascontiguousarray(pcm[:, s * 1280:(s + 1) * 1280]), 1).copy()
            launches.append(eng.ctx.launch_count - n0)
            col = 0
            for h in hs:
                n_out = h["layers"][-1]["W"].shape[1]
                f = np.stack([eng.ctx.get_features(b, h["n_in"]) for b in range(B)])
                r, cn = _head_ratio(h, f, got[:, col:col + n_out], terms)
                worst, worst_c = max(worst, r), max(worst_c, cn)
                col += n_out
    print(f"{kind} heads ({len(hs)} heads): worst ratio {worst:.3g} at C = {C_ROUNDOFF:g}, worst C needed {worst_c:.3g}; "
          f"launches per step {launches}")
    if kind == "in_kernel":
        assert all(k == 1 for k in launches[1:]), launches
    assert worst <= 1.0
