"""-m gpu: the tensor-core embedding-CNN path (cnn_mode = OWW_CNN_TC_WINDOW) against the oracle, layer by
layer (fp16 operands: activations and weights are rounded to fp16, accumulation is fp32), then end to
end on embeddings and scores (1e-3 gate)."""
import numpy as np
import pytest

from helpers import emb_weights, head

pytestmark = pytest.mark.gpu
TC = 2


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _ctx(mode, window_batch=0):
    from openwakeword_b200 import _native, weights as W
    ctx = _native.Context(cnn_mode=mode, window_batch=window_batch)
    ctx.load_mel()
    ctx.load_embedding(W.pack_embedding_blob(emb_weights()))
    return ctx


def _windows(rng, n):
    from oracle import mel
    out = []
    for i in range(n):
        amp = [300, 3000, 12000][i % 3]
        x = np.clip(rng.normal(0, amp, 12400 + 512), -32768, 32767).astype(np.int16)
        out.append(mel.melspectrogram(x)[:76])
    return np.stack(out).astype(np.float32)


@pytest.mark.parametrize("n", [3, 130])
def test_tc_layers_vs_oracle(torch_cuda, built_library, n):
    torch = torch_cuda
    from oracle import embedding
    rng = np.random.default_rng(5)
    wins = _windows(rng, n)
    _, ref_layers = embedding.forward(emb_weights(), wins, return_all=True)
    ctx = _ctx(TC)
    d = torch.from_numpy(wins).cuda()
    worst_rel = 0.0
    for li in range(19):
        ref = ref_layers[li]
        out = torch.empty(ref.shape, dtype=torch.float32, device="cuda")
        ctx.debug_layer(d, n, li, out)
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        err = np.abs(got - ref)
        scale = np.abs(ref).max()
        print(f"layer {li:2d} shape {ref.shape} max|ref| {scale:7.3f} max err {err.max():.4e} mean err {err.mean():.3e}")
        assert np.isfinite(got).all(), f"layer {li} has non-finite values"
        # fp16-operand budget: gates at ~2x the worst max err (1.7e-3 x scale) and mean err (4.3e-4) of this path
        assert err.max() < 4e-3 * max(scale, 1.0), f"layer {li}: max err {err.max()}"
        assert err.mean() < 9e-4, f"layer {li}: mean err {err.mean()}"
        worst_rel = max(worst_rel, err.max() / max(scale, 1.0))
    emb = torch.empty((n, 96), dtype=torch.float32, device="cuda")
    ctx.embed_windows(d, n, emb)
    torch.cuda.synchronize()
    e = np.abs(emb.cpu().numpy() - embedding.embed_windows(emb_weights(), wins))
    print("embedding max err", e.max(), "worst relative layer err", worst_rel)
    assert e.max() < 7e-3                       # measured 3.4e-3


def test_tc_scores_vs_fp32_and_oracle(torch_cuda, built_library):
    from openwakeword_b200.engine import StreamEngine
    from oracle import streaming, heads as oheads
    rng = np.random.default_rng(9)
    B, steps = 300, 6
    hs = [head("alexa_v0.1"), head("hey_mycroft_v0.1"), head("timer_v0.1"), head("big_v0.1")]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    pcm = np.clip(rng.normal(0, 2500, (B, steps * 1280)), -32768, 32767).astype(np.int16)
    pcm[::3] = rng.integers(-1000, 1000, (len(pcm[::3]), steps * 1280))
    res = {}
    for mode in (0, TC):
        eng = StreamEngine(hs, B, embedding=emb_weights(), feature_init=fi, cnn_mode=mode)
        res[mode] = np.stack([eng.step_host(np.ascontiguousarray(pcm[:, s * 1280:(s + 1) * 1280]), 1).copy()
                              for s in range(steps)], 1)
    d = np.abs(res[0] - res[TC])
    print("max |score_tc - score_fp32| =", d.max(), " mean", d.mean())
    assert d.max() < 1e-3
    # and both against the oracle on a sample of streams
    worst = {0: 0.0, TC: 0.0}
    for b in list(range(0, B, 13)):
        o = streaming.OracleAudioFeatures(emb_weights(), feature_init=fi)
        for s in range(steps):
            o(pcm[b, s * 1280:(s + 1) * 1280])
            ref = np.concatenate([oheads.forward(h, o.get_features(h["n_in"]))[0] for h in hs])
            for mode in (0, TC):
                worst[mode] = max(worst[mode], float(np.abs(ref - res[mode][b, s]).max()))
    print("max |score - oracle|: fp32", worst[0], " tc", worst[TC])
    assert worst[0] < 2e-5 and worst[TC] < 1e-3


def test_tc_incremental_vs_window_modes(torch_cuda, built_library):
    """cnn_mode 3 (fused incremental kernel, tails in HBM) against cnn_mode 2 (full window, same fp16
    quantisation points) and cnn_mode 0 (fp32): ragged group (B % 4 != 0), a 2-chunk step, a mid-stream
    reset of two streams (forces a re-prime) and the first-chunk-of-5-rows case."""
    from openwakeword_b200.engine import StreamEngine
    rng = np.random.default_rng(21)
    B = 37
    hs = [head("alexa_v0.1"), head("timer_v0.1")]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    plan = [1, 1, 1, 2, 1, 1, 1, 1, 1]
    pcm = np.clip(rng.normal(0, 2500, (B, sum(plan) * 1280)), -32768, 32767).astype(np.int16)
    pcm[::4] = rng.integers(-1000, 1000, (len(pcm[::4]), pcm.shape[1]))
    pcm[1::4, : pcm.shape[1] // 2] = 0
    out, feats, mels = {}, {}, {}
    for mode in (0, 2, 3, 13):        # 13 = mode 3 with the steady-state step kept as separate launches
        eng = StreamEngine(hs, B, embedding=emb_weights(), feature_init=fi, cnn_mode=mode % 10, max_chunks=2,
                           fuse_step=mode != 13)
        pos, rows = 0, []
        for si, n in enumerate(plan):
            if si == 6:
                eng.reset(fi, stream_ids=[3, 36])
            rows.append(eng.step_host(np.ascontiguousarray(pcm[:, pos:pos + n * 1280]), n).copy())
            pos += n * 1280
        out[mode] = np.stack(rows, 1)
        feats[mode] = np.stack([eng.ctx.get_features(b, 12) for b in (0, 3, 35, 36)])
    d32 = np.abs(out[3] - out[2])
    print("max |score_inc - score_window_tc| =", d32.max(), "  max |feat diff| =", np.abs(feats[3] - feats[2]).max())
    print("max |score_inc - score_fp32| =", np.abs(out[3] - out[0]).max())
    print("fused step vs separate launches: max |score diff| =", np.abs(out[3] - out[13]).max(),
          " max |feat diff| =", np.abs(feats[3] - feats[13]).max())
    assert np.abs(feats[3] - feats[2]).max() < 2e-3
    # same embeddings bit for bit; the scores differ only by the heads' arithmetic (in-kernel fp32 FMA chain when fused,
    # tensor-core hi/lo-split first layer when the heads run as their own launch): fp32 round-off
    assert np.array_equal(feats[3], feats[13]) and np.abs(out[3] - out[13]).max() < 2e-5
    assert d32.max() < 2e-4
    assert np.abs(out[3] - out[0]).max() < 1e-3


@pytest.mark.gpu
def test_fused_step_heads_with_awkward_shapes(torch_cuda, built_library):
    """The in-kernel heads phase (first layer through the smem ring in 96-row chunks, later layers in
    head_rows() chunks, tensors re-aligned to 16 bytes on upload) against the stand-alone heads kernel and the
    oracle, for widths that are not multiples of 4, a single-Linear head, a wide 256-unit later layer, softmax
    outputs and different n_in per head."""
    from openwakeword_b200.engine import StreamEngine
    from openwakeword_b200 import weights as W
    from oracle import heads as oh
    rng = np.random.default_rng(5)
    hs = [W.synthetic_head(n_in=16, hidden=30, n_blocks=1, n_out=1, seed=3),
          W.synthetic_head(n_in=3, hidden=7, n_blocks=2, n_out=3, layernorm=False, final="softmax", seed=4),
          W.synthetic_head(n_in=16, hidden=128, n_blocks=0, n_out=1, seed=5),
          W.synthetic_head(n_in=28, hidden=96, n_blocks=1, n_out=5, final="relu_softmax", seed=6)]
    single = W.synthetic_head(n_in=16, hidden=128, n_blocks=0, n_out=1, seed=7)
    single["layers"] = [dict(single["layers"][0])]                    # one Linear(1536, 1) + sigmoid
    single["layers"][0]["W"] = (rng.standard_normal((1536, 1)) / 40).astype(np.float32)
    single["layers"][0]["b"] = np.zeros(1, np.float32)
    single["layers"][0]["ln"] = None
    hs.append(single)
    wide = W.synthetic_head(n_in=16, hidden=128, n_blocks=1, n_out=2, final="softmax", seed=8)
    lw = wide["layers"]
    lw[1]["W"] = (rng.standard_normal((128, 256)) / np.sqrt(128)).astype(np.float32)
    lw[1]["b"] = rng.normal(0, 0.1, 256).astype(np.float32)
    lw[1]["ln"] = (rng.uniform(0.7, 1.3, 256).astype(np.float32), rng.normal(0.1, 0.2, 256).astype(np.float32))
    lw[2]["W"] = (rng.standard_normal((256, 2)) * 3 / 16).astype(np.float32)
    hs.append(wide)
    B = 19
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    pcm = np.clip(rng.normal(0, 2500, (B, 7 * 1280)), -32768, 32767).astype(np.int16)
    out, feats = {}, {}
    for fuse in (True, False):
        # split_from=20: plain fp16 everywhere, i.e. the configuration in which the heads run INSIDE the fused step kernel
        eng = StreamEngine(hs, B, embedding=emb_weights(), feature_init=fi, cnn_mode=3, fuse_step=fuse, split_from=20)
        out[fuse] = np.stack([eng.step_host(np.ascontiguousarray(pcm[:, k * 1280:(k + 1) * 1280]), 1).copy() for k in range(6)], 1)
        n0 = eng.ctx.launch_count
        last = eng.step_host(np.ascontiguousarray(pcm[:, 6 * 1280:]), 1).copy()
        assert (eng.ctx.launch_count - n0 == 1) == fuse            # the steady-state step really is one launch when fused
        out[fuse] = np.concatenate([out[fuse], last[:, None]], 1)
        feats[fuse] = np.stack([eng.ctx.get_features(b, 28) for b in range(B)])
    assert np.array_equal(feats[True], feats[False])
    print("awkward heads, fused vs separate launches: max |score diff| =", np.abs(out[True] - out[False]).max())
    assert np.abs(out[True] - out[False]).max() < 2e-5       # in-kernel fp32 heads vs tensor-core / heads.cu launch
    # the last step's scores from the device features through the NumPy heads
    col = 0
    for h in hs:
        n_in, n_out = h["n_in"], h["layers"][-1]["W"].shape[1]
        ref = oh.forward(h, feats[True][:, -n_in:])
        assert np.abs(out[True][:, -1, col:col + n_out] - ref).max() < 2e-5
        col += n_out


def _mixes(rng, n, length):
    """SURVEY.md 8d signal mixes: +-1000 noise, full scale, gated bursts (onset inside a call), silence, tone."""
    out = np.empty((n, length), np.int16)
    for i in range(n):
        k = i % 5
        if k == 0:
            x = rng.integers(-1000, 1000, length)
        elif k == 1:
            x = rng.uniform(-1, 1, length) * 32767
        elif k == 2:
            x = rng.normal(0, 8000, length) * ((np.arange(length) // 4000) % 2)
        elif k == 3:
            x = np.zeros(length)
        else:
            t = np.arange(length); x = 12000 * np.sin(2 * np.pi * 440 * t / 16000) + rng.normal(0, 20, length)
        out[i] = np.clip(x, -32768, 32767).astype(np.int16)
    return out


# launches of a steady one-chunk step in the default (precise) mode 3: fused frontend + conv 0-10 kernel, 9 split conv
# launches + 2 pools of the incremental late layers, ring append (2), heads (1-2)
@pytest.mark.parametrize("B,n_heads,max_launches", [(1024, 1, 16), (2048, 1, 16), (8192, 3, 16)])
def test_fused_step_bench_configs_vs_oracle(torch_cuda, built_library, B, n_heads, max_launches):
    """The configurations bench.py measures, checked against the ORACLE (not against another CUDA mode):
    default cnn_mode 3 (fused frontend + early-layer kernel, split-operand late layers) at B = 1024 and B = 2048
    (ragged last groups) and B = 8192 (configs[2]'s stream count, many rounds of groups per SM).
    14 calls: steady one-chunk steps (ONE launch each - asserted), a 2-chunk call, a mid-run reset of a stream subset
    (re-prime through the full-window kernels), then steady state again.  Scores of >= 64 sampled streams (first
    group, last ragged group, the reset streams, random others) must match the NumPy oracle within 1e-3, the mel ring
    within 5e-3 and the feature ring within the fp16-operand budget."""
    from openwakeword_b200.engine import StreamEngine
    from oracle import streaming, heads as oheads
    rng = np.random.default_rng(100 + B)
    hs = [head("alexa_v0.1"), head("timer_v0.1"), head("big_v0.1")][:n_heads]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    plan = [1, 1, 1, 1, 1, 2, 1, 1, 1, 1, 1, 1, 1, 1]
    reset_at = 9
    base = _mixes(rng, 40, sum(plan) * 1280)
    pick = rng.integers(0, 40, B)
    pcm = base[pick]                                            # [B, T] (40 distinct signals, scattered)
    G = 7
    last_group = list(range((B - 1) // G * G, B))
    reset_ids = sorted(set([3, B // 2, B - 1] + list(rng.integers(0, B, 5))))
    sample = sorted(set(list(range(G)) + last_group + reset_ids + list(rng.integers(0, B, 64))))
    assert len(sample) >= 64
    eng = StreamEngine(hs, B, embedding=emb_weights(), feature_init=fi, max_chunks=2)      # default mode = 3, fused
    oracles = {b: streaming.OracleAudioFeatures(emb_weights(), feature_init=fi) for b in sample}
    pos, worst, steady_steps = 0, 0.0, 0
    for si, nch in enumerate(plan):
        if si == reset_at:
            eng.reset(fi, stream_ids=reset_ids)
            for b in reset_ids:
                oracles[b].reset(feature_init=fi)
        x = np.ascontiguousarray(pcm[:, pos:pos + nch * 1280])
        pos += nch * 1280
        n0 = eng.ctx.launch_count
        got = eng.step_host(x, nch)
        steady_steps += int(eng.ctx.launch_count - n0 <= max_launches)
        for b in sample:
            assert oracles[b](x[b]) == nch * 1280
            ref = []
            for h in hs:
                g = [oheads.forward(h, oracles[b].get_features(h["n_in"], -h["n_in"] - i))[0] for i in range(nch - 1, -1, -1)]
                ref.append(np.max(np.stack(g), axis=0))
            d = float(np.abs(np.concatenate(ref) - got[b]).max())
            assert d < 1e-3, (si, b, d)
            worst = max(worst, d)
    print(f"B={B}: max |score - oracle| over {len(sample)} sampled streams x {len(plan)} calls = {worst:.3e}; "
          f"{steady_steps} of {len(plan)} calls took <= {max_launches} launch(es)")
    # every one-chunk step really ran as the fused step kernel (one launch; with head sets too large for the in-kernel
    # heads phase: fused frontend+CNN launch + heads launches) - also the first step and the step after the reset
    # (fresh streams start from the tails template): everything but the 2-chunk call
    assert steady_steps >= len(plan) - 1
    for b in (0, last_group[-1], reset_ids[0]):
        assert np.abs(eng.ctx.get_mel(b, 76) - oracles[b].melspectrogram_buffer[-76:]).max() < 5e-3
        assert np.abs(eng.ctx.get_features(b, 40) - oracles[b].feature_buffer[-40:]).max() < 8e-3


def _gain_head(gain, seed=1):
    """alexa-shaped head whose last Linear is scaled by `gain` with the bias re-centred, so the scores keep straddling
    0.5 (maximum sigmoid slope) while the logit's sensitivity to embedding error grows with the gain."""
    from openwakeword_b200 import weights as W
    h = W.synthetic_head(n_in=16, hidden=64, n_blocks=1, n_out=1, layernorm=True, final="sigmoid", seed=seed)
    last = h["layers"][-1]
    last["W"] = (last["W"] * gain).astype(np.float32)
    last["b"] = (last["b"] * gain).astype(np.float32)
    return h


# worst |score - oracle| allowed per (cnn_mode, gain): the fp32 path must hold 5e-4 everywhere; the fp16-operand
# tensor-core path is budgeted at 2x its measured error (filled from the first hardware run, see DESIGN.md section 3)
GAIN_BUDGET = {0: {1: 5e-4, 2: 5e-4, 4: 5e-4, 8: 5e-4, 16: 5e-4},
               3: {1: 1e-3, 2: 2e-3, 4: 4e-3, 8: 8e-3, 16: 1.6e-2}}


@pytest.mark.parametrize("mode", [0, 3])
def test_gain_sweep_precision_headroom(torch_cuda, built_library, mode):
    """Adversarial-gain parity: heads whose last Linear is scaled x1..x16 (scores near 0.5), all on one handle, streamed
    for 24 steps on 56 streams (8 groups of 7) against the oracle.  Prints the worst error per gain - the table
    DESIGN.md section 3 quotes - and holds each path to its budget."""
    from openwakeword_b200.engine import StreamEngine
    from oracle import streaming, heads as oheads
    rng = np.random.default_rng(77)
    gains = [1, 2, 4, 8, 16]
    hs = [_gain_head(g) for g in gains]
    B, steps = 56, 24
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    pcm = _mixes(rng, B, steps * 1280)
    pcm[3::5] = np.clip(rng.normal(0, 2500, (len(pcm[3::5]), steps * 1280)), -32768, 32767).astype(np.int16)   # no silence rows
    eng = StreamEngine(hs, B, embedding=emb_weights(), feature_init=fi, cnn_mode=mode)
    oracles = [streaming.OracleAudioFeatures(emb_weights(), feature_init=fi) for _ in range(B)]
    worst = np.zeros(len(gains))
    near = np.zeros(len(gains), int)
    for s in range(steps):
        x = np.ascontiguousarray(pcm[:, s * 1280:(s + 1) * 1280])
        got = eng.step_host(x, 1)
        for b in range(B):
            oracles[b](x[b])
            f = oracles[b].get_features(16)
            for j, h in enumerate(hs):
                ref = oheads.forward(h, f)[0, 0]
                worst[j] = max(worst[j], abs(float(ref) - float(got[b, j])))
                near[j] += int(0.2 < ref < 0.8)
    for g, w, n in zip(gains, worst, near):
        print(f"cnn_mode {mode} gain x{g:<2d}: max |score - oracle| = {w:.3e}   ({n} of {B * steps} reference scores in (0.2, 0.8))")
    assert near[0] > B * steps // 10, "the sweep must exercise the steep part of the sigmoid"
    for g, w in zip(gains, worst):
        assert w <= GAIN_BUDGET[mode][g], (mode, g, w)


def test_tc_heads_vs_oracle_and_cuda_core_heads(torch_cuda, built_library):
    """heads_tc.cu (first layer as a wgmma GEMM on fp16 hi/lo split operands, fp32 accumulate) against the oracle and
    against heads.cu on the same features: stateless (linear source; sample counts that leave a ragged last 128-row
    tile), widths 30 / 64 / 128 with padding to N = 32 / 64 / 128, n_in 3 / 16 / 34, softmax / sigmoid / relu finals.
    The 3-term split must be fp32-grade (2e-5); the 1-term variant is held to the fp16 budget."""
    torch = torch_cuda
    from openwakeword_b200 import _native, weights as W
    from oracle import heads as oh
    rng = np.random.default_rng(12)
    relu_head = W.synthetic_head(n_in=16, hidden=64, n_blocks=1, n_out=4, layernorm=True, final="relu_softmax", seed=13)
    relu_head["final"] = "relu"
    hs = [head("alexa_v0.1"), head("timer_v0.1"), head("big_v0.1"),
          W.synthetic_head(n_in=16, hidden=30, n_blocks=1, n_out=1, seed=3),
          W.synthetic_head(n_in=3, hidden=7, n_blocks=2, n_out=3, layernorm=False, final="softmax", seed=4),
          relu_head]
    worst = {}
    for terms, tc in ((3, True), (1, True), (3, False)):
        ctx = _native.Context(cnn_mode=3, tc_heads=tc, tc_heads_terms=terms)
        ctx.load_mel()
        ctx.load_embedding(W.pack_embedding_blob(emb_weights()))
        ids = [ctx.add_head(*W.head_desc(h), W.pack_head_blob(h)) for h in hs]
        w = 0.0
        for n in (1, 130, 700):
            for hid, h in zip(ids, hs):
                f = rng.normal(0.3, 1.5, (n, h["n_in"], 96)).astype(np.float32)
                f[::7] *= 4.0                                             # a few large-magnitude rows
                d = torch.from_numpy(f).cuda()
                n_out = h["layers"][-1]["W"].shape[1]
                out = torch.full((n, n_out), -7.0, dtype=torch.float32, device="cuda")
                ctx.head_predict(hid, d, n, out)
                torch.cuda.synchronize()
                ref = oh.forward(h, f)
                # unbounded outputs (the relu head) are judged relative to their magnitude
                w = max(w, float((np.abs(out.cpu().numpy() - ref) / np.maximum(1.0, np.abs(ref))).max()))
        worst[(terms, tc)] = w
        ctx.close()
    print("max |score - oracle|: tc 3-term", worst[(3, True)], " tc 1-term", worst[(1, True)], " cuda-core", worst[(3, False)])
    # inputs here reach |x| ~ 25 (4x the usual feature scale): fp32 FMA chains vs NumPy's blocked sums differ by ~1e-5;
    # the tensor core accumulates 3 x K/16 partial products with truncating fp32 adds - a few 1e-5 at this scale
    assert worst[(3, False)] < 3e-5
    assert worst[(3, True)] < 2e-4
    assert worst[(1, True)] < 2e-2


def test_partial_reset_keeps_the_fused_kernel_and_matches_oracle(torch_cuda, built_library):
    """One stream of 1024 is reset before EVERY step (stream-ordered oww_reset_async on the step's stream).  A reset
    writes the tails of the all-ones window into the stream's slots, so the very next step is an ordinary fused step
    for all 1024 streams - checked by parity with the oracle for the reset streams, their group neighbours and random
    others, and by the device time of reset + step (< 0.6 ms; round 1 pushed all 1024 streams through the full-window
    kernels after any reset: ~0.85 ms)."""
    torch = torch_cuda
    from openwakeword_b200.engine import StreamEngine
    from oracle import streaming, heads as oheads
    rng = np.random.default_rng(31)
    B, steps = 1024, 16
    hs = [head("alexa_v0.1")]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    base = _mixes(rng, 40, steps * 1280)
    pcm = base[rng.integers(0, 40, B)]
    eng = StreamEngine(hs, B, embedding=emb_weights(), feature_init=fi)
    reset_of_step = [int(x) for x in rng.integers(0, B, steps)]
    reset_of_step[5] = reset_of_step[4]                                   # the same stream twice in a row
    reset_of_step[9] = B - 1                                              # a stream of the ragged last group
    sample = sorted(set(reset_of_step + [r ^ 1 for r in reset_of_step] + [0, 7, B - 2] + list(rng.integers(0, B, 16))))
    orc = {b: streaming.OracleAudioFeatures(emb_weights(), feature_init=fi) for b in sample}
    dev = [torch.from_numpy(np.ascontiguousarray(pcm[:, s * 1280:(s + 1) * 1280])).cuda() for s in range(steps)]
    for s in range(3):                                                    # prime everything first
        got = eng.step(dev[s], 1)
        torch.cuda.synchronize()
        for b in sample:
            orc[b](pcm[b, s * 1280:(s + 1) * 1280])
    worst = 0.0
    t_steps = []
    for s in range(3, steps):
        r = reset_of_step[s]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        # a device-side delay ahead of e0: the whole reset + step is enqueued before e0 fires, so the events time the
        # device work rather than the host's enqueue after the oracle's CPU work between steps
        torch.cuda._sleep(5_000_000)
        e0.record()
        eng.reset_async(fi, stream_ids=[r])
        got = eng.step(dev[s], 1)
        e1.record()
        torch.cuda.synchronize()
        t_steps.append(e0.elapsed_time(e1))
        orc[r].reset(feature_init=fi)
        g = got.cpu().numpy()
        for b in sample:
            orc[b](pcm[b, s * 1280:(s + 1) * 1280])
            ref = oheads.forward(hs[0], orc[b].get_features(16))[0]
            d = float(np.abs(ref - g[b]).max())
            assert d < 1e-3, (s, b, d)
            worst = max(worst, d)
    ms = float(np.median(t_steps))
    print(f"one-of-{B} reset per step: max |score - oracle| = {worst:.3e}; median step {ms:.3f} ms (reset + step)")
    assert ms < 0.6         # reset + 15-launch step at 1024 streams, device time
    for b in (reset_of_step[-1], B - 1, 0):
        assert np.abs(eng.ctx.get_mel(b, 76) - orc[b].melspectrogram_buffer[-76:]).max() < 5e-3
        assert np.abs(eng.ctx.get_features(b, 30) - orc[b].feature_buffer[-30:]).max() < 8e-3


@pytest.mark.gpu
def test_grouped_heads_match_per_head_kernels(torch_cuda, built_library):
    """heads_grp.cu (one CTA per 128 streams and head, A operand from the fp16 mirror of the
    feature rings) against heads_tc.cu (one CTA per head, fp32 rings) and heads.cu (CUDA cores) on identical stream
    state: 300 streams (ragged third tile), head groups with n_in 16 / 34 / 3, widths 30..128, 1-4 Linear layers,
    LayerNorm on and off, sigmoid / softmax / relu-softmax / relu finals, a gated verifier pair; distinct feature
    histories per stream block (resets with different init rows), single-chunk steps, 3-chunk calls (windows ending
    0, 1, 2 rows back + max over chunks) and a partial reset between steps."""
    from openwakeword_b200.engine import StreamEngine
    from openwakeword_b200 import weights as W
    rng = np.random.default_rng(77)
    relu_head = W.synthetic_head(n_in=16, hidden=64, n_blocks=1, n_out=4, layernorm=True, final="relu_softmax", seed=13)
    relu_head["final"] = "relu"
    single = {"n_in": 16, "final": "softmax",                    # a head that is ONE Linear layer
              "layers": [{"W": (rng.standard_normal((1536, 5)) / 40).astype(np.float32),
                          "b": rng.normal(0, 0.1, 5).astype(np.float32), "ln": None}]}
    hs = [head("alexa_v0.1"), head("timer_v0.1"),
          W.synthetic_gated_head(seed_main=21, seed_verifier=22, threshold=0.5),
          W.synthetic_head(n_in=16, hidden=30, n_blocks=1, n_out=1, seed=3),
          W.synthetic_head(n_in=16, hidden=128, n_blocks=2, n_out=3, layernorm=True, final="softmax", seed=8),
          W.synthetic_head(n_in=3, hidden=7, n_blocks=2, n_out=3, layernorm=False, final="softmax", seed=4),
          relu_head, single]
    B, steps = 300, 6
    pcm = _mixes(rng, B, (steps + 3 * 2) * 1280)
    inits = [rng.normal(0.2, 1.0, (41, 96)).astype(np.float32) for _ in range(5)]
    outs = {}
    for key, kw in (("grp", {}), ("tc", {"group_heads": False}), ("cc", {"tc_heads": False})):
        eng = StreamEngine(hs, B, embedding=emb_weights(), max_chunks=3, **kw)
        for i, fi in enumerate(inits):                          # five blocks of streams with different histories
            eng.reset(fi[: 41 - 7 * i], stream_ids=list(range(i, B, 5)))
        got = []
        at = 0
        for k in range(steps):
            if k == 3:
                eng.reset(inits[1][:20], stream_ids=[0, 7, 129, 299])
            got.append(eng.step_host(np.ascontiguousarray(pcm[:, at:at + 1280]), 1).copy()); at += 1280
        for _ in range(2):
            got.append(eng.step_host(np.ascontiguousarray(pcm[:, at:at + 3 * 1280]), 3).copy()); at += 3 * 1280
        outs[key] = np.stack(got)
        eng.ctx.close()
    cols = outs["cc"].shape[-1]
    scale = np.maximum(1.0, np.abs(outs["cc"]))
    # the gated column switches between two networks at the threshold: skip entries where either side shows a main
    # score within 1e-3 of it (the two kernels may then legitimately decide differently)
    gate_col = 1 + 7
    def err(x, y):
        e = np.abs(x - y) / scale
        near = (np.abs(x[..., gate_col] - 0.5) < 1e-3) | (np.abs(y[..., gate_col] - 0.5) < 1e-3)
        e[..., gate_col] = np.where(near, 0.0, e[..., gate_col])
        return float(e.max())
    e_grp_tc, e_grp_cc, e_tc_cc = err(outs["grp"], outs["tc"]), err(outs["grp"], outs["cc"]), err(outs["tc"], outs["cc"])
    print(f"grouped vs per-head TC {e_grp_tc:.3e}; grouped vs CUDA cores {e_grp_cc:.3e}; per-head TC vs CUDA cores {e_tc_cc:.3e} ({cols} columns)")
    assert e_grp_tc < 5e-5 and e_grp_cc < 2e-4


@pytest.mark.gpu
@pytest.mark.parametrize("split_from,tol", [(15, 1e-3), (20, 1e-3)])
def test_split_from_variants_vs_oracle(torch_cuda, built_library, split_from, tol):
    """The other points of the precision / speed curve bench.py reports as `variants`: conv layers >= 15 on split operands
    (tc_inc_kernel<15> + a 5-layer late chain) and plain fp16 everywhere (one launch per step), against the oracle."""
    from openwakeword_b200.engine import StreamEngine
    from oracle import streaming, heads as oheads
    rng = np.random.default_rng(41)
    B, steps = 300, 12
    hs = [head("alexa_v0.1"), head("timer_v0.1")]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    pcm = _mixes(rng, B, steps * 1280)
    eng = StreamEngine(hs, B, embedding=emb_weights(), feature_init=fi, cnn_mode=3, split_from=split_from)
    got = np.stack([eng.step_host(np.ascontiguousarray(pcm[:, k * 1280:(k + 1) * 1280]), 1).copy() for k in range(steps)])
    eng.ctx.close()
    worst = 0.0
    for b in list(range(0, B, 23)) + [B - 1]:
        o = streaming.OracleAudioFeatures(emb_weights(), feature_init=fi)
        for k in range(steps):
            o(pcm[b, k * 1280:(k + 1) * 1280])
            col = 0
            for h in hs:
                ref = oheads.forward(h, o.get_features(h["n_in"]))[0]
                worst = max(worst, float(np.abs(ref - got[k, b, col:col + ref.size]).max()))
                col += ref.size
    print(f"split_from={split_from}: max |score - oracle| = {worst:.3e}")
    assert worst < tol
