"""-m gpu: configurations of the embedding CNN beside the default one, checked bit for bit against the configuration
whose arithmetic they share by construction (and against the oracle where the arithmetic differs):

* the bulk clip path (oww_predict_clips, one fully convolutional pass per layer) against streaming the same clips, at
  every split point cnn_mode 3 accepts;
* the incremental late chain with and without programmatic dependent launches, at every split point that has one;
* the sub-batching of the window modes over window_batch;
* the bulk clip path with heads that are not on the tensor cores, or cnn_mode 0, and on clips longer than one
  8192-step segment of its frontend."""
import numpy as np
import pytest

from helpers import emb_weights, head

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _signals(rng, n, length):
    """noise of +-1000, full-scale noise, gated bursts, silence, a tone - by row, cyclically."""
    out = np.empty((n, length), np.int16)
    t = np.arange(length)
    for i in range(n):
        k = i % 5
        if k == 0:
            x = rng.integers(-1000, 1000, length)
        elif k == 1:
            x = rng.uniform(-1, 1, length) * 32767
        elif k == 2:
            x = rng.normal(0, 8000, length) * ((t // 4000) % 2)
        elif k == 3:
            x = np.zeros(length)
        else:
            x = 12000 * np.sin(2 * np.pi * (300 + 40 * i) * t / 16000) + rng.normal(0, 20, length)
        out[i] = np.clip(x, -32768, 32767).astype(np.int16)
    return out


def _n_cols(hs):
    return sum(h["layers"][-1]["W"].shape[1] for h in hs)


# ---------------------------------------------------------------------------------------------------- clips
CLIP_SAMPLES, PAD, N_CLIPS = 20800, 16000, 9          # 1.3 s clips, 1 s of zeros on each side: 41 steps
_CLIPS = {}


def _clip_case():
    """Nine equal-length clips, their padded form and the oracle's raw scores for every step of predict_clip."""
    if _CLIPS:
        return _CLIPS
    from oracle import streaming, heads as oheads
    rng = np.random.default_rng(61)
    hs = [head("alexa_v0.1"), head("timer_v0.1")]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    clips = _signals(rng, N_CLIPS, CLIP_SAMPLES)
    z = np.zeros((N_CLIPS, PAD), np.int16)
    padded = np.concatenate([z, clips, z], 1)
    steps = len(range(0, padded.shape[1] - 1280, 1280))
    ref = np.zeros((N_CLIPS, steps, _n_cols(hs)), np.float32)
    for c in range(N_CLIPS):
        o = streaming.OracleAudioFeatures(emb_weights(), feature_init=fi)
        for s in range(steps):
            o(padded[c, s * 1280:(s + 1) * 1280])
            ref[c, s] = np.concatenate([oheads.forward(h, o.get_features(h["n_in"]))[0] for h in hs])
    _CLIPS.update(hs=hs, fi=fi, clips=clips, pad=PAD, padded=padded, steps=steps, ref=ref)
    return _CLIPS


def _predict_clips(torch, c, **kw):
    from openwakeword_b200.engine import StreamEngine
    eng = StreamEngine(c["hs"], 1, embedding=emb_weights(), feature_init=c["fi"], **kw)
    n, length = c["clips"].shape
    d = torch.from_numpy(c["clips"]).cuda()
    out = torch.full((n, c["steps"], eng.n_cols), -7.0, dtype=torch.float32, device="cuda")
    eng.ctx.predict_clips(d, n, length, c["pad"], c["fi"], out)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    eng.ctx.close()
    return got


def _stream_clips(c, **kw):
    """The padded clips streamed one chunk per call through a fresh engine of one stream per clip."""
    from openwakeword_b200.engine import StreamEngine
    eng = StreamEngine(c["hs"], len(c["padded"]), embedding=emb_weights(), feature_init=c["fi"], **kw)
    got = np.stack([eng.step_host(np.ascontiguousarray(c["padded"][:, s * 1280:(s + 1) * 1280]), 1).copy()
                    for s in range(c["steps"])], 1)
    eng.ctx.close()
    return got


@pytest.mark.parametrize("split_from", [3, 7, 11, 15, 20])
def test_bulk_clips_equal_streaming_at_every_split(torch_cuda, built_library, split_from):
    """oww_predict_clips' bulk path (one mel launch, fully convolutional tensor-core passes with split operands from
    split_from on, heads over every window) against the same padded clips streamed one chunk per call through a fresh
    engine at the same split.  Mel, CNN and feature rows are the same arithmetic; the heads may sum their first layer in
    another order (2e-6, as the bulk_predict test).  At 20 the streaming step runs the heads inside the fused kernel
    (fp32 FMA chain): 2e-5.  At 3 / 7 the clip pass runs the 48- and 72-channel split convs too, in the window layout
    (tc_conv_kernel<.,.,3>), against the block-major late chain of the streaming step."""
    torch = torch_cuda
    c = _clip_case()
    bulk = _predict_clips(torch, c, cnn_mode=3, split_from=split_from)
    stream = _stream_clips(c, cnn_mode=3, split_from=split_from)
    d = float(np.abs(bulk - stream).max())
    e_bulk, e_stream = float(np.abs(bulk - c["ref"]).max()), float(np.abs(stream - c["ref"]).max())
    print(f"split_from={split_from}: max |bulk - streaming| = {d:.3e}; max |score - oracle|: bulk {e_bulk:.3e}, "
          f"streaming {e_stream:.3e}")
    assert np.isfinite(bulk).all() and np.isfinite(stream).all()
    assert d <= (2e-5 if split_from == 20 else 2e-6)
    assert e_bulk < 1e-3 and e_stream < 1e-3


@pytest.mark.parametrize("kw", [pytest.param(dict(cnn_mode=3, tc_heads=False), id="mode3-cuda-core-heads"),
                                pytest.param(dict(cnn_mode=3, tc_heads=False, split_from=7), id="mode3-split7-cuda-core-heads"),
                                pytest.param(dict(cnn_mode=0), id="mode0")])
def test_predict_clips_bulk_path_without_tensor_core_heads(torch_cuda, built_library, kw):
    """oww_predict_clips with heads that are not on the tensor cores (tc_heads=False: heads.cu over the sliding windows)
    or with the fp32 CNN (mode 0: fully convolutional fp32 pass, heads.cu).  Bit for bit against streaming the same padded
    clips through a fresh engine of the same configuration (the same heads kernel on the same feature rows), against the
    oracle (1e-3), and against the bulk path of a default handle: CUDA-core vs tensor-core heads, 2e-4 relative (the
    bound of the grouped-heads test)."""
    torch = torch_cuda
    c = _clip_case()
    got = _predict_clips(torch, c, **kw)
    stream = _stream_clips(c, **kw)
    bulk = _predict_clips(torch, c)
    e_ref = float(np.abs(got - c["ref"]).max())
    e_bulk = float((np.abs(got - bulk) / np.maximum(1.0, np.abs(bulk))).max())
    print(f"{kw}: max |score - oracle| = {e_ref:.3e}; max relative |got - default bulk| = {e_bulk:.3e}; "
          f"max |got - streaming| = {np.abs(got - stream).max():.3e}")
    assert np.isfinite(got).all()
    assert np.array_equal(got, stream)
    assert e_ref < 1e-3
    assert e_bulk < 2e-4


@pytest.mark.parametrize("mode", [0, 3])
def test_predict_clips_longer_than_one_frontend_segment(torch_cuda, built_library, mode):
    """Two clips of 8230 steps (about 11 minutes): the bulk frontend runs them as two segments, [0, 8192) and
    [8192, 8230).  The second segment's first mel row is frame 65465, 4 frames into the streaming call (clamp group) of
    frames 65461..65468.  A loud burst covers only the first 4 of those frames and near-silence the rest, so the -80 dB
    clamp of the written frames depends on frames the second segment computes but does not write.  Against the same
    clips streamed through a 2-stream engine: bit for bit in mode 0 (heads.cu on both sides), 2e-6 in mode 3 (grouped
    heads over the clips' feature rows against the fp16 mirror of the rings)."""
    torch = torch_cuda
    rng = np.random.default_rng(83)
    steps = 8230
    length = 1280 * (steps + 1)
    burst = (160 * 65461, 160 * 65465)            # samples seen by frames 65461..65464 and none after them
    quiet = (burst[1], 160 * 65477 + 512)         # the rest of the group and the one after it
    clips = np.clip(rng.normal(0, 1000, (2, length)), -32768, 32767).astype(np.int16)
    clips[:, quiet[0]:quiet[1]] = rng.integers(-2, 3, (2, quiet[1] - quiet[0]))
    clips[:, burst[0]:burst[1]] = np.clip(rng.normal(0, 20000, (2, burst[1] - burst[0])), -32768, 32767)
    clips[1, burst[0]:burst[1]] //= 4
    c = dict(hs=[head("alexa_v0.1"), head("timer_v0.1")], fi=rng.normal(0, 1, (41, 96)).astype(np.float32),
             clips=clips, pad=0, padded=clips, steps=steps)
    got = _predict_clips(torch, c, cnn_mode=mode)
    stream = _stream_clips(c, cnn_mode=mode)
    d = float(np.abs(got - stream).max())
    print(f"cnn_mode {mode}: {steps} steps, max |bulk - streaming| = {d:.3e}")
    assert np.isfinite(got).all() and np.isfinite(stream).all()
    if mode == 0:
        assert np.array_equal(got, stream)
    else:
        assert d <= 2e-6


# ---------------------------------------------------------------------------------------------------- late chain
def _late_run(torch, monkeypatch, B, split_from, pdl=True):
    """10 device-resident calls of B streams (a 2-chunk call, a stream-ordered reset of three streams) -> all scores
    of every call and the feature rings (last 40 rows) of 64 sampled streams."""
    from openwakeword_b200.engine import StreamEngine
    rng = np.random.default_rng(B + split_from)
    hs = [head("alexa_v0.1"), head("timer_v0.1"), head("big_v0.1")]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    plan = [1, 1, 1, 2, 1, 1, 1, 1, 1, 1]
    reset_at, reset_ids = 6, [0, B // 2 + 1, B - 1]
    base = _signals(rng, 40, sum(plan) * 1280)
    pick = rng.integers(0, 40, B)
    fixed = reset_ids + [1, B - 2]
    sample = sorted(fixed + [int(x) for x in rng.permutation(B) if x not in fixed][:64 - len(fixed)])
    # reserved[0] bit 5 (no dependent launches) is read when the handle is created
    monkeypatch.setenv("OWW_FLAGS", "0" if pdl else "32")
    eng = StreamEngine(hs, B, embedding=emb_weights(), feature_init=fi, cnn_mode=3, split_from=split_from, max_chunks=2)
    monkeypatch.delenv("OWW_FLAGS")
    scores, pos = [], 0
    for si, nch in enumerate(plan):
        if si == reset_at:
            eng.reset_async(fi, stream_ids=reset_ids)
        d = torch.from_numpy(np.ascontiguousarray(base[pick, pos:pos + nch * 1280])).cuda()
        pos += nch * 1280
        scores.append(eng.step(d, nch).cpu().numpy())
    feats = np.stack([eng.ctx.get_features(b, 40) for b in sample])
    eng.ctx.close()
    return np.stack(scores), feats


@pytest.mark.parametrize("split_from", [3, 7, 11, 15])
def test_late_chain_pdl_is_bit_identical_at_every_split(torch_cuda, built_library, monkeypatch, split_from):
    """The incremental late layers on 2048 streams with dependent launches (default) against plain launches
    (OWW_FLAGS=32), at every split point that has a late chain (every tc_conv_blk_kernel instance, the fused (1,2) pool
    of layers 6 and 14, the separate (2,2) pools of layers 10 and 18).  Scores and rings must match bit for bit: this is
    the race check of the griddepcontrol chain."""
    torch = torch_cuda
    ref_s, ref_f = _late_run(torch, monkeypatch, 2048, split_from)
    nopdl_s, nopdl_f = _late_run(torch, monkeypatch, 2048, split_from, pdl=False)
    print(f"split_from={split_from}: max |PDL - plain| = {np.abs(ref_s - nopdl_s).max():.3e} "
          f"(features {np.abs(ref_f - nopdl_f).max():.3e})")
    assert np.isfinite(ref_s).all() and np.isfinite(ref_f).all()
    assert np.array_equal(ref_s, nopdl_s) and np.array_equal(ref_f, nopdl_f)


def test_late_chain_pdl_is_bit_identical_at_8192(torch_cuda, built_library, monkeypatch):
    """The dependent-launch chain against plain launches at the stream count of the largest bench configuration (many
    tiles per CTA in every late layer)."""
    torch = torch_cuda
    ref_s, ref_f = _late_run(torch, monkeypatch, 8192, 11)
    nopdl_s, nopdl_f = _late_run(torch, monkeypatch, 8192, 11, pdl=False)
    print(f"B=8192: max |PDL - plain| = {np.abs(ref_s - nopdl_s).max():.3e} (features {np.abs(ref_f - nopdl_f).max():.3e})")
    assert np.isfinite(ref_s).all()
    assert np.array_equal(ref_s, nopdl_s) and np.array_equal(ref_f, nopdl_f)


# ---------------------------------------------------------------------------------------------------- window_batch
def _window_run(mode, window_batch):
    from openwakeword_b200.engine import StreamEngine
    rng = np.random.default_rng(17)
    B = 37
    hs = [head("alexa_v0.1"), head("timer_v0.1")]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    plan = [1, 3, 1, 1, 3, 1]
    reset_at, reset_ids = 3, [0, 17, 36]
    pcm = _signals(rng, B, sum(plan) * 1280)
    eng = StreamEngine(hs, B, embedding=emb_weights(), feature_init=fi, cnn_mode=mode, max_chunks=3,
                       window_batch=window_batch)
    scores, pos = [], 0
    for si, nch in enumerate(plan):
        if si == reset_at:
            eng.reset(fi, stream_ids=reset_ids)
        scores.append(eng.step_host(np.ascontiguousarray(pcm[:, pos:pos + nch * 1280]), nch).copy())
        pos += nch * 1280
    feats = np.stack([eng.ctx.get_features(b, 40) for b in range(B)])
    eng.ctx.close()
    return np.stack(scores), feats


@pytest.mark.parametrize("mode", [0, 2])
def test_window_batch_sub_batches_are_bit_identical(torch_cuda, built_library, mode):
    """The window modes cut a call's B x n_chunks windows into sub-batches of window_batch: whole chunk rows when a
    sub-batch holds at least one, runs of streams inside one chunk row otherwise.  37 streams, 1- and 3-chunk calls and
    a reset, with window_batch 16 (every call split into runs) and 64 (3-chunk calls split into a row and a run) against
    the default (one batch): each window's arithmetic is the same, so scores and rings must match bit for bit."""
    ref_s, ref_f = _window_run(mode, 0)
    for wb in (16, 64):
        s, f = _window_run(mode, wb)
        print(f"cnn_mode {mode} window_batch {wb}: max |score diff| = {np.abs(s - ref_s).max():.3e}, "
              f"max |feature diff| = {np.abs(f - ref_f).max():.3e}")
        assert np.array_equal(s, ref_s) and np.array_equal(f, ref_f), wb


@pytest.mark.parametrize("mode", [0, 2, 3])
def test_embed_windows_sub_batches_are_bit_identical(torch_cuda, built_library, mode):
    """oww_embed_windows of 130 windows in sub-batches of 16 (eight full ones and a ragged one of 2) against one batch."""
    torch = torch_cuda
    from openwakeword_b200 import _native, weights as W
    from oracle import mel
    rng = np.random.default_rng(23)
    wins = np.stack([mel.melspectrogram(np.clip(rng.normal(0, [300, 3000, 12000][i % 3], 12400 + 512), -32768, 32767)
                                        .astype(np.int16))[:76] for i in range(130)]).astype(np.float32)
    d = torch.from_numpy(wins).cuda()
    out = {}
    for wb in (0, 16):
        ctx = _native.Context(cnn_mode=mode, window_batch=wb)
        ctx.load_mel()
        ctx.load_embedding(W.pack_embedding_blob(emb_weights()))
        emb = torch.full((130, 96), np.nan, dtype=torch.float32, device="cuda")
        ctx.embed_windows(d, 130, emb)
        torch.cuda.synchronize()
        out[wb] = emb.cpu().numpy()
        ctx.close()
    assert np.isfinite(out[0]).all()
    assert np.array_equal(out[0], out[16])
