"""-m gpu: the one-chunk step at split_from 11 / 15 runs the log-mel frontend as a launch of its own (mel_kernel, at the
head of the step's dependent-launch chain), then the early-layer kernel on the mel rows it wrote.

* The same call sequence - 1-, 2- and 3-chunk calls, ragged calls (held streams, one-chunk and multi-chunk counts) and a
  partial reset - with the dependent-launch chain on and off (OWW_FLAGS=32), and on the general path (fuse_step=False,
  which runs the same kernels as separate stages): scores, mel rings and feature rings equal bit for bit.  The stream
  count leaves a ragged last group for every group size the planner may pick.
* A steady one-chunk step at 8192 streams x 3 heads takes no more launches than before the frontend left the step kernel
  (the new launch is paid for by the (2,2) pool of layer 18, now fused into its conv's epilogue)."""
import numpy as np
import pytest

from helpers import emb_weights, head

pytestmark = pytest.mark.gpu

# launches of a steady one-chunk step at 8192 streams x 3 heads, split_from 11, before the frontend became its own launch
PARENT_STEP_LAUNCHES = 15


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _signals(rng, n, length):
    out = np.empty((n, length), np.int16)
    t = np.arange(length)
    for i in range(n):
        k = i % 4
        if k == 0:
            x = rng.integers(-1000, 1000, length)
        elif k == 1:
            x = rng.normal(0, 8000, length) * ((t // 3000) % 2)
        elif k == 2:
            x = np.zeros(length)
        else:
            x = 12000 * np.sin(2 * np.pi * 440 * t / 16000) + rng.normal(0, 20, length)
        out[i] = np.clip(x, -32768, 32767).astype(np.int16)
    return out


def _run(torch, monkeypatch, B, split_from, pdl=True, fuse=True):
    """A fixed call sequence on B streams -> (scores of every call, mel rings and feature rings of sampled streams)."""
    from openwakeword_b200.engine import StreamEngine
    rng = np.random.default_rng(7 * B + split_from)
    hs = [head("alexa_v0.1"), head("timer_v0.1")]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    # entries: int = every stream steps that many chunks; list = ragged counts per stream (cycled); "reset" = partial reset
    plan = [1, 1, 2, 1, [0, 1], 3, 1, [1, 0, 2, 3], "reset", 1, [0, 1, 1], 1, 2, 1, 1]
    reset_ids = [0, 5, B // 2, B - 1]
    n_samples = sum(max(p) if isinstance(p, list) else p for p in plan if p != "reset") * 1280
    base = _signals(rng, 24, n_samples)
    pcm = base[rng.integers(0, 24, B)]
    monkeypatch.setenv("OWW_FLAGS", "0" if pdl else "32")          # read when the handle is created
    eng = StreamEngine(hs, B, embedding=emb_weights(), feature_init=fi, cnn_mode=3, split_from=split_from, max_chunks=3,
                       fuse_step=fuse)
    monkeypatch.delenv("OWW_FLAGS")
    scores, pos = [], np.zeros(B, np.int64)
    for p in plan:
        if p == "reset":
            eng.reset_async(fi, stream_ids=reset_ids)
            continue
        counts = np.resize(np.array(p if isinstance(p, list) else [p], np.int32), B)
        n = int(counts.max())
        x = np.zeros((B, n * 1280), np.int16)
        for b in range(B):
            x[b, :counts[b] * 1280] = pcm[b, pos[b]:pos[b] + counts[b] * 1280]
        pos += counts * 1280
        d = torch.from_numpy(x).cuda()
        out = torch.full((B, eng.n_cols), float("nan"), dtype=torch.float32, device="cuda")
        if isinstance(p, list):
            eng.step_ragged(d, counts, out)
        else:
            eng.step(d, n, out)
        scores.append(out.cpu().numpy())
    torch.cuda.synchronize()
    sample = sorted(set(reset_ids + [1, 2, B - 2, B - 3] + [int(v) for v in rng.integers(0, B, 24)]))
    mel = np.stack([eng.ctx.get_mel(b, 76) for b in sample])
    feats = np.stack([eng.ctx.get_features(b, 40) for b in sample])
    eng.ctx.close()
    return np.stack(scores), mel, feats


@pytest.mark.parametrize("split_from", [11, 15])
def test_separate_frontend_chain_on_off_and_general_path(torch_cuda, built_library, monkeypatch, split_from):
    torch = torch_cuda
    B = 1501                                       # 19 x 79: a ragged last group for every group size 2..7
    ref = _run(torch, monkeypatch, B, split_from)
    plain = _run(torch, monkeypatch, B, split_from, pdl=False)
    general = _run(torch, monkeypatch, B, split_from, fuse=False)
    assert np.isfinite(ref[1]).all() and np.isfinite(ref[2]).all()
    for name, got in (("chain off", plain), ("general path", general)):
        for what, a, b in zip(("scores", "mel rings", "feature rings"), ref, got):
            assert np.array_equal(a, b, equal_nan=True), (name, what, float(np.nanmax(np.abs(a - b))))


def test_one_chunk_step_launches(torch_cuda, built_library):
    from openwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    B = 8192
    eng = StreamEngine([head("alexa_v0.1"), head("timer_v0.1"), head("big_v0.1")], B, embedding=emb_weights(),
                       cnn_mode=3, split_from=11, max_chunks=1)
    rng = np.random.default_rng(3)
    d = torch.from_numpy(rng.integers(-1000, 1000, (B, 1280)).astype(np.int16)).cuda()
    out = torch.empty((B, eng.n_cols), dtype=torch.float32, device="cuda")
    for _ in range(3):
        eng.step(d, 1, out)
    n0 = eng.ctx.launch_count
    eng.step(d, 1, out)
    torch.cuda.synchronize()
    n = eng.ctx.launch_count - n0
    print(f"one-chunk step at {B} streams x 3 heads, split_from 11: {n} launches (before: {PARENT_STEP_LAUNCHES})")
    assert n <= PARENT_STEP_LAUNCHES
    eng.ctx.close()
