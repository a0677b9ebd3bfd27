"""-m gpu: the fused step kernel (tc_inc_kernel) at every group size G = 1..7 and at every split_from (3, 7, 11, 15, 20).

The kernel runs each layer as 64-position items spread over four warpgroups, with weight copies issued by one thread
of the CTA; how many items a warpgroup takes (none, one or many), whether the last 64-row tile is partial and whether
the last group of streams is ragged all depend on G.  The stream count of each case is chosen so that the library picks
that G on this device, with a ragged last group; the handle's plan is read back to confirm it.  The padded clips are
streamed one chunk per call and compared with oww_predict_clips_ragged on the same clips, whose CNN runs in
tc_conv_kernel (same per-element arithmetic): feature rows bit for bit at every split; scores bit for bit below 20,
where the heads run as their own launch, and within 2e-5 at 20, where they run inside the fused kernel (the bound of
test_bulk_clips_equal_streaming_at_every_split)."""
import ctypes as C

import numpy as np
import pytest

from helpers import emb_weights, head
from test_gpu_bulk_edges import _padded, _steps, torch_cuda  # noqa: F401  (fixture)
from test_gpu_cnn_configs import _signals

pytestmark = pytest.mark.gpu

LEN, PAD, CHUNK = 12800, 2560, 1280
OWW_EUNSUPPORTED = -4


def _plan_g(built_library, h, G=0, n=0, split=20):
    """group size of the plan: the handle's own (h given, G = 0), or G if the builder accepts that plan, else None"""
    buf = (C.c_int32 * 4096)()
    if h is not None:
        rc = built_library.oww_debug_inc_plan(h, 0, 0, buf, 4096)
    elif split < 20:
        rc = built_library.oww_debug_inc_cut_plan(None, G, n, split, buf, 4096)
    else:
        rc = built_library.oww_debug_inc_plan(None, G, n, buf, 4096)
    if rc == OWW_EUNSUPPORTED:
        return None
    assert rc > 0
    return int(buf[0])


@pytest.mark.parametrize("split", [3, 7, 11, 15, 20])
@pytest.mark.parametrize("G", list(range(1, 8)))
def test_fused_items_every_group_size(torch_cuda, built_library, G, split):
    torch = torch_cuda
    from openwakeword_b200.engine import StreamEngine
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    if _plan_g(built_library, None, G, 1, split) is None:
        pytest.skip(f"G={G} does not fit shared memory at split_from={split}")
    # (G - 1) full rounds of SMs plus part of one more, so that G - 1 would need a second round; n % G != 0 leaves a
    # ragged last group
    n = sm // 2 + 1 if G == 1 else sm * (G - 1) + sm // 2 + 1
    if G > 1 and n % G == 0:
        n += 1
    rng = np.random.default_rng(1000 + G)
    clips = _signals(rng, n, LEN)
    hs = [head("alexa_v0.1"), head("hey_jarvis_v0.1"), head("timer_v0.1")]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    cfg = dict(cnn_mode=3, split_from=split)
    S = _steps(LEN + 2 * PAD)

    eng = StreamEngine(hs, n, embedding=emb_weights(), feature_init=fi, **cfg)
    assert _plan_g(built_library, eng.ctx.h) == G, n
    padded = _padded(clips, PAD)
    stream = np.stack([eng.step_host(np.ascontiguousarray(padded[:, s * CHUNK:(s + 1) * CHUNK]), 1).copy()
                       for s in range(S)], 1)
    feats = np.stack([eng.ctx.get_features(b, S) for b in range(n)])       # [n, S, 96]: the rows these steps appended
    eng.ctx.close()

    ref = StreamEngine(hs, 1, embedding=emb_weights(), **cfg)
    d = torch.from_numpy(np.ascontiguousarray(clips).reshape(-1)).cuda()
    off = np.arange(n + 1, dtype=np.int64) * LEN
    scores = torch.full((n * S, ref.n_cols), np.nan, dtype=torch.float32, device="cuda")
    emb = torch.full((n * S, 96), np.nan, dtype=torch.float32, device="cuda")
    ref.ctx.predict_clips_ragged(d, off, PAD, CHUNK, fi, scores, None, emb)
    torch.cuda.synchronize()
    bulk = scores.cpu().numpy().reshape(n, S, -1)
    bulk_f = emb.cpu().numpy().reshape(n, S, 96)
    ref.ctx.close()

    ds, df = float(np.abs(bulk - stream).max()), float(np.abs(bulk_f - feats).max())
    print(f"G={G} split_from={split}: {n} streams, {-(-n // G)} groups; max |bulk - streaming|: scores {ds:.3e}, "
          f"feature rows {df:.3e}")
    assert np.isfinite(bulk).all() and np.isfinite(stream).all() and np.isfinite(bulk_f).all()
    assert np.array_equal(bulk_f, feats)
    if split == 20:
        assert ds <= 2e-5
    else:
        assert np.array_equal(bulk, stream)
