"""-m gpu: per-stream head banks (heads_tc.cu, oww_add_head_bank) against ordinary heads of the same weights (bit for
bit), the oracle, ragged steps, the bulk clip path, scale and the ABI's refusals."""
import numpy as np
import pytest

from helpers import emb_weights, head
from openwakeword_b200 import weights as W

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _bank_heads(n, seed0=100, **kw):
    """n synthetic heads of one shape (alexa's by default)."""
    spec = dict(n_in=16, hidden=64, n_blocks=1, n_out=1, layernorm=True, final="sigmoid")
    spec.update(kw)
    return [W.synthetic_head(seed=seed0 + i, **spec) for i in range(n)]


# ---------------------------------------------------------------- 1. stateless equality
SHAPES = {
    "h32": dict(n_in=16, hidden=32, n_blocks=1, n_out=1, layernorm=True, final="sigmoid"),
    "h128x2": dict(n_in=16, hidden=128, n_blocks=2, n_out=1, layernorm=True, final="sigmoid"),
    "no_ln": dict(n_in=16, hidden=64, n_blocks=1, n_out=1, layernorm=False, final="sigmoid"),
    "timer": dict(n_in=34, hidden=128, n_blocks=1, n_out=7, layernorm=False, final="relu_softmax"),
}


@pytest.mark.parametrize("terms", [3, 1])
@pytest.mark.parametrize("mode", [2, 3])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_bank_predict_equals_head_predict(torch_cuda, built_library, shape, mode, terms):
    from openwakeword_b200 import _native
    torch = torch_cuda
    hs = [W.synthetic_head(seed=7 + i, **SHAPES[shape]) for i in range(3)]
    ctx = _native.Context(cnn_mode=mode, tc_heads_terms=terms)
    n_in, dims, ln, fin = W.head_desc(hs[0])
    bank = ctx.add_head_bank(n_in, dims, ln, fin, 5)
    rng = np.random.default_rng(1)
    x = torch.from_numpy((rng.normal(0, 1.5, (300, n_in, 96))).astype(np.float32)).cuda()
    for i, h in enumerate(hs):
        hid = ctx.add_head(n_in, dims, ln, fin, W.pack_head_blob(h))
        ctx.load_bank_head(bank, 4 - i, W.pack_head_blob(h))
        ref = torch.empty((300, dims[-1]), dtype=torch.float32, device="cuda")
        got = torch.full_like(ref, float("nan"))
        ctx.head_predict(hid, x, 300, ref)
        ctx.bank_head_predict(bank, 4 - i, x, 300, got)
        torch.cuda.synchronize()
        assert torch.equal(got, ref), (shape, i, (got - ref).abs().max().item())


# ---------------------------------------------------------------- 2-4. streaming
STREAMS = 151
PLAN = [1, 1, 1, 2, 1, 3, 1, 1, 2, 1, 1]
RESET_AT, SWAP_AT = 5, 7
CONFIGS = [(2, 11), (3, 11), (3, 20)]       # (cnn_mode, split_from); at 20 the ordinary heads run inside the fused kernel


def _streaming_setup():
    rng = np.random.default_rng(151)
    cands = _bank_heads(7)                  # slots 0..5 loaded at the start; candidate 6 replaces slot 2 at SWAP_AT
    # shared slots (0: every 4th stream, 1: every 5th), singletons (slots 3, 4, 5), the rest on 2 or none
    slots = np.full(STREAMS, -1, np.int32)
    slots[::4] = 0
    slots[1::5] = 1
    slots[[7, 150, 63]] = [3, 4, 5]
    slots[(np.arange(STREAMS) % 7 == 2) & (slots < 0)] = 2
    swap_ids = np.array([0, 3, 7, 22, 150], np.int32)
    swap_slots = np.array([-1, 2, 1, 3, 0], np.int32)
    reset_ids = np.array([1, 2, 75, 150], np.int32)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    pcm = np.clip(rng.normal(0, 4000, (STREAMS, sum(PLAN) * 1280)), -32768, 32767).astype(np.int16)
    return cands, slots, swap_ids, swap_slots, reset_ids, fi, pcm


ORDINARY = ["alexa_v0.1", "timer_v0.1", "hey_jarvis_v0.1"]


def _run_streaming(torch, mode, split_from, kind, group_heads=False):
    """kind: "bank" (ordinary heads + the bank), "plain" (ordinary heads only), "ref" (ordinary heads + the 7 candidates
    as ordinary heads).  -> (scores [steps, B, cols] raw, per step the candidate of every stream (-1 none), bank column)"""
    from openwakeword_b200.engine import StreamEngine
    cands, slots, swap_ids, swap_slots, reset_ids, fi, pcm = _streaming_setup()
    heads = [head(n) for n in ORDINARY] + (cands if kind == "ref" else [])
    eng = StreamEngine(heads, STREAMS, embedding=emb_weights(), feature_init=fi, cnn_mode=mode, max_chunks=3,
                       split_from=split_from, group_heads=group_heads)
    cand_of_slot = list(range(6))
    bank = col = None
    if kind == "bank":
        bank, col, _ = eng.add_head_bank(cands[0], 8)
        for k in range(6):
            eng.load_bank_head(bank, k, cands[k])
        eng.assign_bank_head(bank, slots)
    cur = slots.copy()
    out, who, pos = [], [], 0
    for i, n in enumerate(PLAN):
        if i == RESET_AT:
            eng.reset(fi, stream_ids=reset_ids)
        if i == SWAP_AT:
            cand_of_slot[2] = 6
            cur[swap_ids] = swap_slots
            if kind == "bank":
                eng.load_bank_head(bank, 2, cands[6])
                eng.assign_bank_head(bank, swap_slots, stream_ids=swap_ids)
        x = torch.from_numpy(np.ascontiguousarray(pcm[:, pos:pos + n * 1280])).cuda()
        out.append(eng.step(x, n).cpu().numpy())
        who.append(np.array([cand_of_slot[k] if k >= 0 else -1 for k in cur]))
        pos += n * 1280
    return np.stack(out), np.stack(who), col, eng


def _oracle_stream(b, who):
    """raw per-step scores of every candidate on stream b (the oracle's feature pipeline, max over chunk windows)."""
    from oracle.streaming import OracleAudioFeatures
    from oracle import heads as OH
    cands, slots, swap_ids, swap_slots, reset_ids, fi, pcm = _streaming_setup()
    pre = OracleAudioFeatures(emb_weights(), feature_init=fi)
    res, pos = [], 0
    for i, n in enumerate(PLAN):
        if i == RESET_AT and b in reset_ids:
            pre.reset(feature_init=fi)
        n_s = pre(pcm[b, pos:pos + n * 1280])
        pos += n * 1280
        k = who[i, b]
        if k < 0:
            res.append(0.0)
            continue
        h = cands[k]
        g = [OH.forward(h, pre.get_features(16, -16 - j))[0] for j in range(n_s // 1280 - 1, -1, -1)] \
            if n_s > 1280 else [OH.forward(h, pre.get_features(16))[0]]
        res.append(float(np.max(np.stack(g), axis=0)[0]))
    return np.array(res, np.float32)


@pytest.mark.parametrize("mode,split_from", CONFIGS)
def test_bank_streaming_vs_ordinary_and_oracle(torch_cuda, built_library, mode, split_from):
    torch = torch_cuda
    got, who, col, eng = _run_streaming(torch, mode, split_from, "bank")
    ref, _, _, ref_eng = _run_streaming(torch, mode, split_from, "ref")
    plain, _, _, plain_eng = _run_streaming(torch, mode, split_from, "plain")
    n_ord = plain.shape[2]
    bank_col = got[:, :, col]
    # unassigned streams read exactly 0; every other stream its candidate's column of the reference handle
    assert np.all(bank_col[who < 0] == 0.0)
    cand_cols = [ref_eng.columns[len(ORDINARY) + k][0] for k in range(7)]
    want = np.where(who >= 0, np.take_along_axis(ref[:, :, cand_cols], np.maximum(who, 0)[..., None], 2)[..., 0], 0.0)
    diff = np.abs(bank_col - want).max()
    print(f"mode {mode} split {split_from}: max |bank - ordinary head| = {diff:.3e}")
    if split_from != 20:     # the ordinary heads run heads_tc_kernel on the fp32 rings: the same bits
        assert np.array_equal(bank_col, want)
    else:                    # they run inside the fused kernel, in its own summation order
        assert diff <= 1e-4
    # the ordinary columns do not change when a bank is added
    assert np.array_equal(got[:, :, :n_ord], plain)
    # oracle on sampled streams: shared, singleton, swapped, reset and unassigned ones
    worst = 0.0
    for b in [0, 1, 7, 22, 63, 75, 150, 3]:
        o = _oracle_stream(b, who)
        worst = max(worst, float(np.abs(o - bank_col[:, b]).max()))
    print(f"mode {mode} split {split_from}: max |bank - oracle| over sampled streams = {worst:.3e}")
    assert worst <= 1e-3


def test_bank_streaming_grouped_handle(torch_cuda, built_library):
    """default handle (ordinary heads on the grouped mirror kernel): ordinary columns unchanged bit for bit, bank
    columns within fp32-grade distance of the reference handle's."""
    torch = torch_cuda
    got, who, col, _ = _run_streaming(torch, 3, 11, "bank", group_heads=True)
    plain, _, _, _ = _run_streaming(torch, 3, 11, "plain", group_heads=True)
    assert np.array_equal(got[:, :, :plain.shape[2]], plain)
    ref, _, _, ref_eng = _run_streaming(torch, 3, 11, "ref", group_heads=False)
    cand_cols = [ref_eng.columns[len(ORDINARY) + k][0] for k in range(7)]
    want = np.where(who >= 0, np.take_along_axis(ref[:, :, cand_cols], np.maximum(who, 0)[..., None], 2)[..., 0], 0.0)
    assert np.array_equal(got[:, :, col], want)


def test_bank_assign_is_stream_ordered_and_launches(torch_cuda, built_library):
    torch = torch_cuda
    from openwakeword_b200.engine import StreamEngine
    cands = _bank_heads(2)
    rng = np.random.default_rng(3)
    pcm = torch.from_numpy(np.clip(rng.normal(0, 4000, (40, 1280 * 8)), -32768, 32767).astype(np.int16)).cuda()
    eng = StreamEngine([head("alexa_v0.1")], 40, embedding=emb_weights(), cnn_mode=3, group_heads=False)
    bare = StreamEngine([head("alexa_v0.1")], 40, embedding=emb_weights(), cnn_mode=3, group_heads=False)
    bank, col, _ = eng.add_head_bank(cands[0], 2)
    eng.load_bank_head(bank, 0, cands[0])
    eng.load_bank_head(bank, 1, cands[1])
    # a handle without a bank keeps its launches per step; the bank adds one launch per step
    c0, d0 = eng.ctx.launch_count, bare.ctx.launch_count
    eng.step(pcm[:, :1280]); bare.step(pcm[:, :1280])
    torch.cuda.synchronize()
    assert eng.ctx.launch_count - c0 == bare.ctx.launch_count - d0 + 1
    # an assignment enqueued between two steps takes effect at the second, not the first
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        a = eng.step(pcm[:, 1280:2560])
        eng.assign_bank_head(bank, np.ones(40, np.int32))
        b = eng.step(pcm[:, 2560:3840])
    torch.cuda.synchronize()
    assert torch.all(a[:, col] == 0)
    assert torch.all(b[:, col] > 0)


# ---------------------------------------------------------------- 4. ragged
def test_bank_ragged_matches_lockstep(torch_cuda, built_library):
    """oww_step_ragged with 0/1/2 counts: bank columns equal a lockstep handle's bit for bit; held rows untouched."""
    torch = torch_cuda
    from openwakeword_b200.engine import StreamEngine
    B = 30
    cands = _bank_heads(3)
    rng = np.random.default_rng(5)
    counts = [rng.integers(0, 3, B).astype(np.int32) for _ in range(6)]
    counts[0][:] = 1
    counts[2][4] = 0                                   # stream 4: held, then fresh for a while
    pcm = np.clip(rng.normal(0, 4000, (B, 1280 * 2 * len(counts))), -32768, 32767).astype(np.int16)
    slots = np.array([b % 4 - 1 for b in range(B)], np.int32)
    for split_from in (11, 20):
        eng = StreamEngine([head("alexa_v0.1")], B, embedding=emb_weights(), cnn_mode=3, max_chunks=2,
                           split_from=split_from, group_heads=False)
        bank, col, _ = eng.add_head_bank(cands[0], 3)
        for k in range(3):
            eng.load_bank_head(bank, k, cands[k])
        eng.assign_bank_head(bank, slots)
        pos = np.zeros(B, np.int64)
        rows = []
        for c in counts:
            x = np.zeros((B, 2560), np.int16)
            for b in range(B):
                x[b, :c[b] * 1280] = pcm[b, pos[b]:pos[b] + c[b] * 1280]
            out = torch.full((B, eng.n_cols), -7.0, device="cuda")
            eng.step_ragged(torch.from_numpy(x).cuda(), c, out)
            o = out.cpu().numpy()
            assert np.all(o[c == 0] == -7.0)          # held rows are not written
            rows.append(o[:, col])
            pos += c * 1280
        for b in (0, 4, 5, 9, 14):             # each against a one-stream handle stepped by its own counts
            twin = StreamEngine([head("alexa_v0.1")], 1, embedding=emb_weights(), cnn_mode=3, max_chunks=2,
                                split_from=split_from, group_heads=False)
            tb, tcol, _ = twin.add_head_bank(cands[0], 3)
            for k in range(3):
                twin.load_bank_head(tb, k, cands[k])
            twin.assign_bank_head(tb, slots[b:b + 1])
            p = 0
            for i, c in enumerate(counts):
                if c[b] == 0:
                    continue
                x = torch.from_numpy(np.ascontiguousarray(pcm[b:b + 1, p:p + c[b] * 1280])).cuda()
                r = twin.step(x, int(c[b])).cpu().numpy()[0, tcol]
                p += c[b] * 1280
                assert r == rows[i][b], (split_from, b, i, r, rows[i][b])


# ---------------------------------------------------------------- 5. bulk
def test_bank_bulk_clip_slot(torch_cuda, built_library):
    torch = torch_cuda
    from openwakeword_b200.engine import StreamEngine
    cands = _bank_heads(2)
    rng = np.random.default_rng(9)
    lens = [16000, 23000, 9000, 30000]
    pad = 16000
    clips = [np.clip(rng.normal(0, 4000, n), -32768, 32767).astype(np.int16) for n in lens]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    eng = StreamEngine([head("alexa_v0.1")], len(clips), embedding=emb_weights(), feature_init=fi, cnn_mode=3,
                       group_heads=False)
    bank, col, _ = eng.add_head_bank(cands[0], 2)
    eng.load_bank_head(bank, 1, cands[1])
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    d = torch.from_numpy(np.concatenate(clips)).cuda()
    from openwakeword_b200 import _native
    rows = sum(_native.clip_schedule(1280, n + 2 * pad).size for n in lens)

    def bulk():
        sc = torch.full((rows, eng.n_cols), -5.0, device="cuda")
        st = torch.zeros(rows, dtype=torch.uint8, device="cuda")
        eng.ctx.predict_clips_ragged(d, off, pad, 1280, fi, sc, st, None, torch.cuda.current_stream().cuda_stream)
        return sc.cpu().numpy()

    z = bulk()
    assert np.all(z[:, col] == 0.0)                     # clip slot -1: zeros
    eng.set_head_bank_clip_slot(bank, 1)
    got = bulk()
    # streaming the padded clips on streams assigned slot 1
    eng.assign_bank_head(bank, np.ones(len(clips), np.int32))
    eng.reset(fi)
    L = max(lens) + 2 * pad
    padded = np.zeros((len(clips), L), np.int16)
    for i, c in enumerate(clips):
        padded[i, pad:pad + c.size] = c
    r0 = 0
    per = []
    for s in range((L - 1) // 1280):
        x = torch.from_numpy(np.ascontiguousarray(padded[:, s * 1280:(s + 1) * 1280])).cuda()
        per.append(eng.step(x).cpu().numpy()[:, col])
    per = np.stack(per, 1)
    for i, n in enumerate(lens):
        k = _native.clip_schedule(1280, n + 2 * pad).size
        assert np.array_equal(got[r0:r0 + k, col], per[i, :k]), i
        r0 += k


# ---------------------------------------------------------------- 6. scale
def test_bank_scale(torch_cuda, built_library):
    """8192 streams x 7 networks plus a bank with 1024 distinct slots; and 300 distinct models on 320 streams."""
    torch = torch_cuda
    from openwakeword_b200.engine import StreamEngine
    from oracle import heads as OH
    B = 8192
    heads7 = [head("alexa_v0.1"), head("hey_mycroft_v0.1"), head("timer_v0.1"), head("hey_jarvis_v0.1"),
              W.synthetic_head(seed=51), W.synthetic_head(seed=52)]
    eng = StreamEngine(heads7, B, embedding=emb_weights(), cnn_mode=3)
    cands = _bank_heads(1024, seed0=1000)
    bank, col, _ = eng.add_head_bank(cands[0], 1024)
    for k, h in enumerate(cands):
        eng.load_bank_head(bank, k, h)
    rng = np.random.default_rng(11)
    slots = rng.integers(0, 1024, B).astype(np.int32)
    eng.assign_bank_head(bank, slots)
    pcm = torch.from_numpy(np.clip(rng.normal(0, 4000, (B, 1280)), -32768, 32767).astype(np.int16)).cuda()
    for _ in range(3):
        out = eng.step(pcm).cpu().numpy()
    sample = rng.choice(B, 16, replace=False)
    worst = 0.0
    for b in sample:
        f = eng.ctx.get_features(int(b), 16)
        ref = OH.forward(cands[slots[b]], f[None])[0][0]
        worst = max(worst, abs(float(ref) - float(out[b, col])))
    print(f"8192 streams, 1024 slots: max |bank - oracle| over 16 streams = {worst:.3e}")
    assert worst <= 1e-3
    del eng
    # 300 distinct models: more than oww_add_head allows on one handle
    eng = StreamEngine([], 320, embedding=emb_weights(), cnn_mode=3)
    cands = _bank_heads(300, seed0=5000)
    bank, col, _ = eng.add_head_bank(cands[0], 300)
    for k, h in enumerate(cands):
        eng.load_bank_head(bank, k, h)
    slots = np.array([b % 300 for b in range(320)], np.int32)
    eng.assign_bank_head(bank, slots)
    p = torch.from_numpy(np.clip(rng.normal(0, 4000, (320, 1280)), -32768, 32767).astype(np.int16)).cuda()
    out = eng.step(p).cpu().numpy()
    for b in (0, 17, 299, 319):
        ref = OH.forward(cands[slots[b]], eng.ctx.get_features(b, 16)[None])[0][0]
        assert abs(float(ref) - float(out[b, col])) <= 1e-3


# ---------------------------------------------------------------- 7. ABI edges
def test_bank_refusals(torch_cuda, built_library):
    from openwakeword_b200 import _native
    h = _bank_heads(1)[0]
    n_in, dims, ln, fin = W.head_desc(h)
    c0 = _native.Context(cnn_mode=0)
    with pytest.raises(_native.NativeError, match="cnn_mode 0"):
        c0.add_head_bank(n_in, dims, ln, fin, 4)
    ctx = _native.Context(cnn_mode=3)
    wide = W.synthetic_head(hidden=192, seed=3)
    with pytest.raises(_native.NativeError, match="128"):
        ctx.add_head_bank(*W.head_desc(wide), 4)
    bank = ctx.add_head_bank(n_in, dims, ln, fin, 4)
    with pytest.raises(_native.NativeError, match="floats"):
        ctx.load_bank_head(bank, 0, W.pack_head_blob(W.synthetic_head(hidden=32, seed=3)))
    with pytest.raises(_native.NativeError, match="slot"):
        ctx.load_bank_head(bank, 4, W.pack_head_blob(h))
    with pytest.raises(_native.NativeError, match="bank"):
        ctx.load_bank_head(bank + 1, 0, W.pack_head_blob(h))
    ctx.load_bank_head(bank, 0, W.pack_head_blob(h))
    ctx.load_mel()
    ctx.load_embedding(W.pack_embedding_blob(emb_weights()))
    ctx.set_streams(8)
    with pytest.raises(_native.NativeError, match="stream id"):
        ctx.assign_bank_head(bank, [8], [0])
    with pytest.raises(_native.NativeError, match="slot"):
        ctx.assign_bank_head(bank, [1], [4])
    with pytest.raises(_native.NativeError, match="holds no head"):
        ctx.assign_bank_head(bank, [1], [2])
    with pytest.raises(_native.NativeError, match="slot"):
        ctx.set_head_bank_clip_slot(bank, -2)
    ctx.assign_bank_head(bank, [1, 2], [0, -1])
    ctx.set_head_bank_clip_slot(bank, 0)
    assert ctx.n_outputs == 1
