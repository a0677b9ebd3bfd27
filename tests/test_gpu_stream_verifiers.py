"""-m gpu: custom verifiers on per-stream head banks (oww_add_bank_verifier_bank): streaming bit for bit against the
unverified run and oww_verifier_predict, ragged steps, launch counts, the bulk path with per-clip streams
(oww_predict_clips_streams) against the clip-slot path, Model.predict_clips(streams=) against streaming, enrollment
against each stream's own model, and the ABI's refusals."""
import copy
import os

import numpy as np
import pytest

from helpers import GOLDEN, emb_weights, head
from openwakeword_b200 import weights as W
from test_gpu_verifier import _fit

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


STREAMS = 151
PLAN = [1, 1, 1, 2, 1, 3, 1, 1, 2, 1, 1]
RESET_AT, SWAP_AT = 5, 7
CONFIGS = [(2, 11), (3, 11), (3, 20)]


def _cands(n=6):
    return [W.synthetic_head(seed=300 + i, n_in=16, hidden=64, n_blocks=1, n_out=1, layernorm=True, final="sigmoid")
            for i in range(n)]


def _setup():
    rng = np.random.default_rng(77)
    hslots = np.full(STREAMS, -1, np.int32)
    hslots[::4] = 0
    hslots[1::5] = 1
    hslots[[7, 150, 63]] = [3, 4, 5]
    hslots[(np.arange(STREAMS) % 7 == 2) & (hslots < 0)] = 2
    vslots = np.where(np.arange(STREAMS) % 3 == 0, -1, np.arange(STREAMS) % 4).astype(np.int32)
    vslots[[2, 5, 11]] = [0, 1, 2]                  # some verified streams have no model (slot -1 of the bank)
    hslots[[2, 5, 11]] = -1
    swap_ids = np.array([0, 3, 7, 22, 150, 11], np.int32)
    swap_h = np.array([-1, 2, 1, 3, 0, 1], np.int32)
    swap_v = np.array([1, -1, 3, 2, 0, 0], np.int32)
    reset_ids = np.array([1, 2, 75, 150], np.int32)
    vers = [_fit(rng, 16), _fit(rng, 16, 2.0), _fit(rng, 16, 0.5), _fit(rng, 16)]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    pcm = np.clip(rng.normal(0, 4000, (STREAMS, sum(PLAN) * 1280)), -32768, 32767).astype(np.int16)
    return hslots, vslots, swap_ids, swap_h, swap_v, reset_ids, vers, fi, pcm


def _engine(mode, split_from, thr, verified, n_streams=STREAMS, fi=None, ordinary_verifier=True):
    """alexa + a bank of the 6 candidates; verified: a verifier bank on the bank and one on alexa (both at thr)"""
    from openwakeword_b200.custom_verifier_model import linear_verifier_params
    from openwakeword_b200.engine import StreamEngine
    hslots, vslots, _, _, _, _, vers, fi0, _ = _setup()
    eng = StreamEngine([head("alexa_v0.1")], n_streams, embedding=emb_weights(), feature_init=fi0 if fi is None else fi,
                       cnn_mode=mode, max_chunks=3, split_from=split_from)
    bank, col, _ = eng.add_head_bank(_cands()[0], 8)
    for k, h in enumerate(_cands()):
        eng.load_bank_head(bank, k, h)
    eng.assign_bank_head(bank, hslots[:n_streams])
    vb = ob = None
    if verified:
        vb = eng.add_bank_verifier_bank(bank, 4, thr)
        for k, v in enumerate(vers):
            eng.ctx.load_verifier(vb, k, *linear_verifier_params(v))
        eng.assign_verifier(vb, vslots[:n_streams])
        if ordinary_verifier:
            ob = eng.add_verifier_bank(0, 4, thr)
            eng.ctx.load_verifier(ob, 0, *linear_verifier_params(vers[3]))
            eng.assign_verifier(ob, np.zeros(n_streams, np.int32))
    return eng, bank, col, vb, ob


def _run(torch, mode, split_from, thr, verified):
    hslots, vslots, swap_ids, swap_h, swap_v, reset_ids, vers, fi, pcm = _setup()
    eng, bank, col, vb, ob = _engine(mode, split_from, thr, verified)
    cur_h, cur_v = hslots.copy(), vslots.copy()
    out, hs, vs, feats, pos = [], [], [], [], 0
    for i, n in enumerate(PLAN):
        if i == RESET_AT:
            eng.reset(fi, stream_ids=reset_ids)
        if i == SWAP_AT:
            eng.assign_bank_head(bank, swap_h, stream_ids=swap_ids)
            cur_h[swap_ids] = swap_h
            if verified:
                eng.assign_verifier(vb, swap_v, swap_ids)
            cur_v[swap_ids] = swap_v
        x = torch.from_numpy(np.ascontiguousarray(pcm[:, pos:pos + n * 1280])).cuda()
        out.append(eng.step(x, n).cpu().numpy())
        hs.append(cur_h.copy())
        vs.append(cur_v.copy())
        if verified:
            feats.append(np.stack([eng.ctx.get_features(b, 16) for b in range(STREAMS)]))
        pos += n * 1280
    return np.stack(out), np.stack(hs), np.stack(vs), feats, eng, vb, ob, col


@pytest.mark.parametrize("thr", [0.0, 0.3])
@pytest.mark.parametrize("mode,split_from", CONFIGS)
def test_streaming_bank_verifiers_bit_for_bit(torch_cuda, built_library, mode, split_from, thr):
    torch = torch_cuda
    got, hs, vs, feats, eng, vb, ob, col = _run(torch, mode, split_from, thr, True)
    plain = _run(torch, mode, split_from, thr, False)[0]
    t = np.float32(thr)
    n_ver = 0
    for k in range(len(PLAN)):
        p_bank = {s: eng.ctx.verifier_predict_host(vb, s, feats[k]) for s in range(4)}
        p_ord = eng.ctx.verifier_predict_host(ob, 0, feats[k])
        for b in range(STREAMS):
            g, p = got[k, b, col], plain[k, b, col]
            if hs[k, b] < 0:
                assert g == 0.0 and p == 0.0, (k, b)             # no model: never verified, whatever the threshold
            elif vs[k, b] < 0 or p < t:
                assert g == p, (k, b)
            else:
                assert g == p_bank[int(vs[k, b])][b], (k, b)
                n_ver += 1
            want0 = p_ord[b] if plain[k, b, 0] >= t else plain[k, b, 0]
            assert got[k, b, 0] == want0, (k, b)
    # float64 oracle on sampled streams (shared and singleton slots, no model with a verifier, swapped, reset): its
    # heads on its features, the max over a call's chunk windows, then the verifier rule.  Scores within the path's
    # distance of the threshold may take the other side of it: those elements are left out.
    worst = 0.0
    for b in ORACLE_STREAMS:
        o = _oracle_stream(b, hs[:, b], vs[:, b], thr)
        for c, oc in ((col, 0), (0, 1)):
            clear = np.abs(plain[:, b, c] - t) > 2e-3
            worst = max(worst, float(np.abs(got[clear, b, c] - o[clear, oc]).max(initial=0.0)))
    print(f"mode {mode} split {split_from} thr {thr}: {n_ver} bank scores verified; max |device - float64 oracle| over "
          f"{len(ORACLE_STREAMS)} streams = {worst:.2e}")
    assert n_ver > 0
    assert worst <= 1e-3


ORACLE_STREAMS = [0, 1, 2, 3, 7, 11, 22, 63, 75, 150]
_oracle_cache = {}


def _oracle_raw(b):
    """per call of PLAN on stream b: (max over its chunk windows of every candidate [6], of alexa, the newest window)"""
    if b not in _oracle_cache:
        from oracle.streaming import OracleAudioFeatures
        from oracle import heads as OH
        _, _, _, _, _, reset_ids, _, fi, pcm = _setup()
        cands, alexa = _cands(), head("alexa_v0.1")
        pre = OracleAudioFeatures(emb_weights(), feature_init=fi, dtype=np.float64)
        res, pos = [], 0
        for i, n in enumerate(PLAN):
            if i == RESET_AT and b in reset_ids:
                pre.reset(feature_init=fi)
            pre(pcm[b, pos:pos + n * 1280])
            pos += n * 1280
            wins = [pre.get_features(16, -16 - j) for j in range(n - 1, -1, -1)] if n > 1 else [pre.get_features(16)]
            best = lambda h: np.max([OH.forward(h, w, np.float64)[0, 0] for w in wins])   # noqa: E731
            res.append(([best(h) for h in cands], best(alexa), pre.get_features(16)))
        _oracle_cache[b] = res
    return _oracle_cache[b]


def _oracle_stream(b, hs, vs, thr):
    """float64 oracle of stream b's bank column and alexa column per call, verified as verifier.cu specifies"""
    from oracle.verifier import verifier_proba
    vers = _setup()[6]
    t = np.float32(thr)
    out = []
    for (cand, alexa, newest), h, v in zip(_oracle_raw(b), hs, vs):
        if h < 0:
            bank = 0.0
        elif v >= 0 and np.float32(cand[h]) >= t:
            bank = float(verifier_proba(vers[v], newest)[0])
        else:
            bank = cand[h]
        ordinary = float(verifier_proba(vers[3], newest)[0]) if np.float32(alexa) >= t else alexa
        out.append((bank, ordinary))
    return np.array(out)


def _bench_heads():
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "bench_mod", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    return list(bench.bench_heads("c3").values())


def test_scale_8192_streams(torch_cuda, built_library):
    """8192 streams x the 7 benchmark networks with verifier banks on two ordinary heads, a bank of 1024 slots and 8192
    distinct stream verifiers: 16 sampled streams within 1e-3 of the float64 oracle."""
    torch = torch_cuda
    from oracle.streaming import OracleAudioFeatures
    from oracle import heads as OH
    from openwakeword_b200.custom_verifier_model import linear_verifier_params
    from openwakeword_b200.engine import StreamEngine
    B, D, thr = 8192, 1024, 0.0
    heads = _bench_heads()
    rng = np.random.default_rng(8192)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    eng = StreamEngine(heads, B, embedding=emb_weights(), feature_init=fi, cnn_mode=3, max_chunks=2)
    cands = [W.synthetic_head(seed=1000 + k, n_in=16, hidden=64, n_blocks=1, n_out=1, layernorm=True, final="sigmoid")
             for k in range(D)]
    bank, col, _ = eng.add_head_bank(cands[0], D)
    for k, h in enumerate(cands):
        eng.load_bank_head(bank, k, h)
    ids = np.arange(B)
    hslot = np.where(ids % 61 == 0, -1, ids % D).astype(np.int32)
    vslot = np.where(ids % 53 == 0, -1, ids).astype(np.int32)
    eng.assign_bank_head(bank, hslot)
    # ordinary verifier banks on alexa (head 0) and timer (the last entry) share the launch
    ords = [_fit(rng, 16), _fit(rng, 16, 2.0)]
    ob = eng.add_verifier_bank(0, 2, thr)
    for k, v in enumerate(ords):
        eng.ctx.load_verifier(ob, k, *linear_verifier_params(v))
    eng.assign_verifier(ob, (ids % 2).astype(np.int32))
    tb = eng.add_verifier_bank(len(heads) - 1, 1, thr)
    eng.ctx.load_verifier(tb, 0, *linear_verifier_params(_fit(rng, 34)))
    eng.assign_verifier(tb, np.zeros(B, np.int32))
    vb = eng.add_bank_verifier_bank(bank, B, thr)
    mean = rng.normal(0, 1, (B, 16 * 96)).astype(np.float32)
    weight = rng.normal(0, 0.02, (B, 16 * 96)).astype(np.float32)
    bias = rng.normal(0, 0.5, B).astype(np.float32)
    dev = torch.device("cuda")
    eng.ctx.load_verifiers(vb, ids.astype(np.int32), torch.from_numpy(mean).to(dev), torch.from_numpy(weight).to(dev),
                           torch.from_numpy(bias).to(dev))
    eng.assign_verifier(vb, vslot)
    plan = [1, 2, 1, 1]
    pcm = np.clip(rng.normal(0, 4000, (B, sum(plan) * 1280)), -32768, 32767).astype(np.int16)
    got, pos = [], 0
    for n in plan:
        got.append(eng.step(torch.from_numpy(np.ascontiguousarray(pcm[:, pos:pos + n * 1280])).cuda(), n).cpu().numpy())
        pos += n * 1280
    got = np.stack(got)
    sample = [0, 1, 53, 61, 1023, 1024, 2047, 3181, 4096, 5000, 6100, 7000, 7321, 8000, 8190, 8191]
    alexa = heads[0]
    from oracle.verifier import verifier_proba
    worst = 0.0
    for b in sample:
        pre = OracleAudioFeatures(emb_weights(), feature_init=fi, dtype=np.float64)
        pos = 0
        for k, n in enumerate(plan):
            pre(pcm[b, pos:pos + n * 1280])
            pos += n * 1280
            wins = [pre.get_features(16, -16 - j) for j in range(n - 1, -1, -1)] if n > 1 else [pre.get_features(16)]
            newest = pre.get_features(16).astype(np.float64).reshape(-1)
            if hslot[b] < 0:
                want = 0.0
            else:
                raw = max(OH.forward(cands[hslot[b]], w, np.float64)[0, 0] for w in wins)
                if vslot[b] >= 0 and np.float32(raw) >= np.float32(thr):
                    z = float(bias[b]) + float((newest - mean[b].astype(np.float64)) @ weight[b].astype(np.float64))
                    want = 1.0 / (1.0 + np.exp(-z))
                else:
                    want = raw
            a_raw = max(OH.forward(alexa, w, np.float64)[0, 0] for w in wins)
            a_want = float(verifier_proba(ords[b % 2], newest.reshape(1, 16, 96))[0]) if np.float32(a_raw) >= thr \
                else a_raw
            worst = max(worst, abs(float(got[k, b, col]) - want), abs(float(got[k, b, 0]) - a_want))
    print(f"8192 streams: max |device - float64 oracle| over {len(sample)} streams = {worst:.2e}")
    assert worst <= 1e-3
    assert (got[:, hslot < 0, col] == 0.0).all()


def test_ragged_steps_equal_lockstep(torch_cuda, built_library):
    torch = torch_cuda
    _, _, _, _, _, _, _, fi, pcm = _setup()
    rag, _, col, _, _ = _engine(3, 20, 0.0, True)
    lock, _, _, _, _ = _engine(3, 20, 0.0, True)
    rng = np.random.default_rng(5)
    pos_r = np.zeros(STREAMS, np.int64)
    pos_l = 0
    for _ in range(4):
        counts = rng.integers(0, 3, STREAMS).astype(np.int32)
        counts[0] = 2
        n = int(counts.max())
        x = np.zeros((STREAMS, n * 1280), np.int16)
        for b in range(STREAMS):
            x[b, :counts[b] * 1280] = pcm[b, pos_r[b]:pos_r[b] + counts[b] * 1280]
        sentinel = torch.full((STREAMS, rag.ctx.n_outputs), -7.0, device="cuda")
        got = rag.step_ragged(torch.from_numpy(x).cuda(), counts, out=sentinel).cpu().numpy()
        pos_r += counts * 1280
        held = counts == 0
        assert (got[held] == -7.0).all()                     # held rows are not written
        # the lockstep handle steps every stream by 2 chunks: streams that stepped 2 chunks from the same samples
        lx = torch.from_numpy(np.ascontiguousarray(pcm[:, pos_l:pos_l + 2 * 1280])).cuda()
        ref = lock.step(lx, 2).cpu().numpy()
        pos_l += 2 * 1280
        same = (pos_r == pos_l) & (counts == 2)
        assert same.sum() > 0
        assert np.array_equal(got[same], ref[same])


def test_launch_count(torch_cuda, built_library):
    torch = torch_cuda
    from openwakeword_b200.custom_verifier_model import linear_verifier_params
    x = torch.zeros((64, 1280), dtype=torch.int16, device="cuda")

    def per_step(eng):
        eng.step(x); torch.cuda.synchronize()
        n0 = eng.ctx.launch_count
        eng.step(x); torch.cuda.synchronize()
        return eng.ctx.launch_count - n0
    both = _engine(3, 11, 0.0, True, n_streams=64)[0]
    ordinary = _engine(3, 11, 0.0, False, n_streams=64)[0]
    ob = ordinary.add_verifier_bank(0, 4, 0.0)
    ordinary.ctx.load_verifier(ob, 0, *linear_verifier_params(_setup()[6][3]))
    assert per_step(both) == per_step(ordinary)


def _clips(rng, n):
    lens = rng.integers(100, 40000, n)
    lens[:3] = [0, 700, 2 * 16000]
    return [np.clip(rng.normal(0, 5000, int(L)), -32768, 32767).astype(np.int16) for L in lens]


@pytest.mark.parametrize("chunk", [1280, 2000])
@pytest.mark.parametrize("mode,split_from", [(2, 11), (3, 11)])
def test_bulk_clip_streams_equal_clip_slot_path(torch_cuda, built_library, mode, split_from, chunk):
    """oww_predict_clips_streams on clips of mixed streams equals, clip by clip, the one-clip-slot path with the clip
    slots set to that clip's stream's slots (the path the existing tests pin to streaming), bit for bit.  The clips span
    several slabs; at chunk_size 1280 the 40 equal clips at the end form slabs of their own, which take the direct path
    (every call one step, the heads writing the score rows in place)."""
    torch = torch_cuda
    from openwakeword_b200.model import _concat_clips
    hslots, vslots, *_ = _setup()
    eng, bank, col, vb, ob = _engine(mode, split_from, 0.0, True)
    rng = np.random.default_rng(11)
    clips = _clips(rng, 90) + [np.clip(rng.normal(0, 5000, 60000), -32768, 32767).astype(np.int16) for _ in range(40)]
    streams = rng.choice([0, 1, 2, 4, 5, 7, 11, 14, 63, 150], len(clips)).astype(np.int32)
    streams[:70:2] = 4                               # > 64 rows on one slot
    pcm, off = _concat_clips(clips)
    fi = _setup()[7]
    ctx = eng.ctx
    n_out = ctx.n_outputs
    from openwakeword_b200 import _native
    calls = np.array([_native.clip_schedule(chunk, len(c) + 32000).size for c in clips])
    row_off = np.concatenate([[0], np.cumsum(calls)])
    steps = calls * chunk // 1280
    assert _native.clip_slab_plan(steps[steps > 0])[0] > 1
    # the equal clips lead the longest-first order, more than 5 % longer than every other clip: no other clip joins
    # their slabs, so each of those slabs holds consecutive clips of one step count
    assert steps[90:].min() == steps[90:].max() and 20 * (steps[90] - steps[:90].max()) > steps[90]
    d = torch.from_numpy(pcm).cuda()

    def run(offsets, cs):
        rows = int(sum(_native.clip_schedule(chunk, int(offsets[i + 1] - offsets[i]) + 32000).size
                       for i in range(len(offsets) - 1)))
        raw = torch.full((rows, n_out), -5.0, device="cuda")
        st = torch.zeros(rows, dtype=torch.uint8, device="cuda")
        ctx.predict_clips_ragged(d, offsets, 16000, chunk, fi, raw, st, None, clip_streams=cs)
        return raw.cpu().numpy(), st.cpu().numpy()
    got, stepped = run(off, streams)
    for s in np.unique(streams):
        ctx.set_head_bank_clip_slot(bank, int(hslots[s]))
        ctx.set_verifier_clip_slot(vb, int(vslots[s]))
        ctx.set_verifier_clip_slot(ob, 0)
        for i in np.nonzero(streams == s)[0]:
            ref, st = run(np.array([off[i], off[i + 1]], np.int64), None)
            g = got[row_off[i]:row_off[i + 1]]
            m = st.astype(bool)
            assert np.array_equal(stepped[row_off[i]:row_off[i + 1]].astype(bool), m)
            assert np.array_equal(g[m], ref[m]), (s, i)


def test_model_predict_clips_streams_equal_streaming(torch_cuda, built_library):
    """Model.predict_clips(clips, streams=) equals streaming the padded clips on those streams, bit for bit, with
    calls that step no chunk (chunk_size 640, re-verified on the host) and multi-chunk calls (2000)."""
    from openwakeword_b200 import Model
    from helpers import emb_weights as _emb
    rng = np.random.default_rng(21)
    B = 12
    cands = _cands()
    vers = _setup()[6]
    fi = _setup()[7]
    sm = {b: cands[b % 3] for b in range(B) if b % 4 != 3}
    sv = {b: vers[b % 4] for b in range(B) if b % 5 != 4}
    for chunk in (640, 2000):
        m = Model(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")}], embedding_model_path=_emb(),
                  feature_init=fi, n_streams=B, max_chunks=3, stream_models={"mine": sm},
                  stream_verifiers={"mine": sv}, custom_verifier_threshold=0.0)
        clips = np.clip(rng.normal(0, 5000, (B, 30000)), -32768, 32767).astype(np.int16)
        streams = np.arange(B)
        bulk = m.predict_clips(list(clips), padding=1, chunk_size=chunk, streams=streams)
        m.reset(fi)
        data = np.concatenate([np.zeros((B, 16000), np.int16), clips, np.zeros((B, 16000), np.int16)], axis=1)
        for j, i in enumerate(range(0, data.shape[1] - chunk, chunk)):
            r = m.predict(data[:, i:i + chunk])
            for b in range(B):
                assert bulk[b][j]["mine"] == r["mine"][b], (chunk, j, b)
                assert bulk[b][j]["alexa"] == r["alexa"][b], (chunk, j, b)
        assert all(bulk[b][j]["mine"] == 0.0 for b in range(3, B, 4) for j in range(len(bulk[b])))


def _golden_head(g):
    h = copy.deepcopy(head("alexa_v0.1"))
    last = h["layers"][-1]
    last["b"] = ((last["b"] + np.float32(g["bias_shift"])) * np.float32(g["spread"])).astype(np.float32)
    last["W"] = (last["W"] * np.float32(g["spread"])).astype(np.float32)
    return h


def test_train_stream_verifiers(torch_cuda, built_library, tmp_path):
    """Enrollment against each stream's own model: the golden's head in a bank slot gives the golden's passes and
    windows; batched users equal users enrolled alone; streaming afterwards equals a Model built from the pickles;
    refusals."""
    from openwakeword_b200 import Model
    from openwakeword_b200.custom_verifier_model import dumps_verifier, enrollment_passes
    g = np.load(os.path.join(GOLDEN, "enroll_alexa.npz"))
    assert float(g["nearest"]) >= 2e-3
    gh = _golden_head(g)
    emb = emb_weights(int(g["emb_seed"]))
    # one user against the golden: the golden head sits in slot 1 of a bank, stream 3 on it
    from openwakeword_b200.custom_verifier_model import enroll
    others = _cands(2)
    m = Model(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")}], embedding_model_path=emb, cnn_mode=3,
              n_streams=4, stream_models={"mine": {0: others[0], 3: gh}})
    # seeded after the construction: assigning the stream models resets the streams, which draws a noise feature_init
    # of its own; the reference draws one, then the pass offsets
    pos, neg = [g["pos0"], g["pos1"]], [g["neg0"]]
    np.random.seed(int(g["seed"]))
    fi = m.preprocessor._get_embeddings(np.random.randint(-1000, 1000, 16000 * 4).astype(np.int16))
    r = enroll(m, "mine", [(pos, neg)], feature_init=fi, streams=[3])[0]
    assert [o for p_, _, o, _ in r["passes"] if p_] == g["offsets"].tolist()
    assert r["counts"].tolist() == g["counts"].tolist()
    np.random.seed(int(g["seed"]))
    res = m.train_stream_verifiers("mine", {3: (pos, neg)})
    pipe, st = res[3]
    assert st in (0, 1)
    assert np.array_equal(pipe.steps[2][1].coef_, r["pipeline"].steps[2][1].coef_)
    p = pipe.predict_proba(g["probe"])[:, 1]
    d = np.abs(p - g["probe_p"]).max()
    print(f"golden enrollment through a bank slot: max |p - reference| = {d:.2e}")
    assert d <= 1e-3
    assert m.stream_verifiers["mine"] == {3: pipe}
    # batched: 48 of 64 streams, several slots, one shared
    rng = np.random.default_rng(3)
    B = 64
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    slot_heads = [gh, copy.deepcopy(gh), gh]
    slot_heads[1]["layers"][-1]["b"] = (slot_heads[1]["layers"][-1]["b"] + np.float32(0.5)).astype(np.float32)
    sm = {b: slot_heads[b % 3] for b in range(B)}
    kw = dict(wakeword_models=[{"name": "alexa", "head": head("alexa_v0.1")}], embedding_model_path=emb,
              feature_init=fi)
    src = np.concatenate([g["pos0"], g["pos1"]])
    users = {}
    for b in rng.permutation(B)[:48]:
        L = int(rng.integers(16000, min(32000, len(src))))
        a = int(rng.integers(0, len(src) - L + 1))
        users[int(b)] = ([src[a:a + L]], [g["neg0"][:16000]])
    m = Model(n_streams=B, stream_models={"mine": sm}, **kw)
    np.random.seed(99)
    res = m.train_stream_verifiers("mine", users)
    assert all(st == 0 for _, st in res.values())
    np.random.seed(99)
    for b, (pos, neg) in users.items():
        state = np.random.get_state()
        one = Model(n_streams=1, stream_models={"mine": {0: slot_heads[b % 3]}}, **kw)
        r1 = one.train_stream_verifiers("mine", {0: (pos, neg)})[0][0]
        assert np.array_equal(r1.steps[2][1].coef_, res[b][0].steps[2][1].coef_), b
        assert np.array_equal(r1.steps[1][1].mean_, res[b][0].steps[1][1].mean_), b
        np.random.set_state(state)
        enrollment_passes([len(c) for c in pos], [len(c) for c in neg])
    pickles = {}
    for b in users:
        (tmp_path / f"{b}.pkl").write_bytes(dumps_verifier(res[b][0]))
        pickles[b] = str(tmp_path / f"{b}.pkl")
    ref = Model(n_streams=B, stream_models={"mine": sm}, stream_verifiers={"mine": pickles},
                custom_verifier_threshold=0.3, **kw)
    m.custom_verifier_threshold = 0.3
    pcm = np.clip(rng.normal(0, 3000, (B, 30 * 1280)), -32768, 32767).astype(np.int16)
    pcm[:, :len(src[:30 * 1280])] += src[:30 * 1280][None] // 2
    for s in range(30):
        a = m.predict(pcm[:, s * 1280:(s + 1) * 1280])["mine"]
        b_ = ref.predict(pcm[:, s * 1280:(s + 1) * 1280])["mine"]
        assert np.array_equal(a, b_), s
    # refusals
    sub = {next(iter(users)): users[next(iter(users))]}
    bare = Model(n_streams=2, stream_models={"mine": {0: gh}}, **kw)
    with pytest.raises(ValueError):
        bare.train_stream_verifiers("mine", {1: sub[next(iter(sub))]})     # stream 1 has no model
    multi = Model(n_streams=2, stream_models={"t": {0: head("timer_v0.1")}}, **kw)
    with pytest.raises(ValueError):
        multi.train_stream_verifiers("t", {0: sub[next(iter(sub))]})
    with pytest.raises(ValueError):
        m.train_stream_verifiers("nope", sub)
    with pytest.raises(ValueError):
        m.train_stream_verifiers("mine", sub, N=4)
    with pytest.raises(ValueError):
        m.train_stream_verifiers("mine", sub, threshold=0.4)


def test_abi_refusals(torch_cuda, built_library):
    torch = torch_cuda
    from openwakeword_b200 import _native
    eng, bank, col, vb, ob = _engine(3, 11, 0.0, True, n_streams=8)
    ctx = eng.ctx
    with pytest.raises(_native.NativeError):
        ctx.add_bank_verifier_bank(5, 4, 0.1)                # no such head bank
    with pytest.raises(_native.NativeError):
        ctx.add_bank_verifier_bank(bank, 4, 0.1)             # a second verifier bank on the same head bank
    with pytest.raises(_native.NativeError):
        ctx.add_bank_verifier_bank(bank, 0, 0.1)             # capacity
    bank2, _, _ = eng.add_head_bank(_cands()[0], 2)
    with pytest.raises(_native.NativeError):
        ctx.add_bank_verifier_bank(bank2, (1 << 20) + 1, 0.1)
    pcm = torch.zeros(4000, dtype=torch.int16, device="cuda")
    off = np.array([0, 2000, 4000], np.int64)
    raw = torch.zeros((8, ctx.n_outputs), device="cuda")
    st = torch.zeros(8, dtype=torch.uint8, device="cuda")
    with pytest.raises(_native.NativeError):
        ctx.predict_clips_ragged(pcm, off, 0, 1280, None, raw, st, None, clip_streams=[0, 8])    # stream out of range
    with pytest.raises(_native.NativeError):
        ctx._check(ctx.lib.oww_predict_clips_streams(ctx.h, _native._ptr(pcm), _native._ptr(off), 2, 0, 1280, None, 41,
                                                     _native._ptr(raw), _native._ptr(st), None, None, None))
