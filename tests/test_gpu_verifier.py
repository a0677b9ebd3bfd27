"""-m gpu: custom verifier models on the device (verifier.cu) against scikit-learn, the reference goldens, the oracle
and the host path; bulk against streaming; launch counts and ABI errors."""
import os

import numpy as np
import pytest

import fake_backend
from helpers import GOLDEN, VERIFIER_CASES, case_model as _model, emb_weights, head, load_case, verifier_pipeline as _pipeline

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _fit(rng, n_in, scale=1.0):
    """a verifier of the reference's form on random windows (C = 0.001 as train_verifier_model uses)."""
    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import FunctionTransformer, StandardScaler
    from openwakeword_b200.custom_verifier_model import flatten_features
    off, sc = rng.normal(0, 2, 96), rng.uniform(0.2, 3, 96) * scale
    x = (rng.normal(0, 1, (60, n_in, 96)) * sc + off).astype(np.float32)
    y = np.array([1] * 20 + [0] * 40)
    x[:20] += rng.normal(0, 0.5, 96).astype(np.float32)
    return make_pipeline(FunctionTransformer(flatten_features), StandardScaler(),
                         LogisticRegression(random_state=0, max_iter=2000, C=0.001)).fit(x, y)


def test_verifier_predict_vs_sklearn(torch_cuda, built_library):
    from openwakeword_b200.engine import StreamEngine
    rng = np.random.default_rng(0)
    eng = StreamEngine([head("alexa_v0.1"), head("timer_v0.1")], 4, embedding=emb_weights())
    for hi, tag in ((0, "alexa"), (1, "timer")):
        v = _pipeline(tag)
        n_in = v.steps[-1][1].coef_.shape[1] // 96
        bank = eng.add_verifier_bank(hi, 3, 0.5)
        eng.load_verifier(bank, 2, v)
        x = (rng.normal(0, 1, (4096, n_in, 96)) * rng.uniform(0.5, 3, 96) + rng.normal(0, 2, 96)).astype(np.float32)
        got = eng.ctx.verifier_predict_host(bank, 2, x)
        ref = v.predict_proba(x)[:, -1]
        print(f"{tag}: max |device - predict_proba| over 4096 windows = {np.abs(got - ref).max():.2e}")
        assert np.abs(got - ref).max() <= 1e-5


@pytest.mark.parametrize("mode", [0, 3])
@pytest.mark.parametrize("tag", VERIFIER_CASES)
def test_verifier_golden_on_gpu(torch_cuda, built_library, tag, mode):
    c = load_case(tag)
    parent, thr = str(c["parent"]), float(c["threshold"])
    m = _model(c, cnn_mode=mode, custom_verifier_models={parent: os.path.join(GOLDEN, str(c["verifier"]))},
               custom_verifier_threshold=thr)
    assert parent in m._vbanks
    reads = []
    real = m.preprocessor.ctx.get_features
    m.preprocessor.ctx.get_features = lambda *a, **k: reads.append(a) or real(*a, **k)
    res = m.predict_clip(c["pcm"], padding=1, chunk_size=int(c["chunk"]))
    got = np.array([[r[lab] for lab in c["labels"]] for r in res], np.float32)
    assert not reads                                    # every call ran a step: verified on the device
    plain = _model(c, cnn_mode=mode).predict_clip(c["pcm"], padding=1, chunk_size=int(c["chunk"]))
    plain = np.array([[r[lab] for lab in c["labels"]] for r in plain], np.float32)
    n_ver = int((plain >= np.float32(thr)).sum())
    err = np.abs(got - c["scores"]).max()
    print(f"{tag} mode {mode}: max |device - reference| = {err:.2e}, verified {n_ver} (reference {int(c['n_verified'])})")
    assert n_ver == int(c["n_verified"])
    assert err <= 1e-3


STREAMS = 151
PLAN = [1, 1, 1, 2, 1, 3, 1, 1, 2, 1, 1]
RESET_AT, SWAP_AT = 6, 8
CONFIGS = [(0, 11), (2, 11), (3, 11), (3, 20)]      # (cnn_mode, split_from): mode 3 heads outside / inside the fused kernel
_oracle_cache = {}


def _setup_151():
    rng = np.random.default_rng(151)
    heads = [head("alexa_v0.1"), head("timer_v0.1"), head("hey_jarvis_v0.1")]
    n_ins = [16, 34, 16]
    pool = [(0, _fit(rng, 16)), (0, _fit(rng, 16, 2.0)), (1, _fit(rng, 34)), (1, _fit(rng, 34, 0.5)), (2, _fit(rng, 16))]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    pcm = np.clip(rng.normal(0, 4000, (STREAMS, sum(PLAN) * 1280)), -32768, 32767).astype(np.int16)
    # slots per parent bank: stream b (b % 3 != 0) uses pool verifier (b // 3) % (verifiers of that parent)
    per_parent = {p: [i for i, (q, _) in enumerate(pool) if q == p] for p in range(3)}
    assign = {p: np.array([-1 if b % 3 == 0 else (b + p) % len(per_parent[p]) for b in range(STREAMS)], np.int32)
              for p in range(3)}
    swap_ids = np.arange(1, 151, 15)[:10]
    swapped = {p: np.where(a[swap_ids] < 0, 0, -1).astype(np.int32) for p, a in assign.items()}
    reset_ids = [0, 2, 75, 150]
    return heads, n_ins, pool, per_parent, assign, swap_ids, swapped, reset_ids, fi, pcm


def _thresholds(heads, fi, pcm):
    """per parent: the median of its score columns over the run, without verifiers (cnn_mode 0)."""
    from openwakeword_b200.engine import StreamEngine
    import torch
    eng = StreamEngine(heads, STREAMS, embedding=emb_weights(), feature_init=fi, cnn_mode=0, max_chunks=3)
    out, pos = [], 0
    for n in PLAN:
        out.append(eng.step(torch.from_numpy(np.ascontiguousarray(pcm[:, pos:pos + n * 1280])).cuda(), n).cpu().numpy())
        pos += n * 1280
    out = np.stack(out)
    return [float(np.median(out[..., c0:c0 + n])) for c0, n in eng.columns]


def _run_151(torch, mode, split_from, with_banks=True, fake=None):
    heads, n_ins, pool, per_parent, assign, swap_ids, swapped, reset_ids, fi, pcm = _setup_151()
    if "thr" not in _oracle_cache:
        _oracle_cache["thr"] = _thresholds(heads, fi, pcm)
    thr = _oracle_cache["thr"]
    if fake is None:
        from openwakeword_b200.engine import StreamEngine
        eng = StreamEngine(heads, STREAMS, embedding=emb_weights(), feature_init=fi, cnn_mode=mode, max_chunks=3,
                           split_from=split_from)
        ctx, step = eng.ctx, lambda x, n: eng.step(torch.from_numpy(np.ascontiguousarray(x)).cuda(), n).cpu().numpy()
        reset = lambda ids: eng.reset_async(fi, stream_ids=ids)
        assign_fn = lambda bank, ids, slots: eng.assign_verifier(bank, slots, ids)
    else:
        ctx = fake
        def step(x, n):
            out = np.zeros((x.shape[0], ctx.n_outputs), np.float32)
            ctx.step_host(np.ascontiguousarray(x), n, out)
            return out
        reset = lambda ids: ctx.reset(ids, fi)
        assign_fn = lambda bank, ids, slots: ctx.assign_verifier(bank, ids, slots)
    rows = fake.rows if fake is not None else np.arange(STREAMS)
    banks = []
    if with_banks:
        head_ids = [0, 1, 2]                       # add_head order: alexa 0, timer 1, jarvis main 2 (its verifier net 3)
        for p in range(3):
            bank = ctx.add_verifier_bank(head_ids[p], STREAMS, thr[p])
            for k, i in enumerate(per_parent[p]):
                from openwakeword_b200.custom_verifier_model import linear_verifier_params
                ctx.load_verifier(bank, k, *linear_verifier_params(pool[i][1]))
            assign_fn(bank, None, assign[p][rows])
            banks.append(bank)
    scores, feats, pos = [], [], 0
    for k, n in enumerate(PLAN):
        if k == RESET_AT:
            ids = [j for j, b in enumerate(rows) if b in reset_ids]
            if ids:
                reset(ids)
        if k == SWAP_AT and with_banks:
            sel = [j for j, b in enumerate(rows) if b in swap_ids]
            if sel:
                for p, bank in enumerate(banks):
                    assign_fn(bank, sel, swapped[p][[list(swap_ids).index(rows[j]) for j in sel]])
        scores.append(step(pcm[rows, pos:pos + n * 1280], n))
        feats.append(None if fake is not None or with_banks else
                     [[ctx.get_features(b, n_ins[p]) for b in range(STREAMS)] for p in range(3)])
        pos += n * 1280
    return np.stack(scores), feats, (assign, swap_ids, swapped, pool, per_parent, thr)


@pytest.mark.parametrize("mode,split_from", CONFIGS)
def test_151_streams_vs_oracle_and_host_path(torch_cuda, built_library, mode, split_from):
    torch = torch_cuda
    from openwakeword_b200 import weights as W
    got, _, (assign, swap_ids, swapped, pool, per_parent, thr) = _run_151(torch, mode, split_from)
    # host path on the same engine: the unverified scores, then predict_proba of the stream's verifier on its window
    plain, feats, _ = _run_151(torch, mode, split_from, with_banks=False)
    cols = [(0, 1), (1, 7), (8, 1)]
    want = plain.copy()
    for k in range(len(PLAN)):
        for p, (c0, nc) in enumerate(cols):
            a = assign[p].copy()
            if k >= SWAP_AT:
                a[swap_ids] = swapped[p]
            for b in range(STREAMS):
                blk = want[k, b, c0:c0 + nc]
                if a[b] < 0 or not (blk >= np.float32(thr[p])).any():
                    continue
                v = pool[per_parent[p][a[b]]][1]
                blk[blk >= np.float32(thr[p])] = v.predict_proba(feats[k][p][b][None])[0, -1]
    n_verified = int((got != plain).sum())
    err_host = np.abs(got - want).max()
    # oracle: the fake context (NumPy graphs + the kernel's verifier arithmetic) on sampled streams
    if "oracle" not in _oracle_cache:
        sample = sorted({0, 1, 2, 3, 75, 76, 150} | set(swap_ids[:3].tolist()))
        fake = fake_backend.FakeContext()
        fake.rows = np.array(sample)
        fake.load_embedding(W.pack_embedding_blob(emb_weights()))
        for h in (head("alexa_v0.1"), head("timer_v0.1")):
            fake.add_head(h["n_in"], W.head_desc(h)[1], W.head_desc(h)[2], W.head_desc(h)[3], W.pack_head_blob(h))
        g = head("hey_jarvis_v0.1")
        ids = [fake.add_head(16, W.head_desc(g[q])[1], W.head_desc(g[q])[2], W.head_desc(g[q])[3],
                             W.pack_head_blob(g[q])) for q in ("main", "verifier")]
        fake.add_gate(ids[0], ids[1], g["threshold"])
        fake.set_streams(len(sample))
        fake.reset(None, _setup_151()[8])
        _oracle_cache["oracle"] = (sample, _run_151(torch, 0, 11, fake=fake)[0])
    sample, ref = _oracle_cache["oracle"]
    # scores within the path's distance to the oracle of a threshold may take the other side of it there: compare the
    # elements whose unverified score is clear of their parent's threshold
    clear = np.ones(plain.shape, bool)
    for p, (c0, nc) in enumerate(cols):
        clear[..., c0:c0 + nc] = np.abs(plain[..., c0:c0 + nc] - np.float32(thr[p])) > 2e-3
    err_oracle = np.abs(got[:, sample] - ref)[clear[:, sample]].max()
    print(f"mode {mode} split {split_from}: {n_verified} verified scores; max |device - host path| = {err_host:.2e}, "
          f"max |device - oracle| ({len(sample)} streams) = {err_oracle:.2e}")
    assert n_verified > 0 and (got == plain).any()
    assert err_host <= 1e-5
    assert err_oracle <= 1e-3


@pytest.mark.parametrize("mode", [0, 3])
def test_predict_clips_equals_streaming_predict_clip(torch_cuda, built_library, mode):
    """The bulk path of oww_predict_clips with the tensor-core CNN and heads (cnn_mode 3) and with the fp32 CNN and
    heads.cu (cnn_mode 0) applies stream 0's verifier (the clip slot) and must equal predict_clip after a reset bit for
    bit."""
    c = load_case("verifier_alexa_c1280")
    parent, thr = str(c["parent"]), float(c["threshold"])
    m = _model(c, cnn_mode=mode, custom_verifier_models={parent: os.path.join(GOLDEN, str(c["verifier"]))},
               custom_verifier_threshold=thr)
    rng = np.random.default_rng(9)
    clips = np.stack([c["pcm"]] + [np.clip(rng.normal(0, a, c["pcm"].shape[0]), -32768, 32767).astype(np.int16)
                                   for a in (500, 3000, 9000)])
    bulk, labels = m.predict_clips_array(clips, padding=1, feature_init=c["feature_init"])
    for i, clip in enumerate(clips):
        m.reset(c["feature_init"])
        res = m.predict_clip(clip, padding=1)
        stream = np.array([[r[lab] for lab in labels] for r in res], np.float32)
        assert np.array_equal(stream, bulk[i]), (i, np.abs(stream - bulk[i]).max())
    np.testing.assert_allclose(bulk[0], c["scores"], atol=1e-3)
    m.set_custom_verifier(parent, None)
    unverified, _ = m.predict_clips_array(clips, padding=1, feature_init=c["feature_init"])
    assert (unverified != bulk).any() and (unverified == bulk).any()


def test_launch_counts_and_abi_errors(torch_cuda, built_library):
    import torch
    from openwakeword_b200 import _native
    from openwakeword_b200.engine import StreamEngine
    hs = [head("alexa_v0.1"), head("timer_v0.1")]
    x = torch.zeros((64, 1280), dtype=torch.int16, device="cuda")

    def per_step(eng):
        eng.step(x); torch.cuda.synchronize()
        n0 = eng.ctx.launch_count
        eng.step(x); torch.cuda.synchronize()
        return eng.ctx.launch_count - n0
    plain = StreamEngine(hs, 64, embedding=emb_weights())
    banked = StreamEngine(hs, 64, embedding=emb_weights())
    bank = banked.add_verifier_bank(0, 4, 0.0)
    assert per_step(banked) == per_step(plain) + 1          # one verifier launch for every bank, nothing without
    v = _pipeline("alexa")
    with pytest.raises(_native.NativeError):
        banked.add_verifier_bank(0, 4, 0.1)                  # a second bank on the same head
    with pytest.raises(ValueError):
        banked.load_verifier(bank, 0, _pipeline("timer"))    # D of another head
    with pytest.raises(ValueError):
        banked.load_verifier(bank, 0, (np.zeros(100, np.float32), np.zeros(1536, np.float32), 0.0))
    with pytest.raises(_native.NativeError):
        banked.ctx.add_verifier_bank(5, 4, 0.1)              # no such head
    with pytest.raises(_native.NativeError):
        banked.ctx.add_verifier_bank(0, 0, 0.1)              # capacity
    with pytest.raises(_native.NativeError):
        banked.load_verifier(bank, 4, v)                     # slot == capacity
    with pytest.raises(_native.NativeError):
        banked.load_verifier(7, 0, v)                        # no such bank
    with pytest.raises(_native.NativeError):
        banked.assign_verifier(bank, [0], [64])              # stream id out of range
    with pytest.raises(_native.NativeError):
        banked.assign_verifier(bank, [4], [1])               # slot out of range
    with pytest.raises(_native.NativeError):
        banked.ctx.set_verifier_clip_slot(bank, 4)
    with pytest.raises(_native.NativeError):
        banked.ctx.verifier_predict_host(bank, -1, np.zeros((2, 16, 96), np.float32))
    # oww_set_streams drops the assignments; oww_reset keeps them
    banked.load_verifier(bank, 1, v)
    banked.assign_verifier(bank, [1, 1], [3, 1])
    banked.reset()
    plain.reset()
    got = banked.step(x).cpu().numpy()
    ref = plain.step(x).cpu().numpy()
    p1 = banked.ctx.verifier_predict_host(bank, 1, np.stack([banked.ctx.get_features(b, 16) for b in (3, 1)]))
    assert got[3, 0] == p1[0] and got[1, 0] == p1[1] and np.array_equal(np.delete(got, [1, 3], 0), np.delete(ref, [1, 3], 0))
    banked.ctx.set_streams(64)
    banked.reset()
    plain.reset()
    assert np.array_equal(banked.step(x).cpu().numpy(), plain.step(x).cpu().numpy())


@pytest.mark.parametrize("mode", [0, 3])
def test_calls_longer_than_max_chunks_on_gpu(torch_cuda, built_library, mode):
    """Calls split into several device steps run them without the banks and verify the max once, on the newest window."""
    from openwakeword_b200 import Model
    from oracle.verifier import VerifiedOracleModel
    c = load_case("verifier_alexa_c1280")
    name = c["names"][0]
    rng = np.random.default_rng(12)
    plan = [1280] * 6 + [5 * 1280, 1280, 7 * 1280, 640, 640, 3 * 1280]
    pcm = np.clip(rng.normal(0, 3000, sum(plan)), -32768, 32767).astype(np.int16)
    specs = [{"name": name, "head": head(name)}]
    thr = 0.06
    kw = dict(wakeword_models=specs, embedding_model_path=emb_weights(), feature_init=c["feature_init"], max_chunks=2,
              cnn_mode=mode)
    m = Model(custom_verifier_models={name: os.path.join(GOLDEN, "verifier_alexa.pkl")}, custom_verifier_threshold=thr, **kw)
    plain = Model(**kw)
    om = VerifiedOracleModel(emb_weights(), {name: head(name)}, verifiers={name: _pipeline("alexa")}, threshold=thr,
                             feature_init=c["feature_init"])
    got, raw, ref, pos = [], [], [], 0
    for n in plan:
        got.append(m.predict(pcm[pos:pos + n])[name])
        raw.append(plain.predict(pcm[pos:pos + n])[name])
        ref.append(om.predict(pcm[pos:pos + n])[name])
        pos += n
    got, raw, ref = (np.array(a, np.float32) for a in (got, raw, ref))
    clear = np.abs(raw - np.float32(thr)) > 2e-3             # same side of the threshold as the oracle
    print(f"mode {mode}: device {got}, oracle {ref}; max |device - oracle| = {np.abs(got - ref)[clear].max():.2e}")
    long = [k for k, n in enumerate(plan) if n > 2 * 1280]
    assert (got[long] != raw[long]).any()
    assert np.abs(got - ref)[clear].max() <= 1e-3


def test_host_path_steps_see_assignments_and_loads(torch_cuda, built_library):
    """assign_verifier / load_verifier before step_host and submit (the handle's own stream) take effect at that step."""
    from openwakeword_b200.engine import StreamEngine
    rng = np.random.default_rng(4)
    hs = [head("alexa_v0.1")]
    B = 256
    pcm = np.clip(rng.normal(0, 3000, (B, 4 * 1280)), -32768, 32767).astype(np.int16)
    eng = StreamEngine(hs, B, embedding=emb_weights())
    ref = StreamEngine(hs, B, embedding=emb_weights())
    bank = eng.add_verifier_bank(0, 2, 0.0)
    v0, v1 = _pipeline("alexa"), _fit(rng, 16)
    eng.load_verifier(bank, 0, v0)
    for k in range(4):
        chunk = np.ascontiguousarray(pcm[:, k * 1280:(k + 1) * 1280])
        want_slot = np.full(B, -1)
        if k == 1:
            eng.assign_verifier(bank, np.zeros(B // 2, np.int32), np.arange(0, B, 2))
        if k == 2:
            eng.load_verifier(bank, 1, v1)
            eng.assign_verifier(bank, np.ones(B // 2, np.int32), np.arange(1, B, 2))
        if k >= 1:
            want_slot[0::2] = 0
        if k >= 2:
            want_slot[1::2] = 1
        got = eng.collect(eng.submit(chunk)) if k % 2 else eng.step_host(chunk)
        r = ref.step_host(chunk)
        feats = np.stack([ref.ctx.get_features(b, 16) for b in range(B)])
        want = r[:, 0].copy()
        for s, v in ((0, v0), (1, v1)):
            sel = want_slot == s
            if sel.any():
                want[sel] = v.predict_proba(feats[sel])[:, -1]
        assert np.abs(got[:, 0] - want).max() <= 1e-5, k


def test_predict_clips_warns_about_host_only_verifiers(torch_cuda, built_library, tmp_path):
    import pickle
    from test_abi_and_host import _ConstVerifier
    c = load_case("verifier_alexa_c1280")
    p = str(tmp_path / "const.pkl")
    with open(p, "wb") as f:
        pickle.dump(_ConstVerifier(0.7), f)
    m = _model(c, custom_verifier_models={c["names"][0]: p})
    with pytest.warns(UserWarning, match="not device-runnable"):
        m.predict_clips(c["pcm"][None])
