"""-m gpu: verifier training on the device (verifier_fit.cu, oww_fit_verifiers / oww_load_verifiers) against the float64
Newton solve and scikit-learn; batch invariance bit for bit; per-user statuses and refusals; train_custom_verifier end
to end."""
import copy

import numpy as np
import pytest

from helpers import emb_weights, head
from verifier_fit_ref import fit_verifier_f64, linear_proba

pytestmark = pytest.mark.gpu
sklearn = pytest.importorskip("sklearn")

# max |p_device - p_f64| on training and held-out windows.  Measured on an H100 80GB HBM3 at a 700 W limit: 3.2e-10
# at C = 1e-3, 3.1e-7 at C = 1, 3.0e-5 at C = 100 (the stopping rule max |g| <= tol*C*n loosens with C); the C = 100
# bound is the smallest power of two at least 4x above its worst case.
BOUND = {1e-3: 1e-6, 1.0: 1e-6, 100.0: 2.0 ** -13}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


@pytest.fixture(scope="module")
def ctx(torch_cuda, built_library):
    from openwakeword_b200 import _native
    return _native.Context(device=0, cnn_mode=_native.CNN_FP32_WINDOW, max_chunks=1)


def _case(rng, n_in, n_pos, n_neg, kind):
    sc = rng.uniform(0.2, 3, 96)
    x = (rng.normal(0, 1, (n_pos + n_neg, n_in, 96)) * sc + rng.normal(0, 2, 96)).astype(np.float32)
    x[:n_pos] += rng.normal(0, 0.4, 96).astype(np.float32)
    if kind == "separable":
        x[:n_pos, 0, 0] += 50.0
    elif kind == "duplicates":
        x[n_pos // 2:n_pos] = x[:n_pos - n_pos // 2]
        x[-5:] = x[-10:-5]
    elif kind == "constant":
        x[:, 2, 10:20] = 1.25
        x[:, -1, :3] = 0.0
    elif kind == "offset":
        x += np.float32(1e3)
    y = np.array([1] * n_pos + [0] * n_neg)
    perm = rng.permutation(len(y))
    return x[perm], y[perm]


CASES = [  # (n_in, n_pos, n_neg, kind)
    (16, 1, 1, "plain"), (16, 60, 640, "plain"), (16, 30, 1500, "plain"),   # 1:50 imbalance
    (16, 1500, 1500, "plain"), (16, 80, 320, "separable"), (16, 90, 300, "duplicates"),
    (16, 70, 400, "constant"), (16, 100, 600, "offset"), (34, 120, 580, "plain"), (34, 40, 260, "offset"),
]


def _fit_dev(ctx, torch, xs, ys, C, max_iter=100, tol=1e-10):
    """users with windows xs[u] [n_u, n_in, 96] as plain arrays (first_row = i*n_in) in one call -> host dict"""
    n_in = xs[0].shape[1]
    rows = np.concatenate([x.reshape(-1, 96) for x in xs]) if xs else np.zeros((0, 96), np.float32)
    off = np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int64)
    first = np.arange(off[-1], dtype=np.int64) * n_in
    lab = np.concatenate([np.asarray(y) != 0 for y in ys]).astype(np.uint8)
    dev = torch.device("cuda", 0)
    out = ctx.fit_verifiers(torch.from_numpy(rows).to(dev), n_in, torch.from_numpy(first).to(dev), off,
                            torch.from_numpy(lab).to(dev), C, max_iter, tol)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("C", [1e-3, 1.0, 100.0])
def test_fit_against_f64(ctx, torch_cuda, C):
    rng = np.random.default_rng(int(C * 1000) + 1)
    worst = 0.0
    for n_in in (16, 34):
        cases = [_case(rng, *c) for c in CASES if c[0] == n_in]
        fit = _fit_dev(ctx, torch_cuda, [x for x, _ in cases], [y for _, y in cases], C)
        for u, (x, y) in enumerate(cases):
            assert fit["status"][u] == 0, (n_in, u, fit["status"][u], fit["iters"][u])
            ref = fit_verifier_f64(x, y, C=C)
            np.testing.assert_allclose(fit["mean"][u], ref["mean"], rtol=1e-12, atol=1e-300)
            np.testing.assert_allclose(fit["var"][u], ref["var"], rtol=1e-12, atol=1e-300)
            scale = np.where(ref["scale"] == 1.0, 1.0, np.sqrt(fit["var"][u]))
            held, _ = _case(np.random.default_rng(u), n_in, 500, 500, "plain")
            if np.abs(x).max() > 500:
                held += np.float32(1e3)
            for z in (x, held):
                p_dev = linear_proba(fit["mean"][u], scale, fit["coef"][u], fit["intercept"][u], z)
                p_ref = linear_proba(ref["mean"], ref["scale"], ref["coef"], ref["intercept"], z)
                worst = max(worst, float(np.abs(p_dev - p_ref).max()))
    print(f"C = {C}: max |p_device - p_f64| = {worst:.3e} (bound {BOUND[C]:.3e})")
    assert worst <= BOUND[C]


def test_train_verifier_model_against_sklearn(torch_cuda, built_library):
    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import FunctionTransformer, StandardScaler
    from openwakeword_b200.custom_verifier_model import flatten_features, linear_verifier_params, train_verifier_model
    rng = np.random.default_rng(11)
    for n_in, n_pos, n_neg in ((16, 60, 140), (16, 200, 1300), (34, 50, 400)):
        x, y = _case(rng, n_in, n_pos, n_neg, "plain")
        dev = train_verifier_model(x, y)
        sk = make_pipeline(FunctionTransformer(flatten_features), StandardScaler(),
                           LogisticRegression(random_state=0, max_iter=2000, C=0.001)).fit(x, y)
        held, _ = _case(np.random.default_rng(1), n_in, 500, 500, "plain")
        for z in (x, held):
            d = np.abs(dev.predict_proba(z)[:, 1] - sk.predict_proba(z)[:, 1]).max()
            print(f"n_in {n_in}, n {len(x)}: max |p_device - p_sklearn| = {d:.2e}")
            assert d <= 1e-3
            mean, w, b = linear_verifier_params(dev)
            p_lin = 1.0 / (1.0 + np.exp(-(b + (z.reshape(len(z), -1) - mean).astype(np.float64) @ w)))
            assert np.abs(p_lin - dev.predict_proba(z)[:, 1]).max() <= 1e-5
        lr, sc = dev.steps[2][1], dev.steps[1][1]
        assert lr.coef_.shape == (1, n_in * 96) and lr.coef_.dtype == np.float64 and list(lr.classes_) == [0, 1]
        assert sc.mean_.dtype == np.float64 and sc.n_samples_seen_ == len(x)


def test_batch_invariance(ctx, torch_cuda):
    """64 users fitted alone equal the same users inside a batch of 8192 (random order, mixed n_u, overlapping windows
    into one row array), bit for bit."""
    torch = torch_cuda
    rng = np.random.default_rng(21)
    n_in, R, U = 16, 200_000, 8192
    rows = rng.normal(0, 1, (R, 96)).astype(np.float32)
    n_u = rng.integers(2, 800, U)
    off = np.concatenate([[0], np.cumsum(n_u)]).astype(np.int64)
    first = rng.integers(0, R - n_in + 1, int(off[-1])).astype(np.int64)
    lab = (rng.uniform(0, 1, int(off[-1])) < 0.3).astype(np.uint8)
    for u in range(U):                        # both classes
        lab[off[u]] = 1; lab[off[u] + 1] = 0
    rows[first[lab == 1]] += np.float32(0.3)
    dev = torch.device("cuda", 0)
    d_rows = torch.from_numpy(rows).to(dev)
    t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    big = ctx.fit_verifiers(d_rows, n_in, torch.from_numpy(first).to(dev), off, torch.from_numpy(lab).to(dev))
    t1.record()
    torch.cuda.synchronize()
    print(f"{U} users, {int(off[-1])} windows: {t0.elapsed_time(t1):.1f} ms (first call, {torch.cuda.get_device_name(0)})")
    big = {k: v.cpu().numpy() for k, v in big.items()}
    assert (big["status"] == 0).all(), np.unique(big["status"], return_counts=True)
    for u in rng.choice(U, 64, replace=False):
        s = slice(off[u], off[u + 1])
        one = ctx.fit_verifiers(d_rows, n_in, torch.from_numpy(first[s].copy()).to(dev),
                                np.array([0, n_u[u]], np.int64), torch.from_numpy(lab[s].copy()).to(dev))
        for k, v in one.items():
            assert np.array_equal(v.cpu().numpy()[0], big[k][u]), (u, k)


def test_statuses_and_refusals(ctx, torch_cuda):
    torch = torch_cuda
    rng = np.random.default_rng(4)
    n_in, R = 4, 400
    rows = rng.normal(0, 1, (R, 96)).astype(np.float32)
    rows[50, 7] = np.nan
    # users: ok | one class | empty | NaN row | window past n_rows | ok
    firsts = [np.arange(0, 40), np.arange(0, 10), np.arange(0), np.arange(45, 60), np.array([10, R - n_in + 1]),
              np.arange(100, 160)]
    labs = [np.arange(40) % 2, np.ones(10), np.zeros(0), np.arange(15) % 2, np.array([0, 1]), np.arange(60) % 3 == 0]
    off = np.concatenate([[0], np.cumsum([len(f) for f in firsts])]).astype(np.int64)
    dev = torch.device("cuda", 0)
    d_rows = torch.from_numpy(rows).to(dev)
    first = torch.from_numpy(np.concatenate(firsts).astype(np.int64)).to(dev)
    lab = torch.from_numpy(np.concatenate(labs).astype(np.uint8)).to(dev)
    out = ctx.fit_verifiers(d_rows, n_in, first, off, lab)
    assert out["status"].cpu().tolist() == [0, 2, 2, 3, 3, 0]
    assert (out["coef"][1:5] == 0).all() and (out["iters"][1:5] == 0).all()
    assert ctx.fit_verifiers(d_rows, n_in, first, off, lab, max_iter=1)["status"].cpu().tolist() == [1, 2, 2, 3, 3, 1]
    torch.cuda.synchronize()
    # refusals leave the outputs untouched
    U, D = len(firsts), n_in * 96
    outs = [torch.full((U, D), 7.0, dtype=torch.float64, device=dev) for _ in range(3)]
    outs += [torch.full((U,), 7.0, dtype=torch.float64, device=dev), torch.full((U,), 7, dtype=torch.int32, device=dev),
             torch.full((U,), 7, dtype=torch.int32, device=dev)]
    ptrs = [o.data_ptr() for o in outs]

    def call(n_in_=n_in, offs=off, Cv=1e-3, it=10, tol=1e-10):
        o = np.ascontiguousarray(offs, np.int64)
        return ctx.lib.oww_fit_verifiers(ctx.h, d_rows.data_ptr(), R, n_in_, first.data_ptr(), o.ctypes.data,
                                         lab.data_ptr(), len(o) - 1, Cv, it, tol, *ptrs, None)
    bad_off = off.copy(); bad_off[3] = bad_off[2] - 1
    for kw in (dict(Cv=0.0), dict(Cv=-1.0), dict(Cv=float("nan")), dict(Cv=float("inf")), dict(n_in_=0),
               dict(n_in_=121), dict(offs=bad_off), dict(it=0), dict(tol=-1.0)):
        assert call(**kw) == -1, kw
    torch.cuda.synchronize()
    for o in outs:
        assert (o == 7).all()
    assert call() == 0


def test_load_verifiers(torch_cuda, built_library):
    """oww_load_verifiers from device memory equals oww_load_verifier from the host, bit for bit in verifier_predict."""
    from openwakeword_b200 import _native
    torch = torch_cuda
    h = head("alexa_v0.1")
    from openwakeword_b200 import weights as W
    ctx = _native.Context(device=0)
    n_in, dims, ln, fin = W.head_desc(h)
    hid = ctx.add_head(n_in, dims, ln, fin, W.pack_head_blob(h))
    banks = [ctx.add_verifier_bank(hid, 8, 0.5)]
    ctx2 = _native.Context(device=0)
    ctx2.add_head(n_in, dims, ln, fin, W.pack_head_blob(h))
    banks.append(ctx2.add_verifier_bank(0, 8, 0.5))
    rng = np.random.default_rng(2)
    D = n_in * 96
    mean = rng.normal(0, 1, (3, D)).astype(np.float32)
    w = rng.normal(0, 0.05, (3, D)).astype(np.float32)
    b = rng.normal(0, 1, 3).astype(np.float32)
    slots = [5, 0, 7]
    dev = torch.device("cuda", 0)
    ctx.load_verifiers(banks[0], slots, *(torch.from_numpy(a).to(dev) for a in (mean, w, b)))
    for i, s in enumerate(slots):
        ctx2.load_verifier(banks[1], s, mean[i], w[i], float(b[i]))
    x = rng.normal(0, 1, (257, n_in, 96)).astype(np.float32)
    for s in slots:
        np.testing.assert_array_equal(ctx.verifier_predict_host(banks[0], s, x), ctx2.verifier_predict_host(banks[1], s, x))
    with pytest.raises(_native.NativeError):
        ctx.load_verifiers(banks[0], [1, 1], *(torch.from_numpy(a[:2]).to(dev) for a in (mean, w, b)))
    with pytest.raises(_native.NativeError):
        ctx.load_verifiers(banks[0], [8], *(torch.from_numpy(a[:1]).to(dev) for a in (mean, w, b)))
    with pytest.raises(_native.ArgumentError):
        ctx.load_verifiers(banks[0], [1], *(torch.from_numpy(a[:1]).to(dev) for a in (mean, w, b[:0])))


def test_train_custom_verifier_end_to_end(torch_cuda, built_library, tmp_path):
    """train_custom_verifier (bulk capture + device fit) against get_reference_clip_features driven through a streaming
    Model's predict loop + train_verifier_model, from the same seed: same windows, same offsets, same verifier."""
    import openwakeword_b200 as ow
    from openwakeword_b200 import Model
    from openwakeword_b200.custom_verifier_model import get_reference_clip_features, load_verifier, train_verifier_model
    h = copy.deepcopy(head("alexa_v0.1"))                               # helpers.head shares its dicts between tests
    h["layers"][-1]["b"] = h["layers"][-1]["b"] + np.float32(4.0)       # scores mostly above 0.5: positives captured
    emb = emb_weights()
    rng = np.random.default_rng(8)
    pos = [np.clip(rng.normal(0, 3000, L), -32768, 32767).astype(np.int16) for L in (16000 * 2, 23000)]
    neg = [np.clip(rng.normal(0, 2000, L), -32768, 32767).astype(np.int16) for L in (16000 * 3, 9000)]
    kw = dict(wakeword_models=[{"name": "alexa", "head": h}], embedding_model_path=emb, cnn_mode=0)
    np.random.seed(77)
    out = tmp_path / "v.pkl"
    got = ow.train_custom_verifier(pos, neg, str(out), "alexa", **kw)
    after = np.random.randint(0, 1 << 30)
    np.random.seed(77)
    m = Model(**kw)
    m.preprocessor._feature_init = m.preprocessor._get_embeddings(np.random.randint(-1000, 1000, 16000 * 4).astype(np.int16))
    m.reset()
    P = np.vstack([get_reference_clip_features(c, m, "alexa", N=5) for c in pos])
    Nf = np.vstack([get_reference_clip_features(c, m, "alexa", threshold=0.0, N=1) for c in neg])
    assert np.random.randint(0, 1 << 30) == after
    ref = train_verifier_model(np.vstack([P, Nf]), np.array([1] * len(P) + [0] * len(Nf)))
    assert got.steps[1][1].n_samples_seen_ == len(P) + len(Nf) and len(P) > 0
    loaded = load_verifier(str(out))
    probe = np.vstack([P, Nf]).astype(np.float32)
    d = np.abs(loaded.predict_proba(probe)[:, 1] - ref.predict_proba(probe)[:, 1]).max()
    print(f"{len(P)} positive / {len(Nf)} negative windows; max |p_bulk - p_streaming| = {d:.2e}")
    assert d <= 1e-4
    with pytest.raises(KeyError):
        ow.train_custom_verifier(pos, neg, str(out), "nope", **kw)


def _golden_head(g):
    """alexa_v0.1 with the golden maker's output-layer shift and spread (tests/golden/make_enroll_golden.py)"""
    h = copy.deepcopy(head("alexa_v0.1"))
    last = h["layers"][-1]
    last["b"] = ((last["b"] + np.float32(g["bias_shift"])) * np.float32(g["spread"])).astype(np.float32)
    last["W"] = (last["W"] * np.float32(g["spread"])).astype(np.float32)
    return h


@pytest.mark.parametrize("mode,tol", [(3, 1e-3), (0, 1e-4)])
def test_enrollment_against_reference_golden(torch_cuda, built_library, tmp_path, mode, tol):
    """the unmodified reference train_custom_verifier (tests/golden/enroll_alexa.npz): same offsets, same windows per
    pass, and its pipeline's p on the probe windows within 1e-3 (default split) / 1e-4 (fp32 CNN)."""
    import os
    import openwakeword_b200 as ow
    from openwakeword_b200 import Model
    from openwakeword_b200.custom_verifier_model import enroll
    from helpers import GOLDEN
    g = np.load(os.path.join(GOLDEN, "enroll_alexa.npz"))
    assert float(g["nearest"]) >= 2e-3
    kw = dict(wakeword_models=[{"name": "alexa_v0.1", "head": _golden_head(g)}],
              embedding_model_path=emb_weights(int(g["emb_seed"])), cnn_mode=mode)
    pos, neg = [g["pos0"], g["pos1"]], [g["neg0"]]
    np.random.seed(int(g["seed"]))
    m = Model(**kw)
    fi = m.preprocessor._get_embeddings(np.random.randint(-1000, 1000, 16000 * 4).astype(np.int16))
    r = enroll(m, "alexa_v0.1", [(pos, neg)], feature_init=fi)[0]
    assert [o for p, _, o, _ in r["passes"] if p] == g["offsets"].tolist()
    assert r["counts"].tolist() == g["counts"].tolist()
    p = r["pipeline"].predict_proba(g["probe"])[:, 1]
    d = np.abs(p - g["probe_p"]).max()
    print(f"cnn_mode {mode}: {int(g['counts'].sum())} windows; max |p - reference| on the probe set = {d:.2e}")
    assert d <= 1e-3            # the reference's pipeline carries scikit-learn's lbfgs stopping error (up to ~6e-4)
    # the capture itself: scikit-learn's own fit on this package's captured windows (the same solver and stopping
    # point as the reference) gives the reference's p within `tol`
    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import FunctionTransformer, StandardScaler
    from openwakeword_b200.custom_verifier_model import flatten_features, get_reference_clip_features
    np.random.seed(int(g["seed"]))
    s = Model(**kw)
    s.preprocessor._feature_init = s.preprocessor._get_embeddings(np.random.randint(-1000, 1000, 16000 * 4).astype(np.int16))
    P = np.vstack([get_reference_clip_features(c, s, "alexa_v0.1", N=5) for c in pos])
    Q = np.vstack([get_reference_clip_features(c, s, "alexa_v0.1", threshold=0.0, N=1) for c in neg])
    assert len(P) + len(Q) == int(g["counts"].sum())
    sk = make_pipeline(FunctionTransformer(flatten_features), StandardScaler(),
                       LogisticRegression(random_state=0, max_iter=2000, C=0.001)).fit(
        np.vstack([P, Q]), np.array([1] * len(P) + [0] * len(Q)))
    d_sk = np.abs(sk.predict_proba(g["probe"])[:, 1] - g["probe_p"]).max()
    np.testing.assert_allclose(sk.steps[1][1].mean_, g["mean"], rtol=1e-3, atol=tol)
    print(f"cnn_mode {mode}: scikit-learn on the captured windows vs reference: max |p| difference = {d_sk:.2e}")
    assert d_sk <= tol
    np.random.seed(int(g["seed"]))
    pipe = ow.train_custom_verifier(pos, neg, str(tmp_path / "v.pkl"), "alexa_v0.1", **kw)
    assert np.array_equal(pipe.steps[2][1].coef_, r["pipeline"].steps[2][1].coef_)


def test_train_custom_verifiers_batched(torch_cuda, built_library, tmp_path):
    """Model.train_custom_verifiers on 48 of 64 streams: each equals a single-user train_custom_verifier run, bit for
    bit; streaming afterwards equals a Model built from the pickles; other streams keep what they had; a Model that
    already verifies captures the unverified scores; refusals."""
    import os
    import openwakeword_b200 as ow
    from openwakeword_b200 import Model
    from openwakeword_b200.custom_verifier_model import dumps_verifier, enrollment_passes
    from helpers import GOLDEN
    g = np.load(os.path.join(GOLDEN, "enroll_alexa.npz"))
    rng = np.random.default_rng(3)
    B, name = 64, "alexa_v0.1"
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    kw = dict(wakeword_models=[{"name": name, "head": _golden_head(g)}],
              embedding_model_path=emb_weights(int(g["emb_seed"])), feature_init=fi)
    src = np.concatenate([g["pos0"], g["pos1"]])
    users = {}
    for b in rng.permutation(B)[:48]:
        L = int(rng.integers(16000, min(32000, len(src))))
        a = int(rng.integers(0, len(src) - L + 1))
        Ln = min(16000, len(g["neg0"]))
        n0 = int(rng.integers(0, len(g["neg0"]) - Ln + 1))
        users[int(b)] = ([src[a:a + L]], [g["neg0"][n0:n0 + Ln]])
    m = Model(n_streams=B, **kw)
    keep = next(b for b in range(B) if b not in users)
    np.random.seed(5)
    m_prev = ow.train_custom_verifier([src[:30000]], [g["neg0"][:16000]], str(tmp_path / "prev.pkl"), name, **kw)
    m.set_custom_verifier(name, m_prev, [keep])
    np.random.seed(99)
    res = m.train_custom_verifiers(name, users)
    assert all(st == 0 for _, st in res.values())
    # each user alone, from the RNG state before its draws
    np.random.seed(99)
    for b, (pos, neg) in users.items():
        state = np.random.get_state()
        one = ow.train_custom_verifier(pos, neg, str(tmp_path / f"{b}.pkl"), name, **kw)
        for k in (1, 2):
            for att in ("mean_", "var_", "coef_", "intercept_"):
                if hasattr(one.steps[k][1], att):
                    assert np.array_equal(getattr(one.steps[k][1], att), getattr(res[b][0].steps[k][1], att)), (b, att)
        np.random.set_state(state)
        enrollment_passes([len(c) for c in pos], [len(c) for c in neg])
    # streaming equals a Model built from the pickles; the stream outside the enrollments keeps its verifier
    pickles = {b: str(tmp_path / f"{b}.pkl") for b in users}
    (tmp_path / "keep.pkl").write_bytes(dumps_verifier(m_prev))
    pickles[keep] = str(tmp_path / "keep.pkl")
    ref = Model(n_streams=B, custom_verifier_models={name: pickles}, custom_verifier_threshold=0.3, **kw)
    m.custom_verifier_threshold = 0.3
    assert set(m.custom_verifier_models[name]) == set(pickles)
    pcm = np.clip(rng.normal(0, 3000, (B, 40 * 1280)), -32768, 32767).astype(np.int16)
    pcm[:, :len(src[:40 * 1280])] += src[:40 * 1280][None] // 2
    for s in range(40):
        a = m.predict(pcm[:, s * 1280:(s + 1) * 1280])[name]
        b_ = ref.predict(pcm[:, s * 1280:(s + 1) * 1280])[name]
        assert np.array_equal(a, b_), s
    # a Model that already verifies `name` captures what a fresh one does
    sub = dict(list(users.items())[:4])
    np.random.seed(99)
    again = m.train_custom_verifiers(name, sub)
    for b in sub:
        assert np.array_equal(again[b][0].steps[2][1].coef_, res[b][0].steps[2][1].coef_)
    # refusals
    timer = Model(wakeword_models=[{"name": "timer_v0.1", "head": head("timer_v0.1")}],
                  embedding_model_path=emb_weights(), feature_init=fi)
    with pytest.raises(ValueError):
        timer.train_custom_verifiers("timer_v0.1", {0: sub[next(iter(sub))]})
    with pytest.raises(ValueError):
        m.train_custom_verifiers("nope", sub)
