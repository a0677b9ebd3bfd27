"""-m gpu: stream records (oww_export_streams / oww_import_streams).

* A move continues bit for bit: handles A and C run one schedule (1-, 2-, 3-chunk calls, ragged calls with held
  streams, a mid-run reset); after it a subset of A's streams - among them freshly reset streams and streams held in the
  last call - is imported into scattered slots of D, a handle with another stream count and max_chunks (other group
  size, late block size and ring sizes) and a history of its own, which gives those slots A's head-bank and verifier
  assignments.  From then on D's imported slots and C's originals get the same samples and give the same score rows,
  feature rows, mel rows and counts, at every split point of mode 3 and in modes 0 and 2.  D's other streams equal E,
  which ran D's schedule without the import.
* A self import changes nothing and a permuted import equals the permuted control; a handle grows by export,
  set_streams, import; exports are stream ordered (device steps and host submits); refusals; launch counts; two GPUs;
  and Model.export_streams / import_streams with patience and debounce."""
import os

import numpy as np
import pytest

from helpers import GOLDEN, emb_weights, head

pytestmark = pytest.mark.gpu

MC = 4                      # max_chunks of A and C
D_STREAMS, D_MC = 230, 9    # D: other G, late block and ring sizes (mel 256 / feature 256 rows instead of 128 / 128)
SRC = 151
VER = os.path.join(GOLDEN, "verifier_alexa.pkl")


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _mixes(rng, n, length):
    """+-1000 noise, full scale, gated bursts, silence, tone (the ragged-step test's inputs)."""
    out = np.empty((n, length), np.int16)
    t = np.arange(length)
    for i in range(n):
        k = (i + int(rng.integers(0, 5))) % 5
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


def _seven():
    from openwakeword_b200 import weights as W
    hs = []
    for i in range(5):
        hs.append(W.synthetic_gated_head(seed_main=10 + i, seed_verifier=40 + i, threshold=0.5) if i == 2
                  else W.synthetic_head(seed=10 + i))
    hs.append(W.synthetic_head(n_in=34, hidden=128, n_out=7, layernorm=False, final="relu_softmax", seed=20))
    return hs


def _bank_heads():
    from openwakeword_b200 import weights as W
    return [W.synthetic_head(seed=300 + i, n_in=16, hidden=64, n_out=1) for i in range(3)]


class Handle:
    """A StreamEngine with the seven bench networks, a verifier bank (slot 0 on even sources) and, outside mode 0, a
    head bank of three slots (slot source % 3)."""

    def __init__(self, B, mc, fi, **kw):
        from openwakeword_b200.engine import StreamEngine
        self.eng = StreamEngine(_seven(), B, embedding=emb_weights(), feature_init=fi, max_chunks=mc, **kw)
        self.vb = self.eng.add_verifier_bank(0, 1, 0.0)
        self.eng.load_verifier(self.vb, 0, VER)
        self.hb = None
        if kw.get("cnn_mode", 3) != 0:
            bh = _bank_heads()
            self.hb, _, _ = self.eng.add_head_bank(bh[0], 3)
            for k, h in enumerate(bh):
                self.eng.load_bank_head(self.hb, k, h)
        self.assign(np.arange(B), np.arange(B))

    def assign(self, ids, src):
        ids, src = np.asarray(ids, np.int32), np.asarray(src)
        self.eng.assign_verifier(self.vb, np.where(src % 2 == 0, 0, -1).astype(np.int32), stream_ids=ids)
        if self.hb is not None:
            self.eng.assign_bank_head(self.hb, (src % 3).astype(np.int32), stream_ids=ids)

    def step(self, torch, x, counts):
        return self.eng.step_ragged(torch.from_numpy(np.ascontiguousarray(x)).cuda(), np.asarray(counts, np.int32)).cpu().numpy()


def _counts(rng, B, kind, mc_call=3):
    if kind == "rag":
        c = rng.integers(0, mc_call + 1, B).astype(np.int32)
        c[rng.choice(B, max(3, B // 8), replace=False)] = 0        # held streams
        c[-1] = mc_call
        return c
    return np.full(B, kind, np.int32)


def _state(eng, b):
    c, b = eng.ctx, int(b)
    return (c.get_counts(b), c.get_mel(b, 76), c.get_features(b, 120), c.get_features(b, 100, 20),
            c.get_features(b, 16, 3))


def _same_state(e1, b1, e2, b2, what):
    s1, s2 = _state(e1, b1), _state(e2, b2)
    assert s1[0] == s2[0], (what, b1, b2, s1[0], s2[0])
    for k in range(1, len(s1)):
        assert np.array_equal(s1[k], s2[k]), (what, b1, b2, k, np.abs(s1[k] - s2[k]).max())


def _launches_per_step(torch, eng):
    n0 = eng.ctx.launch_count
    eng.step(torch.zeros((eng.n_streams, 1280), dtype=torch.int16, device="cuda"))
    return eng.ctx.launch_count - n0


MOVE_CONFIGS = {
    "mode3_split3": dict(cnn_mode=3, split_from=3),
    "mode3_split7": dict(cnn_mode=3, split_from=7),
    "mode3_split11": dict(cnn_mode=3, split_from=11),
    "mode3_split15": dict(cnn_mode=3, split_from=15),
    "mode3_split20": dict(cnn_mode=3, split_from=20),
    "mode0": dict(cnn_mode=0),
    "mode2": dict(cnn_mode=2),
}
PRE = [1, 2, "rag", "reset", 3, "rag", 1, "rag"]     # A and C; after the last call a subset is reset, then the move
POST = [1, "rag", 2, "rag", 3, "rag", 1, "rag", "rag", 2]


@pytest.mark.parametrize("config", list(MOVE_CONFIGS))
def test_move_continues_bit_for_bit(torch_cuda, built_library, config):
    torch = torch_cuda
    kw = MOVE_CONFIGS[config]
    rng = np.random.default_rng(list(MOVE_CONFIGS).index(config) + 11)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    A, C = Handle(SRC, MC, fi, **kw), Handle(SRC, MC, fi, **kw)
    D, E = Handle(D_STREAMS, D_MC, fi, **kw), Handle(D_STREAMS, D_MC, fi, **kw)
    if kw.get("split_from") == 20:
        # the heads run inside the fused kernel on both sides (its own summation order): the same choice, the same launches
        assert _launches_per_step(torch, C.eng) == _launches_per_step(torch, D.eng) == _launches_per_step(torch, E.eng)
        _launches_per_step(torch, A.eng)
    for kind in PRE:                                     # D and E: a history of their own
        if kind == "reset":
            ids = rng.choice(D_STREAMS, 20, replace=False)
            D.eng.reset_async(fi, stream_ids=ids); E.eng.reset_async(fi, stream_ids=ids)
            continue
        x, c = _mixes(rng, D_STREAMS, 4 * 1280), _counts(rng, D_STREAMS, kind)
        assert np.array_equal(D.step(torch, x, c), E.step(torch, x, c), equal_nan=True)
    held = None
    for kind in PRE:
        if kind == "reset":
            ids = rng.choice(SRC, 12, replace=False)
            A.eng.reset_async(fi, stream_ids=ids); C.eng.reset_async(fi, stream_ids=ids)
            continue
        x, c = _mixes(rng, SRC, 4 * 1280), _counts(rng, SRC, kind)
        assert np.array_equal(A.step(torch, x, c), C.step(torch, x, c), equal_nan=True)
        held = np.nonzero(c == 0)[0]
    fresh = rng.choice(np.setdiff1d(np.arange(SRC), held), 3, replace=False)
    A.eng.reset_async(fi, stream_ids=fresh); C.eng.reset_async(fi, stream_ids=fresh)
    src = np.unique(np.concatenate([fresh, held[:4], rng.choice(SRC, 30, replace=False), [0, SRC - 1]]))
    dst = np.sort(rng.choice(D_STREAMS, src.size, replace=False))[rng.permutation(src.size)]
    rec = A.eng.export_streams(src)
    D.eng.import_streams(dst, rec)
    D.assign(dst, src)
    assert D.eng.ctx.stream_state_rejected() == 0
    for s, d in zip(src, dst):
        _same_state(C.eng, s, D.eng, d, "after import")
    others = np.setdiff1d(np.arange(D_STREAMS), dst)
    for t, kind in enumerate(POST):
        xc, cc = _mixes(rng, SRC, 4 * 1280), _counts(rng, SRC, kind)
        xd, cd = _mixes(rng, D_STREAMS, 4 * 1280), _counts(rng, D_STREAMS, kind)
        xd[dst], cd[dst] = xc[src], cc[src]
        oc, od, oe = C.step(torch, xc, cc), D.step(torch, xd, cd), E.step(torch, xd, cd)
        assert np.array_equal(oc[src], od[dst], equal_nan=True), (t, kind, np.nanmax(np.abs(oc[src] - od[dst])))
        assert np.array_equal(od[others], oe[others], equal_nan=True), t
        if t == 0:
            for s, d in zip(fresh, dst[np.searchsorted(src, fresh)]):
                assert C.eng.ctx.get_counts(int(s))[0] == 76 + 5 and D.eng.ctx.get_counts(int(d))[0] == 76 + 5
    for s, d in zip(src, dst):
        _same_state(C.eng, int(s), D.eng, int(d), "end")
    for b in others[::7]:
        _same_state(D.eng, int(b), E.eng, int(b), "untouched")


def _pair(torch, B=64, mc=MC, **kw):
    rng = np.random.default_rng(B)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    A, C = Handle(B, mc, fi, **kw), Handle(B, mc, fi, **kw)
    for kind in [1, "rag", 2, "rag"]:
        x, c = _mixes(rng, B, 4 * 1280), _counts(rng, B, kind)
        A.step(torch, x, c); C.step(torch, x, c)
    return rng, fi, A, C


def test_self_and_permuted_import(torch_cuda, built_library):
    torch = torch_cuda
    rng, fi, A, C = _pair(torch)
    B = A.eng.n_streams
    A.eng.import_streams(np.arange(B), A.eng.export_streams(np.arange(B)))
    perm = rng.permutation(B)
    A.eng.import_streams(perm, A.eng.export_streams(np.arange(B)))       # A's stream perm[i] is C's stream i
    A.assign(perm, np.arange(B))
    for kind in [1, "rag", 3, "rag"]:
        x, c = _mixes(rng, B, 4 * 1280), _counts(rng, B, kind)
        xa, ca = np.empty_like(x), np.empty_like(c)
        xa[perm], ca[perm] = x, c
        oc, oa = C.step(torch, x, c), A.step(torch, xa, ca)
        assert np.array_equal(oa[perm], oc, equal_nan=True)
    for i in range(0, B, 5):
        _same_state(C.eng, i, A.eng, int(perm[i]), "permuted")


def test_grow(torch_cuda, built_library):
    torch = torch_cuda
    rng, fi, A, C = _pair(torch, B=SRC)
    rec = A.eng.export_streams(np.arange(SRC)).cpu()                     # through the host
    A.eng.set_streams(400, fi)
    A.eng.import_streams(np.arange(SRC), rec)
    A.assign(np.arange(SRC), np.arange(SRC))
    for kind in [1, "rag", 2, "rag", 3]:
        x, c = _mixes(rng, SRC, 4 * 1280), _counts(rng, SRC, kind)
        xa, ca = np.zeros((400, 4 * 1280), np.int16), np.zeros(400, np.int32)
        xa[:SRC], ca[:SRC] = x, c
        ca[SRC:] = c[0]
        oc, oa = C.step(torch, x, c), A.step(torch, xa, ca)
        assert np.array_equal(oa[:SRC], oc, equal_nan=True)
    for i in range(0, SRC, 9):
        _same_state(C.eng, i, A.eng, i, "grown")


def test_export_is_stream_ordered(torch_cuda, built_library):
    """step k, export, step k + 1 without a host synchronisation: the records are those of a synchronised export after
    step k - on a device stream, and between host submits on the handle's own stream."""
    torch = torch_cuda
    rng, fi, A, C = _pair(torch)
    B = A.eng.n_streams
    ids = np.arange(0, B, 3)
    x1, x2 = [torch.from_numpy(_mixes(rng, B, 1280)).cuda() for _ in range(2)]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        A.eng.step(x1)
        got = A.eng.export_streams(ids)
        A.eng.step(x2)
    C.eng.step(x1)
    torch.cuda.synchronize()
    want = C.eng.export_streams(ids)
    assert torch.equal(got, want)
    torch.cuda.synchronize()
    p1, p2 = _mixes(rng, B, 1280), _mixes(rng, B, 1280)
    t1 = A.eng.submit(p1)
    got = A.eng.export_streams(ids)
    t2 = A.eng.submit(p2)
    A.eng.collect(t1); A.eng.collect(t2)
    C.eng.step(x2)
    C.eng.step_host(p1)
    assert torch.equal(got, C.eng.export_streams(ids))


def test_refusals_and_rejected_records(torch_cuda, built_library):
    torch = torch_cuda
    from openwakeword_b200 import _native
    rng, fi, A, C = _pair(torch, B=20)
    lib, h = A.eng.ctx.lib, A.eng.ctx.h
    n_bytes, _ = A.eng.ctx.stream_state_info()
    buf = torch.zeros((21, n_bytes), dtype=torch.uint8, device="cuda")
    ids = lambda *v: np.array(v, np.int32)                              # noqa: E731
    for call in (lib.oww_export_streams, lib.oww_import_streams):
        for bad in (ids(20), ids(-1)):
            assert call(h, bad.ctypes.data, 1, buf.data_ptr(), None) == -1
        assert call(h, np.arange(21, dtype=np.int32).ctypes.data, 21, buf.data_ptr(), None) == -1
    assert lib.oww_import_streams(h, ids(3, 3).ctypes.data, 2, buf.data_ptr(), None) == -1
    assert lib.oww_export_streams(h, ids(3, 3).ctypes.data, 2, buf.data_ptr(), None) == 0
    fresh = _native.Context(max_chunks=MC)
    assert fresh.lib.oww_export_streams(fresh.h, ids(0).ctypes.data, 1, buf.data_ptr(), None) == -1
    assert fresh.lib.oww_stream_state_info(fresh.h, None, None) == -1
    # records of another split point and of other weights: rejected on the device, the target stays bit-identical
    from openwakeword_b200.engine import StreamEngine
    other_split = StreamEngine(_seven(), 20, embedding=emb_weights(), feature_init=fi, max_chunks=MC, split_from=7)
    other_w = StreamEngine(_seven(), 20, embedding=emb_weights(1), feature_init=fi, max_chunks=MC)
    before = A.eng.export_streams(ids(4, 5))
    for o in (other_split, other_w):
        rec = o.export_streams(ids(0, 1))
        with pytest.raises(ValueError):
            A.eng.import_streams(ids(4, 5), rec)
        if rec.shape[1] == n_bytes:
            A.eng.ctx.import_streams(ids(4, 5), rec)
        else:                                           # same size, wrong size field: still a device-side refusal
            r = torch.zeros((2, n_bytes), dtype=torch.uint8, device="cuda")
            r[:, :min(n_bytes, rec.shape[1])] = rec[:, :min(n_bytes, rec.shape[1])]
            A.eng.ctx.import_streams(ids(4, 5), r)
        assert A.eng.ctx.stream_state_rejected() == 2
        assert A.eng.ctx.stream_state_rejected() == 0
        assert torch.equal(A.eng.export_streams(ids(4, 5)), before)
    _same_state(A.eng, 4, C.eng, 4, "after rejected records")


def test_import_keeps_launch_count(torch_cuda, built_library):
    torch = torch_cuda
    rng, fi, A, C = _pair(torch)
    A.eng.import_streams(np.arange(10), C.eng.export_streams(np.arange(10, 20)))
    assert _launches_per_step(torch, A.eng) == _launches_per_step(torch, C.eng)


def test_move_between_gpus(torch_cuda, built_library):
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from openwakeword_b200.engine import StreamEngine
    rng = np.random.default_rng(2)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    mk = lambda dev: StreamEngine(_seven(), 32, embedding=emb_weights(), feature_init=fi, max_chunks=MC, device_index=dev)  # noqa: E731
    A, C, D = mk(0), mk(0), mk(1)
    for n in (1, 2, 1):
        x = torch.from_numpy(_mixes(rng, 32, n * 1280))
        A.step(x.cuda(0), n); C.step(x.cuda(0), n)
    with torch.cuda.device(1):
        D.import_streams(np.arange(32), A.export_streams(np.arange(32)))
    for n in (1, 3, 1):
        x = torch.from_numpy(_mixes(rng, 32, n * 1280))
        oc = C.step(x.cuda(0), n).cpu()
        with torch.cuda.device(1):
            od = D.step(x.cuda(1), n).cpu()
        assert torch.equal(oc, od)


@pytest.mark.parametrize("post", ["patience", "debounce"])
def test_model_move(torch_cuda, built_library, post):
    """Two Models of one configuration: streams moved from A to B (within the first-5 zeroing, holding remainders) return
    what A's unmoved streams return, through predict and predict_ragged."""
    import openwakeword_b200 as owb
    rng = np.random.default_rng(7)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    names = ["alexa_v0.1", "timer_v0.1", "hey_jarvis_v0.1"]
    thr = {n: 0.3 for n in names}
    kw = dict(patience={"alexa_v0.1": 2, "hey_jarvis_v0.1": 3}, threshold=thr) if post == "patience" else \
        dict(debounce_time=0.5, threshold=thr)
    mk = lambda B: owb.Model(wakeword_models=[{"name": n, "head": head(n)} for n in names],  # noqa: E731
                             embedding_model_path=emb_weights(), feature_init=fi, n_streams=B, max_chunks=2)
    a, b = mk(6), mk(9)
    pcm = lambda lens: [rng.integers(-3000, 3000, n).astype(np.int16) for n in lens]  # noqa: E731
    lengths = lambda B: [[0, 700, 1280, 2000, 3500][int(k)] for k in rng.integers(0, 5, B)]  # noqa: E731
    for _ in range(6):
        b.predict_ragged(pcm(lengths(9)), **kw)
    a.predict(np.stack(pcm([900] * 6)), **kw)
    a.predict_ragged(pcm([300, 1500, 0, 1279, 2600, 40]), **kw)
    src, dst = [0, 2, 3, 5], [8, 1, 4, 6]
    b.import_streams(dst, a.export_streams(src))
    for t in range(30):
        if t % 6 == 0:
            n = [700, 1280, 2000, 3500][t % 4]
            xa, xb = pcm([n] * 6), pcm([n] * 9)
        else:
            xa, xb = pcm(lengths(6)), pcm(lengths(9))
        for s, d in zip(src, dst):
            xb[d] = xa[s]
        ga = a.predict(np.stack(xa), **kw) if t % 6 == 0 else a.predict_ragged(xa, **kw)
        gb = b.predict(np.stack(xb), **kw) if t % 6 == 0 else b.predict_ragged(xb, **kw)
        for lab in ga:
            for s, d in zip(src, dst):
                assert ga[lab][s] == gb[lab][d], (t, lab, s, d)


def test_record_size(torch_cuda, built_library):
    """Mode 3 at split_from 11: 32 B header, 960 B PCM tail, 76 mel rows (9728 B), 120 feature rows (46080 B), the
    fused kernel's conv tails (930 units, 14880 B) and the late layers' (X_12, X_14: 240 units, X_16, X_18: 144, X_19:
    96; 13824 B).  Modes 0 and 2: no conv tails."""
    from openwakeword_b200 import _native
    c = _native.Context(max_chunks=MC)
    c.load_mel()
    from openwakeword_b200 import weights as W
    c.load_embedding(W.pack_embedding_blob(emb_weights()))
    c.set_streams(8)
    n, key = c.stream_state_info()
    assert n == 56800 + 14880 + 13824, n
    c0 = _native.Context(max_chunks=MC, cnn_mode=0)
    c0.load_mel()
    c0.load_embedding(W.pack_embedding_blob(emb_weights()))
    c0.set_streams(8)
    n0, key0 = c0.stream_state_info()
    assert n0 == 56800 and key0 != key
    print(f"record bytes: mode 3 split 11 {n}, mode 0 {n0}")
