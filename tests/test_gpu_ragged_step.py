"""-m gpu: ragged steps (oww_step_ragged), every stream at its own pace in one device call.

* Holds are invisible, bit for bit: streams that follow one base schedule of chunk counts, each with zero-count calls
  inserted at its own random places, end with the scores, feature rings, mel rings and counts of a lockstep engine that
  ran the base schedule - at every split point of cnn_mode 3, in the window modes, with the heads inside and outside the
  fused kernel, with the grouped-mirror heads and without, and with a verifier bank and a gate.  A mid-run reset of a
  stream subset lands at the same position of each stream's own schedule, and some of those streams are held right
  after it (a fresh stream stays fresh while held).
* Truly ragged counts against the oracle.
* The edges of the call: held rows untouched, all-zero and all-equal counts, launch counts, rejected arguments, and
  the host-buffer forms."""
import os

import numpy as np
import pytest

from helpers import GOLDEN, emb_weights, head

pytestmark = pytest.mark.gpu

BASE = [1, 1, 2, 1, 3, 1, 4, 1, 1, 2, 1, 1]      # the lockstep schedule (max_chunks = 4)
RESET_AT = 6                                     # the subset is reset after its 6th stepping call


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _mixes(rng, n, length):
    """+-1000 noise, full scale, gated bursts (onset inside a call), silence, tone."""
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


def _seven():
    """The seven head networks of the bench workload: five wake words (one a gated pair) and a 7-class timer."""
    from openwakeword_b200 import weights as W
    hs = []
    for i in range(5):
        hs.append(W.synthetic_gated_head(seed_main=10 + i, seed_verifier=40 + i, threshold=0.5) if i == 2
                  else W.synthetic_head(seed=10 + i))
    hs.append(W.synthetic_head(n_in=34, hidden=128, n_out=7, layernorm=False, final="relu_softmax", seed=20))
    return hs


def _schedules(rng, B, n_zero, held_after_reset):
    """Per stream: BASE with n_zero zero-count calls at random places (streams in held_after_reset get one right after
    their RESET_AT-th stepping call)."""
    K = len(BASE)
    sched = np.zeros((B, K + n_zero), np.int32)
    for b in range(B):
        gaps = rng.multinomial(n_zero, np.ones(K + 1) / (K + 1))
        if b in held_after_reset and gaps[RESET_AT] == 0:
            j = int(np.argmax(gaps))
            gaps[j] -= 1
            gaps[RESET_AT] += 1
        row = []
        for i in range(K):
            row += [0] * int(gaps[i]) + [BASE[i]]
        sched[b] = row + [0] * int(gaps[K])
    return sched


def _engine(hs, B, fi, verifier, **kw):
    from openwakeword_b200.engine import StreamEngine
    eng = StreamEngine(hs, B, embedding=emb_weights(), feature_init=fi, max_chunks=4, **kw)
    if verifier:
        bank = eng.add_verifier_bank(0, 1, 0.0)            # threshold 0: every assigned stream is verified at every step
        eng.load_verifier(bank, 0, os.path.join(GOLDEN, "verifier_alexa.pkl"))
        eng.assign_verifier(bank, np.where(np.arange(B) % 2 == 0, 0, -1).astype(np.int32))
    return eng


def _holds_invisible(torch, B, hs, seed, verifier=False, n_zero=5, **kw):
    rng = np.random.default_rng(seed)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(BASE)]) * 1280
    sig = _mixes(rng, 64, int(off[-1]))
    pick = rng.integers(0, 64, B)
    reset_ids = sorted(set(rng.choice(B, max(4, B // 20), replace=False).tolist()))
    sched = _schedules(rng, B, n_zero, set(reset_ids[::2]))
    K = len(BASE)

    lock = _engine(hs, B, fi, verifier, **kw)
    ref = []
    for j, n in enumerate(BASE):
        if j == RESET_AT:
            lock.reset_async(fi, stream_ids=reset_ids)
        ref.append(lock.step(torch.from_numpy(np.ascontiguousarray(sig[pick, off[j]:off[j + 1]])).cuda(), n).cpu().numpy())

    rag = _engine(hs, B, fi, verifier, **kw)
    got = np.zeros((B, K, rag.n_cols), np.float32)
    done = np.zeros(B, np.int64)
    was_reset = np.zeros(B, bool)
    held_fresh = 0
    for t in range(sched.shape[1]):
        c = sched[:, t]
        due = [b for b in reset_ids if done[b] == RESET_AT and not was_reset[b]]
        if due:
            rag.reset_async(fi, stream_ids=due)
            was_reset[due] = True
            held_fresh += int((c[due] == 0).sum())
        x = np.zeros((B, 4 * 1280), np.int16)
        for b in np.nonzero(c)[0]:
            x[b, :c[b] * 1280] = sig[pick[b], off[done[b]]:off[done[b]] + c[b] * 1280]
        o = rag.step_ragged(torch.from_numpy(x).cuda(), c).cpu().numpy()
        assert np.isnan(o[c == 0]).all(), "a held stream's score row was written"
        st = np.nonzero(c)[0]
        got[st, done[st]] = o[st]
        done[st] += 1
    assert (done == K).all() and was_reset[reset_ids].all() and held_fresh > 0
    for j in range(K):
        bad = np.nonzero(~(got[:, j] == ref[j]).all(axis=1))[0]
        assert bad.size == 0, f"step {j}: streams {bad[:8].tolist()} differ by {np.abs(got[bad, j] - ref[j][bad]).max():.3e}"
    sample = range(B) if B <= 300 else sorted(set(reset_ids[:16] + list(range(B - 7, B)) + rng.integers(0, B, 48).tolist()))
    for b in sample:
        b = int(b)
        assert rag.ctx.get_counts(b) == lock.ctx.get_counts(b), b
        assert np.array_equal(rag.ctx.get_mel(b, 76), lock.ctx.get_mel(b, 76)), b
        assert np.array_equal(rag.ctx.get_features(b, 120), lock.ctx.get_features(b, 120)), b
    rag.ctx.close()
    lock.ctx.close()


HOLD_CONFIGS = {
    "mode3_split3": dict(cnn_mode=3, split_from=3),
    "mode3_split7": dict(cnn_mode=3, split_from=7),
    "mode3_split11": dict(cnn_mode=3, split_from=11),
    "mode3_split15": dict(cnn_mode=3, split_from=15),
    "mode3_split20": dict(cnn_mode=3, split_from=20),
    "mode0": dict(cnn_mode=0),
    "mode2": dict(cnn_mode=2),
    "heads_in_fused_kernel": dict(cnn_mode=3, split_from=20, heads="one"),
    "heads_tc_no_mirror": dict(cnn_mode=3, group_heads=False),
    "verifier_bank_and_gate": dict(cnn_mode=3, heads="verifier"),
}


@pytest.mark.parametrize("config", list(HOLD_CONFIGS))
def test_holds_are_invisible_b300(torch_cuda, built_library, config):
    """B = 300: a ragged last group of the fused kernel and three 128-stream tiles of the feature mirror."""
    kw = dict(HOLD_CONFIGS[config])
    which = kw.pop("heads", "seven")
    hs = {"seven": _seven, "one": lambda: [head("alexa_v0.1")],
          "verifier": lambda: [head("alexa_v0.1"), head("hey_jarvis_v0.1"), head("timer_v0.1")]}[which]()
    _holds_invisible(torch_cuda, 300, hs, seed=list(HOLD_CONFIGS).index(config), verifier=which == "verifier", **kw)


def test_holds_are_invisible_b8192(torch_cuda, built_library):
    """The bench's size: 8192 streams x 7 head networks, default mode 3."""
    _holds_invisible(torch_cuda, 8192, _seven(), seed=8192, n_zero=4)


def test_ragged_counts_vs_oracle(torch_cuda, built_library):
    """Independent per-stream counts in 0..4 for 20 calls: scores of >= 64 sampled streams within 1e-3 of per-stream
    oracles fed the same samples, mel ring within 5e-3, feature ring within the fp16-operand budget."""
    from oracle import streaming, heads as oheads
    torch = torch_cuda
    rng = np.random.default_rng(7)
    B, calls = 160, 20
    hs = [head("alexa_v0.1"), head("timer_v0.1")]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    cnt = rng.integers(0, 5, (calls, B)).astype(np.int32)
    sig = _mixes(rng, B, int(cnt.sum(0).max()) * 1280)
    eng = _engine(hs, B, fi, False)
    sample = sorted(set(list(range(8)) + list(range(B - 8, B)) + rng.choice(B, 60, replace=False).tolist()))
    assert len(sample) >= 64
    oracles = {b: streaming.OracleAudioFeatures(emb_weights(), feature_init=fi) for b in sample}
    pos = np.zeros(B, np.int64)
    worst = 0.0
    for t in range(calls):
        c = cnt[t]
        x = np.zeros((B, 4 * 1280), np.int16)
        for b in range(B):
            x[b, :c[b] * 1280] = sig[b, pos[b]:pos[b] + c[b] * 1280]
        got = eng.step_ragged(torch.from_numpy(x).cuda(), c).cpu().numpy()
        for b in sample:
            if c[b] == 0:
                assert np.isnan(got[b]).all()
                continue
            assert oracles[b](x[b, :c[b] * 1280]) == c[b] * 1280
            ref = [np.max(np.stack([oheads.forward(h, oracles[b].get_features(h["n_in"], -h["n_in"] - i))[0]
                                    for i in range(c[b])]), axis=0) for h in hs]
            d = float(np.abs(np.concatenate(ref) - got[b]).max())
            assert d < 1e-3, (t, b, d)
            worst = max(worst, d)
        pos += c * 1280
    print(f"max |score - oracle| over {len(sample)} streams x {calls} ragged calls = {worst:.3e}")
    for b in sample:
        assert np.abs(eng.ctx.get_mel(b, 76) - oracles[b].melspectrogram_buffer[-76:]).max() < 5e-3
        assert np.abs(eng.ctx.get_features(b, 40) - oracles[b].feature_buffer[-40:]).max() < 8e-3


def test_ragged_edges(torch_cuda, built_library):
    from openwakeword_b200._native import NativeError
    torch = torch_cuda
    rng = np.random.default_rng(3)
    B = 40
    hs = [head("alexa_v0.1"), head("timer_v0.1")]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    sig = _mixes(rng, B, 40 * 1280)
    rag, twin = _engine(hs, B, fi, False), _engine(hs, B, fi, False)
    pos = 0

    def chunk(n, width=4):
        x = np.zeros((B, width * 1280), np.int16)
        x[:, :n * 1280] = sig[:, pos:pos + n * 1280]
        return torch.from_numpy(x).cuda()

    # rejected arguments: nothing enqueued, the next valid step unaffected
    n0 = rag.ctx.launch_count
    for bad in (np.full(B, 5), np.r_[np.ones(B - 1), -1]):
        with pytest.raises(NativeError):
            rag.step_ragged(chunk(1), bad.astype(np.int32))
    with pytest.raises(NativeError):                           # stride 1280 for a 2-chunk stream
        rag.step_ragged(chunk(1, width=1), np.r_[np.full(B - 1, 1), 2].astype(np.int32))
    with pytest.raises(ValueError):
        rag.step_ragged(chunk(1), np.ones(B + 1, np.int32))
    # all zero: nothing launched, nothing written
    out = rag.step_ragged(chunk(1), np.zeros(B, np.int32))
    assert rag.ctx.launch_count == n0 and torch.isnan(out).all()
    # all equal: the lockstep step, same launches, same bits
    for n in (1, 2, 1):
        a0, b0 = twin.ctx.launch_count, rag.ctx.launch_count
        ref = twin.step(chunk(n), n).cpu().numpy()
        got = rag.step_ragged(chunk(n), np.full(B, n, np.int32)).cpu().numpy()
        assert rag.ctx.launch_count - b0 == twin.ctx.launch_count - a0
        assert np.array_equal(got, ref)
        pos += n * 1280
    for b in (0, B - 1):
        assert np.array_equal(rag.ctx.get_features(b, 120), twin.ctx.get_features(b, 120))
        assert np.array_equal(rag.ctx.get_mel(b, 76), twin.ctx.get_mel(b, 76))
    # a 0/1 call: at most three launches beyond the lockstep one-chunk step
    c = (np.arange(B) % 3 != 0).astype(np.int32)
    a0 = twin.ctx.launch_count
    twin.step(chunk(1), 1)
    lock_launches = twin.ctx.launch_count - a0
    b0 = rag.ctx.launch_count
    rag.step_ragged(chunk(1), c)
    assert rag.ctx.launch_count - b0 <= lock_launches + 3, (rag.ctx.launch_count - b0, lock_launches)
    torch.cuda.synchronize()

    # host forms against the device form on twin handles: same bits, held rows keep the caller's values
    dev, host = _engine(hs, B, fi, False), _engine(hs, B, fi, False)
    p = np.zeros(B, np.int64)
    for t in range(6):
        c = rng.integers(0, 4, B).astype(np.int32)
        x = np.zeros((B, 3 * 1280), np.int16)
        for b in range(B):
            x[b, :c[b] * 1280] = sig[b, p[b]:p[b] + c[b] * 1280]
        p += c * 1280
        ref = dev.step_ragged(torch.from_numpy(x).cuda(), c).cpu().numpy()
        out = np.full((B, host.n_cols), 7.0, np.float32)
        if t % 2:
            host.step_host_ragged(x, c, out)
        else:
            host.collect(host.submit_ragged(x, c), out)
        assert (out[c == 0] == 7.0).all()
        assert np.array_equal(out[c > 0], ref[c > 0])
    # every stream held: no row of the caller's buffer is written, a collect without a buffer gives NaN rows
    zero = np.zeros(B, np.int32)
    out = np.full((B, host.n_cols), 7.0, np.float32)
    host.step_host_ragged(x, zero, out)
    assert (out == 7.0).all()
    host.collect(host.submit_ragged(x, zero), out)
    assert (out == 7.0).all()
    assert np.isnan(host.collect(host.submit_ragged(x, zero))).all()
    for e in (rag, twin, dev, host):
        e.ctx.close()


def _ragged_lengths(rng, B, n_calls, max_chunks):
    pick = [0, 1, 2, 3, 4]
    out = []
    for _ in range(n_calls):
        ks = rng.choice(pick, B)
        out.append([[0, int(rng.integers(1, 401)), 1280, int(rng.integers(1281, 4000)),
                     int(rng.integers(max_chunks * 1280 + 1, 6 * 1280))][k] for k in ks])
    return out


def test_model_predict_ragged_gpu_equals_cpu_fake(torch_cuda, built_library, monkeypatch):
    """Model.predict_ragged (per-stream accumulation, ragged device steps, host post-processing) on the GPU against the
    same Model on the CPU stand-in of the handle, fed the same arrays, interleaved with lockstep predict calls and a
    reset_streams: every label within 1e-3."""
    import openwakeword_b200 as owb
    from openwakeword_b200 import _native
    import fake_backend
    from helpers import NAMES, class_mapping
    rng = np.random.default_rng(21)
    B, mc = 7, 2
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    specs = [{"name": n, "head": head(n), "class_mapping": class_mapping([n]).get(n)} for n in NAMES]
    kw = dict(wakeword_models=specs, embedding_model_path=emb_weights(), feature_init=fi, n_streams=B, max_chunks=mc)
    monkeypatch.setattr(_native, "Context", fake_backend.FakeContext)
    cpu = owb.Model(**kw)
    monkeypatch.undo()
    gpu = owb.Model(**kw)
    pp = dict(patience={"alexa_v0.1": 2}, threshold={n: 0.3 for n in NAMES})
    worst = 0.0
    for t, lens in enumerate(_ragged_lengths(rng, B, 24, mc)):
        if t == 13:
            gpu.reset_streams([0, 5])
            cpu.reset_streams([0, 5])
        if t % 6 == 5:
            xs = [rng.integers(-3000, 3000, 1280).astype(np.int16) for _ in range(B)]
            a, b = gpu.predict(np.stack(xs), **pp), cpu.predict(np.stack(xs), **pp)
        else:
            xs = [rng.integers(-3000, 3000, n).astype(np.int16) for n in lens]
            a, b = gpu.predict_ragged(xs, **pp), cpu.predict_ragged(xs, **pp)
        assert list(a) == list(b)
        for lab in a:
            d = float(np.abs(a[lab] - b[lab]).max())
            assert d <= 1e-3, (t, lab, d)
            worst = max(worst, d)
    print(f"max |GPU - CPU stand-in| = {worst:.2e}")


def test_model_predict_ragged_custom_verifiers(torch_cuda, built_library):
    """custom_verifier_models through Model.predict_ragged against per-stream VerifiedOracleModels: stepping streams are
    verified on the device; streams with fewer than 1280 samples prepared re-verify their previous prediction and
    streams whose call exceeds max_chunks verify the max, on the host, as predict does."""
    from openwakeword_b200 import Model
    from oracle.verifier import VerifiedOracleModel
    from helpers import load_case, verifier_pipeline as _pipeline
    c = load_case("verifier_alexa_c1280")
    name = c["names"][0]
    rng = np.random.default_rng(17)
    B, mc, thr = 5, 2, 0.06
    kw = dict(wakeword_models=[{"name": name, "head": head(name)}], embedding_model_path=emb_weights(),
              feature_init=c["feature_init"], max_chunks=mc, n_streams=B)
    m = Model(custom_verifier_models={name: os.path.join(GOLDEN, "verifier_alexa.pkl")}, custom_verifier_threshold=thr, **kw)
    plain = Model(**kw)
    oms = [VerifiedOracleModel(emb_weights(), {name: head(name)}, verifiers={name: _pipeline("alexa")}, threshold=thr,
                               feature_init=c["feature_init"]) for _ in range(B)]
    got, raw, ref, short = [], [], [], []
    for lens in _ragged_lengths(rng, B, 24, mc):
        xs = [np.clip(rng.normal(0, 3000, n), -32768, 32767).astype(np.int16) for n in lens]
        got.append(m.predict_ragged(xs)[name])
        raw.append(plain.predict_ragged(xs)[name])
        ref.append([oms[b].predict(xs[b])[name] for b in range(B)])
        short.append([n < 1280 for n in lens])
    got, raw, ref, short = (np.array(a) for a in (got, raw, ref, short))
    clear = np.abs(raw - np.float32(thr)) > 2e-3
    print(f"max |device - oracle| = {np.abs(got - ref)[clear].max():.2e}; verified entries {(got != raw).sum()}")
    assert np.abs(got - ref)[clear].max() <= 1e-3
    assert (got != raw).any() and ((got != raw) & short).any()     # verification ran, also for held / short calls
