"""-m gpu: the bulk clip path (oww_predict_clips, oww_embed_clips) at its edges: more than one slab of clips (outer loop
of oww_predict_clips, inner loop of the mode-0 clip pass), more than one 128-clip tile of the grouped heads, every heads
kernel over sliding windows, clip geometries that are not whole chunks, feature-init row counts around and below the
heads' windows, and the steps > 65535 fallback of the grouped heads.

Every predict_clips case is checked twice:
* against the same padded clips streamed one 1280-sample chunk per call through a fresh engine of the same
  configuration with one stream per clip (ring, incremental CNN and mirror code the bulk path does not share): bit for
  bit.  Both sides run the same mel, CNN and heads arithmetic on the same feature rows; the grouped heads read the
  same fp16 hi/lo split of them from the per-slab mirror as from the ring mirror, heads_tc and heads.cu read them
  directly.  Measured on an H100: equal in every case below, in every mode and heads configuration;
* against the float64 oracle (oracle.streaming + oracle.heads) on the clips at every boundary the call crosses: the
  first clip, clips 127 / 128 / 129, the last clip of each slab and the first of the next, the last clip.
Each test prints its worst errors, and the slabs and tiles it ran."""
import numpy as np
import pytest

from helpers import emb_weights, head
from test_gpu_cnn_configs import _signals

pytestmark = pytest.mark.gpu

CHUNK = 1280
BAND = 2e-3           # a gate or verifier threshold this close to the oracle's score: either branch is accepted


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


# ---------------------------------------------------------------------------------------------------- slab arithmetic
# Host-side restatement of clip_slab (api.cu) and oww_tc_act_units_T (cnn_tc.cu), used only to pick clip counts and
# the boundary clips to sample.  Whether a boundary was crossed is proved by the launch count of the call.
_LAYERS = [(3, 24, 0, 0), (1, 24, 0, 0), (3, 24, 2, 2), (1, 48, 0, 0), (3, 48, 0, 0), (1, 48, 0, 0), (3, 48, 1, 2),
           (1, 72, 0, 0), (3, 72, 0, 0), (1, 72, 0, 0), (3, 72, 2, 2), (1, 96, 0, 0), (3, 96, 0, 0), (1, 96, 0, 0),
           (3, 96, 1, 2), (1, 96, 0, 0), (3, 96, 0, 0), (1, 96, 0, 0), (3, 96, 2, 2), (3, 96, 0, 0)]   # kh cout pool


def _tc_units(T, split_from=11):
    best, W = 0, 32
    for li, (kh, cout, pt, pf) in enumerate(_LAYERS):
        mult = 2 if li + 1 >= split_from else 1
        T -= kh - 1
        best = max(best, cout // 8 * mult * ((8 + T * (W + 1) + 384 + 7) & ~7))
        if pt:
            T, W = T // pt, W // pf
            best = max(best, cout // 8 * mult * ((8 + T * (W + 1) + 384 + 7) & ~7))
    return best + 64


def _outer_slab(T):
    """clips per slab of oww_predict_clips / oww_embed_clips: 1 GiB of fp16 planes per buffer"""
    return max(1, (1 << 26) // _tc_units(T))


def _mode0_slab(T):
    """clips per slab of the mode-0 clip pass of a fresh handle: layer-1 output of 512 windows (window_batch)"""
    per = (T - 2) * 32 * 24
    return max(per, 512 * 74 * 32 * 24) // per


def _mode0_launches_fit(l1, ln, outer, inner):
    """a 1-clip call launches l1 kernels: one fp32 pyramid of P launches and l1 - P others, all run once per outer slab.
    The n-clip call must have launched exactly outer * (l1 - P) + inner * P for one P in [1, l1]."""
    P = (ln - outer * l1) / (inner - outer) if inner > outer else None
    return P is not None and P == int(P) and 1 <= P <= l1


def _boundaries(n, *slabs):
    out = {0, n - 1}
    out.update(c for c in (127, 128, 129) if c < n)
    for s in slabs:
        for k in range(s, n, s):
            out.update((k - 1, k))
    return sorted(out)


# ---------------------------------------------------------------------------------------------------- runs
def _steps(L):
    return len(range(0, L - CHUNK, CHUNK))


def _padded(clips, pad):
    z = np.zeros((clips.shape[0], pad), np.int16)
    return np.concatenate([z, clips, z], 1)


def _verifier(rng, n_in):
    """a custom verifier bank on entry 0 of the head set, slot 2 of 3 (slot 0 holds a decoy)"""
    D = n_in * 96
    return dict(head=0, thr=0.07, slot=2, mean=rng.normal(0, 1, D).astype(np.float32),
                weight=rng.normal(0, 0.03, D).astype(np.float32), bias=np.float32(0.2))


def _engine(hs, n_streams, fi, cfg, ver):
    from openwakeword_b200.engine import StreamEngine
    eng = StreamEngine(hs, n_streams, embedding=emb_weights(), feature_init=fi, **cfg)
    bank = None
    if ver is not None:
        bank = eng.add_verifier_bank(ver["head"], 3, ver["thr"])
        eng.load_verifier(bank, 0, (ver["mean"] + 1, -ver["weight"], -3.0))
        eng.load_verifier(bank, ver["slot"], (ver["mean"], ver["weight"], float(ver["bias"])))
    return eng, bank


def _bulk(torch, hs, clips, pad, fi, cfg, ver=None, count=True):
    """oww_predict_clips on all clips -> (scores [n, steps, cols], launches of a 1-clip call, launches of the n-clip
    call; count=False: no 1-clip calls, None, None).  Unwritten scores stay NaN."""
    eng, bank = _engine(hs, 1, None, cfg, ver)
    if ver is not None:
        eng.ctx.set_verifier_clip_slot(bank, ver["slot"])
    n, length = clips.shape
    steps = _steps(length + 2 * pad)
    d = torch.from_numpy(np.ascontiguousarray(clips)).cuda()
    one = torch.full((1, steps, eng.n_cols), np.nan, dtype=torch.float32, device="cuda")
    out = torch.full((n, steps, eng.n_cols), np.nan, dtype=torch.float32, device="cuda")
    n0 = n1 = 0
    if count:
        eng.ctx.predict_clips(d, 1, length, pad, fi, one)      # first call: lazy set-up of the handle
        torch.cuda.synchronize()
        n0 = eng.ctx.launch_count
        eng.ctx.predict_clips(d, 1, length, pad, fi, one)
        torch.cuda.synchronize()
        n1 = eng.ctx.launch_count
    eng.ctx.predict_clips(d, n, length, pad, fi, out)
    torch.cuda.synchronize()
    ln = eng.ctx.launch_count - n1
    got = out.cpu().numpy()
    eng.ctx.close()
    return (got, n1 - n0, ln) if count else (got, None, None)


def _stream(hs, clips, pad, fi, cfg, ver=None):
    """the padded clips streamed one chunk per call through a fresh engine of one stream per clip"""
    n = clips.shape[0]
    eng, bank = _engine(hs, n, fi, cfg, ver)
    if ver is not None:
        eng.assign_verifier(bank, np.full(n, ver["slot"], np.int32))
    padded = _padded(clips, pad)
    got = np.stack([eng.step_host(np.ascontiguousarray(padded[:, s * CHUNK:(s + 1) * CHUNK]), 1).copy()
                    for s in range(_steps(padded.shape[1]))], 1)
    eng.ctx.close()
    return got


def _n_cols(hs):
    from openwakeword_b200 import weights as W
    return sum(2 if W.is_gated(h) else h["layers"][-1]["W"].shape[1] for h in hs)


def _oracle(hs, padded, fi, ver=None, hits=None):
    """float64 oracle of one padded clip -> (ref, alt) [steps, cols]: the engine's columns (a gated pair: the gated score,
    then its verifier network's raw score) with the verifier bank applied; alt is the other branch where the oracle's
    score is within BAND of a gate or bank threshold (else = ref).  NaN where the window reaches below the first
    feature row (the oracle cannot run it).  hits: a list that gains one entry per bank decision (1: replaced)."""
    from oracle import streaming, heads as oh
    from openwakeword_b200 import weights as W
    f64 = np.float64
    steps = _steps(padded.shape[0])
    ref = np.full((steps, _n_cols(hs)), np.nan)
    alt = ref.copy()
    o = streaming.OracleAudioFeatures(emb_weights(), feature_init=fi, dtype=f64)
    for s in range(steps):
        o(padded[s * CHUNK:(s + 1) * CHUNK])
        col = 0
        for k, h in enumerate(hs):
            gated = W.is_gated(h)
            width = 2 if gated else h["layers"][-1]["W"].shape[1]
            if o.feature_buffer.shape[0] < h["n_in"]:
                col += width
                continue
            x = o.get_features(h["n_in"]).astype(f64)
            if gated:
                m = oh.forward(h["main"], x, f64)[0, 0]
                v = oh.forward(h["verifier"], x, f64)[0, 0]
                thr = h["threshold"]
                ref[s, col] = v if m > thr else m
                alt[s, col] = (m if m > thr else v) if abs(m - thr) < BAND else ref[s, col]
                ref[s, col + 1] = alt[s, col + 1] = v
            else:
                r = oh.forward(h, x, f64)[0].astype(f64)
                ref[s, col:col + width] = alt[s, col:col + width] = r
                if ver is not None and ver["head"] == k:
                    z = float(ver["bias"]) + np.dot(x.ravel() - ver["mean"].astype(f64), ver["weight"].astype(f64))
                    p = 1.0 / (1.0 + np.exp(-z))
                    for j in range(width):
                        hit = r[j] >= np.float32(ver["thr"])
                        if hits is not None:
                            hits.append(int(hit))
                        ref[s, col + j] = p if hit else r[j]
                        if abs(r[j] - ver["thr"]) < BAND:
                            alt[s, col + j] = r[j] if hit else p
                        else:
                            alt[s, col + j] = ref[s, col + j]
            col += width
    return ref, alt


def _report(what, err, bound, clip_ids=None):
    """max of err [clips, steps, cols] (NaN: not compared), printed with the first (clip, step, col) beyond bound"""
    e = np.nan_to_num(err, nan=0.0)
    w = float(e.max()) if e.size else 0.0
    bad = np.argwhere(e > bound)
    msg = f"  {what}: max {w:.3e} (bound {bound:g})"
    if len(bad):
        c, s, j = (int(v) for v in bad[0])
        msg += f"; {len(bad)} beyond, first at clip {clip_ids[c] if clip_ids is not None else c} step {s} col {j}"
    print(msg)
    return w


def _vs_oracle(got, ref, alt, relative=False):
    e = np.minimum(np.abs(got - ref), np.abs(got - alt))
    if relative:
        e = e / np.maximum(1.0, np.abs(ref))
    return e


# ---------------------------------------------------------------------------------------------------- A. slabs, tiles
A_LEN, A_PAD = 32000, 16000                    # 2 s clips, 1 s of zeros on each side: 49 steps, T = 460 mel rows
_A = {}


def _case_a():
    if not _A:
        rng = np.random.default_rng(101)
        T = 76 + 8 * (_steps(A_LEN + 2 * A_PAD) - 1)
        outer = _outer_slab(T)
        n = outer + outer // 7                # two outer slabs, the last one ragged, in every mode
        hs = [head("alexa_v0.1"), head("hey_jarvis_v0.1"), head("timer_v0.1")]
        _A.update(hs=hs, fi=rng.normal(0, 1, (41, 96)).astype(np.float32), clips=_signals(rng, n, A_LEN),
                  ver=_verifier(rng, 16), T=T, outer=outer, oracle={})
    return _A


@pytest.mark.parametrize("mode", [0, 2, 3])
def test_bulk_slabs_and_tiles(torch_cuda, built_library, mode):
    """More clips than one slab of oww_predict_clips (2 s clips, 1 s padding: ~1440 per slab) with a ragged last slab;
    in mode 0 also many slabs of the fp32 clip pass (82 clips each).  A plain head, a gated pair and a verifier bank with
    a clip slot; more than 128 clips per slab, so the grouped heads run several tiles."""
    torch = torch_cuda
    c = _case_a()
    hs, fi, clips, ver = c["hs"], c["fi"], c["clips"], c["ver"]
    n = len(clips)
    cfg = dict(cnn_mode=mode)
    got, l1, ln = _bulk(torch, hs, clips, A_PAD, fi, cfg, ver)
    outer = -(-n // c["outer"])
    inner = -(-min(n, c["outer"]) // _mode0_slab(c["T"])) + -(-max(0, n - c["outer"]) // _mode0_slab(c["T"]))
    print(f"\nA mode {mode}: {n} clips x {got.shape[1]} steps; launches: 1 clip {l1}, {n} clips {ln}; "
          f"outer slabs {outer} of {c['outer']} clips" + (f", mode-0 clip-pass slabs {inner}" if mode == 0 else "")
          + (f", heads tiles per slab {-(-c['outer'] // 128)}" if mode else ""))
    assert ln > l1
    if mode:                                  # every launch of the call is per slab: the ratio is the slab count
        assert ln % l1 == 0 and ln // l1 == outer >= 2, (l1, ln)
    else:
        assert outer >= 2 and _mode0_launches_fit(l1, ln, outer, inner), (l1, ln)
    assert np.isfinite(got).all()
    stream = _stream(hs, clips, A_PAD, fi, cfg, ver)
    _report("max |bulk - streaming|", np.abs(got - stream), 0.0)
    s0 = _mode0_slab(c["T"])                  # first boundary of the mode-0 clip pass in each outer slab
    sample = sorted(set(_boundaries(n, c["outer"])) | {s0 - 1, s0, c["outer"] + s0 - 1, c["outer"] + s0})
    for k in sample:
        if k not in c["oracle"]:
            hits = []
            c["oracle"][k] = _oracle(hs, _padded(clips[k:k + 1], A_PAD)[0], fi, ver, hits)
            c["hits"] = c.get("hits", 0) + sum(hits)
    ref = np.stack([c["oracle"][k][0] for k in sample])
    alt = np.stack([c["oracle"][k][1] for k in sample])
    o_bound = 2e-5 if mode == 0 else 1e-3
    e_o = _report(f"max |bulk - oracle| on clips {sample}", _vs_oracle(got[sample], ref, alt), o_bound, sample)
    print(f"  the verifier bank replaced {c['hits']} of {ref[..., 0].size} sampled oracle scores")
    assert c["hits"] > 0
    assert np.array_equal(got, stream)
    assert e_o < o_bound


# ---------------------------------------------------------------------------------------------------- B. geometry
# (n_samples, pad): 1, 2 and 5 steps; L % 1280 in {0, 1, 159, 160, 161, 1279}; bodies shorter than one 512-sample frame;
# pads of 0, 1, 160 and 16000 samples
GEOMETRIES = [(1281, 0), (2560, 0), (2559, 1), (3520, 160), (6239, 160), (6560, 0), (6559, 1), (7679, 0), (3839, 0),
              (1, 16000), (300, 16000), (511, 16000), (300, 1280)]
_B = {}


@pytest.mark.parametrize("mode", [0, 3])
def test_bulk_clip_geometry(torch_cuda, built_library, mode):
    """Clips of 1 step (T = 76: a single window), 2 and 5 steps, lengths that are not whole chunks, bodies shorter than
    one frame and pads that are not whole mel hops."""
    torch = torch_cuda
    hs = [head("alexa_v0.1"), head("timer_v0.1")]
    rng = np.random.default_rng(7)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    worst_s = worst_o = 0.0
    o_bound = 2e-5 if mode == 0 else 1e-3
    print()
    for n_samples, pad in GEOMETRIES:
        L = n_samples + 2 * pad
        key = (n_samples, pad)
        if key not in _B:
            clips = _signals(np.random.default_rng(n_samples * 7 + pad), 5, n_samples)
            _B[key] = (clips, [_oracle(hs, p, fi) for p in _padded(clips, pad)])
        clips, orc = _B[key]
        got = _bulk(torch, hs, clips, pad, fi, dict(cnn_mode=mode), count=False)[0]
        stream = _stream(hs, clips, pad, fi, dict(cnn_mode=mode))
        assert got.shape[1] == _steps(L) >= 1 and np.isfinite(got).all(), key
        print(f"B mode {mode}: n_samples {n_samples} pad {pad} (L % 1280 = {L % CHUNK}, {got.shape[1]} steps; one slab, "
              f"one heads tile)")
        e_s = _report("max |bulk - streaming|", np.abs(got - stream), 0.0)
        ref = np.stack([r for r, _ in orc])
        alt = np.stack([a for _, a in orc])
        e_o = _report("max |bulk - oracle|", _vs_oracle(got, ref, alt), o_bound)
        assert np.array_equal(got, stream), key
        assert e_o < o_bound, key
        worst_s, worst_o = max(worst_s, e_s), max(worst_o, e_o)
    print(f"B mode {mode}: worst |bulk - streaming| {worst_s:.3e}, worst |bulk - oracle| {worst_o:.3e}")


# ---------------------------------------------------------------------------------------------------- C. feature init
C_STEPS, C_CLIPS = 40, 4
_C = {}


def _c_heads():
    from openwakeword_b200 import weights as W
    return [W.synthetic_head(n_in=3, hidden=32, n_blocks=1, n_out=2, layernorm=False, final="softmax", seed=21),
            head("alexa_v0.1"), head("timer_v0.1")]


C_CONFIGS = {"grouped": dict(), "heads_tc": dict(group_heads=False), "heads_cu": dict(tc_heads=False)}


@pytest.mark.parametrize("config", list(C_CONFIGS))
def test_bulk_feature_init_rows(torch_cuda, built_library, config):
    """feature_init of 0, 1, 15, 16, 17, 41 and 128 rows and None, with heads of n_in 3, 16 and 34: windows that reach
    below the first row read zeros there, as the streaming ring does.  The oracle checks each head from the step at
    which its window lies inside the rows.  200 rows give the same scores as their newest 128 and newest 34."""
    torch = torch_cuda
    hs = _c_heads()
    cfg = C_CONFIGS[config]
    rng = np.random.default_rng(55)
    clips = _signals(rng, C_CLIPS, CHUNK * (C_STEPS + 1))
    print()
    for n_rows in (0, 1, 15, 16, 17, 41, 128, None):
        fi = None if n_rows is None else np.random.default_rng(n_rows).normal(0, 1, (n_rows, 96)).astype(np.float32)
        got = _bulk(torch, hs, clips, 0, fi, cfg, count=False)[0]
        stream = _stream(hs, clips, 0, fi, cfg)
        if n_rows not in _C:
            _C[n_rows] = [_oracle(hs, p, fi) for p in clips[:2]]
        ref = np.stack([r for r, _ in _C[n_rows]])
        alt = np.stack([a for _, a in _C[n_rows]])
        print(f"C {config}: n_rows {n_rows} ({C_CLIPS} clips x {C_STEPS} steps: one slab, one heads tile)")
        assert np.isfinite(got).all()
        _report("max |bulk - streaming|", np.abs(got - stream), 0.0)
        e_o = _report(f"max |bulk - oracle| ({int(np.isnan(ref).sum())} of {ref.size} entries below the first row)",
                      _vs_oracle(got[:2], ref, alt), 1e-3)
        assert np.array_equal(got, stream), n_rows
        assert e_o < 1e-3, n_rows
    fi200 = np.random.default_rng(200).normal(0, 1, (200, 96)).astype(np.float32)
    g200, g128, g34 = (_bulk(torch, hs, clips, 0, f, cfg, count=False)[0] for f in (fi200, fi200[-128:], fi200[-34:]))
    print(f"C {config}: 200 rows vs newest 128 / 34: max diff {np.abs(g200 - g128).max():.3e} / "
          f"{np.abs(g200 - g34).max():.3e}")
    assert np.isfinite(g200).all()
    assert np.array_equal(g200, g128) and np.array_equal(g200, g34)


# ---------------------------------------------------------------------------------------------------- D. heads kernels
D_CLIPS, D_STEPS = 140, 8
_D = {}


def _d_heads():
    """widths 30 / 128 / 256 (256: heads.cu only), 1 to 4 Linear layers, sigmoid / softmax / relu_softmax / relu"""
    from openwakeword_b200 import weights as W
    rng = np.random.default_rng(5)
    hs = [W.synthetic_head(n_in=16, hidden=30, n_blocks=1, n_out=1, seed=3),
          W.synthetic_head(n_in=3, hidden=7, n_blocks=2, n_out=3, layernorm=False, final="softmax", seed=4),
          W.synthetic_head(n_in=34, hidden=128, n_blocks=0, n_out=5, final="relu_softmax", seed=6)]
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
    relu = W.synthetic_head(n_in=16, hidden=64, n_blocks=1, n_out=4, final="relu_softmax", seed=13)
    relu["final"] = "relu"
    hs.append(relu)
    return hs


# config -> bound against the oracle relative to max(1, |score|): 1e-3 as every score test, the fp16 budget of the
# plain-fp16 heads (test_tc_heads_vs_oracle_and_cuda_core_heads) with one term
D_CONFIGS = {"grouped": (dict(), 1e-3), "heads_tc": (dict(group_heads=False), 1e-3),
             "heads_cu": (dict(tc_heads=False), 1e-3), "one_term": (dict(tc_heads_terms=1), 2e-2)}


@pytest.mark.parametrize("config", list(D_CONFIGS))
def test_bulk_heads_kernels(torch_cuda, built_library, config):
    """The same 140 clips through the grouped heads (two tiles), heads_tc over sliding windows (group_heads=False),
    heads.cu (tc_heads=False) and the plain-fp16 grouped variant (tc_heads_terms=1)."""
    torch = torch_cuda
    cfg, o_bound = D_CONFIGS[config]
    if "hs" not in _D:
        rng = np.random.default_rng(77)
        _D.update(hs=_d_heads(), fi=rng.normal(0, 1, (41, 96)).astype(np.float32),
                  clips=_signals(rng, D_CLIPS, CHUNK * (D_STEPS + 1)), oracle={})
    hs, fi, clips = _D["hs"], _D["fi"], _D["clips"]
    got = _bulk(torch, hs, clips, 0, fi, cfg, count=False)[0]
    stream = _stream(hs, clips, 0, fi, cfg)
    sample = _boundaries(D_CLIPS)
    for k in sample:
        if k not in _D["oracle"]:
            _D["oracle"][k] = _oracle(hs, clips[k], fi)
    ref = np.stack([_D["oracle"][k][0] for k in sample])
    alt = np.stack([_D["oracle"][k][1] for k in sample])
    print(f"\nD {config}: {D_CLIPS} clips x {D_STEPS} steps ({-(-D_CLIPS // 128)} heads tiles)")
    assert np.isfinite(got).all()
    _report("max |bulk - streaming|", np.abs(got - stream), 0.0)
    e_o = _report(f"max |bulk - oracle| / max(1, |oracle|) on clips {sample}",
                  _vs_oracle(got[sample], ref, alt, relative=True), o_bound, sample)
    assert np.array_equal(got, stream)
    assert e_o < o_bound


# ---------------------------------------------------------------------------------------------------- E. > 65535 steps
def test_bulk_heads_beyond_65535_steps(torch_cuda, built_library):
    """One clip of 65537 steps: the grouped heads decline (grid.z would exceed 65535) and heads_tc runs every window,
    bit for bit as on a group_heads=False handle.  The first 8230 steps against the default handle on the clip cut to
    8230 steps (grouped heads; causality makes them comparable)."""
    torch = torch_cuda
    steps, cut = 65537, 8230
    rng = np.random.default_rng(65537)
    clip = np.clip(rng.normal(0, 3000, (1, CHUNK * (steps + 1))), -32768, 32767).astype(np.int16)
    clip[0, ::7919] = 20000
    hs = [head("alexa_v0.1"), head("timer_v0.1")]
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    got = _bulk(torch, hs, clip, 0, fi, dict(), count=False)[0]
    tc = _bulk(torch, hs, clip, 0, fi, dict(group_heads=False), count=False)[0]
    short = _bulk(torch, hs, np.ascontiguousarray(clip[:, :CHUNK * (cut + 1)]), 0, fi, dict(), count=False)[0]
    assert got.shape[1] == steps and short.shape[1] == cut
    assert np.isfinite(got).all() and np.isfinite(short).all()
    print(f"\nE: {steps} steps: max |default - group_heads=False| = {np.abs(got - tc).max():.3e}")
    e = _report(f"max |first {cut} steps - default handle on the clip cut to {cut} steps|",
                np.abs(got[:, :cut] - short), 2e-6)
    assert np.array_equal(got, tc)
    assert e <= 2e-6


# ---------------------------------------------------------------------------------------------------- F. embed_clips
F_BIG_T = 83                                   # W = 1 window, (T - 76) % 8 = 7


@pytest.mark.parametrize("mode", [0, 2, 3])
def test_embed_clips_edges(torch_cuda, built_library, mode):
    """oww_embed_clips at T = 76, 79, 83 and 84 mel rows (one window; one window and 7 unused rows; two windows), and at
    T = 83 with more clips than one slab (and, in mode 0, many slabs of the fp32 clip pass).  Against the oracle CNN on
    each clip's windows of its mel (the device mel, itself checked against the oracle mel), and each sampled clip of the
    large call against a call on that clip alone (bit for bit)."""
    torch = torch_cuda
    from openwakeword_b200 import _native, weights as W
    from oracle import embedding, mel as omel
    ctx = _native.Context(cnn_mode=mode)
    ctx.load_mel()
    ctx.load_embedding(W.pack_embedding_blob(emb_weights()))
    bound = 5e-4 if mode == 0 else 8e-3
    big = _outer_slab(76) + 37
    print()
    for T, n in ((76, 5), (79, 5), (84, 5), (F_BIG_T, big)):
        n_samples = 512 + 160 * (T - 1)
        Wn = (T - 76) // 8 + 1
        clips = _signals(np.random.default_rng(T), n, n_samples)
        d = torch.from_numpy(clips).cuda()
        emb = torch.full((n, Wn, 96), np.nan, dtype=torch.float32, device="cuda")
        one = torch.full((1, Wn, 96), np.nan, dtype=torch.float32, device="cuda")
        ctx.embed_clips(d, 1, n_samples, one)
        torch.cuda.synchronize()
        n0 = ctx.launch_count
        ctx.embed_clips(d, 1, n_samples, one)
        torch.cuda.synchronize()
        n1 = ctx.launch_count
        ctx.embed_clips(d, n, n_samples, emb)
        torch.cuda.synchronize()
        ln = ctx.launch_count - n1
        got = emb.cpu().numpy()
        assert np.isfinite(got).all()
        sample = _boundaries(n, _outer_slab(76 + 8 * (Wn - 1)), *([_mode0_slab(76 + 8 * (Wn - 1))] if mode == 0 else []))
        ds = torch.from_numpy(np.ascontiguousarray(clips[sample])).cuda()
        m = torch.empty((len(sample), T, 32), dtype=torch.float32, device="cuda")
        ctx.melspectrogram(ds, len(sample), n_samples, m)
        alone = []
        for k in sample:
            ctx.embed_clips(d[k:k + 1], 1, n_samples, one)
            alone.append(one.cpu().numpy()[0])
        mels = m.cpu().numpy()
        e_mel = max(float(np.abs(mels[i] - omel.melspectrogram(clips[k])).max()) for i, k in enumerate(sample))
        ref = np.stack([embedding.embed_windows(emb_weights(), np.stack([mels[i, 8 * w:8 * w + 76] for w in range(Wn)]),
                                                np.float64) for i in range(len(sample))])
        slabs = -(-n // _outer_slab(76 + 8 * (Wn - 1)))
        inner = sum(-(-min(_outer_slab(76 + 8 * (Wn - 1)), n - c0) // _mode0_slab(76 + 8 * (Wn - 1)))
                    for c0 in range(0, n, _outer_slab(76 + 8 * (Wn - 1))))
        print(f"F mode {mode}: T {T} ({Wn} windows), {n} clips; launches: 1 clip {n1 - n0}, {n} clips {ln}; slabs {slabs}"
              + (f", mode-0 clip-pass slabs {inner}" if mode == 0 else ""))
        e = _report(f"max |embedding - oracle| on clips {sample}", np.abs(got[sample] - ref), bound, sample)
        print(f"  max |device mel - oracle mel| {e_mel:.3e}")
        assert e < bound and e_mel < 5e-3
        assert np.array_equal(got[sample], np.stack(alone))
        if n == big:
            assert slabs >= 2 and ln > n1 - n0
            if mode:
                assert ln % (n1 - n0) == 0 and ln // (n1 - n0) == slabs
            else:
                assert _mode0_launches_fit(n1 - n0, ln, slabs, inner)
    ctx.close()
