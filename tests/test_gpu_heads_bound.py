"""-m gpu: whole wake-word heads and custom verifiers against float64 with the per-element round-off bound of
tests/test_heads_bound.py.

Stateless calls (oww_head_predict) on heads_tc.cu at 3 terms (hi/lo bound) and at 1 term (fp16 bound) and on heads.cu,
at 1, 130 and 700 rows, and oww_bank_head_predict on a head-bank slot: the head zoo (HEAD_SPECS, LayerNorm and
ReLU-only heads of widths 7 to 256 with 2 to 4 Linear layers, every final activation, ill-conditioned LayerNorm rows,
saturated sigmoid and softmax logits) and the rescaled heads (every hidden activation x 2^k, k in {-20, -14, 17}),
judged against the original head's bound.  A head inside the bound (test_heads_bound.outside_bound) must have at least
MIN_JUDGED of its live rows judged.

Streaming, on the windows the streams' rings hold: the grouped heads (the default), heads_tc on the ring
(group_heads=False), heads.cu (tc_heads=False), the fused kernel's heads and gates (split_from=20, one launch per step),
and head-bank and verifier-bank columns; calls of 1 and 3 chunks and a ragged call (counts {0, 1, 3}); gated pairs
(gate_kernel and the in-kernel gates) including a main at exactly the threshold.  Verifiers: oww_verifier_predict on
the edge parameters."""
import contextlib

import numpy as np
import pytest

from helpers import emb_weights
from test_heads_bound import (C_ROUNDOFF, MIN_JUDGED, RESCALE_HEADS, RESCALE_K, _f32, gate_judge, head_zoo,
                              judged_fraction, judged_rows, max_judge, options_ratio, outside_bound, rescaled_head,
                              small_head, verifier_edges, verifier_parts, verifier_pipeline, whole_head_parts, zero_main,
                              zoo_features)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _judge(h, feats, got, terms, name="", check=True):
    """(worst ratio, C needed, judged fraction of the live rows) of device outputs; a head inside the bound must have
    at least MIN_JUDGED of its live rows judged (test_heads_bound.outside_bound)."""
    y, A, B, rho = whole_head_parts(h, feats, terms)
    k = judged_rows(rho)
    frac = judged_fraction(feats, rho)
    assert not check or outside_bound(h, terms, name) or frac >= MIN_JUDGED, (name, frac)
    if not k.any():
        return 0.0, 0.0, frac
    r, cn = options_ratio(np.asarray(got)[k], [(y[k], A[k], B[k])])
    return r, cn, frac


def _cases(tc):
    """(label, head run on the device, head the bound is taken from)."""
    zoo = head_zoo(tc_only=tc)
    out = [(name, h, h) for name, h in zoo.items()]
    for name in RESCALE_HEADS:
        for k in RESCALE_K:
            out.append((name, rescaled_head(zoo[name], k), zoo[name], k))
    return [c if len(c) == 4 else c + (0,) for c in out]


@pytest.mark.parametrize("kind", ["tc3", "tc1", "cuda_core", "bank"])
def test_stateless_heads_within_the_bound(torch_cuda, built_library, kind):
    torch = torch_cuda
    from openwakeword_b200 import _native, weights as W
    terms = {"tc3": 3, "tc1": 1, "cuda_core": 0, "bank": 3}[kind]
    rng = np.random.default_rng(60 + terms)
    blob = W.pack_embedding_blob(emb_weights())
    worst, worst_c, bad = 0.0, 0.0, []
    for name, run, ref, k2 in _cases(terms > 0):          # one handle per head: at most 16 heads per handle
        label = name if k2 == 0 else f"{name} x2^{k2}"
        ctx = _native.Context(cnn_mode=3, tc_heads=terms > 0, tc_heads_terms=max(terms, 1))
        with contextlib.closing(ctx):
            ctx.load_mel()
            ctx.load_embedding(blob)
            n_in, dims, ln, fin = W.head_desc(run)
            if kind == "bank":
                hid = ctx.add_head_bank(n_in, dims, ln, fin, 2)
                ctx.load_bank_head(hid, 1, W.pack_head_blob(run))
            else:
                hid = ctx.add_head(n_in, dims, ln, fin, W.pack_head_blob(run))
            for n in ((130,) if kind == "bank" else (1, 130, 700)):
                f = zoo_features(rng, n, n_in)
                out = torch.full((n, dims[-1]), np.nan, dtype=torch.float32, device="cuda")
                if kind == "bank":
                    ctx.bank_head_predict(hid, 1, torch.from_numpy(f).cuda(), n, out)
                else:
                    ctx.head_predict(hid, torch.from_numpy(f).cuda(), n, out)
                torch.cuda.synchronize()
                r, cn, frac = _judge(ref, f, out.cpu().numpy(), terms, name, check=n > 1)
                print(f"{kind} n={n} {label}: worst ratio {r:.3g} at C = {C_ROUNDOFF:g} (C needed {cn:.3g}), "
                      f"live rows judged {frac:.2f}{' (outside the bound)' if outside_bound(ref, terms, name) else ''}")
                worst, worst_c = max(worst, r), max(worst_c, cn)
                if not r <= 1.0:
                    bad.append((label, n, r))
    print(f"{kind}: worst ratio {worst:.3g}, worst C needed {worst_c:.3g}")
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------- streaming
STREAM_CONFIGS = {                      # name -> (StreamEngine options, bound terms the scores may come from)
    "grouped": ({}, (3,)),                                   # heads_grp.cu, the default
    "per_head": (dict(group_heads=False), (3,)),             # heads_tc.cu on the ring
    "cuda_core": (dict(tc_heads=False), (0,)),               # heads.cu
    "in_kernel": (dict(split_from=20), (0, 3)),              # the fused kernel's heads (tensor-core heads while priming)
    "banks": ({}, (3,)),                                     # head-bank columns and a verifier bank's columns
}
CALLS = [("1-chunk", 1), ("1-chunk", 1), ("3-chunk", 3), ("ragged", (0, 1, 3)), ("1-chunk", 1)]
THR = 0.5


def _entries(config):
    """[(entry for StreamEngine, label, reference)]: an entry is a head or a gated pair; reference the head (or
    (main, verifier) pair) the bound is taken from."""
    zoo = head_zoo(tc_only=True)
    ex, gm, gv, pm, pv = zero_main(3, 42), small_head(41), small_head(43), small_head(44), small_head(45)
    out = [({"main": ex, "verifier": gv, "threshold": THR, "n_in": 3}, "gated, exact-0.5 main", (ex, gv)),
           ({"main": pm, "verifier": pv, "threshold": THR, "n_in": 3}, "gated", (pm, pv)),
           (zoo["alexa_v0.1"], "alexa_v0.1", zoo["alexa_v0.1"]),
           (rescaled_head(zoo["alexa_v0.1"], -20), "alexa_v0.1 x2^-20", zoo["alexa_v0.1"]),
           (rescaled_head(zoo["relu_w7_l3_in16_softmax"], 17), "relu_w7_l3_in16_softmax x2^17",
            zoo["relu_w7_l3_in16_softmax"])]
    if config != "in_kernel":                                # n_in 34: beyond the fused kernel's head limits
        out.append((rescaled_head(zoo["timer_v0.1"], 17), "timer_v0.1 x2^17", zoo["timer_v0.1"]))
    if config == "banks":
        out.append((gm, "verified parent", gm))
        out.append((gm, "parent twin", gm))                  # the device's parent score, bit for bit
    return out


def _windows(eng, B, n_in, backs, cache):
    for k in backs:
        if (n_in, k) not in cache:
            cache[(n_in, k)] = np.stack([eng.ctx.get_features(b, n_in, k) for b in range(B)])
    return [cache[(n_in, k)] for k in backs]


def _head_options(h, wins, terms_opts, name):
    """Options of the max over a call's windows of one head's outputs, and the rows judged in every window."""
    per_win, keep = [], None
    for f in wins:
        opts = []
        for t in terms_opts:
            y, A, B, rho = whole_head_parts(h, f, t)
            assert not outside_bound(h, t, name) and judged_fraction(f, rho) >= MIN_JUDGED, (name, t)
            k = judged_rows(rho)
            keep = k if keep is None else keep & k
            opts.append((y, A, B))
        per_win.append(opts)
    return max_judge(per_win), keep


def _gated_options(main, ver, wins, terms_opts, exact):
    per_win = []
    for f in wins:
        opts = []
        for t in terms_opts:
            m, v = whole_head_parts(main, f, t)[:3], whole_head_parts(ver, f, t)[:3]
            opts += gate_judge(m, v, THR, None, main_exact=exact)
        per_win.append(opts)
    return max_judge(per_win)


@pytest.mark.parametrize("config", list(STREAM_CONFIGS))
def test_streaming_heads_within_the_bound(torch_cuda, built_library, config):
    """130 streams, calls of 1 chunk, 3 chunks (each window gated, then the max) and a ragged call with counts {0, 1, 3}
    (held rows stay NaN), each judged on the windows the streams' rings hold after the call (oww_get_features).  Gated
    pairs include a main that scores exactly 0.5, whose column must keep 0.5.  in_kernel requires every 1-chunk call
    after the first to be one launch, so the heads and gates ran inside the fused kernel.  banks: head-bank columns
    (slots -1 / a x2^17 head / the original, per stream) and a verifier bank on a parent head, whose decision is taken
    from the device's own parent score (a twin head's column) with `>=` as verifier_kernel does."""
    from openwakeword_b200.engine import StreamEngine
    from test_gpu_cnn_configs import _signals
    opts_kw, terms_opts = STREAM_CONFIGS[config]
    entries = _entries(config)
    B = 130
    rng = np.random.default_rng(62)
    fi = rng.normal(0.3, 1.5, (41, 96)).astype(np.float32)
    total = sum(c if isinstance(c, int) else max(c) for _, c in CALLS)
    pcm = _signals(rng, B, total * 1280)
    eng = StreamEngine([e[0] for e in entries], B, embedding=emb_weights(), feature_init=fi, cnn_mode=3, max_chunks=3,
                       **opts_kw)
    zoo = head_zoo(tc_only=True)
    bank_slots = np.array([b % 3 - 1 for b in range(B)], np.int32)
    ver_slots = np.array([0 if b % 2 == 0 else -1 for b in range(B)], np.int32)
    worst, worst_c, bad, launches = 0.0, 0.0, [], []
    with contextlib.closing(eng.ctx):
        if config == "banks":
            shape = zoo["relu_w7_l3_in16_softmax"]
            bank, bcol, bn = eng.add_head_bank(shape, 2)
            eng.load_bank_head(bank, 0, rescaled_head(shape, 17))
            eng.load_bank_head(bank, 1, shape)
            eng.assign_bank_head(bank, bank_slots)
            vrng = np.random.default_rng(63)
            D = 3 * 96
            vmean = _f32(vrng.normal(0.3, 1.5, D)).astype(np.float64)
            vw, vb = vrng.normal(0, 1, D) / np.sqrt(D), 0.1
            vbank = eng.add_verifier_bank(len(entries) - 2, 1, THR)
            eng.load_verifier(vbank, 0, (_f32(vmean), _f32(vw), float(np.float32(vb))))
            eng.assign_verifier(vbank, ver_slots)
        pos = 0
        for ci, (kind, c) in enumerate(CALLS):
            n0 = eng.ctx.launch_count
            if kind == "ragged":
                counts = np.array([c[b % 3] for b in range(B)], np.int32)
                seg = np.ascontiguousarray(pcm[:, pos * 1280:(pos + 3) * 1280])
                got = eng.step_host_ragged(seg, counts).copy()
                pos += 3
            else:
                counts = np.full(B, c, np.int32)
                got = eng.step_host(np.ascontiguousarray(pcm[:, pos * 1280:(pos + c) * 1280]), c).copy()
                pos += c
            launches.append(eng.ctx.launch_count - n0)
            held = counts == 0
            assert np.isnan(got[held]).all()
            cache = {}
            for n_chunks in sorted(set(counts[~held].tolist())):
                rows = counts == n_chunks
                backs = list(range(n_chunks - 1, -1, -1))
                for (entry, label, ref), (col, n_out) in zip(entries, eng.columns):
                    if isinstance(ref, tuple):
                        main, ver = ref
                        wins = [w[rows] for w in _windows(eng, B, 3, backs, cache)]
                        opts = _gated_options(main, ver, wins, terms_opts, exact=label.startswith("gated, exact"))
                        r, cn = options_ratio(got[rows, col:col + 1], opts)
                        vopts, _ = _head_options(ver, wins, terms_opts, "")
                        r2, cn2 = options_ratio(got[rows, col + 1:col + 2], vopts)
                        if label.startswith("gated, exact") and not np.all(got[rows, col] == THR):
                            bad.append((config, ci, label, "the exact-0.5 main was replaced"))
                        r, cn = max(r, r2), max(cn, cn2)
                    elif config == "banks" and label == "verified parent" and n_chunks == 1:
                        wins = [w[rows] for w in _windows(eng, B, 3, backs, cache)]
                        vp, vA, vB = verifier_parts(wins[0], vmean, vw, vb, _f32(vmean), _f32(vw), np.float32(vb))
                        popts, _ = _head_options(ref, wins, terms_opts, label)
                        twin = eng.columns[len(entries) - 1][0]
                        fire = (got[rows, twin] >= THR) & (ver_slots[rows] >= 0)
                        py, pA, pB = popts[0]
                        opt = (np.where(fire, vp, py[:, 0]), np.where(fire, vA, pA[:, 0]), np.where(fire, vB, pB[:, 0]))
                        r, cn = options_ratio(got[rows, col], [opt])
                        print(f"{config} call {ci}: {int(fire.sum())} rows verified")
                    elif config == "banks" and label == "verified parent":
                        continue                                  # verifiers are judged on 1-chunk calls
                    else:
                        wins = [w[rows] for w in _windows(eng, B, ref["n_in"], backs, cache)]
                        opts, keep = _head_options(ref, wins, terms_opts, label.split(" ")[0])
                        r, cn = options_ratio(got[rows, col:col + n_out][keep], [tuple(a[keep] for a in o) for o in opts])
                    print(f"{config} call {ci} ({kind}, {n_chunks} chunks) {label}: worst ratio {r:.3g} (C needed {cn:.3g})")
                    worst, worst_c = max(worst, r), max(worst_c, cn)
                    if not r <= 1.0:
                        bad.append((config, ci, label, r))
                if config == "banks":
                    shape = zoo["relu_w7_l3_in16_softmax"]
                    on = rows & (bank_slots >= 0)
                    assert np.all(got[rows & (bank_slots < 0), bcol:bcol + bn] == 0.0)
                    wins = [w[on] for w in _windows(eng, B, 16, backs, cache)]
                    opts, keep = _head_options(shape, wins, terms_opts, "bank")
                    r, cn = options_ratio(got[on, bcol:bcol + bn][keep], [tuple(a[keep] for a in o) for o in opts])
                    print(f"{config} call {ci} ({kind}, {n_chunks} chunks) bank columns: worst ratio {r:.3g} (C needed {cn:.3g})")
                    worst, worst_c = max(worst, r), max(worst_c, cn)
                    if not r <= 1.0:
                        bad.append((config, ci, "bank", r))
    print(f"{config}: worst ratio {worst:.3g} at C = {C_ROUNDOFF:g}, worst C needed {worst_c:.3g}; launches per call {launches}")
    if config == "in_kernel":
        assert launches[1] == 1, launches
    assert not bad, bad


def test_verifier_predict_within_the_bound(torch_cuda, built_library):
    from openwakeword_b200 import _native, weights as W
    from helpers import head
    ctx = _native.Context(cnn_mode=3)
    worst, worst_c = 0.0, 0.0
    with contextlib.closing(ctx):
        ctx.load_mel()
        ctx.load_embedding(W.pack_embedding_blob(emb_weights()))
        hid = ctx.add_head(*W.head_desc(head("alexa_v0.1")), W.pack_head_blob(head("alexa_v0.1")))
        bank = ctx.add_verifier_bank(hid, 2, 0.5)
        for mean, w, b, x in (verifier_edges(), verifier_pipeline()):
            m32, w32, b32 = _f32(mean), _f32(w), np.float32(b)
            ctx.load_verifier(bank, 1, m32, w32, float(b32))
            got = ctx.verifier_predict_host(bank, 1, x)
            p, A, B = verifier_parts(x, mean, w, b, m32, w32, b32)
            r, cn = options_ratio(got, [(p, A, B)])
            print(f"verifier: worst ratio {r:.3g} at C = {C_ROUNDOFF:g} (C needed {cn:.3g})")
            worst, worst_c = max(worst, r), max(worst_c, cn)
    print(f"verifier_predict: worst ratio {worst:.3g}, worst C needed {worst_c:.3g}")
    assert worst <= 1.0
