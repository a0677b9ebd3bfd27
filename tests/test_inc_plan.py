"""not-gpu: replay the fused incremental-CNN kernel's geometry plan (csrc/cnn_tc_inc.cu) in NumPy.

The plan (buffer pitches, tap offsets, tail regions, pool geometry, smem offsets) is computed on
the host by the library and exported through ``oww_debug_inc_plan`` (cut plans: ``oww_debug_inc_cut_plan``); this test executes the same
data movement the kernel does - position order (t, stream, f), taps as unit shifts, tails loaded
into rows 0..1, new tails written back - with exact float64 arithmetic, and checks that a stream
of incremental steps reproduces the oracle's full 76-row-window embeddings (SURVEY.md F10).
Buffers start as NaN so any read of a unit the kernel would not have written shows up."""
import ctypes as C

import numpy as np
import pytest

from openwakeword_b200 import _native
from oracle import embedding, mel
from helpers import emb_weights

NAMES = ("kh3 final W Wp rows_in T_out M cg_in cgp np cg_out in_buf out_buf in_base tmp_base nx_base in_pitch tap0 tap1 tap2 pool_t pool_f "
         "tmp_pitch nx_buf nx_pitch nx_W nx_Wp nx_rows_new nx_t_off nx_tail_off w_off w_bytes w_smem").split()
LEAK, FLOOR = float(embedding.LEAK), float(embedding.FLOOR)


OWW_EUNSUPPORTED = -4


def get_plan(G, n_streams, built_library, n_layers=0):
    """n_layers 0 = the full 20-layer plan; otherwise the cut plan of split_from = n_layers. None if the builder
    rejects the plan as not fitting (OWW_EUNSUPPORTED)."""
    buf = (C.c_int32 * 4096)()
    if n_layers:
        n = built_library.oww_debug_inc_cut_plan(None, G, n_streams, n_layers, buf, 4096)
    else:
        n = built_library.oww_debug_inc_plan(None, G, n_streams, buf, 4096)
    if n == OWW_EUNSUPPORTED:
        return None
    assert n > 0
    a = np.array(buf[:n])
    hdr = dict(zip("G n_groups tail_units x_units y_units w_total_bytes smem_bytes pad".split(), a[:8]))
    layers = [dict(zip(NAMES, map(int, row))) for row in a[8:8 + 20 * len(NAMES)].reshape(20, len(NAMES))]
    assert int(a[8 + 20 * len(NAMES)]) == (n_layers or 20)       # n_layers: the conv layers inside the kernel
    return hdr, layers


def check_plan_structure(hdr, layers, NL):
    """Structural invariants of a plan with NL layers inside the kernel (the last one pooled and, for NL < 20, cut:
    its unpooled hi/lo output stays in the temp and leaves the kernel).  Offsets are 16-byte units above the 2048-byte
    arena base; weight slots are byte offsets."""
    top = 227 * 1024
    assert hdr["smem_bytes"] <= top
    assert all(L["w_smem"] == 0 for L in layers[NL:])            # no weight slot for a layer outside the kernel
    wsz = [((L["w_bytes"] + 127) & ~127) if 1 <= l < NL else 0 for l, L in enumerate(layers)]
    act_end = [0] * NL
    for l in range(NL):
        L = layers[l]
        cut = l == NL - 1 and NL < 20
        if cut:
            assert L["pool_t"], "a cut plan ends behind a pooled layer"
        # tensors alive while the phase's MMAs run: its input, and its output (the unpooled temp of a pooled layer)
        spans = []
        if l > 0:
            spans.append((L["in_base"], L["in_base"] + layers[l - 1]["nx_pitch"] * layers[l - 1]["cg_out"]))
        if L["pool_t"]:
            spans.append((L["tmp_base"], L["tmp_base"] + L["tmp_pitch"] * L["cg_out"] * (2 if cut else 1)))
        if not L["final"] and not L["pool_t"] and not cut:
            spans.append((L["nx_base"], L["nx_base"] + L["nx_pitch"] * L["cg_out"]))
        spans.sort()
        for (a0, a1), (b0, b1) in zip(spans, spans[1:]):
            assert a1 <= b0, (NL, l, spans)
        if L["pool_t"] and not cut:
            # the pool pass reads the temp while it writes the pooled tensor (over the dead input)
            t0, t1 = L["tmp_base"], L["tmp_base"] + L["tmp_pitch"] * L["cg_out"]
            n0, n1 = L["nx_base"], L["nx_base"] + L["nx_pitch"] * L["cg_out"]
            assert t1 <= n0 or n1 <= t0, (NL, l, (t0, t1), (n0, n1))
            spans.append((n0, n1))
        act_end[l] = 2048 + 16 * max((e for _, e in spans), default=0)
        if l >= 1:
            # weight slot of this layer and the prefetch of the next one: inside the arena, apart, above the activations
            assert 0 < L["w_smem"] and L["w_smem"] + wsz[l] <= top, (NL, l)
            if l + 1 < NL:
                nxt = layers[l + 1]
                assert nxt["w_smem"] + wsz[l + 1] <= L["w_smem"] or L["w_smem"] + wsz[l] <= nxt["w_smem"], (NL, l)
            wl = min(L["w_smem"], layers[l + 1]["w_smem"] if l + 1 < NL else 1 << 30)
            assert act_end[l] <= wl, (NL, l, spans, wl)
            assert act_end[l - 1] <= L["w_smem"], (NL, l)        # slot l is filled during phase l - 1
    return act_end


@pytest.mark.parametrize("n_layers", [3, 7, 11, 15, 20])
@pytest.mark.parametrize("G", list(range(1, 8)))
def test_cut_plans_fit_shared_memory(built_library, n_layers, G):
    """Every cut point mode 3 accepts (split_from 3 / 7 / 11 / 15, and 20 = no cut) and every group size 1..7: the
    plan the library would build keeps its live tensors apart and clear of the weight slots.  Plans the builder
    rejects as not fitting are the ones oww_inc_alloc_streams skips."""
    got = get_plan(G, 151, built_library, n_layers)
    if got is None:
        pytest.skip(f"the builder rejects G={G} at n_layers={n_layers}")
    hdr, layers = got
    assert hdr["G"] == G and hdr["n_groups"] == (151 + G - 1) // G
    check_plan_structure(hdr, layers, n_layers)


def test_cut_plan_has_a_group_size(built_library):
    """Each cut point has at least one feasible group size (else set_streams fails in mode 3)."""
    for n_layers in (3, 7, 11, 15, 20):
        assert any(get_plan(G, 151, built_library, n_layers) is not None for G in range(1, 8)), n_layers


def act(x):
    return np.maximum(np.maximum(LEAK * x, x), FLOOR)


class Emu:
    def __init__(self, hdr, layers, weights):
        self.h, self.L, self.w = hdr, layers, weights
        self.G = int(hdr["G"])
        self.arena = np.full(((227 * 1024 - 2048) // 16, 8), np.nan)      # the activation arena; tensors at plan offsets
        self.tails = np.zeros((int(hdr["tail_units"]), 8))
        self.sb = [embedding.fold_bn(*[np.asarray(p, np.float64) for p in weights["bn"][i]]) for i in range(19)]

    def prime(self, per_stream_layers):
        """tails <- last two rows of the tensors feeding (3,1) convs (what tc_capture_kernel copies)."""
        G = self.G
        for li, L in enumerate(self.L):
            if L["nx_tail_off"] < 0:
                continue
            Wp = L["nx_Wp"]
            for g in range(G):
                x = per_stream_layers[g][li][0]            # [T, W, C] output of layer li (after pool)
                T, W, Cc = x.shape
                for pl in range(L["cg_out"]):
                    for r in range(2):
                        for f in range(Wp):
                            v = x[T - 2 + r, f, pl * 8:pl * 8 + 8] if f < W else np.zeros(8)
                            self.tails[L["nx_tail_off"] + pl * 2 * G * Wp + (r * G + g) * Wp + f] = v

    def step(self, mel10):
        """mel10: [G, 10, 32] last ten mel rows of each stream -> embeddings [G, 96]; tails advance."""
        G = self.G
        tin, tout = self.tails, self.tails.copy()
        emb = np.zeros((G, 96))
        for l, L in enumerate(self.L):
            nx = self.arena[L["nx_base"]:]

            def fill():
                if L["nx_tail_off"] >= 0:
                    per = 2 * G * L["nx_Wp"]
                    for i in range(L["cg_out"] * per):
                        pl, u = divmod(i, per)
                        v = tin[L["nx_tail_off"] + i]
                        nx[pl * L["nx_pitch"] + 1 + u] = v
                        if L["nx_rows_new"] == 1 and u >= G * L["nx_Wp"]:
                            tout[L["nx_tail_off"] + pl * per + (u - G * L["nx_Wp"])] = v
                if not L["final"]:
                    for pl in range(L["cg_out"]):
                        nx[pl * L["nx_pitch"]] = 0.0
            if not L["pool_t"]:
                fill()
            else:
                for pl in range(L["cg_out"]):
                    self.arena[L["tmp_base"] + pl * L["tmp_pitch"]] = 0.0
            if l == 0:
                w0 = self.w["conv"][0].astype(np.float64)[:, :, 0, :]           # [3,3,24]
                s, b = self.sb[0]
                for p in range(8 * G * 33):
                    f = p % 33; tg = p // 33; g = tg % G; t = tg // G
                    if f == 32:
                        for pl in range(3):
                            nx[pl * L["nx_pitch"] + 1 + p] = 0.0
                        continue
                    x = np.zeros((3, 3))
                    for dt in range(3):
                        for df in range(3):
                            ff = f + df - 1
                            if 0 <= ff < 32:
                                x[dt, df] = mel10[g, t + dt, ff]
                    y = act(np.maximum(np.einsum("ab,abc->c", x, w0), 0) * s + b)
                    for pl in range(3):
                        nx[pl * L["nx_pitch"] + 1 + p] = y[pl * 8:pl * 8 + 8]
                continue
            src = self.arena[L["in_base"]:]
            Wt = self.w["conv"][l].astype(np.float64).reshape(3, L["cg_in"] * 8, -1)   # [tap, cin, cout]
            M = L["M"]
            taps = (L["tap0"], L["tap1"], L["tap2"])
            accum = np.zeros((M, Wt.shape[2]))
            for j in range(3):
                for pl in range(L["cg_in"]):
                    A = src[pl * L["in_pitch"] + 1 + taps[j] + np.arange(M)]            # [M, 8]
                    accum += A @ Wt[j, pl * 8:pl * 8 + 8]
            if L["final"]:
                for m in range(M):
                    if m % L["Wp"] == 0:
                        emb[(m // L["Wp"]) % G] = accum[m]
                continue
            s, b = self.sb[l]
            y = act(accum * s + b)
            dst = self.arena[L["tmp_base"]:] if L["pool_t"] else nx
            dpitch = L["tmp_pitch"] if L["pool_t"] else L["nx_pitch"]
            t_off_units = 0 if L["pool_t"] else L["nx_t_off"] * G * L["Wp"]
            tail_start = (L["T_out"] - 2) * G * L["Wp"]
            for m in range(M):
                pad = (m % L["Wp"]) == L["W"]
                for pl in range(L["cg_out"]):
                    v = np.zeros(8) if pad else y[m, pl * 8:pl * 8 + 8]
                    dst[pl * dpitch + 1 + t_off_units + m] = v
                    if not L["pool_t"] and L["nx_tail_off"] >= 0 and m >= tail_start:
                        tout[L["nx_tail_off"] + pl * 2 * G * L["Wp"] + (m - tail_start)] = v
            if L["pool_t"]:
                fill()
                tmp = self.arena[L["tmp_base"]:]
                T2 = L["T_out"] // L["pool_t"]
                per = T2 * G * L["nx_Wp"]
                for i in range(L["cg_out"] * per):
                    pl, p = divmod(i, per)
                    f = p % L["nx_Wp"]; tg = p // L["nx_Wp"]; g = tg % G; t = tg // G
                    res = np.zeros(8)
                    if f < L["nx_W"]:
                        res = np.full(8, -np.inf)
                        for da in range(L["pool_t"]):
                            for db in range(L["pool_f"]):
                                res = np.maximum(res, tmp[pl * L["tmp_pitch"] + 1 + ((t * L["pool_t"] + da) * G + g) * L["Wp"] + f * L["pool_f"] + db])
                    nx[pl * L["nx_pitch"] + 1 + L["nx_t_off"] * G * L["nx_Wp"] + p] = res
                    if L["nx_tail_off"] >= 0:
                        keep = 2 if T2 >= 2 else 1
                        if t >= T2 - keep:
                            tout[L["nx_tail_off"] + pl * 2 * G * L["nx_Wp"] + ((2 - keep + t - (T2 - keep)) * G + g) * L["nx_Wp"] + f] = res
        self.tails = tout
        return emb


@pytest.mark.parametrize("G", [7, 4, 1])
def test_fused_plan_reproduces_full_window_embeddings(built_library, G):
    hdr, layers = get_plan(G, G, built_library)
    # live tensors of a phase never overlap each other or the weight slots in use
    check_plan_structure(hdr, layers, 20)
    w = emb_weights()
    rng = np.random.default_rng(3)
    n_steps = 3
    mels = []
    for g in range(G):
        x = np.clip(rng.normal(0, [300, 3000, 9000, 1000][g % 4], 512 + 160 * (76 + 8 * n_steps)), -32768, 32767).astype(np.int16)
        mels.append(mel.melspectrogram(x)[:76 + 8 * n_steps].astype(np.float64))
    mels = np.stack(mels)                                   # [G, 76+8n, 32]
    emu = Emu(hdr, layers, w)
    per_stream = [embedding.forward(w, mels[g:g + 1, :76], np.float64, return_all=True)[1] for g in range(G)]
    emu.prime(per_stream)
    for s in range(1, n_steps + 1):
        got = emu.step(mels[:, 8 * s + 66:8 * s + 76])
        ref = embedding.forward(w, mels[:, 8 * s:8 * s + 76], np.float64)[:, 0]
        assert np.isfinite(got).all()
        assert np.abs(got - ref).max() < 1e-4, (s, np.abs(got - ref).max())   # float32 cast of the oracle's output
