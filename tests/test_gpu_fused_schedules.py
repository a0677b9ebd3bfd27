"""-m gpu: the fused step kernel (tc_inc_kernel) and the block-major late chain under ragged schedules, at every split
point and every group size G = 1..7.

Each case forces G as test_gpu_fused_items does (the plan is read back) and runs about 30 oww_step_host_ragged calls
in which every stream steps 1, 2 or 3 chunks or is held, with partial resets between calls.  Two kinds of call mix:
fused calls (every stream that steps takes one chunk: the fused launch with the held streams as dead slots) and general
calls (counts 0..3: one CNN launch per chunk, with carry_kernel moving the held streams' tails after each).  The
schedule holds streams for runs of 1 to 4 calls, so that held state is carried across every residue of the late
tensors' 2- and 3-buffer rotation (late_step) and both parities of the G-group tails buffer (inc_cur), holds streams
on the first call and right after their reset, never holds one stream, and resets the first and last stream of a
group, a whole group, the ragged last group, and a whole late-chain block plus one stream of the next.

The reference is the bulk clip path: every (stream, reset segment) becomes one clip of the samples that stream
stepped in that segment, run through oww_predict_clips_ragged with pad 0 and chunk size c*1280 (one call per c), whose
CNN runs in tc_conv_kernel with the same per-element arithmetic.  The rows of each clip's calls are mapped with the
library's own call schedule (oww_clip_schedule).  After every call: the feature rows each stepped stream appended equal
the bulk embeddings bit for bit; its scores too at split_from 3, 7, 11 and 15, and within 2e-5 at 20, where the heads
may run inside the fused kernel (the bound of test_bulk_clips_equal_streaming_at_every_split); a held stream's score
row is not written and its counts do not move.  test_fused_schedules_host.py runs the same schedules and row mapping
on the CPU stand-in of the library."""
import time

import numpy as np
import pytest

from helpers import emb_weights, head
from openwakeword_b200 import weights as W
from test_gpu_fused_items import _plan_g, torch_cuda  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

CHUNK = 1280
MAX_C = 3                     # largest per-stream count of a call (the engines' max_chunks)
CALLS = 30
RESETS = (10, 15, 20)         # partial resets run before these calls
SPLITS = [3, 7, 11, 15, 20]
# the kinds of the calls: F = fused (streams with c != 1 are held), R = general (counts 0..3)
KINDS = "FRFFRFFFRRFRFFRFRRFFFRFRFFRRFR"
assert len(KINDS) == CALLS


def heads():
    return [head("alexa_v0.1"), head("hey_jarvis_v0.1"), head("timer_v0.1")]


def late_layout(split):
    """(layer l, new rows per step, n_buf, S) of every late tensor X_l (the input of conv layer l >= split), by the rule
    of oww_late_alloc (cnn_tc.cu): n_buf 3 for a (3,1) layer on one new row per step, 2 for other (3,1) layers, 1 for
    (1,3) layers; S streams per block fill the 128 accumulator rows, halved while a (3,1) block exceeds 256 units."""
    rows, Wd = 8, 32
    out = []
    for l, (kh, _, _, _, pool_t, pool_f) in enumerate(W.EMBEDDING_LAYERS):
        if l >= split:
            kh3 = kh == 3
            T, Wq = rows + (2 if kh3 else 0), Wd if kh3 else Wd + 1
            S = max(1, 128 // (rows * Wq))
            while kh3 and S > 1 and T * S * Wd > 256:
                S //= 2
            out.append((l, rows, (3 if rows == 1 else 2) if kh3 else 1, S))
        if pool_t:
            rows, Wd = rows // pool_t, Wd // pool_f
    return out


def group_stream_count(G, sm):
    """(G - 1) full rounds of SMs plus part of one more, so that G - 1 would need a second round; n % G != 0 leaves a
    ragged last group (test_gpu_fused_items)"""
    n = sm // 2 + 1 if G == 1 else sm * (G - 1) + sm // 2 + 1
    return n + 1 if G > 1 and n % G == 0 else n


class Schedule:
    """counts [CALLS, n] int32; resets {call: stream ids reset right before it}; seg [CALLS, n]: the reset segment of
    each stream at each call; c {(stream, segment): the stream's count in that segment}.  A stream steps either its
    segment's count or nothing in each call."""

    def __init__(self, n, G, S, seed):
        rng = np.random.default_rng(seed)
        self.n, self.G, self.S = n, G, S
        n_groups = -(-n // G)
        assert n_groups >= 3 and (n % G or G == 1), (n, G)
        grp = lambda k: list(range(k * G, min(n, (k + 1) * G)))   # noqa: E731
        first = [G, 2 * G - 1] + grp(n_groups - 1)                          # first and last of group 1, the ragged group
        late = grp(n_groups // 2)                                            # one whole group
        if S:                                                                # one late-chain block and one more stream
            k = (n // S) // 2
            late += list(range(k * S, min(n, (k + 1) * S + 1)))
        self.steady = min((b for b in range(n) if b not in first + late), key=lambda b: abs(b - n // 2))
        some = rng.choice([b for b in range(n) if b != self.steady], max(2, n // 3), replace=False)
        self.resets = {t: sorted(set(int(b) for b in ids)) for t, ids in zip(RESETS, (first, some, late))}
        self.counts = np.zeros((CALLS, n), np.int32)
        self.seg = np.zeros((CALLS, n), np.int32)
        self.c = {}
        seg = np.zeros(n, np.int32)
        cur = rng.choice([1, 2, 3], n, p=[0.4, 0.3, 0.3]).astype(np.int32)
        cur[self.steady] = 1
        for b in range(n):
            self.c[(b, 0)] = int(cur[b])
        for t in range(CALLS):
            fresh = np.zeros(n, bool)
            for b in self.resets.get(t, []):
                seg[b] += 1
                cur[b] = rng.choice([1, 2, 3], p=[0.4, 0.3, 0.3])
                self.c[(b, int(seg[b]))] = int(cur[b])
                fresh[b] = True
            held = rng.random(n) < 0.2
            held |= fresh & (rng.random(n) < 0.5)                   # half of the reset streams wait a call
            if t == 0:
                held[0] = True
            if KINDS[t] == "F":
                held |= cur != 1
            held[self.steady] = False
            row = np.where(held, 0, cur).astype(np.int32)
            if (row == 1).all():                                    # equal counts would be the lockstep oww_step
                row[self.steady - 1] = 0
            self.counts[t], self.seg[t] = row, seg
        self.runs = self._hold_runs()
        self._check()

    def launches(self):
        """late_step before each call and after the last: one late-chain pass per chunk of the call's largest count (its
        parity is inc_cur's below split_from 20; at 20 a general call may run its one-chunk streams as a launch of their
        own, one flip more)"""
        return np.concatenate([[0], np.cumsum(self.counts.max(1))])

    def _hold_runs(self):
        """(stream, first held call, length) of every run of holds inside a segment that the stream then steps out of"""
        out = []
        for b in range(self.n):
            t0 = None
            for t in range(CALLS):
                if t0 is not None and self.seg[t, b] != self.seg[t0, b]:
                    t0 = None
                if self.counts[t, b] == 0:
                    t0 = t if t0 is None else t0
                elif t0 is not None:
                    out.append((b, t0, t - t0))
                    t0 = None
        return out

    def kinds(self):
        """calls by what the library runs: fused (largest count 1) or general (larger)"""
        m = self.counts.max(1)
        return int((m == 1).sum()), int((m > 1).sum())

    def coverage(self):
        """{run length (5: longer): sorted (late_step mod 2, mod 3) at the call the held stream resumes}"""
        L = self.launches()
        cov = {}
        for _, t0, k in self.runs:
            cov.setdefault(min(k, 5), set()).add((int(L[t0 + k] % 2), int(L[t0 + k] % 3)))
        return {k: sorted(v) for k, v in sorted(cov.items())}

    def _check(self):
        c = self.counts
        assert not (c == c[:, :1]).all(1).any(), "a call with equal counts"
        assert (c[:, self.steady] == 1).all()
        assert c[0, 0] == 0, "no stream held on the first call"
        assert any((c[t, ids] == 0).any() for t, ids in self.resets.items()), "no hold right after a reset"
        assert any(c[t].max() == 3 and (c[t] == 1).any() for t in range(CALLS)), "no count 1 in a call of largest count 3"
        assert all(self.kinds()), self.kinds()
        cov = self.coverage()
        assert all(k in cov for k in (1, 2, 3, 4)), cov
        resumed = set().union(*map(set, cov.values()))
        assert {r for r, _ in resumed} == {0, 1} and {r for _, r in resumed} == {0, 1, 2}, cov
        for (b, s), cb in self.c.items():
            st = c[:, b][self.seg[:, b] == s]
            assert set(st.tolist()) <= {0, cb}, (b, s)


def signals(rng, n, length):
    """noise at a per-stream level, louder every fourth 3000-sample stretch (shifted by stream), so that no stream is
    silent and states differ between neighbours"""
    t = np.arange(length)
    lvl = rng.uniform(300, 5000, n)[:, None] * (1 + 2 * (((t[None] // 3000) + np.arange(n)[:, None]) % 4 == 0))
    return np.clip(rng.standard_normal((n, length), np.float32) * lvl, -32768, 32767).astype(np.int16)


def run_schedule(eng, sched, sig, fi):
    """Drive eng through sched (partial resets with fi before their calls, oww_step_host_ragged on the samples each
    stream has not stepped yet).  Held streams: score row not written, (mel, feature) counts unchanged.
    -> {(stream, segment): (calls, score rows [steps, cols], appended feature rows [steps * c, 96])}"""
    n = sched.n
    pos = np.zeros(n, np.int64)
    acc = {}
    for t in range(CALLS):
        if t in sched.resets:
            eng.reset(fi, stream_ids=sched.resets[t])
        c = sched.counts[t]
        x = np.zeros((n, MAX_C * CHUNK), np.int16)
        for b in np.nonzero(c)[0]:
            x[b, :c[b] * CHUNK] = sig[b, pos[b]:pos[b] + c[b] * CHUNK]
        held = np.nonzero(c == 0)[0]
        before = [eng.ctx.get_counts(int(b)) for b in held]
        out = eng.step_host_ragged(x, c)
        assert np.isnan(out[held]).all(), f"call {t}: a held stream's score row was written"
        after = [eng.ctx.get_counts(int(b)) for b in held]
        assert after == before, f"call {t}: a held stream's counts moved"
        for b in np.nonzero(c)[0]:
            a = acc.setdefault((int(b), int(sched.seg[t, b])), ([], [], []))
            a[0].append(t)
            a[1].append(out[b].copy())
            a[2].append(eng.ctx.get_features(int(b), int(c[b])))     # read before a reset drops them
        pos += c.astype(np.int64) * CHUNK
    return {k: (v[0], np.stack(v[1]), np.concatenate(v[2])) for k, v in acc.items()}


def segment_clips(sched, sig):
    """{(stream, segment): the samples the stream stepped in that segment, holds removed}"""
    out = {}
    pos = np.concatenate([np.zeros((1, sched.n), np.int64), np.cumsum(sched.counts, 0, dtype=np.int64) * CHUNK])
    for (b, s), c in sched.c.items():
        t = np.nonzero(sched.seg[:, b] == s)[0]
        p0, p1 = pos[t[0], b], pos[t[-1] + 1, b]
        if p1 > p0:
            out[(b, s)] = sig[b, p0:p1]
    return out


def clip_rows(c, lengths):
    """The bulk path's rows of clips of these stepped lengths run at chunk size c*1280, each clip extended by one
    unread call of zeros (predict_clip leaves the last chunk_size samples of a clip unstepped).  -> (padded lengths,
    first score row of each clip, [per clip: first embedding row of each call]) from oww_clip_schedule"""
    from openwakeword_b200 import _native
    cs = c * CHUNK
    padded = [L + cs for L in lengths]
    row0, emb0, r, e = [], [], 0, 0
    for L, P in zip(lengths, padded):
        per_call = _native.clip_schedule(cs, P)
        assert np.array_equal(per_call, np.full(L // cs, c)), (c, L, per_call)   # one call per stepping call
        row0.append(r)
        emb0.append(e + np.concatenate([[0], np.cumsum(per_call)[:-1]]).astype(np.int64))
        r += per_call.size
        e += int(per_call.sum())
    return padded, row0, emb0, r, e


def bulk_reference(torch, hs, cfg, fi, sched, clips):
    """{(stream, segment): (score rows, feature rows)} of the segments' clips on the bulk clip path, one call per c"""
    from openwakeword_b200.engine import StreamEngine
    ref = StreamEngine(hs, 1, embedding=emb_weights(), max_chunks=MAX_C, **cfg)
    out = {}
    for c in (1, 2, 3):
        keys = [k for k in clips if sched.c[k] == c]
        if not keys:
            continue
        padded, row0, emb0, rows, embs = clip_rows(c, [clips[k].size for k in keys])
        pcm = np.zeros(sum(padded), np.int16)
        off = np.concatenate([[0], np.cumsum(padded)]).astype(np.int64)
        for i, k in enumerate(keys):
            pcm[off[i]:off[i] + clips[k].size] = clips[k]
        scores = torch.full((rows, ref.n_cols), float("nan"), dtype=torch.float32, device="cuda")
        emb = torch.full((embs, 96), float("nan"), dtype=torch.float32, device="cuda")
        ref.ctx.predict_clips_ragged(torch.from_numpy(pcm).cuda(), off, 0, c * CHUNK, fi, scores, None, emb)
        torch.cuda.synchronize()
        scores, emb = scores.cpu().numpy(), emb.cpu().numpy()
        for i, k in enumerate(keys):
            m = clips[k].size // (c * CHUNK)
            f = np.concatenate([emb[e:e + c] for e in emb0[i]])
            out[k] = (scores[row0[i]:row0[i] + m], f)
    ref.ctx.close()
    return out


def compare(sched, got, ref, score_tol):
    """-> (worst score difference, worst feature difference); fails at the first call and stream that differ, with
    the stream's place in its group and its late-chain block"""
    assert got.keys() == ref.keys()
    worst_s = worst_f = 0.0
    bad = []
    for k, (calls, gs, gf) in got.items():
        rs, rf = ref[k]
        c = sched.c[k]
        assert gs.shape == rs.shape and gf.shape == rf.shape, (k, gs.shape, rs.shape, gf.shape, rf.shape)
        assert np.isfinite(rs).all() and np.isfinite(rf).all() and np.isfinite(gs).all()
        ds = np.abs(gs - rs).max(1)
        df = np.abs(gf - rf).reshape(len(calls), c * 96).max(1)
        worst_s, worst_f = max(worst_s, float(ds.max())), max(worst_f, float(df.max()))
        wrong = (ds > score_tol) | (df > 0)
        if wrong.any():
            j = int(np.argmax(wrong))
            bad.append((calls[j], k[0], k[1], c, float(ds[j]), float(df[j])))
    if bad:
        t, b, s, c, ds, df = min(bad)
        G, S = sched.G, sched.S
        where = f"group {b // G} position {b % G}" + (f", block {b // S} position {b % S} (S = {S})" if S else "")
        raise AssertionError(f"{len(bad)} (stream, segment) pairs differ; first at call {t}: stream {b} ({where}), "
                             f"segment {s}, count {c}, counts of the call {np.bincount(sched.counts[t], minlength=4)}, "
                             f"score diff {ds:.3e}, feature diff {df:.3e}")
    return worst_s, worst_f


@pytest.mark.parametrize("split", SPLITS)
@pytest.mark.parametrize("G", list(range(1, 8)))
def test_fused_schedules(torch_cuda, built_library, G, split):
    torch = torch_cuda
    from openwakeword_b200.engine import StreamEngine
    if _plan_g(built_library, None, G, 1, split) is None:
        pytest.skip(f"G={G} does not fit shared memory at split_from={split}")
    t_start = time.time()
    n = group_stream_count(G, torch.cuda.get_device_properties(0).multi_processor_count)
    lay = late_layout(split)
    S = min(s for *_, s in lay) if lay else None
    sched = Schedule(n, G, S, seed=100 * split + G)
    rng = np.random.default_rng(split * 10 + G)
    fi = rng.normal(0, 1, (41, 96)).astype(np.float32)
    sig = signals(rng, n, int(sched.counts.sum(0).max()) * CHUNK)
    hs = heads()
    cfg = dict(cnn_mode=3, split_from=split)

    eng = StreamEngine(hs, n, embedding=emb_weights(), feature_init=fi, max_chunks=MAX_C, **cfg)
    assert _plan_g(built_library, eng.ctx.h) == G, n
    got = run_schedule(eng, sched, sig, fi)
    eng.ctx.close()
    ref = bulk_reference(torch, hs, cfg, fi, sched, segment_clips(sched, sig))

    fused, general = sched.kinds()
    n3 = ", ".join(f"X_{l}" for l, _, nb, _ in lay if nb == 3)
    print(f"split_from={split} G={G}: {n} streams, {-(-n // G)} groups; S per late layer "
          f"{ {l: s for l, _, _, s in lay} }; {fused} fused + {general} general calls, {len(sched.runs)} hold runs; "
          f"of the 6 (late_step mod 2, mod 3) a held stream resumes at, by run length (5: longer): "
          f"{ {k: len(v) for k, v in sched.coverage().items()} }" + (f"; 3-buffer tensors {n3}" if n3 else ""))
    ws, wf = compare(sched, got, ref, 2e-5 if split == 20 else 0.0)
    print(f"  max |streaming - bulk|: scores {ws:.3e}, feature rows {wf:.3e}; {time.time() - t_start:.1f} s")
