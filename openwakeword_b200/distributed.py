"""Multi-GPU sharding of independent audio streams / clips (SURVEY.md section 8e).

A stream's scores depend only on its own PCM and its own rings, and the weights are a few MB, so
the path shards with NO data-path collective: rank r owns the contiguous block
``shard_range(n, r, world)`` of streams (or clips), weights are replicated, and the only exchange
is one gather of ``float32[n_local, n_labels]`` per step (``gather_scores``: NCCL all-gather over
NVLink/NVSwitch on GPU ranks, gloo in the CPU tests).  One process per GPU (torchrun).

``PeerGather`` removes even that call from the step: every rank's last kernel stores its scores
straight into the gathering rank's memory (peer-mapped over NVLink) and a counter follows them.
"""
import os


def shard_range(n_items, rank, world):
    """Contiguous block [lo, hi) of rank ``rank``; the first n_items % world ranks get one extra."""
    if world < 1 or not (0 <= rank < world):
        raise ValueError("bad rank/world")
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def env_rank_world():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))


def init_process_group(backend=None):
    """torchrun-style init from RANK/WORLD_SIZE/MASTER_*; returns (rank, world, local_rank)."""
    import torch
    import torch.distributed as dist
    rank, world, local = env_rank_world()
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, local


def gather_scores(local_scores, n_total, group=None):
    """All-gather per-rank score blocks [n_local, L] -> [n_total, L] in stream order on every rank.
    Blocks may differ by one row (uneven shard); they are padded to the largest for the collective."""
    import torch
    import torch.distributed as dist
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return local_scores
    world = dist.get_world_size(group)
    sizes = [shard_range(n_total, r, world) for r in range(world)]
    n_max = max(hi - lo for lo, hi in sizes)
    L = local_scores.shape[1]
    pad = local_scores
    if local_scores.shape[0] < n_max:
        pad = torch.zeros((n_max, L), dtype=local_scores.dtype, device=local_scores.device)
        pad[:local_scores.shape[0]] = local_scores
    out = torch.empty((world * n_max, L), dtype=local_scores.dtype, device=local_scores.device)
    dist.all_gather_into_tensor(out, pad.contiguous(), group=group)
    if all(hi - lo == n_max for lo, hi in sizes):
        return out
    return torch.cat([out[r * n_max:r * n_max + (hi - lo)] for r, (lo, hi) in enumerate(sizes)], dim=0)


class PeerGather:
    """Gather of the per-step scores on rank ``root`` through peer memory - no collective call.

    The root owns ``slots`` score buffers ``float32[n_total, n_cols]`` and one arrival counter per rank;
    every rank owns one acknowledgement counter.  Step k (1, 2, ...) uses buffer ``k % slots``:

      every rank   begin(k)    wait until the root has released step k - slots (this buffer's previous use)
                   dest(k)     device address for ``oww_step``'s scores: the rank's rows of the root's buffer
                   publish(k)  arrival counter of this rank on the root <- k (after the step's kernels)
      root only    collect(k)  wait until every rank's counter is >= k -> address of the full [n_total, n_cols]
                   release(k)  after the consumer's work is enqueued: every rank's acknowledgement counter <- k

    All calls are stream-ordered on ``stream`` (nothing blocks the host).  ``ctx`` supplies the peer_* calls of
    ``_native.Context``; ``exchange(obj)`` is an all-gather of small Python objects (``all_gather_object``)."""

    LINE = 16                                   # counters sit on their own 128-byte lines (16 x uint64)

    def __init__(self, ctx, n_total, n_cols, rank, world, exchange, root=0, slots=2, timeout_s=10.0):
        if slots < 2:
            raise ValueError("PeerGather needs at least two buffers (a step's scores land while the previous are read)")
        self.ctx, self.rank, self.world, self.root = ctx, rank, world, root
        self.n_total, self.n_cols, self.slots, self.timeout_s = n_total, n_cols, slots, timeout_s
        self.lo, self.hi = shard_range(n_total, rank, world)
        self._opened = []
        self.slot_bytes = n_total * n_cols * 4
        mine = {}
        self.ack_local, mine["ack"] = ctx.peer_alloc(8 * self.LINE)
        if rank == root:
            self.scores_base, mine["scores"] = ctx.peer_alloc(slots * self.slot_bytes)
            self.arrive_base, mine["arrive"] = ctx.peer_alloc(8 * self.LINE * world)
        everyone = exchange(mine)
        if rank == root:
            self.ack_of = [self.ack_local if r == rank else self._open(everyone[r]["ack"]) for r in range(world)]
        else:
            self.scores_base = self._open(everyone[root]["scores"])
            self.arrive_base = self._open(everyone[root]["arrive"])
        self.my_arrive = self.arrive_base + 8 * self.LINE * rank

    def _open(self, handle):
        addr = self.ctx.peer_open(handle)
        self._opened.append(addr)
        return addr

    def begin(self, k, stream=None):
        if k > self.slots:
            self.ctx.peer_wait(self.ack_local, 1, 1, k - self.slots, self.timeout_s, stream)

    def dest(self, k):
        return self.scores_base + (k % self.slots) * self.slot_bytes + self.lo * self.n_cols * 4

    def publish(self, k, stream=None):
        self.ctx.peer_signal(self.my_arrive, k, stream)

    def collect(self, k, stream=None):
        if self.rank != self.root:
            raise RuntimeError("collect() is the gathering rank's call")
        self.ctx.peer_wait(self.arrive_base, self.world, self.LINE, k, self.timeout_s, stream)
        return self.scores_base + (k % self.slots) * self.slot_bytes

    def release(self, k, stream=None):
        if self.rank != self.root:
            raise RuntimeError("release() is the gathering rank's call")
        for r in range(self.world):
            self.ctx.peer_signal(self.ack_of[r], k, stream)

    def close(self):
        for a in self._opened:
            self.ctx.peer_close(a)
        self._opened = []
        self.ctx.peer_free(self.ack_local)
        if self.rank == self.root:
            self.ctx.peer_free(self.scores_base)
            self.ctx.peer_free(self.arrive_base)


class _DeviceView:
    """Zero-copy torch view of library-owned device memory (``__cuda_array_interface__``)."""

    def __init__(self, addr, shape):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (int(addr), False),
                                         "version": 3, "strides": None}


class GatheredScores:
    """Result of an overlapped gather: ``wait()`` orders the current CUDA stream behind the collective and returns the
    ``[n_total, n_cols]`` tensor (valid until the step after next reuses the buffer)."""

    def __init__(self, tensor, work):
        self._t, self._w = tensor, work

    def wait(self):
        if self._w is not None:
            self._w.wait()
        return self._t


class ShardedStreams:
    """n_total independent streams split over the ranks of the default process group.

    ``engine_factory(n_local, lo, hi)`` builds this rank's step engine (on GPU ranks a
    ``StreamEngine`` bound to LOCAL_RANK); ``step(local_pcm)`` runs it and gathers the scores.

    ``gather``: ``"nccl"`` - all-gather on the compute stream after every step (every rank gets the scores);
    ``"nccl-overlap"`` - the all-gather of step k runs on a side stream while the compute stream already works on
    step k+1 (two score buffers; ``step`` returns a ``GatheredScores`` whose ``wait()`` yields the tensor);
    ``"peer"`` - every rank copies its score block into rank 0's buffer over NVLink, counters follow; no collective
    (tests/test_gpu_multi.py, two GPUs)."""

    def __init__(self, n_total, engine_factory, rank=None, world=None, gather="nccl"):
        r, w, _ = env_rank_world()
        self.rank = r if rank is None else rank
        self.world = w if world is None else world
        self.n_total = n_total
        self.lo, self.hi = shard_range(n_total, self.rank, self.world)
        self.engine = engine_factory(self.hi - self.lo, self.lo, self.hi)
        if gather not in ("nccl", "nccl-overlap", "peer"):
            raise ValueError("gather is 'nccl', 'nccl-overlap' (side-stream all-gather) or 'peer' (peer-memory gather on rank 0)")
        self.peer = None
        self._peer_loc = None
        self._peer_views = {}
        self._k = 0
        self._ov = None
        self.gather_kind = "none (single rank)" if self.world == 1 else gather
        if self.world > 1 and gather == "nccl-overlap" and n_total % self.world != 0:
            self.gather_kind = gather = "nccl"                    # uneven shards need the padded path
        if gather == "peer" and self.world > 1:
            import torch.distributed as dist

            def exchange(obj):
                out = [None] * self.world
                dist.all_gather_object(out, obj)
                return out
            self.peer = PeerGather(self.engine.ctx, n_total, self.engine.n_cols, self.rank, self.world, exchange)
        self._overlap = gather == "nccl-overlap" and self.world > 1

    def _overlap_state(self, dev):
        import torch
        if self._ov is None:
            n_loc, L = self.hi - self.lo, self.engine.n_cols
            self._ov = {"side": torch.cuda.Stream(device=dev),
                        "loc": [torch.empty((n_loc, L), dtype=torch.float32, device=dev) for _ in range(2)],
                        "out": [torch.empty((self.n_total, L), dtype=torch.float32, device=dev) for _ in range(2)],
                        "work": [None, None], "ev": [torch.cuda.Event(), torch.cuda.Event()]}
        return self._ov

    def step(self, local_pcm, n_chunks=1):
        """Scores of all n_total streams: on every rank with the NCCL all-gather ('nccl-overlap': a ``GatheredScores``);
        with gather='peer' on rank 0 only (a view of the gather buffer, valid until the step after next) and None elsewhere."""
        if self.world == 1:
            return self.engine.step(local_pcm, n_chunks)
        if self._overlap:
            import torch
            import torch.distributed as dist
            ov = self._overlap_state(local_pcm.device)
            i = self._k & 1
            self._k += 1
            if ov["work"][i] is not None:
                ov["work"][i].wait()                              # compute stream: buffer i has been gathered (no host block)
            self.engine.step(local_pcm, n_chunks, out=ov["loc"][i])
            ov["ev"][i].record()
            with torch.cuda.stream(ov["side"]):
                ov["side"].wait_event(ov["ev"][i])
                ov["work"][i] = dist.all_gather_into_tensor(ov["out"][i], ov["loc"][i], async_op=True)
            return GatheredScores(ov["out"][i], ov["work"][i])
        if self.peer is None:
            return gather_scores(self.engine.step(local_pcm, n_chunks), self.n_total)
        import torch
        pg = self.peer
        self._k += 1
        k = self._k
        stream = torch.cuda.current_stream(local_pcm.device).cuda_stream
        if self.rank == pg.root and k > 1:
            pg.release(k - 1, stream)             # whatever the caller enqueued on the previous result is ordered before this
        pg.begin(k, stream)
        # the step writes its scores locally (the heads and the verifier gates read-modify-write them); the finished
        # [rows x columns] block then crosses NVLink as ONE copy into this rank's rows of the root's buffer
        if self._peer_loc is None:
            self._peer_loc = torch.empty((self.hi - self.lo, self.engine.n_cols), dtype=torch.float32, device=local_pcm.device)
        self.engine.step(local_pcm, n_chunks, out=self._peer_loc)
        self.engine.ctx.peer_copy(pg.dest(k), self._peer_loc, self._peer_loc.numel() * 4, stream)
        pg.publish(k, stream)
        if self.rank != pg.root:
            return None
        addr = pg.collect(k, stream)
        # one zero-copy view per gather buffer, built once (wrapping a raw device address costs the host ~0.5 ms)
        view = self._peer_views.get(addr)
        if view is None:
            view = torch.as_tensor(_DeviceView(addr, (self.n_total, self.engine.n_cols)), device=local_pcm.device)
            self._peer_views[addr] = view
        return view

    def flush(self):
        """Order the current CUDA stream behind every outstanding overlapped gather."""
        if self._ov is not None:
            for w in self._ov["work"]:
                if w is not None:
                    w.wait()
