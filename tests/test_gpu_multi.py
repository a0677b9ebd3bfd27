"""gpu, needs two devices (skipped on a one-GPU box): the peer-memory score gather (distributed.PeerGather: every rank
copies its score block into rank 0's buffer over NVLink, counters follow) against every rank's own local scores.
Run on a machine with two GPUs: `python -m pytest tests/test_gpu_multi.py -m gpu`; the
protocol is also covered on host memory by tests/test_distributed_cpu.py::test_peer_gather_protocol_threads."""
import os
import socket

import numpy as np
import pytest

from helpers import emb_weights, head


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


def _worker(rank, world, port, n_total, steps, q):
    import torch
    import torch.distributed as dist
    from openwakeword_b200 import distributed as owd
    from openwakeword_b200.engine import StreamEngine
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    owd.init_process_group("gloo")                     # object exchange only; the data path uses no collective
    torch.cuda.set_device(rank)
    hs = [head("alexa_v0.1"), head("timer_v0.1")]

    def factory(n_local, lo, hi):
        return StreamEngine(hs, n_local, embedding=emb_weights(), device_index=rank, cnn_mode=3)
    sh = owd.ShardedStreams(n_total, factory, rank=rank, world=world, gather="peer")
    ref = factory(sh.hi - sh.lo, sh.lo, sh.hi)         # same shard, plain local scores
    rng = np.random.default_rng(11)
    pcm = rng.integers(-2000, 2000, (n_total, steps * 1280)).astype(np.int16)      # same on every rank
    worst, mine = 0.0, []
    for k in range(steps):
        d = torch.from_numpy(np.ascontiguousarray(pcm[sh.lo:sh.hi, k * 1280:(k + 1) * 1280])).cuda()
        full = sh.step(d, 1)
        local = ref.step(d, 1)
        mine.append(local.cpu().numpy())
        if rank == 0:
            got = full.clone()
            torch.cuda.synchronize()
            q.put(("full", k, got.cpu().numpy()))
    q.put(("local", rank, np.stack(mine)))
    dist.barrier()
    sh.peer.close()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("n_total", [12, 13])
def test_peer_gather_two_gpus(torch_cuda, built_library, n_total):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    steps, world = 9, 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_worker, args=(r, world, port, n_total, steps, q)) for r in range(world)]
    [p.start() for p in ps]
    items = [q.get(timeout=300) for _ in range(steps + world)]
    [p.join(60) for p in ps]
    assert all(p.exitcode == 0 for p in ps)
    local = {r: a for tag, r, a in items if tag == "local"}
    full = {k: a for tag, k, a in items if tag == "full"}
    want = np.concatenate([local[0], local[1]], axis=1)          # [steps, n_total, n_cols] in stream order
    for k in range(steps):
        np.testing.assert_array_equal(full[k], want[k])


@pytest.mark.gpu
def test_two_devices_in_one_process(torch_cuda, built_library):
    """Two handles on two GPUs inside ONE process (the per-device function attributes - dynamic shared memory above
    48 KB for the conv, heads and step kernels - are tracked per handle): both must run the default path and agree."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from openwakeword_b200.engine import StreamEngine
    rng = np.random.default_rng(5)
    hs = [head("alexa_v0.1"), head("timer_v0.1")]
    B, steps = 200, 6
    pcm = rng.integers(-3000, 3000, (B, steps * 1280)).astype(np.int16)
    outs = []
    for dev in (0, 1):
        eng = StreamEngine(hs, B, embedding=emb_weights(), device_index=dev, cnn_mode=3)
        got = []
        with torch.cuda.device(dev):
            for k in range(steps):
                d = torch.from_numpy(np.ascontiguousarray(pcm[:, k * 1280:(k + 1) * 1280])).to(f"cuda:{dev}")
                got.append(eng.step(d, 1).cpu().numpy())
        outs.append(np.stack(got))
        eng.ctx.close()
    np.testing.assert_array_equal(outs[0], outs[1])
