"""world_size-2 gloo test of the data-parallel plumbing (batch sharding + the single flat gradient all-reduce)."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from vmambair_b200.dist import FlatGradAllReduce, broadcast_params, shard_batch


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(rank)  # different init per rank on purpose
    m = torch.nn.Sequential(torch.nn.Linear(4, 3), torch.nn.Linear(3, 2))
    v0 = [p._version for p in m.parameters()]
    broadcast_params(m)
    bumped = [p._version > v for p, v in zip(m.parameters(), v0)]
    gar = FlatGradAllReduce(m.parameters()).attach()
    data = torch.arange(8 * 4, dtype=torch.float32).view(8, 4) / 10
    lo, hi = shard_batch(8, rank, world)
    gar.zero()
    m(data[lo:hi]).square().sum().backward()
    gar.reduce(world)
    q.put((rank, [p.detach().clone() for p in m.parameters()], gar.flat.clone(), (lo, hi), bumped))
    dist.barrier()
    dist.destroy_process_group()


def _run_world(world):
    """spawn `world` gloo ranks on a fresh port; a rendezvous that fails (the probed port taken in between, a slow first import under
    load) is retried on another port"""
    ctx = mp.get_context("spawn")
    last = None
    for _ in range(3):
        port = _free_port()
        q = ctx.Queue()
        ps = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
        [p.start() for p in ps]
        try:
            res = sorted([q.get(timeout=180) for _ in range(world)], key=lambda t: t[0])
            [p.join(60) for p in ps]
            return res
        except Exception as e:  # queue.Empty: a rank died or hung before reporting
            last = e
            for p in ps:
                if p.is_alive():
                    p.terminate()
                p.join(10)
    raise last


def test_two_rank_flat_allreduce_matches_single_process():
    world = 2
    res = _run_world(world)
    assert res[0][3] == (0, 4) and res[1][3] == (4, 8)
    # replicas identical after broadcast, reduced gradients identical on both ranks
    for a, b in zip(res[0][1], res[1][1]):
        assert torch.equal(a, b)
    # the broadcast writes through p.data, which has its own version counter: broadcast_params bumps each parameter's, on every
    # rank, so weight caches keyed on _version (the inference path's) rebuild from the broadcast values
    assert all(res[0][4]) and all(res[1][4]), (res[0][4], res[1][4])
    assert torch.equal(res[0][2], res[1][2])
    # equals the mean over ranks of the per-shard gradients computed in one process
    m = torch.nn.Sequential(torch.nn.Linear(4, 3), torch.nn.Linear(3, 2))
    with torch.no_grad():
        for p, v in zip(m.parameters(), res[0][1]):
            p.copy_(v)
    data = torch.arange(8 * 4, dtype=torch.float32).view(8, 4) / 10
    m(data).square().sum().backward()
    flat = torch.cat([p.grad.flatten() for p in m.parameters()]) / world
    torch.testing.assert_close(res[0][2], flat, rtol=1e-5, atol=1e-6)


def test_shard_batch_covers_everything():
    for gb in (1, 7, 8, 32):
        for w in (1, 2, 4, 8):
            seen = []
            for r in range(w):
                lo, hi = shard_batch(gb, r, w)
                seen += list(range(lo, hi))
            assert seen == list(range(gb))


def test_flat_allreduce_mixed_dtype_and_missing_grads():
    """a parameter whose dtype differs from the flat buffer keeps its own .grad (copied in at reduce time); a parameter without a
    gradient this step contributes zeros instead of the previous step's values (single process: no collective needed)"""
    a = torch.nn.Parameter(torch.ones(3))
    b = torch.nn.Parameter(torch.ones(2, dtype=torch.float64))
    c = torch.nn.Parameter(torch.ones(4))
    gar = FlatGradAllReduce([a, b, c]).attach()
    assert a.grad is gar.views[0] and b.grad is None
    (a.sum() * 2 + b.sum() * 3 + c.sum() * 5).backward()
    gar.reduce(1)
    assert gar.flat.tolist() == [2.0] * 3 + [3.0] * 2 + [5.0] * 4
    assert b.grad.dtype == torch.float64  # untouched: assigning the fp32 view would raise
    c.grad = None
    gar.reduce(1)
    assert gar.flat[5:].tolist() == [0.0] * 4 and gar.flat[:3].tolist() == [2.0] * 3
