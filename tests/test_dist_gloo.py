"""world_size-2 gloo test of the N>1 path's host logic (sharding, seeds, max-over-ranks timing, rank-0 gather, with and
without the names)."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    from panacea_b200 import dist_utils as D
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        seed = D.rank_seed(rank)
        g = torch.Generator().manual_seed(seed)
        x = torch.randn(8, 4, 4, 12, generator=g)            # this rank's "sequence"
        ms = D.max_over_ranks(10.0 + 5.0 * rank, torch.device("cpu"))
        gathered = D.gather_on_rank0(x)
        named = D.gather_named_on_rank0(x, [f"rank{rank}"])
        idx = D.shard_indices(5, rank, world)
        if rank == 0:
            ok = len(gathered) == world and len(named) == world
            for r in range(world):
                ref = torch.randn(8, 4, 4, 12, generator=torch.Generator().manual_seed(D.rank_seed(r)))
                ok = ok and torch.equal(gathered[r], ref) and torch.equal(named[r][0], ref) and named[r][1] == [f"rank{r}"]
            out.put((rank, ok, ms, idx))
        else:
            out.put((rank, gathered is None and named == [], ms, idx))
    finally:
        dist.destroy_process_group()


def test_two_rank_gather_and_timing():
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(r[1] for r in res)
    assert all(abs(r[2] - 15.0) < 1e-9 for r in res)          # max over ranks
    assert res[0][3] == [0, 2, 4] and res[1][3] == [1, 3, 0]  # DistributedSampler(shuffle=False) with wrap-around pad
