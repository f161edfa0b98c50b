"""Multi-GPU plumbing of the data-parallel path: one process per GPU, one BEV sequence per rank, no collective
inside the denoising loop (the reference: inference.py:248-269 DistributedSampler + bs=1; DDP is constructed but
only `model.module.log_images` is called, so no gradient/activation collective ever runs). The only exchange is
the gather of the finished frames/latents on rank 0 (BASELINE.json configs[2])."""
from __future__ import annotations

import torch
import torch.distributed as dist

BASE_SEED = 3407     # inference.py:250: seed = rank + 3407


def rank_seed(rank: int, base: int = BASE_SEED) -> int:
    return base + rank


def shard_indices(n_items: int, rank: int, world: int) -> list[int]:
    """DistributedSampler(shuffle=False) semantics (inference.py:264-266): rank r takes items r, r+world, ...;
    the tail is padded by wrapping around so every rank gets the same count."""
    per = (n_items + world - 1) // world
    idx = list(range(n_items))
    idx += idx[: per * world - n_items]
    return idx[rank: per * world: world]


def max_over_ranks(value_ms: float, device) -> float:
    """Device-timed duration -> max over ranks (how every multi-GPU number here is reported)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return value_ms
    t = torch.tensor([value_ms], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def gather_on_rank0(x: torch.Tensor):
    """Gathers equally-shaped per-rank results on rank 0 (NCCL over NVLink on the GPU box, gloo in CPU tests).
    Returns a list (rank 0) or None."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return [x]
    outs = [torch.empty_like(x) for _ in range(dist.get_world_size())] if dist.get_rank() == 0 else None
    dist.gather(x, outs, dst=0)
    return outs


def gather_named_on_rank0(x: torch.Tensor, names):
    """`gather_on_rank0` of `x`, with each rank's `names` (any picklable value, e.g. its frame file names) gathered
    alongside. Returns [(x of rank r, names of rank r) for every rank r] on rank 0 and [] elsewhere."""
    gathered = gather_on_rank0(x.contiguous())
    all_names = [None] * dist.get_world_size()
    dist.all_gather_object(all_names, names)
    return [] if gathered is None else list(zip(gathered, all_names))
