"""Data-parallel plumbing: one process per GPU (torchrun), NCCL over NVLink 4 / NVSwitch.

Replaces the reference's thread-queue "devices" and Python gradient averaging
(distributed/utils.py:8-226, distributed/hybrid_distributed.py:303-354,430-452,495-522).  The DP
contract it defined is kept: every rank processes its own `batch_size` sequences, gradients are the
unweighted mean over ranks (sum all-reduce here, 1/world folded into the optimizer's fused
gradient scale), the logged loss is token-weighted.

Because parameters/gradients live in one shape-grouped flat buffer (flat.ParamStore) the exchange
step is a single all-reduce of one contiguous tensor per optimizer update (not per micro-batch).
CPU tests run the same code over gloo.
"""
from __future__ import annotations

import os
from typing import List, Tuple

import torch
import torch.distributed as dist


def env_rank_world() -> Tuple[int, int, int]:
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")),
            int(os.environ.get("LOCAL_RANK", "0")))


def init_process_group(device: torch.device) -> None:
    if dist.is_initialized():
        return
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29500")
    backend = "nccl" if device.type == "cuda" else "gloo"
    kwargs = {"device_id": device} if device.type == "cuda" else {}
    dist.init_process_group(backend=backend, **kwargs)


def world_size() -> int:
    return dist.get_world_size() if dist.is_initialized() else 1


def all_reduce_sum_(t: torch.Tensor) -> torch.Tensor:
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t


def broadcast_(t: torch.Tensor, src: int = 0) -> torch.Tensor:
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.broadcast(t, src=src)
    return t


def barrier() -> None:
    if dist.is_initialized():
        dist.barrier()


def shard_batch(batch: torch.Tensor, rank: int, world: int) -> torch.Tensor:
    """Contiguous split of a global batch; the last shard takes the remainder
    (distribute_batch, hybrid_distributed.py:440-450)."""
    n = batch.shape[0]
    per = n // world
    lo = rank * per
    hi = n if rank == world - 1 else lo + per
    return batch[lo:hi]


def token_weighted_loss(loss_sum_and_ntok: torch.Tensor) -> float:
    """[sum(loss_i * ntok_i), sum(ntok_i)] -> mean loss after a sum all-reduce."""
    all_reduce_sum_(loss_sum_and_ntok)
    return float(loss_sum_and_ntok[0] / loss_sum_and_ntok[1])


def partition_by_cost(costs: List[float], world: int) -> List[int]:
    """Static greedy bin-packing (largest first): owner rank per item.  Used by the
    owner-computes Newton-Schulz mode, echoing ModalDistributedOptimizer's size-balanced chunks
    (modal/modal_cuda_utils.py:468-490)."""
    order = sorted(range(len(costs)), key=lambda i: -costs[i])
    load = [0.0] * world
    owner = [0] * len(costs)
    for i in order:
        r = min(range(world), key=lambda k: load[k])
        owner[i] = r
        load[r] += costs[i]
    return owner


def chunk_ranges(batch: int, world: int) -> Tuple[int, List[Tuple[int, int]]]:
    """Owner-computes split of one shape group's `batch` matrices: equal chunks of c = ceil(batch/world)
    consecutive matrices (the tail ranks may own fewer or none).  Returns (c, [(lo, hi) per rank]).
    Groups smaller than the world are handled by `small_group_owner` + broadcast instead, so that a
    single 32003 x 1024 embedding is not gathered world-size times."""
    c = -(-batch // world)
    return c, [(min(r * c, batch), min((r + 1) * c, batch)) for r in range(world)]


def small_group_owner(index: int, world: int) -> int:
    """Owner of matrix `index` of a group with fewer matrices than ranks: filled from the LAST rank
    down, because chunk_ranges leaves the tail ranks with the least work."""
    return world - 1 - (index % world)


def balanced_ranges(groups: List[Tuple[int, float]], world: int) -> List[List[Tuple[int, int, int]]]:
    """Cost-balanced contiguous ownership over the concatenation of all shape groups.
    groups[g] = (batch_g, cost_per_matrix_g).  Matrix i (global order) goes to rank
    floor(midpoint_i / (total / world)), so every rank owns ONE contiguous run that crosses few group
    boundaries: few, large batched launches per rank instead of a sliver of every group (the equal-chunk
    split an NCCL all-gather needs).  Returns per rank a list of (group, lo, hi).  Needs an exchange that
    accepts arbitrary ownership (the peer-memory epilogue stores)."""
    total = sum(b * c for b, c in groups)
    target = total / world if total > 0 else 1.0
    out: List[List[Tuple[int, int, int]]] = [[] for _ in range(world)]
    prefix = 0.0
    for g, (batch, cost) in enumerate(groups):
        run_rank, run_lo = None, 0
        for i in range(batch):
            r = min(world - 1, int((prefix + 0.5 * cost) / target))
            prefix += cost
            if r != run_rank:
                if run_rank is not None:
                    out[run_rank].append((g, run_lo, i))
                run_rank, run_lo = r, i
        if run_rank is not None:
            out[run_rank].append((g, run_lo, batch))
    return out


def all_gather_chunks_(full: torch.Tensor, chunk_elems: int, async_op: bool = False):
    """In-place all-gather: rank r contributes full[r*chunk : (r+1)*chunk], every rank ends with all
    world*chunk elements.  Returns the work handle when async_op (None on a single process)."""
    if not (dist.is_initialized() and dist.get_world_size() > 1):
        return None
    r = dist.get_rank()
    w = dist.get_world_size()
    assert full.numel() >= w * chunk_elems, "gather buffer smaller than world * chunk"
    out = full[:w * chunk_elems]
    mine = out[r * chunk_elems:(r + 1) * chunk_elems]
    if full.device.type == "cpu":   # gloo: no in-place gather; clone the contribution
        mine = mine.clone()
    return dist.all_gather_into_tensor(out, mine, async_op=async_op)


def broadcast_async_(t: torch.Tensor, src: int):
    if dist.is_initialized() and dist.get_world_size() > 1:
        return dist.broadcast(t, src=src, async_op=True)
    return None


def destroy() -> None:
    if dist.is_initialized():
        dist.destroy_process_group()
