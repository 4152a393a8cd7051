"""Column dealing for one process per GPU over torch.distributed (NCCL over NVLink between H100s; gloo on CPU for the
host-logic tests), as `bench.py --gpus N` runs a proof.

A proof is ~100 independent MSM(n) and several hundred independent NTTs: `column_owner` deals whole columns to ranks
round-robin, every rank holds the whole SRS table, and the per-rank results are all-gathered (96 B per commitment) and put
back in column order.  No op is split across ranks; splitting one MSM or one NTT across devices is the library's job
(`b200_init_multi`, DESIGN.md §6).
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist


def init_distributed(backend: str | None = None):
    """Reads RANK / WORLD_SIZE / LOCAL_RANK / MASTER_* from the environment (torchrun).  Returns (rank, world, local)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, local


def column_owner(index: int, world: int) -> int:
    """Round-robin deal of independent units (columns / ops) to ranks."""
    return index % world


def my_columns(count: int, rank: int, world: int):
    return [i for i in range(count) if column_owner(i, world) == rank]


def allgather_columns(local: torch.Tensor, counts):
    """All-gather variable-count per-rank results [m_r, w] -> list of per-rank tensors (padded exchange)."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    if world == 1:
        return [local]
    mx = max(counts)
    pad = torch.zeros((mx, local.shape[1]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    outs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(outs, pad)
    return [o[:c] for o, c in zip(outs, counts)]


def interleave_columns(per_rank, total: int):
    """Inverse of the round-robin deal: per_rank[r][j] is global column r + j*world."""
    world = len(per_rank)
    out = [None] * total
    for r in range(world):
        for j in range(per_rank[r].shape[0]):
            out[r + j * world] = per_rank[r][j]
    return torch.stack(out) if total else per_rank[0][:0]
