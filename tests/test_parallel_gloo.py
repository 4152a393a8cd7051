"""World-size-2 gloo test (CPU) of the column-dealing layer's host logic: the round-robin column deal, the padded all-gather
of per-rank results and its inverse interleave — the plumbing bench.py --gpus N uses."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from ezkl_b200 import parallel as par


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, total):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    r, w, _ = par.init_distributed("gloo")
    assert (r, w) == (rank, world)
    mine = par.my_columns(total, rank, world)
    # each "column result" is a 16-word row tagged with its global column index
    local = torch.tensor([[c * 1000 + j for j in range(16)] for c in mine], dtype=torch.int64).reshape(len(mine), 16)
    counts = [len(par.my_columns(total, q, world)) for q in range(world)]
    per_rank = par.allgather_columns(local, counts)
    full = par.interleave_columns(per_rank, total)
    assert full.shape == (total, 16)
    for c in range(total):
        assert int(full[c, 0]) == c * 1000 and int(full[c, 15]) == c * 1000 + 15
    dist.barrier()
    dist.destroy_process_group()


def test_column_deal_allgather_world2():
    port = _free_port()
    mp.spawn(_worker, args=(2, port, 7), nprocs=2, join=True)


def test_column_owner():
    assert [par.column_owner(i, 4) for i in range(6)] == [0, 1, 2, 3, 0, 1]
