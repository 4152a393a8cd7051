"""One-process-per-GPU sharding of the prover hot path over torch.distributed (NCCL over NVLink between H100s; gloo on
CPU for the host-logic tests).

The reference has no multi-GPU layer at all (SURVEY.md §2.3); this is the multi-GPU addition the north star asks for:
  * column level  — a proof is ~100 independent MSM(n) and several hundred independent NTTs: `column_owner` deals whole
    columns to ranks, the SRS table is replicated, results are all-gathered (96 B per commitment).  No data-path
    collective inside an op.
  * inside one MSM — `ShardedMsm`: the (scalar, base) pairs are split into contiguous slices, each rank runs the local
    Pippenger pipeline on its slice, the per-rank XYZZ partial sums (128 B each) are all-gathered and added locally in
    rank order (NCCL has no group-law reduction), so every rank ends with the same normalised point.
"""
from __future__ import annotations

import os

import numpy as np
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


def slice_bounds(n: int, rank: int, world: int):
    """Contiguous split of n pairs across ranks (remainder to the low ranks)."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


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


class ShardedMsm:
    """MSM split across ranks by base slice; one all-gather of XYZZ partials + a local add."""

    def __init__(self, d_bases_full_or_slice: torch.Tensor, n_total: int, already_sliced: bool = False, window_bits: int = 0):
        from . import device as dev
        self.rank = dist.get_rank() if dist.is_initialized() else 0
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self.n_total = n_total
        self.lo, self.hi = slice_bounds(n_total, self.rank, self.world)
        sl = d_bases_full_or_slice if already_sliced else d_bases_full_or_slice[self.lo:self.hi].contiguous()
        assert sl.shape[0] == self.hi - self.lo
        self.bases = dev.DeviceBases(sl, window_bits)

    def partial(self, scalars_local: torch.Tensor) -> torch.Tensor:
        """scalars_local [batch, hi-lo, 4] -> this rank's XYZZ partials [batch, 16]."""
        from . import device as dev
        return dev.msm_batch(self.bases, scalars_local)

    def combine(self, partial: torch.Tensor) -> torch.Tensor:
        """all-gather [batch,16] partials and add them in rank order -> [batch,16], identical on every rank."""
        from . import device as dev
        if self.world == 1:
            return partial
        outs = [torch.empty_like(partial) for _ in range(self.world)]
        dist.all_gather(outs, partial)
        stacked = torch.stack(outs, dim=1).contiguous()      # [batch, world, 16]
        return dev.g1_sum(stacked)

    def __call__(self, scalars_full: torch.Tensor) -> np.ndarray:
        """scalars_full [batch, n_total, 4] (every rank holds the column) -> normalised Jacobian wire [batch, 12]."""
        from . import device as dev
        if scalars_full.dim() == 2:
            scalars_full = scalars_full.unsqueeze(0)
        local = scalars_full[:, self.lo:self.hi].contiguous()
        return dev.normalize(self.combine(self.partial(local)))


# ------------------------------------------------------------------------------------------------------------------
class ShardedNtt:
    """Six-step NTT of one size-2^k polynomial split across `world` ranks with ONE all-to-all (north star: k >= 22).

    N = N1*N2, input index i = i1*N2 + i2, output index j = j1 + N1*j2.
      layout in : rank r holds the columns i2 in [r*N2/G, (r+1)*N2/G), all i1, as a local [N1, N2/G] array (row-major)
      step A    : local size-N1 NTTs over i1 (one per local column) and the twiddle omega^(j1*i2)
      step B    : all-to-all transpose — rank r keeps rows j1 in [r*N1/G, (r+1)*N1/G) for ALL i2
      step C    : local size-N2 NTTs over i2 (contiguous rows)
      layout out: rank r holds X[j1 + N1*j2] for its j1 range and all j2, as a local [N1/G, N2] array
    Input and output layouts are the same kind ("index mod the inner factor is block-distributed"), so element-wise column
    ops compose without further exchanges; `scatter` / `gather` convert from / to the natural order for tests.
    The local transforms and the twiddle product run in libezkl_b200.so; torch provides permutes and the NCCL collective.
    `local_ntt(batch_rows, log_m, omega)` and `mul(a, b)` are injectable so the index logic is testable on CPU (gloo)."""

    def __init__(self, k: int, omega_int: int, local_ntt=None, mul=None, make_twiddles=None):
        from . import fields as F
        self.rank = dist.get_rank() if dist.is_initialized() else 0
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self.k = k
        self.log_n1 = (k + 1) // 2
        self.log_n2 = k - self.log_n1
        self.N1, self.N2 = 1 << self.log_n1, 1 << self.log_n2
        G = self.world
        assert self.N1 % G == 0 and self.N2 % G == 0, "world size must divide both factors"
        self.c2, self.r1 = self.N2 // G, self.N1 // G          # local columns (step A) / local rows (step C)
        r = F.FR_MODULUS
        self.omega = omega_int % r
        self.omega_n1 = pow(self.omega, self.N2, r)            # root of the size-N1 transforms
        self.omega_n2 = pow(self.omega, self.N1, r)            # root of the size-N2 transforms
        self._local_ntt = local_ntt or self._dev_ntt
        self._mul = mul or self._dev_mul
        self._tw = (make_twiddles or self._dev_twiddles)()

    # ---- device implementations --------------------------------------------------------------------------------
    def _dev_ntt(self, rows, log_m, omega_int):
        from . import device as dev
        from . import fields as F
        return dev.ntt(rows.contiguous(), log_m, F.fr_to_limbs(omega_int))

    def _dev_mul(self, a, b):
        from . import device as dev
        return dev.poly_op("mul", a.contiguous(), b)

    def _dev_twiddles(self):
        """T[i2l][j1] = omega^(j1 * i2): each row is the running product of a constant row (exclusive scan, init 1)."""
        from . import device as dev
        from . import fields as F
        r = F.FR_MODULUS
        one = F.fr_to_limbs(1)
        out = torch.empty((self.c2, self.N1, 4), dtype=torch.int64, device="cuda")
        row = torch.empty((self.N1, 4), dtype=torch.int64, device="cuda")
        for i2l in range(self.c2):
            i2 = self.rank * self.c2 + i2l
            ratio = torch.from_numpy(F.fr_to_limbs(pow(self.omega, i2, r)).view(np.int64)).cuda()
            row[:] = ratio
            dev.prefix_scan(row, one, True, out=out[i2l])
        return out

    # ---- layout helpers (natural order <-> distributed), used by tests and by callers that start from a full vector ----
    def scatter(self, full):
        """full [N, w] natural order -> this rank's input block [N1, N2/G, w]."""
        w = full.shape[-1]
        return full.reshape(self.N1, self.N2, w)[:, self.rank * self.c2:(self.rank + 1) * self.c2].contiguous()

    def gather(self, local_out):
        """local_out [N1/G, N2, w] -> full [N, w] natural order on every rank (all-gather; test helper)."""
        w = local_out.shape[-1]
        if self.world > 1:
            parts = [torch.empty_like(local_out) for _ in range(self.world)]
            dist.all_gather(parts, local_out.contiguous())
        else:
            parts = [local_out]
        stacked = torch.cat(parts, dim=0)                      # [N1, N2, w] indexed [j1][j2]
        return stacked.permute(1, 0, 2).reshape(self.N1 * self.N2, w).contiguous()     # j = j1 + N1*j2

    # ---- the transform -----------------------------------------------------------------------------------------------
    def forward(self, local_in):
        """local_in [N1, N2/G, w] -> local_out [N1/G, N2, w]."""
        G, w = self.world, local_in.shape[-1]
        cols = local_in.permute(1, 0, 2).contiguous()                          # [c2, N1, w]: one contiguous polynomial per column
        y = self._mul(self._local_ntt(cols, self.log_n1, self.omega_n1), self._tw)     # step A (+ twiddle)
        if G > 1:
            send = y.reshape(self.c2, G, self.r1, w).permute(1, 0, 2, 3).contiguous()  # [dest][i2l][j1l]
            recv = torch.empty_like(send)
            dist.all_to_all_single(recv, send)                                 # step B: recv[src][i2l][j1l]
        else:
            recv = y.reshape(self.c2, 1, self.r1, w).permute(1, 0, 2, 3).contiguous()
        rows = recv.permute(2, 0, 1, 3).reshape(self.r1, self.N2, w).contiguous()      # [j1l][i2 = src*c2 + i2l]
        return self._local_ntt(rows, self.log_n2, self.omega_n2)               # step C
