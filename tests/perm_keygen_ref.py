"""halo2's own algorithm for the permutation sigma columns (plonk/permutation/keygen.rs, Assembly::build_pk), restated on the host with the
oracle's field arithmetic: omega^i by running products, the table delta^j * omega^i row by row on the host threads, then the gather.  It
shares nothing with the device's two-level power table, and is what the device's sigma columns are checked against."""
import numpy as np

from oracle import oracle as orc
from oracle import pyref

DELTA = pow(7, 1 << 28, pyref.R)           # Fr::DELTA = GENERATOR^(2^S)


def _wire(x: int) -> np.ndarray:
    x = pyref.to_mont(x % pyref.R, pyref.R)
    return np.array([(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], np.uint64)


def deltaomega(n_columns: int, k: int, threads: int | None = None) -> np.ndarray:
    """[n_columns, 2^k, 4]: row j = delta^j * [1, omega, omega^2, ...]."""
    threads = threads or orc.host_threads()
    n = 1 << k
    omega_powers = orc.prefix_scan(np.tile(orc.omega(k), (n, 1)), orc.fr_one(), True)      # exclusive running product: omega^i
    delta = _wire(DELTA)
    table = np.empty((n_columns, n, 4), np.uint64)
    cur = orc.fr_one()
    for j in range(n_columns):
        table[j] = orc.poly_op("scale", omega_powers, s=cur, threads=threads)
        cur = orc.field_op("fr", "mul", cur[None], delta[None])[0]
    return table


def perm_sigmas(mapping, k: int, table: np.ndarray | None = None) -> np.ndarray:
    """mapping [P, 2^k, 2] (column, row) per cell -> [P, 2^k, 4] sigma columns; `table` = deltaomega(P, k) when the caller has it."""
    m = np.asarray(mapping)
    if table is None:
        table = deltaomega(m.shape[0], k)
    return table[m[..., 0].astype(np.int64), m[..., 1].astype(np.int64)]


def sigma_int(column: int, row: int, k: int) -> int:
    """One cell's value as a python int (canonical): DELTA^column * omega^row."""
    return pow(DELTA, column, pyref.R) * pow(pyref.omega_for(k), row, pyref.R) % pyref.R


def mapping_of(kind: str, n_columns: int, k: int, seed: int = 0) -> np.ndarray:
    """A copy-constraint mapping [n_columns, 2^k, 2] uint32: `identity`, a `random` permutation of all cells, one `long_cycle` through every
    cell of every column, or `two_cycles` (cells swapped in random pairs)."""
    n = 1 << k
    N = n_columns * n
    rng = np.random.default_rng(seed)
    if kind == "identity":
        nxt = np.arange(N, dtype=np.int64)
    elif kind == "random":
        nxt = rng.permutation(N)
    elif kind == "long_cycle":
        order = rng.permutation(N)
        nxt = np.empty(N, np.int64)
        nxt[order] = np.roll(order, -1)
    elif kind == "two_cycles":
        order = rng.permutation(N)
        nxt = np.arange(N, dtype=np.int64)
        a, b = order[0:N - N % 2:2], order[1:N - N % 2:2]
        nxt[a], nxt[b] = b, a
    else:
        raise ValueError(kind)
    return np.stack([nxt // n, nxt % n], axis=-1).astype(np.uint32).reshape(n_columns, n, 2)
