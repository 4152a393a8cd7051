"""MSM digit recoding with shared-memory bucket counters (k_digits_tile): the tile policy msm_pick_recode, and MSMs on both
sides of its selection rule (a column's whole bucket set in shared memory, nb <= 2^15, or the global-atomic k_digits) against
the oracle.  The base-split offset (base_off != 0), which the product only uses across several devices, runs on one device through
the test hook b200_debug_msm_base_off (msm.cu linked into the debug library)."""
import ctypes as C
import random

import numpy as np
import pytest

from ezkl_b200 import _native as nat
from oracle import oracle as orc
from oracle import pyref
from tests import helpers as H

THREADS = orc.host_threads()
MAX_BUCKETS = 1 << 15
CTA = 1024
L2_BYTES = 16 << 20


def windows(c):
    return (255 + c - 1) // c


def recode_plan(n, batch, nb, W, sms):
    out = np.zeros(2, np.uint32)
    nat.check(nat.dbg_lib().b200_debug_msm_recode_plan(C.c_size_t(n), C.c_int(batch), C.c_uint32(nb), C.c_int(W), C.c_int(sms),
                                                       out.ctypes.data_as(C.c_void_p)))
    return int(out[0]), int(out[1])


def expected_plan(n, batch, nb, W, sms):
    """The policy restated (msm.cuh): enough tiles that the columns in flight scatter into <= 16 MiB of entry list and a small batch
    still fills the SMs; at least nb / W scalars per tile; a multiple of the CTA size."""
    if n == 0 or nb == 0 or nb > MAX_BUCKETS:
        return 0, 0
    tiles = max(-(-sms * n * W * 4 // L2_BYTES), -(-sms // batch))
    tile = max(-(-n // tiles), -(-nb // W))
    tile = -(-tile // CTA) * CTA
    return tile, -(-n // tile)


def level_counts(c):
    """Every windows-per-level count s that msm_pick_levels can produce for window c (one per distinct level count)."""
    W = windows(c)
    first = {}
    for s in range(1, W + 1):
        first.setdefault(-(-W // s), s)
    return sorted(first.values())


# ---- CPU tier ---------------------------------------------------------------------------------------------------------
def test_recode_plan_properties():
    batches = [1, 2, 3, 7, 20, 26, 60, 116, 1000, 4096, 65535]
    for k in range(1, 27):
        n = 1 << k
        for c in sorted({4, 8, 10, 13, 15, 16, 17, 18, 20, 22}):
            W = windows(c)
            for s in level_counts(c):
                nb = s << (c - 1)
                for batch in batches:
                    for sms in (114, 132):
                        tile, tiles = recode_plan(n, batch, nb, W, sms)
                        assert (tile, tiles) == expected_plan(n, batch, nb, W, sms), (k, c, s, batch, sms)
                        if nb > MAX_BUCKETS:                            # global-atomic recoding
                            assert tile == 0 and tiles == 0
                            continue
                        assert tile > 0 and tile % CTA == 0, (k, c, s, batch, sms, tile)
                        assert (tiles - 1) * tile < n <= tiles * tile    # the tiles cover the column, none of them empty
                        assert tile * W >= nb                            # no fewer entries per tile than counters to clear / publish
                        assert tiles * nb <= n * W + nb                  # count matrix within msm_workspace_per_column's bound
                        assert tile * W < 1 << 32                        # a 32-bit counter cannot overflow inside a tile
                        assert tiles < 1 << 31                           # grid.x


def test_recode_selection_threshold():
    """c = 16 (2^15 buckets) takes the shared path, c = 17 (2^16) the global one; a reduced table's s bucket sets count together."""
    n = 1 << 17
    assert recode_plan(n, 60, 1 << 15, 16, 132) == (2048, 64)          # the k = 17 bench shape
    assert recode_plan(n, 1, 1 << 15, 16, 132) == (2048, 64)
    assert recode_plan(n, 60, 1 << 16, 15, 132) == (0, 0)
    assert recode_plan(n, 8, 1 << 17, 15, 132) == (0, 0)              # k = 20, c = 18
    assert recode_plan(n, 4, 2 << 15, 16, 132) == (0, 0)              # c = 16 with s = 2
    assert recode_plan(n, 4, 2 << 9, 26, 132)[0] > 0                  # c = 10 with s = 2
    for bad in ((0, 1, 8, 4, 132), (100, 0, 8, 4, 132), (100, 1, 0, 4, 132), (100, 1, 8, 0, 132), (100, 1, 8, 4, 0)):
        assert recode_plan(*bad) == (0, 0), bad


# ---- GPU tier ---------------------------------------------------------------------------------------------------------
def jac_to_affine(j):
    j = np.asarray(j, np.uint64).reshape(-1, 12)
    out = j[:, :8].copy()
    for i in range(j.shape[0]):
        if not j[i, 8:].any():
            out[i] = 0
    return out


@pytest.fixture(scope="module")
def gpu():
    nat.init(-1)
    yield


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def make_bases(bases_np, c, levels=None):
    from ezkl_b200 import halo2 as h2
    n = bases_np.shape[0]
    return h2.Bases(bases_np, window_bits=c, max_table_bytes=0 if levels is None else levels * n * 64)


def top_digit_scalar(c):
    """Every window digit +2^(c-1) (the last bucket of a set), as many windows as stay below r."""
    x, w = 0, 0
    while c * (w + 1) <= 250:
        x += (1 << (c - 1)) << (c * w)
        w += 1
    return x


def low_digit_scalar(c):
    """Every window digit -(2^(c-1) - 1): c-bit values 2^(c-1) + 1 with the carry of the previous window."""
    x, w = 0, 0
    while c * (w + 1) <= 250:
        x += ((1 << (c - 1)) + (1 if w == 0 else 0)) << (c * w)
        w += 1
    return x


# (window bits, stored levels or None for the full table, n, batch).  c = 16 is the largest shared bucket set, c = 17 the smallest
# global one; c = 4 and 10 with s > 1 are reduced tables on the shared path.  n below one tile, ragged over several tiles, and batch
# 1 / 2 / 60.
SHARED_CASES = [
    (16, None, 1000, 1), (16, None, 5000, 2), (16, None, 9001, 60),
    (17, None, 1000, 1), (17, None, 5000, 2), (17, None, 9001, 60),
    (4, 2, 3001, 2), (10, 3, 5000, 1), (10, 3, 2500, 60), (13, None, 4097, 2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("c,levels,n,batch", SHARED_CASES)
def test_recode_msm_vs_oracle(gpu, c, levels, n, batch):
    from ezkl_b200 import halo2 as h2
    bases_np = orc.gen_bases(n, seed=500 + n + c)
    b = make_bases(bases_np, c, levels)
    info = b.info()
    nb = info["windows_per_level"] << (c - 1)
    tile, tiles = recode_plan(n, batch, nb, windows(c), sm_count())
    assert (tile > 0) == (nb <= MAX_BUCKETS)
    if tile:
        assert tiles == 1 or n % tile != 0, (tile, tiles)              # ragged: a short last tile or a single short tile
    cols = [orc.gen_scalars(n, seed=11 * n + j + c) for j in range(batch)]
    got = jac_to_affine(h2.best_multiexp_batch(cols, b))
    for j in range(batch):
        assert np.array_equal(got[j], orc.msm(cols[j], bases_np, THREADS)), (c, levels, n, batch, j)
    b.release()


@pytest.mark.gpu
@pytest.mark.parametrize("c,levels", [(16, None), (17, None), (10, 3)])
def test_recode_degenerate_scalars(gpu, c, levels):
    """Columns whose digits pile into few buckets: all zero, all equal (every digit of a tile in one bucket per window), r - 1, and
    digits at the ends of the range, +2^(c-1) and -(2^(c-1) - 1); with a few random columns in the same batch."""
    from ezkl_b200 import halo2 as h2
    n = 4500
    bases_np = orc.gen_bases(n, seed=90 + c)
    b = make_bases(bases_np, c, levels)
    rng = random.Random(c)
    eq = rng.randrange(pyref.R)
    cols = {
        "zeros": np.zeros((n, 4), np.uint64),
        "equal_small": H.fr_array([0x1234567] * n),
        "equal_random": np.tile(H.fr_wire(eq), (n, 1)),
        "r_minus_1": np.tile(H.fr_wire(pyref.R - 1), (n, 1)),
        "top_digits": np.tile(H.fr_wire(top_digit_scalar(c)), (n, 1)),
        "low_digits": np.tile(H.fr_wire(low_digit_scalar(c)), (n, 1)),
        "mixed_ends": H.fr_array([(top_digit_scalar(c), low_digit_scalar(c), pyref.R - 1)[i % 3] for i in range(n)]),
        "random": orc.gen_scalars(n, seed=c),
    }
    got = jac_to_affine(h2.best_multiexp_batch(list(cols.values()), b))
    for (name, sc), g in zip(cols.items(), got):
        assert np.array_equal(g, orc.msm(sc, bases_np, THREADS)), name
    assert not got[0].any()
    m = 1500                                                            # fewer scalars than registered bases
    assert np.array_equal(jac_to_affine(h2.best_multiexp(cols["equal_random"][:m], b))[0], orc.msm(cols["equal_random"][:m], bases_np[:m], THREADS))
    b.release()


@pytest.mark.gpu
@pytest.mark.parametrize("c,levels,kernels", [(16, None, ("k_digits_tile", "k_tile_prefix")), (17, None, ("k_digits<",)),
                                              (10, 3, ("k_digits_tile", "k_tile_prefix"))])
def test_recode_launch_count_matches_profiler(gpu, c, levels, kernels):
    """b200_launch_count against the k_* kernels torch.profiler records, on each side of the selection rule, and the recoding
    kernels of that side are the ones that ran."""
    import re

    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from ezkl_b200 import device as dev
    n = 3000
    d_pts = dev.generate_bases(n, seed=71)
    d_sc = dev.from_host(np.stack([orc.gen_scalars(n, seed=72 + j) for j in range(3)]))
    b = dev.DeviceBases(d_pts, window_bits=c, max_table_bytes=0 if levels is None else levels * n * 64)
    dev.msm_batch(b, d_sc)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        torch.zeros(1, device="cuda")           # the profiler can lose the first kernel of a window that starts the moment it opens:
        torch.cuda.synchronize()                # open it with an uncounted kernel and a wait, so every counted kernel comes later
        l0 = nat.launch_count()
        dev.msm_batch(b, d_sc)
        dev.msm_batch(b, d_sc[:1])
        torch.cuda.synchronize()
        launched = nat.launch_count() - l0
    b.release()
    names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA and re.search(r"(^|[\s:])k_\w", e.name)]
    assert launched == len(names), (launched, len(names), sorted(set(names)))
    for k in kernels:
        assert sum(k in x for x in names) >= 2, (k, sorted(set(names)))
    other = "k_digits<" if kernels[0] == "k_digits_tile" else "k_digits_tile"
    assert not any(other in x for x in names), sorted(set(names))


def msm_base_off(cols, bases_np, c, base_off, levels=None):
    """b200_debug_msm_base_off: affine sum_i cols[b][i] * bases[base_off + i] for every column b."""
    sc = np.ascontiguousarray(np.stack(cols), dtype=np.uint64)
    bases_np = np.ascontiguousarray(bases_np, dtype=np.uint64)
    batch, n = sc.shape[0], sc.shape[1]
    out = np.zeros((batch, 8), np.uint64)
    budget = 0 if levels is None else levels * bases_np.shape[0] * 64
    nat.check(nat.dbg_lib().b200_debug_msm_base_off(nat.ptr(sc), C.c_size_t(n), C.c_int(batch), nat.ptr(bases_np), C.c_size_t(bases_np.shape[0]),
                                                    C.c_int(c), C.c_size_t(budget), C.c_size_t(base_off), nat.ptr(out)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("c,levels", [(16, None), (17, None), (10, 3)])
def test_recode_base_off_vs_oracle(gpu, c, levels):
    """A range of pairs that starts inside the table: the entries carry base_off + i on the shared path (c = 16; c = 10 with s = 9)
    and the global one (c = 17), over several tiles (n = 5000, ragged) and inside one short tile (n = 900, at the end of the table)."""
    table_n = 7000
    bases_np = orc.gen_bases(table_n, seed=300 + c)
    rng = random.Random(400 + c)
    for n, base_off, batch in ((5000, 1999, 2), (900, table_n - 900, 1), (3000, 1, 3)):
        cols = [orc.gen_scalars(n, seed=rng.randrange(1 << 30)) for _ in range(batch)]
        if batch == 3:
            cols[2] = np.tile(H.fr_wire(pyref.R - 1), (n, 1))          # every digit of a tile in one bucket per window
        got = msm_base_off(cols, bases_np, c, base_off, levels)
        for j in range(batch):
            assert np.array_equal(got[j], orc.msm(cols[j], bases_np[base_off:base_off + n], THREADS)), (c, n, base_off, j)


@pytest.mark.gpu
def test_recode_concurrent_bucket_counts(gpu):
    """Host threads (each with its own stream and scratch) run shared-path MSMs with different bucket counts at the same time:
    c = 16 (128 KiB of counters per CTA), c = 8 and c = 10 with s = 3.  Every result stays exact."""
    import threading
    from ezkl_b200 import halo2 as h2
    n = 5000
    bases_np = orc.gen_bases(n, seed=808)
    tables = [make_bases(bases_np, 16), make_bases(bases_np, 8), make_bases(bases_np, 10, 3)]
    cols = [[orc.gen_scalars(n, seed=810 + 3 * i + j) for j in range(2)] for i in range(len(tables))]
    exp = [[orc.msm(col, bases_np, THREADS) for col in cs] for cs in cols]
    errs = []

    def worker(i):
        try:
            for _ in range(8):
                got = jac_to_affine(h2.best_multiexp_batch(cols[i], tables[i]))
                for j in range(2):
                    assert np.array_equal(got[j], exp[i][j]), (i, j)
        except Exception as e:      # noqa: BLE001
            errs.append((i, repr(e)))

    ts = [threading.Thread(target=worker, args=(i,)) for i in range(len(tables))]
    [t.start() for t in ts]
    [t.join() for t in ts]
    for b in tables:
        b.release()
    assert not errs, errs
