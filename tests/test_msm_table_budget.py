"""Memory-bounded MSM base tables: the level policy, the sub-window digit routing, and reduced-table MSMs (s > 1 windows per
stored level, one bucket set per window of a level, a Horner fold at the end) against the oracle, up to k = 26 commitments."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from ezkl_b200 import _native as nat
from oracle import oracle as orc
from oracle import pyref
from tests import helpers as H

THREADS = orc.host_threads()
GIB = 1 << 30
DEFAULT_BUDGET = 16 * GIB


def default_window(n):
    """msm_default_window (msm.cu)."""
    k = max(n.bit_length() - 1, 0)
    c = 8 if k <= 10 else (k - 2 if k <= 13 else (k - 1 if k <= 17 else (17 if k <= 19 else (18 if k <= 21 else 20))))
    return min(max(c, 4), 22)


def windows(c):
    return (255 + c - 1) // c


def pick_levels(n, c, budget):
    s, L = C.c_int(0), C.c_int(0)
    nat.check(nat.dbg_lib().b200_debug_msm_pick_levels(C.c_size_t(n), C.c_int(c), C.c_size_t(budget), C.byref(s), C.byref(L)))
    return s.value, L.value


def expected_levels(n, c, budget):
    """The policy restated: smallest s whose ceil(W / s) levels of n * 64 B fit, else one level."""
    W = windows(c)
    for s in range(1, W + 1):
        if -(-W // s) * n * 64 <= budget:
            return s, -(-W // s)
    return W, 1


# ---- CPU tier ---------------------------------------------------------------------------------------------------------
def test_pick_levels_properties():
    budgets = [1, 64, 1 << 20, 256 << 20, GIB, 4 * GIB, 13 * GIB, DEFAULT_BUDGET, 52 * GIB, 1 << 50]
    for k in range(1, 27):
        n = 1 << k
        for c in sorted({4, 8, 10, 13, 16, 20, 22, 24, default_window(n)}):
            W = windows(c)
            for budget in budgets:
                s, L = pick_levels(n, c, budget)
                assert 1 <= s <= W and L == -(-W // s), (k, c, budget, s, L)
                assert L * n * 64 <= budget or L == 1, (k, c, budget, s, L)             # fits, or only the bases are kept
                if s > 1:                                                              # minimal: s - 1 does not fit
                    assert -(-W // (s - 1)) * n * 64 > budget, (k, c, budget, s)
                assert (s, L) == expected_levels(n, c, budget)
        if k <= 24:
            assert pick_levels(n, default_window(n), DEFAULT_BUDGET) == (1, windows(default_window(n))), k
    assert pick_levels(1 << 25, 20, DEFAULT_BUDGET) == (2, 7)
    assert pick_levels(1 << 26, 20, DEFAULT_BUDGET) == (4, 4)


def test_bare_int_above_2_32_reaches_a_size_t_intact():
    """The declared argtypes pass a plain Python int at the full width of size_t; untyped, ctypes passes it as a 32-bit int.  The budget
    is chosen so that cutting n to 5, the budget to 4096, or both, each gives a different level count than the intact call."""
    n, budget = (1 << 33) + 5, (3 << 40) + 4096
    s, L = C.c_int(0), C.c_int(0)
    nat.check(nat.dbg_lib().b200_debug_msm_pick_levels(n, 16, budget, C.byref(s), C.byref(L)))
    assert (s.value, L.value) == expected_levels(n, 16, budget) == (3, 6)
    assert (3, 6) not in {expected_levels(5, 16, budget), expected_levels(n, 16, 4096), expected_levels(5, 16, 4096)}


@pytest.mark.parametrize("c", [4, 7, 10, 13, 16, 20, 24])
def test_digit_slots(c):
    """(level, bucket set, bucket, sign) of every digit, for each windows-per-level count: sum_r 2^(c r) sum_j 2^(c s j) d_(js+r) == x,
    and every index lies inside the table (level < L) and inside its own bucket set."""
    rng = random.Random(100 + c)
    xs = [rng.randrange(pyref.R) for _ in range(60)] + [0, 1, 2, pyref.R - 1, pyref.R - 2, 1 << 253, (1 << c) - 1, 1 << (c - 1), (1 << (c - 1)) + 1]
    can = np.stack([H.int_to_limbs(x) for x in xs])
    W = windows(c)
    half = 1 << (c - 1)
    for s in sorted({1, 2, 3, W - 1, W} - {0}):
        L = -(-W // s)
        out = np.zeros((len(xs), W, 4), np.int32)
        nat.check(nat.dbg_lib().b200_debug_digit_slots_host(nat.ptr(can), C.c_size_t(len(xs)), C.c_int(c), C.c_int(s), out.ctypes.data_as(C.c_void_p)))
        for i, x in enumerate(xs):
            total = 0
            for w in range(W):
                lvl, r, bucket, sign = (int(v) for v in out[i, w])
                assert lvl == w // s and r == w % s and 0 <= lvl < L, (c, s, w)
                if sign == 0:
                    assert bucket == -1
                    continue
                assert r * half <= bucket < (r + 1) * half <= s * half, (c, s, w, bucket)
                d = sign * (bucket - r * half + 1)
                total += d << (c * r) << (c * s * lvl)
            assert total == x, (c, s, i)


@pytest.mark.parametrize("value", ["abc", "0", "-5", "12x", "", "99999999999999999999"])
def test_bad_table_budget_env_is_an_error(value):
    """B200_MSM_TABLE_MB is parsed in b200_init before any device is touched: a bad value fails with -1 and names the variable."""
    code = ("import ctypes, sys\n"
            "sys.path.insert(0, %r)\n"
            "from ezkl_b200 import _native as nat\n"
            "rc = nat.lib().b200_init(-1)\n"
            "print(rc, nat.lib().b200_last_error().decode())\n") % H.ROOT
    env = dict(os.environ, B200_MSM_TABLE_MB=value)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    rc, msg = r.stdout.strip().split(" ", 1)
    assert rc == "-1" and "B200_MSM_TABLE_MB" in msg, r.stdout


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


def budget_for(levels, n):
    return levels * n * 64


# (window bits, budget in levels, n, batch): L = 1, 2, W - 1, W, and c = 10 (W = 26) at 3 levels, where s = 9 leaves the last
# level with 8 of its 9 windows.  Ragged n throughout.
MSM_CASES = [
    (4, 1, 1000, 2), (4, 2, 777, 1), (4, 63, 129, 1),
    (10, 1, 3001, 5), (10, 2, 3001, 1), (10, 3, 2049, 2), (10, 25, 3001, 2), (10, 26, 3001, 1),
    (13, 2, 4099, 2), (16, 1, 1025, 1), (16, 15, 4097, 5), (16, 16, 1500, 2), (20, 4, 3000, 1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("c,levels,n,batch", MSM_CASES)
def test_reduced_table_msm_vs_oracle(gpu, c, levels, n, batch):
    from ezkl_b200 import halo2 as h2
    bases_np = orc.gen_bases(n, seed=1000 + n)
    b = h2.Bases(bases_np, window_bits=c, max_table_bytes=budget_for(levels, n))
    info = b.info()
    s, L = expected_levels(n, c, budget_for(levels, n))
    assert (info["windows_per_level"], info["levels"], info["windows"]) == (s, L, windows(c))
    assert info["table_bytes"] == L * n * 64 and info["n"] == n and info["window_bits"] == c
    cols = [orc.gen_scalars(n, seed=7 * n + j + c) for j in range(batch)]
    got = jac_to_affine(h2.best_multiexp_batch(cols, b))
    for j in range(batch):
        assert np.array_equal(got[j], orc.msm(cols[j], bases_np, THREADS)), (c, levels, j)
    b.release()


@pytest.mark.gpu
@pytest.mark.parametrize("levels", [1, 3, 26])
def test_reduced_table_degenerate_inputs(gpu, levels):
    """The distributions of the full-table degenerate test, on full and reduced tables (c = 10, W = 26)."""
    from ezkl_b200 import halo2 as h2
    n = 3000
    bases_np = orc.gen_bases(n, seed=77)
    bases = h2.Bases(bases_np, window_bits=10, max_table_bytes=budget_for(levels, n))
    assert bases.info()["levels"] == levels
    rng = random.Random(1)
    cols = {
        "zeros": np.zeros((n, 4), np.uint64),
        "ones": np.tile(orc.fr_one(), (n, 1)),
        "small": H.fr_array([rng.randrange(1 << 8) for _ in range(n)]),
        "half_zero": H.fr_array([0 if i % 2 else rng.randrange(pyref.R) for i in range(n)]),
        "r_minus_1": H.fr_array([pyref.R - 1] * n),
        "equal": H.fr_array([0x1234567] * n),
        "two_values": H.fr_array([(1, pyref.R - 5)[i % 2] for i in range(n)]),
        "dominant": H.fr_array([0xABCDEF if i % 10 else rng.randrange(pyref.R) for i in range(n)]),
    }
    got = h2.best_multiexp_batch(list(cols.values()), bases)
    for (name, sc), g in zip(cols.items(), got):
        assert np.array_equal(jac_to_affine(g)[0], orc.msm(sc, bases_np, THREADS)), name
    assert np.array_equal(got[0], np.array([0] * 4 + list(H.fq_wire(1)) + [0] * 4, np.uint64))
    m = 1234                                                # fewer scalars than registered bases (ParamsKZG::commit slicing)
    assert np.array_equal(jac_to_affine(h2.best_multiexp(cols["small"][:m], bases))[0], orc.msm(cols["small"][:m], bases_np[:m], THREADS))
    bases.release()
    dup = bases_np.copy()                                   # repeated and identity bases
    dup[1::2] = dup[0::2]
    dup[::7] = 0
    b2 = h2.Bases(dup, window_bits=10, max_table_bytes=budget_for(levels, n))
    for name in ("ones", "small", "half_zero", "r_minus_1"):
        assert np.array_equal(jac_to_affine(h2.best_multiexp(cols[name], b2))[0], orc.msm(cols[name], dup, THREADS)), name
    b2.release()


@pytest.mark.gpu
def test_reduced_table_geometry_rows(gpu):
    """c = 16 with s = 2 (8 of 16 levels): batch x 2 x 2^15 buckets crosses every reduction-geometry threshold (2^15, 2^18, 5 * 2^17,
    37 * 2^15) on both sides; full and reduced registrations of the same vector give the same normalised points."""
    from ezkl_b200 import halo2 as h2
    n = 1 << 11
    bases_np = orc.gen_bases(n, seed=901)
    full = h2.Bases(bases_np, window_bits=16)
    red = h2.Bases(bases_np, window_bits=16, max_table_bytes=budget_for(8, n))
    assert full.info()["levels"] == 16 and red.info()["windows_per_level"] == 2
    rng = random.Random(5)
    for batch in (1, 4, 5, 10, 11, 18, 19):
        cols = []
        for j in range(batch):
            if j % 3 == 1:
                cols.append(H.fr_array([rng.randrange(1 << 10) for _ in range(n)]))
            elif j % 3 == 2:
                cols.append(H.fr_array([pyref.R - 1 - (i % 3) for i in range(n)]))
            else:
                cols.append(orc.gen_scalars(n, seed=3000 * batch + j))
        a, b = h2.best_multiexp_batch(cols, full), h2.best_multiexp_batch(cols, red)
        assert np.array_equal(a, b), batch
    assert np.array_equal(jac_to_affine(b[-1])[0], orc.msm(cols[-1], bases_np, THREADS))
    full.release()
    red.release()


@pytest.mark.gpu
def test_reduced_table_device_path_matches_host(gpu):
    """b200_msm_batch_dev's XYZZ partials, normalised, against the host path, on a reduced table built from device points."""
    from ezkl_b200 import device as dev
    from ezkl_b200 import halo2 as h2
    n = (1 << 15) + 5
    d_pts = dev.generate_bases(n, seed=41)
    pts = dev.to_host(d_pts)
    budget = budget_for(3, n)
    db = dev.DeviceBases(d_pts, window_bits=13, max_table_bytes=budget)
    hb = h2.Bases(pts, window_bits=13, max_table_bytes=budget)
    assert hb.info()["levels"] == 3 and hb.info()["windows_per_level"] == 7
    cols = [orc.gen_scalars(n, seed=50 + j) for j in range(3)]
    d_sc = dev.from_host(np.stack(cols))
    assert np.array_equal(dev.normalize(dev.msm_batch(db, d_sc)), h2.best_multiexp_batch(cols, hb))
    assert np.array_equal(jac_to_affine(h2.best_multiexp(cols[1], hb))[0], orc.msm(cols[1], pts, THREADS))
    db.release()
    hb.release()


@pytest.mark.gpu
def test_reduced_table_launch_count_matches_profiler(gpu):
    """b200_launch_count against the k_* kernels torch.profiler records for a reduced-table registration and MSMs, so the table
    levels and the fold kernel are counted."""
    import re

    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from ezkl_b200 import device as dev
    n = 4000
    d_pts = dev.generate_bases(n, seed=61)
    d_sc = dev.from_host(np.stack([orc.gen_scalars(n, seed=62 + j) for j in range(2)]))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        torch.zeros(1, device="cuda")           # the profiler can lose the first kernel of a window that starts the moment it opens:
        torch.cuda.synchronize()                # open it with an uncounted kernel and a wait, so every counted kernel comes later
        l0 = nat.launch_count()
        b = dev.DeviceBases(d_pts, window_bits=10, max_table_bytes=budget_for(5, n))
        dev.msm_batch(b, d_sc)
        dev.msm_batch(b, d_sc[:1])
        torch.cuda.synchronize()
        launched = nat.launch_count() - l0
    b.release()
    kernels = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA and re.search(r"(^|[\s:])k_\w", e.name)]
    assert any("k_subwindow_fold" in k for k in kernels)
    assert launched == len(kernels), (launched, len(kernels), sorted(set(kernels)))


@pytest.mark.gpu
def test_budget_below_one_level_keeps_the_bases(gpu):
    from ezkl_b200 import halo2 as h2
    n = 500
    bases_np = orc.gen_bases(n, seed=3)
    b = h2.Bases(bases_np, window_bits=8, max_table_bytes=1)
    info = b.info()
    assert info["levels"] == 1 and info["windows_per_level"] == 32 and info["table_bytes"] == n * 64
    sc = orc.gen_scalars(n, seed=4)
    assert np.array_equal(jac_to_affine(h2.best_multiexp(sc, b))[0], orc.msm(sc, bases_np, THREADS))
    b.release()


def _free_gib():
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0] / GIB


@pytest.mark.gpu
@pytest.mark.parametrize("k", [25, 26])
def test_large_k_commitment_known_discrete_logs(gpu, k):
    """g[i] = [t^i] G for a trapdoor t (ParamsKZG.setup, on the device), so commit(p) = [p(t)] G with p(t) from the oracle's Horner:
    no CPU MSM.  At the full-window one-level table and at the default budget (k = 25: s = 2, L = 7; k = 26: s = 4, L = 4)."""
    import torch
    from ezkl_b200 import device as dev
    from ezkl_b200 import fields as F
    n = 1 << k
    need = (16 + 4 + 2 + 8) * n / (1 << 26)                 # GiB: default table, points, scalars, MSM workspace at 2^26
    free = _free_gib()
    if free < need:
        pytest.skip("needs %.0f GiB of free device memory, %.1f GiB free" % (need, free))
    t = 0x1D3C_5A17_9E3779B9_7F4A7C15
    one = F.fr_to_limbs(1)
    t_pows = dev.prefix_scan(dev.constant_column(t, n), one, True)
    g = dev.fixed_base_mul(t_pows)
    del t_pows
    p = dev.random_scalars(n, seed=k)
    p_host = dev.to_host(p)
    p_t = orc.eval_polynomial(p_host, H.fr_wire(t))
    del p_host
    gen = np.concatenate([F.fq_to_limbs(1), F.fq_to_limbs(2)]).reshape(1, 8)
    want = orc.g1_scalar_mul(gen, p_t.reshape(1, 4))[0]
    for budget, (s_want, L_want) in ((1, (13, 1)), (0, {25: (2, 7), 26: (4, 4)}[k])):
        b = dev.DeviceBases(g, max_table_bytes=budget)
        info = b.info()
        assert (info["windows_per_level"], info["levels"], info["window_bits"]) == (s_want, L_want, 20), info
        got = jac_to_affine(dev.normalize(dev.msm_batch(b, p)))[0]
        b.release()
        assert np.array_equal(got, want), (k, budget)
    del g, p
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_k26_two_vectors_fit_the_default_budget(gpu):
    """Both SRS vectors of k = 26 at the default budget: the two tables add at most 2 x 16 GiB (plus allocator slack) to the device."""
    import torch
    from ezkl_b200 import device as dev
    n = 1 << 26
    free = _free_gib()
    if free < 2 * 16 + 4 + 2:
        pytest.skip("needs 38 GiB of free device memory (two 16 GiB tables and 4 GiB of points), %.1f GiB free" % free)
    pts = dev.generate_bases(n, seed=26)
    torch.cuda.synchronize()
    before = torch.cuda.mem_get_info()[0]
    g = dev.DeviceBases(pts)
    gl = dev.DeviceBases(pts)
    torch.cuda.synchronize()
    used = before - torch.cuda.mem_get_info()[0]
    for b in (g, gl):
        info = b.info()
        assert info["levels"] == 4 and info["table_bytes"] == 16 * GIB, info
    g.release()
    gl.release()
    del pts
    torch.cuda.empty_cache()
    print("k = 26, two vectors at the default budget: %.2f GiB of device memory" % (used / GIB))
    assert used <= 2 * 16 * GIB + (256 << 20), used / GIB
