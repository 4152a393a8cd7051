"""The MSM pipeline of msm_run stage by stage: its launch geometry (msm_plan: chunk cap, chunk and heavy-list strides, bucket-reduction
rows, k_final width, recoding plan, workspace bytes) restated and checked over every window and table shape, and on the device every
window 4..24, every chunk cap, the light / heavy split of k_combine / k_combine_heavy and both loops of the latter, both sides of the
scatter's skew threshold, buckets of only P and -P, and the batch splits of msm_dev_on, each case asserting the branch it reaches
before it compares with the oracle (or with a known discrete log)."""
import ctypes as C
import random

import numpy as np
import pytest

from ezkl_b200 import _native as nat
from oracle import oracle as orc
from oracle import pyref
from tests import helpers as H
from tests.test_msm_recode import expected_plan as expected_recode
from tests.test_msm_recode import level_counts, windows

THREADS = orc.host_threads()
HEAVY_CHUNKS = 32
TREE_THREADS = 256
GIB = 1 << 30
FIELDS = ("cap", "chunk_stride", "heavy_stride", "reduce_m", "reduce_threads", "nparts", "final_threads", "tile", "tiles",
          "counts_bytes", "tile_counts_bytes", "offs_bytes", "ents_bytes", "subs_bytes", "sums_bytes", "ws_per_column")
XYZZ_BYTES = 128


def msm_plan(n, batch, c, s, sms, reduce_m=0, reduce_threads=0):
    """b200_debug_msm_plan as a dict, or None where msm_run rejects the shape."""
    out = np.zeros(len(FIELDS), np.uint64)
    rc = nat.dbg_lib().b200_debug_msm_plan(C.c_size_t(n), C.c_int(batch), C.c_int(c), C.c_int(s), C.c_int(sms), C.c_int(reduce_m),
                                           C.c_int(reduce_threads), out.ctypes.data_as(C.c_void_p))
    if rc == -1:
        return None
    nat.check(rc)
    return dict(zip(FIELDS, (int(v) for v in out)))


def expected_cap(total_entries, sms):
    target = total_entries // (sms * 512 * 4)
    cap = 16
    while cap < 512 and cap < target:
        cap <<= 1
    return cap


def expected_plan(n, batch, c, s, sms, reduce_m=0, reduce_threads=0):
    """The policy restated (msm.cuh msm_plan): a chunk cap from the entries of the whole call, the reduction rows from its bucket count
    (latency-bound small calls take fewer buckets per thread), the tuning overrides, and the buffers msm_run carves its workspace into."""
    W = windows(c)
    half, nb = 1 << (c - 1), s << (c - 1)
    ents = n * W
    cap = expected_cap(ents * batch, sms)
    chunk_stride = nb + ents // cap + 1
    heavy_stride = ents // (cap * HEAVY_CHUNKS) + 2
    buckets = batch * nb
    m, t = ((4, 128) if buckets <= 1 << 15 else (8, 128) if buckets <= 1 << 18 else (16, 256) if buckets <= 5 << 17
            else (32, 128) if buckets < 37 << 15 else (32, 256))
    while m > 1 and m > half:
        m >>= 1
    if 1 <= reduce_m <= 4096:
        m = reduce_m
    if reduce_threads in (32, 64, 128, 256):
        t = reduce_threads
    per_cta = -(-half // m)
    nparts = -(-per_cta // t)
    final = 32
    while final < TREE_THREADS and final < nparts:
        final <<= 1
    tile, tiles = expected_recode(n, batch, nb, W, sms)
    n_len, n_off = batch * (cap + 1), batch * (nb + 1)
    vcols = batch * s
    ws_col = (ents * 4 + (nb + ents // 16 + 1) * (12 + XYZZ_BYTES) + nb * (XYZZ_BYTES + 24) + 65536 * s
              + ((ents + nb) * 4 if nb <= 1 << 15 else 0))
    return dict(cap=cap, chunk_stride=chunk_stride, heavy_stride=heavy_stride, reduce_m=m, reduce_threads=t, nparts=nparts,
                final_threads=final, tile=tile, tiles=tiles,
                counts_bytes=(2 * batch * nb + 2 * n_len + batch * heavy_stride) * 4,
                tile_counts_bytes=batch * tiles * nb * 4 if tile else 0,
                offs_bytes=(2 * n_off + n_len + batch) * 4, ents_bytes=batch * ents * 4, subs_bytes=batch * chunk_stride * 12,
                sums_bytes=XYZZ_BYTES * (batch * chunk_stride + batch * nb + vcols * nparts + (vcols if s > 1 else 0)),
                ws_per_column=ws_col)


def most_chunks(ents, nb, cap):
    """The most chunks of <= cap entries that ents entries in nb buckets can make: one entry opens a bucket's first chunk, every
    further chunk of that bucket needs cap more."""
    k = min(nb, ents)
    return k + (ents - k) // cap


def plan_bytes(p):
    return p["counts_bytes"] + p["tile_counts_bytes"] + p["offs_bytes"] + p["ents_bytes"] + p["subs_bytes"] + p["sums_bytes"]


# ---- CPU tier ---------------------------------------------------------------------------------------------------------
SWEEP_N = sorted({1 << k for k in range(27)} | {3, 1000, 3001, 4097, (1 << 16) + 1, 3 << 20, (1 << 26) - 1})
SWEEP_BATCH = (1, 2, 3, 5, 17, 34, 67, 116, 1000, 1023, 1024, 4096, 4097, 65535)


@pytest.mark.parametrize("c", range(4, 25))
def test_msm_plan_matches_policy_and_invariants(c):
    """Every window, every level count msm_pick_levels can give it, n = 1 .. 2^26, batch 1 .. 65535, 114 and 132 SMs, and the reduction
    overrides: the hook equals the restated policy, and the plan keeps the invariants the kernels rely on."""
    W = windows(c)
    half = 1 << (c - 1)
    for s in level_counts(c):
        nb = s * half
        for n in SWEEP_N:
            ents = n * W
            for batch in SWEEP_BATCH:
                for sms in (114, 132):
                    for rm, rt in ((0, 0), (1, 32), (3, 64), (4096, 256), (5000, 100)):
                        where = (n, batch, c, s, sms, rm, rt)
                        p = msm_plan(n, batch, c, s, sms, rm, rt)
                        if batch * s > 65535 or ents >= 1 << 32:
                            assert p is None, where
                            continue
                        assert p == expected_plan(n, batch, c, s, sms, rm, rt), where
                        cap = p["cap"]
                        assert 16 <= cap <= 512 and cap & (cap - 1) == 0, where
                        assert p["chunk_stride"] >= most_chunks(ents, nb, cap), where
                        # a heavy bucket holds > 32 * cap entries: the list has room for every one of them after its count word
                        assert p["heavy_stride"] - 1 >= ents // (HEAVY_CHUNKS * cap + 1), where
                        assert p["nparts"] * p["reduce_threads"] * p["reduce_m"] >= half, where
                        assert p["nparts"] < 1 << 31 and p["reduce_threads"] in (32, 64, 128, 256), where
                        ft = p["final_threads"]
                        assert ft & (ft - 1) == 0 and 32 <= ft <= TREE_THREADS and ft >= min(p["nparts"], TREE_THREADS), where
                        assert p["ws_per_column"] * batch >= plan_bytes(p), where          # what msm_dev_on's batch split relies on


def test_msm_plan_rejects_what_msm_run_rejects():
    ok = (3000, 1, 16, 1, 132, 0, 0)
    assert msm_plan(*ok) is not None
    for bad in ((0, 1, 16, 1, 132, 0, 0), (3000, 0, 16, 1, 132, 0, 0), (3000, 1, 3, 1, 132, 0, 0), (3000, 1, 25, 1, 132, 0, 0),
                (3000, 1, 16, 0, 132, 0, 0), (3000, 1, 16, 17, 132, 0, 0), (3000, 1, 16, 1, 0, 0, 0), (3000, 1024, 4, 64, 132, 0, 0),
                (1 << 26, 1, 4, 1, 132, 0, 0)):
        assert msm_plan(*bad) is None, bad
    assert msm_plan(3000, 1023, 4, 64, 132) is not None                # 1023 x 64 = 65472 bucket sets fit one grid
    assert msm_plan((1 << 26) - 1, 1, 4, 1, 132) is not None            # n * W = 2^32 - 64


def test_msm_plan_reaches_every_branch():
    """The shapes the GPU tier below builds reach what it claims: k_final's strided loop at c >= 23, each cap on both SM counts
    within 67 columns of 2^16 at c = 16, and cap 16 for the heavy-bucket columns."""
    for c in range(4, 25):
        p = msm_plan(3001, 1, c, 1, 132)
        assert (p["nparts"] > TREE_THREADS) == (c >= 23), (c, p["nparts"])
        assert (p["tile"] > 0) == (c <= 16)
    for sms in (114, 132):
        caps = {msm_plan(1 << 16, b, 16, 1, sms)["cap"] for b in range(1, 68)}
        assert caps == {16, 32, 64, 128, 256, 512}, (sms, caps)
    assert msm_plan(30000, 1, 16, 1, 132)["cap"] == msm_plan(30000, 1, 16, 1, 114)["cap"] == 16


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


def free_gib():
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0] / GIB


def skip_unless_free(p, batch, table_bytes, what):
    need = (plan_bytes(p) + table_bytes) / GIB + 0.25
    free = free_gib()
    if free < need:
        pytest.skip("%s needs %.2f GiB of free device memory (workspace and table), %.1f GiB free" % (what, need, free))


def bucket_counts(scalars_int, c, s):
    """Host digit histogram of one column (b200_debug_digit_slots_host): entries per bucket of the column's s bucket sets."""
    can = np.stack([H.int_to_limbs(x) for x in scalars_int])
    W = windows(c)
    out = np.zeros((len(scalars_int), W, 4), np.int32)
    nat.check(nat.dbg_lib().b200_debug_digit_slots_host(nat.ptr(can), C.c_size_t(len(scalars_int)), C.c_int(c), C.c_int(s),
                                                        out.ctypes.data_as(C.c_void_p)))
    b = out[:, :, 2].reshape(-1)
    return np.bincount(b[b >= 0], minlength=s << (c - 1))


def generator():
    from ezkl_b200 import fields as F
    return np.concatenate([F.fq_to_limbs(1), F.fq_to_limbs(2)]).reshape(1, 8)


TRAPDOOR = 0x2B5E_1F0D_7C4A_9E3779B9_7F4A7C15


def srs_g(n):
    """g[i] = [t^i] G on the device (ParamsKZG.setup's g), so sum_i p_i g[i] = [p(t)] G."""
    from ezkl_b200 import device as dev
    from ezkl_b200 import fields as F
    return dev.fixed_base_mul(dev.prefix_scan(dev.constant_column(TRAPDOOR, n), F.fr_to_limbs(1), True))


def known_dlog(cols_host):
    """[p_j(t)] G for every column p_j (host wire [batch, n, 4]), affine."""
    pts = np.stack([orc.eval_polynomial(col, H.fr_wire(TRAPDOOR)) for col in cols_host])
    return orc.g1_scalar_mul(np.repeat(generator(), len(cols_host), axis=0), pts)


@pytest.mark.gpu
@pytest.mark.parametrize("c", range(4, 25))
def test_every_window_vs_oracle(gpu, c):
    """Full tables of every window the ABI accepts, n = 3001: a uniform column and one whose digits all sit at the top of their set.
    c <= 16 recodes with shared counters, c >= 17 with global atomics; at c >= 23 nparts exceeds k_final's 256 threads."""
    from ezkl_b200 import halo2 as h2
    n, batch = 3001, 2
    p = msm_plan(n, batch, c, 1, sm_count())
    assert (p["tile"] > 0) == (c <= 16)
    assert (p["nparts"] > p["final_threads"]) == (c >= 23), p
    skip_unless_free(p, batch, n * windows(c) * 64, "c = %d" % c)
    bases_np = orc.gen_bases(n, seed=2400 + c)
    b = h2.Bases(bases_np, window_bits=c)
    assert (b.info()["window_bits"], b.info()["levels"]) == (c, windows(c))
    top = (1 << (c - 1)) * sum(1 << (c * w) for w in range(250 // c))
    cols = [orc.gen_scalars(n, seed=2500 + c), H.fr_array([top + i for i in range(n)])]
    got = jac_to_affine(h2.best_multiexp_batch(cols, b))
    b.release()
    for j in range(batch):
        assert np.array_equal(got[j], orc.msm(cols[j], bases_np, THREADS)), (c, j)


@pytest.mark.gpu
def test_every_window_one_column_2_16(gpu):
    """One column of 2^16 against g[i] = [t^i] G under every window 4..24: every normalised result is [p(t)] G."""
    from ezkl_b200 import device as dev
    n = 1 << 16
    g = srs_g(n)
    p = dev.random_scalars(n, seed=216)
    want = known_dlog(dev.to_host(p)[None])[0]
    for c in range(4, 25):
        plan = msm_plan(n, 1, c, 1, sm_count())
        skip_unless_free(plan, 1, n * windows(c) * 64, "c = %d at n = 2^16" % c)
        b = dev.DeviceBases(g, window_bits=c)
        got = jac_to_affine(dev.normalize(dev.msm_batch(b, p)))[0]
        b.release()
        assert np.array_equal(got, want), c


@pytest.mark.gpu
def test_cap_ladder(gpu):
    """n = 2^16 at c = 16: for each chunk cap 16 .. 512 the smallest batch that reaches it on this device, every column against its
    known discrete log."""
    import torch
    from ezkl_b200 import device as dev
    n, c, sms = 1 << 16, 16, sm_count()
    first = {}
    for batch in range(1, 200):
        first.setdefault(msm_plan(n, batch, c, 1, sms)["cap"], batch)
    assert sorted(first) == [16, 32, 64, 128, 256, 512], first
    top = max(first.values())
    g = srs_g(n)
    b = dev.DeviceBases(g, window_bits=c)
    sc = dev.random_scalars(n, batch=top, seed=1616)
    want = known_dlog(dev.to_host(sc).reshape(top, n, 4))
    one_run = None
    for cap, batch in sorted(first.items()):
        if cap > 16:
            assert msm_plan(n, batch - 1, c, 1, sms)["cap"] == cap // 2          # the first batch of its cap
        torch.cuda.synchronize()
        l0 = nat.launch_count()
        out = dev.msm_batch(b, sc[:batch].contiguous())
        launched = nat.launch_count() - l0
        one_run = one_run or launched
        assert launched == one_run, (cap, batch, launched)                    # the whole batch is one msm_run, with this cap
        assert np.array_equal(jac_to_affine(dev.normalize(out)), want[:batch]), (cap, batch)
    b.release()
    del g, sc
    torch.cuda.empty_cache()


def hot_column(hot, fill, seed, c=16):
    """Scalars as python ints: hot = {value: count} (values below 2^(c-1): one window-0 digit, i.e. one entry of bucket value - 1), then
    `fill` uniform scalars that leave those buckets exactly at their count."""
    rng = random.Random(seed)
    fillers = []
    while len(fillers) < fill:
        x = rng.randrange(pyref.R)
        if set(bucket_counts([x], c, 1).nonzero()[0]) & {v - 1 for v in hot}:
            continue
        fillers.append(x)
    xs = [v for v, k in hot.items() for _ in range(k)] + fillers
    rng.shuffle(xs)
    return xs


# (entries of the hot bucket, chunks it makes at cap 16): a bucket at the light / heavy edge (32 | 33 chunks), a full chunk and a full
# chunk plus a length-1 chunk, and k_combine_heavy's loop over chunks for one trip (256) and two (257)
HEAVY_EDGES = [(512, 32), (513, 33), (16, 1), (17, 2), (4096, 256), (4097, 257)]


@pytest.mark.gpu
@pytest.mark.parametrize("count,chunks", HEAVY_EDGES)
def test_heavy_bucket_edges(gpu, count, chunks):
    from ezkl_b200 import halo2 as h2
    c, value = 16, 1000 + count
    xs = hot_column({value: count}, 600, seed=count)
    n = len(xs)
    assert msm_plan(n, 1, c, 1, sm_count())["cap"] == 16
    cnt = bucket_counts(xs, c, 1)
    assert cnt[value - 1] == count and -(-cnt[value - 1] // 16) == chunks
    assert int((-(-cnt // 16) > HEAVY_CHUNKS).sum()) == (1 if chunks > HEAVY_CHUNKS else 0)    # this bucket is the only heavy one, or none is
    sc = H.fr_array(xs)
    bases_np = orc.gen_bases(n, seed=3000 + count)
    b = h2.Bases(bases_np, window_bits=c)
    got = jac_to_affine(h2.best_multiexp(sc, b))[0]
    b.release()
    assert np.array_equal(got, orc.msm(sc, bases_np, THREADS)), (count, chunks)


@pytest.mark.gpu
def test_forty_heavy_buckets(gpu):
    """40 heavy buckets in one column, more than k_combine_heavy's 32 CTAs: its grid-stride loop over the heavy list takes a second
    round.  Their sizes differ (513 .. 1100 entries), so a bucket summed into another's slot shows."""
    from ezkl_b200 import halo2 as h2
    c = 16
    hot = {2000 + 37 * i: 513 + 15 * i for i in range(40)}
    xs = hot_column(hot, 500, seed=40)
    n = len(xs)
    p = msm_plan(n, 1, c, 1, sm_count())
    assert p["cap"] == 16 and p["heavy_stride"] - 1 >= 40
    cnt = bucket_counts(xs, c, 1)
    assert int((-(-cnt // 16) > HEAVY_CHUNKS).sum()) == 40
    sc = H.fr_array(xs)
    bases_np = orc.gen_bases(n, seed=4040)
    b = h2.Bases(bases_np, window_bits=c)
    got = jac_to_affine(h2.best_multiexp(sc, b))[0]
    b.release()
    assert np.array_equal(got, orc.msm(sc, bases_np, THREADS))


def skewed(cnt):
    """k_scan_buckets' rule: a column takes the warp-aggregated scatter when its largest bucket exceeds 16 x (its mean share + 1)."""
    return int(cnt.max()) > 16 * (int(cnt.sum()) // cnt.size + 1)


@pytest.mark.gpu
@pytest.mark.parametrize("c,levels", [(17, None), (16, 8)])
def test_skew_threshold(gpu, c, levels):
    """Global-atomic recoding (c = 17; c = 16 with s = 2 bucket sets): one column whose largest bucket sits exactly at the skew threshold
    (plain scatter) and one with a single entry more (aggregated scatter), in one batch, both against the oracle."""
    from ezkl_b200 import halo2 as h2
    n = 3000
    bases_np = orc.gen_bases(n, seed=5000 + c)
    b = h2.Bases(bases_np, window_bits=c, max_table_bytes=0 if levels is None else levels * n * 64)
    s = b.info()["windows_per_level"]
    assert s == (1 if levels is None else 2)
    assert msm_plan(n, 2, c, s, sm_count())["tile"] == 0
    half = 1 << (c - 1)
    cols, flags = [], []
    for extra in (0, 1):
        rng = random.Random(10 * c + extra)
        xs = [rng.randrange(pyref.R) for _ in range(n)]
        cnt = bucket_counts(xs, c, s)
        hot = int(np.argmin(cnt[:half])) + 1           # an empty bucket of the first set; the scalar `hot` is one entry of it
        assert cnt[hot - 1] == 0
        k = 16 * (int(cnt.sum()) // cnt.size + 1) + extra
        xs = [hot] * k + xs[k:]
        cnt = bucket_counts(xs, c, s)
        assert int(cnt.max()) == int(cnt[hot - 1]) == 16 * (int(cnt.sum()) // cnt.size + 1) + extra
        flags.append(skewed(cnt))
        cols.append(H.fr_array(xs))
    assert flags == [False, True]
    got = jac_to_affine(h2.best_multiexp_batch(cols, b))
    b.release()
    for j in range(2):
        assert np.array_equal(got[j], orc.msm(cols[j], bases_np, THREADS)), (c, levels, j)


@pytest.mark.gpu
@pytest.mark.parametrize("c,levels", [(8, None), (10, 3), (17, None)])
def test_plus_minus_p_accumulation(gpu, c, levels):
    """Bases that are only P and -P: equal scalars (every chunk and bucket sum passes through the identity, the total is 0 or +-xP) and
    mixed ones (sums pass through 2P and doubling), on full and reduced tables; against the oracle and against [sum e_i s_i] P."""
    from ezkl_b200 import halo2 as h2
    n = 3000
    P = orc.gen_bases(1, seed=77)[0]
    x, y = H.g1_unwire(P)
    negP = H.g1_wire((x, pyref.P - y))
    rng = random.Random(c)
    signs = [1 if i % 2 == 0 else -1 for i in range(n - 200)] + [rng.choice((1, -1)) for _ in range(200)]
    bases_np = np.stack([P if e > 0 else negP for e in signs])
    b = h2.Bases(bases_np, window_bits=c, max_table_bytes=0 if levels is None else levels * n * 64)
    v = rng.randrange(pyref.R)
    cols = {
        "equal": [v] * n,
        "equal_balanced": [v] * (n - 200) + [0] * 200,                    # the alternating part cancels exactly: the identity
        "mixed": [rng.randrange(pyref.R) for _ in range(n)],
        "few_values": [(3, pyref.R - 3, 1 << 200)[i % 3] for i in range(n)],
    }
    arrs = [H.fr_array(xs) for xs in cols.values()]
    got = jac_to_affine(h2.best_multiexp_batch(arrs, b))
    b.release()
    for (name, xs), arr, g in zip(cols.items(), arrs, got):
        k = sum(e * s for e, s in zip(signs, xs)) % pyref.R
        want = orc.g1_scalar_mul(P.reshape(1, 8), H.fr_wire(k).reshape(1, 4))[0]
        assert np.array_equal(g, want), (name, c, levels)
        assert np.array_equal(g, orc.msm(arr, bases_np, THREADS)), (name, c, levels)
    assert not got[1].any()


def msm_dev_strided(b, cols, stride):
    """b200_msm_batch_dev over columns laid out `stride` scalars apart (the gap holds other values), normalised; and its launch count."""
    from ezkl_b200 import device as dev
    import torch
    batch, n = cols.shape[0], cols.shape[1]
    buf = orc.gen_scalars(batch * stride, seed=stride).reshape(batch, stride, 4)
    buf[:, :n] = cols
    d_sc = dev.from_host(np.ascontiguousarray(buf))
    out = torch.empty((batch, 16), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    l0 = nat.launch_count()
    nat.check(nat.lib().b200_msm_batch_dev(b.handle, d_sc.data_ptr(), n, stride, batch, out.data_ptr(), dev._stream()))
    torch.cuda.synchronize()
    return jac_to_affine(dev.normalize(out)), nat.launch_count() - l0


# (window bits, table budget in bytes or 0 for the full table, batch): one past msm_dev_on's 4096-column split on a full table, and
# one past its 65535 / s split on a one-level c = 4 table (s = 64: 1023 columns per msm_run)
CLAMP_CASES = [(8, 0, 4097), (4, 1, 65535 // 64 + 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("c,budget,batch", CLAMP_CASES)
def test_batch_clamps(gpu, c, budget, batch):
    from ezkl_b200 import halo2 as h2
    n = 3
    bases_np = orc.gen_bases(n, seed=6000 + c)
    b = h2.Bases(bases_np, window_bits=c, max_table_bytes=budget)
    s = b.info()["windows_per_level"]
    assert s == (64 if budget else 1)
    per_run = min(4096, 65535 // s)
    assert batch == per_run + 1
    cols = orc.gen_scalars(n * batch, seed=6100 + c).reshape(batch, n, 4)
    want = np.stack([orc.msm(col, bases_np, 1) for col in cols])
    got_host = jac_to_affine(h2.best_multiexp_batch(list(cols), b))
    _, one = msm_dev_strided(b, cols[:1], n + 2)
    got_dev, launches = msm_dev_strided(b, cols, n + 2)
    b.release()
    assert launches == 2 * one, (launches, one)                       # two msm_run calls: per_run columns, then one
    bad = [j for j in range(batch) if not (np.array_equal(got_host[j], want[j]) and np.array_equal(got_dev[j], want[j]))]
    assert not bad, bad[:10]


@pytest.mark.gpu
def test_window_bits_outside_4_to_24_rejected(gpu):
    """Registration takes window_bits 0 (automatic) or 4..24; 3 and 25 fail with -1 and say why, and leave no table behind."""
    bases_np = orc.gen_bases(16, seed=7)
    pts = np.ascontiguousarray(bases_np)
    for wb in (3, 25):
        h = C.c_uint64(0)
        assert nat.lib().b200_bases_register_ex(nat.ptr(pts), 16, wb, 0, C.byref(h)) == -1, wb
        assert "window_bits %d" % wb in nat.lib().b200_last_error().decode()
        assert h.value == 0


@pytest.mark.gpu
def test_entry_index_limit_rejected(gpu):
    """L * n must stay below 2^31 (an entry carries a 31-bit table index and a sign bit): 2^25 points at c = 4 with all 64 levels
    (L * n = 2^31) are refused with -1 before the table is allocated."""
    import torch
    n = 1 << 25
    d_pts = torch.empty((n, 8), dtype=torch.int64, device="cuda")      # never read: the check precedes the allocation and the copy
    h = C.c_uint64(0)
    assert nat.lib().b200_bases_register_ex_dev(d_pts.data_ptr(), n, 4, 1 << 50, C.byref(h)) == -1
    assert "31-bit" in nat.lib().b200_last_error().decode()
    assert h.value == 0
    del d_pts
    torch.cuda.empty_cache()
