"""Column kernels (poly.cu, lookup.cu, the evaluate_h interpreter in quotient.cu) against plain references, from one element to 2^24.

What each group is built to reach:
  * scans / evaluation / kate division: chunk (16) and tile (4096) edges, 1024 vs 1025 block values (one carry thread handles one block value,
    then several), a clipped last carry thread, kate's n - 1 shifting each edge by one; strided batches and in-place scans;
  * element-wise kernels: sizes on both sides of the grid clamp (SM count * 16 blocks of 256), so the grid-stride loop takes a second trip;
  * batch inversion: zero patterns around the 64-element chunks that share one inversion;
  * multiplicities: every capacity edge, absent cells mixed with present ones inside a warp, keys that all hash to one probe chain;
  * the interpreter: hand-assembled programs for every opcode and operand kind (the instruction set is the ABI, not what the Python compiler
    happens to emit), every slot-file size, wrapping rotations, the shared-memory limit and every validation branch.
The references are the C oracle (serial, exact), big-integer arithmetic from the definitions at sampled indices, and closed forms (a column of
ones, a root of unity) that do not go through the oracle at all.  Everything is compared bit for bit.
"""
import ctypes as C
import random

import numpy as np
import pytest

from ezkl_b200 import _native as nat
from oracle import oracle as orc
from oracle import pyref
from tests import helpers as H

gpu_test = pytest.mark.gpu
R = pyref.R
CHUNK, TILE, INV_CHUNK = 16, 4096, 64
THREADS = orc.host_threads()
ZERO = np.zeros(4, np.uint64)
ONE = orc.fr_one()


@pytest.fixture(scope="module")
def gpu():
    nat.init(-1)
    yield


# ---- the device calls under test: thin wrappers over the C ABI on resident tensors ---------------------------------------------------------
def _dev():
    from ezkl_b200 import device
    return device


def up(a):
    return _dev().from_host(np.ascontiguousarray(a, np.uint64))


def down(t):
    return _dev().to_host(t)


def sm_count() -> int:
    import torch
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _p(t):
    return nat.dev(t.data_ptr()) if t is not None else None


def g_scan(t_a, init, product, inplace=False):
    d = _dev()
    return d.prefix_scan(t_a, init, product, out=t_a if inplace else None)


def g_scan_batch(t_a, a_stride, n, batch, inits, product, t_out, out_stride) -> int:
    iv = np.ascontiguousarray(inits, np.uint64)
    return nat.lib().b200_prefix_scan_batch_dev(C.c_int(int(product)), _p(t_a), C.c_size_t(a_stride), C.c_size_t(n), C.c_size_t(batch), nat.ptr(iv), _p(t_out),
                                                C.c_size_t(out_stride), _dev()._stream())


def g_eval(t_polys, stride, n, xs, batch) -> np.ndarray:
    import torch
    xs = np.ascontiguousarray(xs, np.uint64).reshape(batch, 4)
    out = torch.zeros((batch, 4), dtype=torch.int64, device="cuda")
    nat.check(nat.lib().b200_poly_eval_batch_dev(_p(t_polys), C.c_size_t(stride), C.c_size_t(n), nat.ptr(xs), C.c_size_t(batch), _p(out), _dev()._stream()))
    return down(out)


def g_kate(t_a, b):
    return _dev().kate_division(t_a, b)


def g_poly_op(op, t_a, t_b=None, s=None, out=None):
    return _dev().poly_op(op, t_a, t_b, s, out)


def g_lincomb(ts, scalars, n):
    out = up(orc.gen_scalars(n, seed=77))                     # not zeros: count = 0 has to overwrite it
    ptrs = (C.c_void_p * max(1, len(ts)))(*[t.data_ptr() for t in ts])
    sc = np.ascontiguousarray(scalars, np.uint64).reshape(-1, 4)
    nat.check(nat.lib().b200_poly_lincomb_dev(ptrs if ts else None, nat.ptr(sc) if ts else None, C.c_size_t(len(ts)), C.c_size_t(n), _p(out), _dev()._stream()))
    return out


def g_scale_cycle(t_a, consts):
    return _dev().scale_cycle(t_a, consts)


def g_invert(t_a):
    return _dev().batch_invert(t_a)


def g_lookup(t_table, n_table, t_inputs, n_rows, want_missing=True):
    import torch
    m = up(orc.gen_scalars(n_table, seed=78))
    ptrs = (C.c_void_p * len(t_inputs))(*[t.data_ptr() for t in t_inputs])
    missing = C.c_uint64(0xDEAD)
    nat.check(nat.lib().b200_lookup_multiplicities_dev(_p(t_table), C.c_size_t(n_table), ptrs, C.c_size_t(len(t_inputs)), C.c_size_t(n_rows), _p(m),
                                                       C.byref(missing) if want_missing else None, _dev()._stream()))
    torch.cuda.synchronize()
    return m, (missing.value if want_missing else None)


def h_lookup(table, inputs, n_rows, want_missing=True):
    """b200_lookup_multiplicities on host arrays"""
    table, cols = np.ascontiguousarray(table), [np.ascontiguousarray(c) for c in inputs]
    m = np.zeros((table.shape[0], 4), np.uint64)
    missing = C.c_uint64(0xDEAD)
    nat.check(nat.lib().b200_lookup_multiplicities(nat.ptr(table), C.c_size_t(table.shape[0]), nat.ptr_array(cols), C.c_size_t(len(cols)), C.c_size_t(n_rows), nat.ptr(m),
                                                   C.byref(missing) if want_missing else None))
    return m, (missing.value if want_missing else None)


def g_quotient(t_cols, k, ext_k, loads, consts, prog, t_out=None, n_columns=None):
    """Raw b200_quotient_eval_dev: returns (rc, out tensor)."""
    import torch
    loads, consts, prog = _program_arrays(loads, consts, prog)
    if t_out is None:
        t_out = torch.zeros((1 << ext_k, 4), dtype=torch.int64, device="cuda")
    ptrs = (C.c_void_p * max(1, len(t_cols)))(*[t.data_ptr() for t in t_cols])
    rc = nat.lib().b200_quotient_eval_dev(ptrs, C.c_size_t(len(t_cols) if n_columns is None else n_columns), C.c_uint32(k), C.c_uint32(ext_k),
                                          loads.ctypes.data_as(C.c_void_p), C.c_size_t(loads.shape[0]), nat.ptr(consts) if consts.size else None,
                                          C.c_size_t(consts.shape[0]), prog.ctypes.data_as(C.c_void_p), C.c_size_t(prog.shape[0]), _p(t_out), _dev()._stream())
    return rc, t_out


def _program_arrays(loads, consts, prog):
    loads = np.ascontiguousarray(np.asarray(loads, dtype=np.int64).reshape(-1, 2).astype(np.int32))
    consts = np.ascontiguousarray(np.asarray(consts, dtype=np.uint64).reshape(-1, 4))
    prog = np.ascontiguousarray(np.asarray(prog, dtype=np.int64).reshape(-1, 4).astype(np.uint32))
    return loads, consts, prog


# ---- comparison helpers ---------------------------------------------------------------------------------------------------------------
def assert_same(got, exp, what, tile=TILE, chunk=CHUNK):
    """Bit-exact comparison of two columns; on failure names the first differing element by the coordinates the kernels work in."""
    got, exp = np.asarray(got, np.uint64).reshape(-1, 4), np.asarray(exp, np.uint64).reshape(-1, 4)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    if np.array_equal(got, exp):
        return
    bad = np.flatnonzero((got != exp).any(axis=1))
    i, j = int(bad[0]), int(bad[-1])
    pytest.fail("%s: %d of %d elements differ; first at %d (tile %d, thread %d, element %d of its chunk; carry group of 1024: %d), last at %d"
                % (what, bad.size, got.shape[0], i, i // tile, (i % tile) // chunk, i % chunk, i // tile // 1024, j))


def mont_sum(a) -> int:
    """Big-integer sum of wire elements, reduced: the wire integer of their field sum (Montgomery form is linear)."""
    a = np.asarray(a, np.uint64).reshape(-1, 4)
    lo = (a & np.uint64(0xFFFFFFFF)).sum(axis=0, dtype=np.uint64)
    hi = (a >> np.uint64(32)).sum(axis=0, dtype=np.uint64)
    return sum((int(lo[l]) + (int(hi[l]) << 32)) << (64 * l) for l in range(4)) % R


def eval_at_small_root(a, log_order: int) -> int:
    """a(w) for w of order 2^log_order, from the definition: sum_r w^r * (sum of the coefficients with index = r mod order)."""
    order, w = 1 << log_order, pyref.omega_for(log_order)
    return sum(pow(w, r, R) * pyref.from_mont(mont_sum(a[r::order]), R) for r in range(order)) % R


def counting_column(n: int, start: int) -> np.ndarray:
    """wire form of start, start + 1, ..., start + n - 1"""
    c = np.zeros((n, 4), np.uint64)
    c[:, 0] = np.arange(start, start + n, dtype=np.uint64)
    return orc.fr_to_mont(c)


def edge_indices(n: int):
    cand = [0, CHUNK, TILE, TILE * 1024, TILE * 1025, (n // 2) // TILE * TILE, (n - 1) // TILE * TILE, n - 1]
    return sorted({i for i in cand if 0 <= i < n})


def check_scan_spans(a, got, product, what):
    """got[hi] == got[lo] (*|+) a[lo .. hi-1] in big integers, on short spans laid across chunk, tile and carry-group edges."""
    n = a.shape[0]
    for i in edge_indices(n):
        lo, hi = max(i - 20, 0), min(i + 20, n - 1)
        acc = H.fr_unwire(got[lo])
        for v in H.fr_list(a[lo:hi]):
            acc = acc * v % R if product else (acc + v) % R
        assert acc == H.fr_unwire(got[hi]), "%s: span [%d, %d] around %d disagrees with big-integer arithmetic" % (what, lo, hi, i)


def check_kate_spans(a, b_int, q, what):
    """q[lo] == sum_{lo <= f < hi} a[f+1] b^(f-lo) + b^(hi-lo) q[hi], and the top coefficient q[m-1] == a[m]."""
    m = a.shape[0] - 1
    assert np.array_equal(q[m - 1], a[m]), what
    for i in edge_indices(m):
        lo, hi = max(i - 20, 0), min(i + 20, m - 1)
        acc = H.fr_unwire(q[hi])
        for v in reversed(H.fr_list(a[lo + 1:hi + 1])):
            acc = (acc * b_int + v) % R
        assert acc == H.fr_unwire(q[lo]), "%s: span [%d, %d] around %d disagrees with big-integer arithmetic" % (what, lo, hi, i)


# ---- 1. scans, evaluation, kate division over the size ladder ------------------------------------------------------------------------------
SIZES = [1, 2, 15, 16, 17, 4095, 4096, 4097, 2 * 4096 + 1, 1 << 20, 1 << 22, (1 << 22) + 1, (1 << 22) + 2, (1 << 22) + 4096 + 5, 1 << 23,
         3 * (1 << 22) + 7, 1 << 24]


@gpu_test
@pytest.mark.parametrize("n", SIZES)
def test_scan_eval_kate_sizes(gpu, n):
    a = orc.gen_scalars(n, seed=1000 + n % 9973)
    t_a = up(a)
    init = orc.gen_scalars(1, seed=11)[0]
    for product in (False, True):
        got = down(g_scan(t_a, init, product))
        assert_same(got, orc.prefix_scan(a, init, product), "prefix_scan(product=%s, n=%d)" % (product, n))
        check_scan_spans(a, got, product, "prefix_scan(product=%s, n=%d)" % (product, n))
    # closed forms that do not involve the oracle's scan: 5 + i, and init * g^i with g of order TILE (so the column has period TILE)
    ones = up(np.tile(ONE, (n, 1)))
    assert_same(down(g_scan(ones, H.fr_wire(5), False)), counting_column(n, 5), "running sum of ones, n=%d" % n)
    g = orc.omega(12)
    period = orc.prefix_scan(np.tile(g, (min(n, TILE), 1)), init, True)
    got = down(g_scan(up(np.tile(g, (n, 1))), init, True))
    assert_same(got, np.resize(period, (n, 4)), "running product of a root of unity of order 4096, n=%d" % n)
    del ones

    # evaluation: x random, x of order 16 (x^CHUNK = 1) and of order 4096 (x^TILE = 1), 0 and 1
    xs = [orc.gen_scalars(1, seed=12)[0], orc.omega(4), orc.omega(12), ZERO, ONE]
    for i, x in enumerate(xs):
        got = g_eval(t_a, n, n, x, 1)[0]
        assert np.array_equal(got, orc.eval_polynomial(a, x)), "eval_polynomial n=%d x#%d" % (n, i)
    assert H.fr_unwire(g_eval(t_a, n, n, orc.omega(4), 1)[0]) == eval_at_small_root(a, 4), "eval at a 16th root of unity vs the definition, n=%d" % n
    assert np.array_equal(g_eval(t_a, n, n, ZERO, 1)[0], a[0]) and H.limbs_to_int(g_eval(t_a, n, n, ONE, 1)[0]) == mont_sum(a), n

    # kate division: b random, 0, 1, and of order 4096
    if n == 1:
        return                                                    # a constant has an empty quotient (test_argument_boundaries)
    for i, b in enumerate([orc.gen_scalars(1, seed=13)[0], ZERO, ONE, orc.omega(12)]):
        q = down(g_kate(t_a, b))
        assert_same(q, orc.kate_division(a, b), "kate_division n=%d b#%d" % (n, i))
        check_kate_spans(a, H.fr_unwire(b), q, "kate_division n=%d b#%d" % (n, i))
        if i == 1:
            assert_same(q, a[1:], "kate_division by X, n=%d" % n)


@gpu_test
@pytest.mark.parametrize("n", [17, 4097, (1 << 22) + 2])
def test_scan_eval_kate_host_pointers(gpu, n):
    from ezkl_b200 import halo2 as h2
    a = orc.gen_scalars(n, seed=1100 + n % 9973)
    init, x = orc.gen_scalars(2, seed=14)
    for product in (False, True):
        assert_same(h2.prefix_scan(a, init, product), orc.prefix_scan(a, init, product), "b200_prefix_scan(product=%s, n=%d)" % (product, n))
    for xx in (x, orc.omega(12)):
        assert np.array_equal(h2.eval_polynomial(a, xx), orc.eval_polynomial(a, xx)), n
        assert_same(h2.kate_division(a, xx), orc.kate_division(a, xx), "b200_kate_division n=%d" % n)


# ---- 2. batched and strided calls, in place ----------------------------------------------------------------------------------------------------
@gpu_test
# batch 9000: 9000 scan initial values (32 B each) and 9000 evaluation parameter sets (96 B each) are both larger than one 256 KiB
# slot of the parameter staging ring (StagingRing::SLOT), so both go through its overflow buffer
@pytest.mark.parametrize("n,batch", [(5000, 1), (5000, 3), (5000, 7), ((1 << 22) + 4096 + 5, 3), (5, 9000)])
def test_scan_and_eval_batched(gpu, n, batch):
    a_stride, out_stride = n + 3, n + 7
    cols = [orc.gen_scalars(n, seed=2000 + 10 * batch + p) for p in range(batch)]
    pad = H.fr_wire(0xBADC0FFEE)
    flat = np.tile(pad, (batch * a_stride, 1))
    for p in range(batch):
        flat[p * a_stride:p * a_stride + n] = cols[p]
    inits = orc.gen_scalars(batch, seed=2100 + batch)
    t_src = up(flat)
    for product in (False, True):
        exp = [orc.prefix_scan(cols[p], inits[p], product) for p in range(batch)]
        t_out = up(np.tile(pad, (batch * out_stride, 1)))
        nat.check(g_scan_batch(t_src, a_stride, n, batch, inits, product, t_out, out_stride))
        got = down(t_out)
        for p in range(batch):
            assert_same(got[p * out_stride:p * out_stride + n], exp[p], "batched scan(product=%s) column %d of %d, n=%d" % (product, p, batch, n))
            assert (got[p * out_stride + n:(p + 1) * out_stride] == pad).all(), "batched scan wrote into the padding after column %d" % p
        assert np.array_equal(down(t_src), flat), "batched scan changed its input"
        # in place: the result replaces the column, the padding between columns stays
        t_io = up(flat)
        nat.check(g_scan_batch(t_io, a_stride, n, batch, inits, product, t_io, a_stride))
        got = down(t_io)
        for p in range(batch):
            assert_same(got[p * a_stride:p * a_stride + n], exp[p], "in-place batched scan(product=%s) column %d of %d, n=%d" % (product, p, batch, n))
            assert (got[p * a_stride + n:(p + 1) * a_stride] == pad).all(), p
        del t_io, t_out
    # single-column entry point in place
    t_one = up(cols[0])
    assert_same(down(g_scan(t_one, inits[0], True, inplace=True)), orc.prefix_scan(cols[0], inits[0], True), "in-place prefix_scan n=%d" % n)
    # evaluation with stride > n: a distinct point per polynomial, 0 and 1 among them; the padding must not be read as coefficients
    xs = orc.gen_scalars(batch, seed=2200)
    xs[0] = ZERO
    xs[-1] = ONE
    got = g_eval(t_src, a_stride, n, xs, batch)
    for p in range(batch):
        assert np.array_equal(got[p], orc.eval_polynomial(cols[p], xs[p])), "eval_batch stride > n: polynomial %d of %d, n=%d" % (p, batch, n)


# ---- 3. element-wise kernels on both sides of the grid clamp ----------------------------------------------------------------------------------
def _ew_sizes():
    # resolved at run time (the clamp is SM count * 16 blocks of 256 threads); the ids stay the same on every device
    return ["1", "255", "256", "257", "clamp-1", "clamp", "clamp+1", "2^22+3"]


def _ew_n(tag: str) -> int:
    clamp = sm_count() * 16 * 256
    return {"clamp-1": clamp - 1, "clamp": clamp, "clamp+1": clamp + 1, "2^22+3": (1 << 22) + 3}.get(tag) or int(tag)


@gpu_test
@pytest.mark.parametrize("size", _ew_sizes())
def test_elementwise_grid_stride(gpu, size):
    n = _ew_n(size)
    a, b = orc.gen_scalars(n, seed=3001), orc.gen_scalars(n, seed=3002)
    s = orc.gen_scalars(1, seed=3003)[0]
    t_a, t_b = up(a), up(b)
    for op in ("add", "sub", "mul", "scale", "axpy"):
        needs_b, needs_s = op != "scale", op in ("scale", "axpy")
        got = down(g_poly_op(op, t_a, t_b if needs_b else None, s if needs_s else None))
        assert_same(got, orc.poly_op(op, a, b if needs_b else None, s if needs_s else None, THREADS), "poly_op %s n=%d" % (op, n), tile=256, chunk=1)
    # aliasing: out is b; a, b and out all one buffer
    t = up(b)
    assert_same(down(g_poly_op("sub", t_a, t, out=t)), orc.poly_op("sub", a, b, threads=THREADS), "poly_op sub, out is b, n=%d" % n, tile=256, chunk=1)
    t = up(b)
    assert_same(down(g_poly_op("axpy", t_a, t, s, out=t)), orc.poly_op("axpy", a, b, s, THREADS), "poly_op axpy, out is b, n=%d" % n, tile=256, chunk=1)
    for op in ("mul", "add"):
        t = up(a)
        assert_same(down(g_poly_op(op, t, t, out=t)), orc.poly_op(op, a, a, threads=THREADS), "poly_op %s, a is b is out, n=%d" % (op, n), tile=256, chunk=1)
    assert np.array_equal(down(t_a), a) and np.array_equal(down(t_b), b), "poly_op changed an input it was not given as out"

    # linear combinations: 0 terms (zeros), 1, 7, 40; the 40 pointers cycle over 5 columns, which sums their scalars per column
    pool = [a, b] + [orc.gen_scalars(n, seed=3010 + i) for i in range(3)]
    t_pool = [t_a, t_b] + [up(p) for p in pool[2:]]
    for count in (0, 1, 7, 40):
        sc = orc.gen_scalars(max(count, 1), seed=3020 + count)[:count]
        got = down(g_lincomb([t_pool[j % 5] for j in range(count)], sc, n))
        exp = np.zeros((n, 4), np.uint64)
        for c in range(min(count, 5)):
            exp = orc.poly_op("axpy", exp, pool[c], H.fr_wire(sum(H.fr_unwire(sc[j]) for j in range(c, count, 5))), THREADS)
        assert_same(got, exp, "lincomb of %d terms, n=%d" % (count, n), tile=256, chunk=1)
    del t_pool
    # 7000 distinct columns, the windows [j, j + n) of one tensor: the pointer table and scalars, 40 B per term, are larger than one
    # 256 KiB slot of the parameter staging ring (StagingRing::SLOT holds at most 6552 terms), so they go through its overflow buffer
    if n <= 257:
        count = 7000
        window = orc.gen_scalars(count + n - 1, seed=3030)
        sc = orc.gen_scalars(count, seed=3031)
        t_window = up(window)
        got = down(g_lincomb([t_window[j:j + n] for j in range(count)], sc, n))
        exp = np.zeros((n, 4), np.uint64)
        for j in range(count):
            exp = orc.poly_op("axpy", exp, window[j:j + n], sc[j])
        assert_same(got, exp, "lincomb of %d distinct columns, n=%d" % (count, n), tile=256, chunk=1)
        del t_window

    # cyclic constants: the product with the constants repeated down the column
    for period in (1, 2, 3, 8, 1024):
        consts = orc.gen_scalars(period, seed=3100 + period)
        got = down(g_scale_cycle(up(a), consts))
        assert_same(got, orc.poly_op("mul", a, np.resize(consts, (n, 4)), threads=THREADS), "scale_cycle period %d, n=%d" % (period, n), tile=256, chunk=1)


# ---- 4. batch inversion ---------------------------------------------------------------------------------------------------------------------------
def _zero_patterns(n):
    mid = (n // INV_CHUNK // 2) * INV_CHUNK
    yield "none", np.zeros(n, bool)
    yield "all", np.ones(n, bool)
    one = np.ones(n, bool)
    one[n // 3] = False
    yield "one non-zero", one
    chunk = np.zeros(n, bool)
    chunk[mid:mid + INV_CHUNK] = True
    yield "a whole chunk", chunk
    ends = np.zeros(n, bool)
    ends[[mid, min(mid + INV_CHUNK - 1, n - 1), 0, n - 1]] = True
    yield "chunk ends", ends
    yield "every other", np.arange(n) % 2 == 0


@gpu_test
@pytest.mark.parametrize("n", [1, 63, 64, 65, 128 * 64, 128 * 64 + 1, (1 << 20) + 3])
def test_batch_invert_patterns(gpu, n):
    base = orc.gen_scalars(n, seed=4000 + n % 9973)
    for name, zeros in _zero_patterns(n):
        a = base.copy()
        a[zeros] = 0
        t = up(a)
        got = down(g_invert(t))
        assert_same(got, orc.batch_invert(a), "batch_invert n=%d zeros: %s" % (n, name), tile=128 * INV_CHUNK, chunk=INV_CHUNK)
        assert not got[zeros].any(), "zeros stay zero (%s)" % name
        prod = down(g_poly_op("mul", t, up(a)))
        assert (prod[~zeros] == ONE).all() and not prod[zeros].any(), "a * a^-1 == 1 on the non-zeros, n=%d zeros: %s" % (n, name)
    for i in {0, n // 2, n - 1}:
        assert H.fr_unwire(got[i]) == (pow(H.fr_unwire(a[i]), -1, R) if a[i].any() else 0), i


# ---- 5-7. mv-lookup multiplicities ---------------------------------------------------------------------------------------------------------------
def multiplicity_reference(table_ids, input_ids):
    """first-row map {value -> smallest table row}, one count per input cell; cells whose value is not in the table are counted as missing.
    Values are given by integer id (equal id <=> equal field element)."""
    uniq, first = np.unique(np.asarray(table_ids), return_index=True)      # np.unique returns the first occurrence
    cells = np.concatenate([np.asarray(c).reshape(-1) for c in input_ids]) if len(input_ids) else np.zeros(0, np.int64)
    pos = np.searchsorted(uniq, cells)
    pos[pos == uniq.size] = 0
    present = uniq[pos] == cells if cells.size else np.zeros(0, bool)
    counts = np.bincount(first[pos[present]], minlength=len(table_ids))
    m = np.zeros((len(table_ids), 4), np.uint64)
    m[:, 0] = counts
    return orc.fr_to_mont(m), int((~present).sum())


def run_lookup(pool, table_ids, input_ids, n_rows, host=False, want_missing=True):
    table = pool[np.asarray(table_ids)]
    ins = [pool[np.asarray(c)] if n_rows else pool[:1] for c in input_ids]
    exp_m, exp_missing = multiplicity_reference(table_ids, [c[:n_rows] for c in input_ids])
    if host:
        got_m, got_missing = h_lookup(table, ins, n_rows, want_missing)
    else:
        t_m, got_missing = g_lookup(up(table), len(table_ids), [up(c) for c in ins], n_rows, want_missing)
        got_m = down(t_m)
    return got_m, got_missing, exp_m, exp_missing


# (64, 5, 32769): the table of 32769 input pointers (8 B each) is 8 B larger than one 256 KiB slot of the parameter staging ring
# (StagingRing::SLOT), so it goes through the ring's overflow buffer
LOOKUP_SHAPES = [(1, 100, 1), (32, 1000, 2), (33, 1000, 2), (4096, 0, 1), (1 << 16, 1 << 16, 4), (1 << 12, (1 << 20) + 17, 3), (1 << 20, 1 << 20, 2),
                 (64, 5, 32769)]


@gpu_test
@pytest.mark.parametrize("n_table,n_rows,n_inputs", LOOKUP_SHAPES)
def test_multiplicities_shapes(gpu, n_table, n_rows, n_inputs):
    rng = np.random.default_rng(5000 + n_table + n_rows)
    pool = orc.gen_scalars(n_table, seed=5001)                                          # full-width, pairwise distinct field elements
    distinct = np.arange(n_table)
    repeated = np.minimum(distinct, max(n_table * 3 // 4 - 1, 0))                       # the last quarter repeats one row: the first gets the count
    rows = max(n_rows, 1)
    dists = {
        "uniform": (distinct, [rng.integers(0, n_table, rows) for _ in range(n_inputs)]),
        "every cell equal": (distinct, [np.full(rows, n_table // 2) for _ in range(n_inputs)]),
        "exponential skew": (distinct, [np.minimum(rng.exponential(50.0, rows).astype(np.int64), n_table - 1) for _ in range(n_inputs)]),
        "repeated table rows": (repeated, [rng.integers(0, n_table, rows) for _ in range(n_inputs)]),
    }
    for name, (t_ids, in_ids) in dists.items():
        in_ids = [t_ids[c] for c in in_ids]                                              # every cell is a table value
        for host in ((False, True) if (n_table, n_rows) in ((33, 1000), (1 << 16, 1 << 16)) else (False,)):
            got_m, got_missing, exp_m, exp_missing = run_lookup(pool, t_ids, in_ids, n_rows, host=host)
            what = "multiplicities %s, table %d, %d x %d cells, %s" % (name, n_table, n_inputs, n_rows, "host pointers" if host else "device")
            assert exp_missing == 0 and got_missing == 0, what
            assert_same(got_m, exp_m, what, tile=256, chunk=32)
            assert mont_sum(got_m) == H.limbs_to_int(H.fr_wire(n_inputs * n_rows)), what


@gpu_test
@pytest.mark.parametrize("n_rows", [32 * 40 + 13, (1 << 19) + 77])
def test_multiplicities_missing_cells(gpu, n_rows):
    """Cells absent from the table, by warp: none, all 32, the odd lanes, one lane, and a ragged last warp; few distinct present values
    per warp so that present lanes share counters while their neighbours are absent."""
    n_table = 1000
    pool = orc.gen_scalars(2 * n_table, seed=5101)                                      # ids >= n_table are not in the table
    rng = np.random.default_rng(5102)
    lane, warp = np.arange(n_rows) % 32, np.arange(n_rows) // 32
    cols = []
    for shift in (0, 2):
        kind = (warp + shift) % 5
        absent = (kind == 1) | ((kind == 2) & (lane % 2 == 1)) | ((kind == 3) & (lane == 7)) | ((kind == 4) & (lane % 3 == 0))
        ids = (warp * 7 + rng.integers(0, 4, n_rows)) % n_table                           # four distinct present values per warp
        ids[absent] = n_table + rng.integers(0, n_table, int(absent.sum()))
        cols.append(ids)
    for want_missing in (True, False):
        got_m, got_missing, exp_m, exp_missing = run_lookup(pool, np.arange(n_table), cols, n_rows, want_missing=want_missing)
        assert exp_missing > n_rows // 4
        assert_same(got_m, exp_m, "multiplicities with absent cells, %d rows, missing %s" % (n_rows, "read" if want_missing else "NULL"), tile=256, chunk=32)
        assert got_missing == (exp_missing if want_missing else None), (got_missing, exp_missing)
    got_m, got_missing, exp_m, exp_missing = run_lookup(pool, np.arange(n_table), [np.arange(n_rows) % n_table + n_table], n_rows)
    assert got_missing == n_rows == exp_missing and not got_m.any(), "every cell absent"


def colliding_keys(count: int, shared: int) -> np.ndarray:
    """Raw field elements (below the modulus: the top 32-bit limb stays under 2^28) that agree in 32-bit limbs 0, 1, 3 and 6 and differ in
    2, 4, 5 and 7.  The function only compares elements, so any bytes below the modulus are valid input."""
    i = np.arange(count, dtype=np.uint64)
    s = np.uint64(shared)
    k = np.zeros((count, 4), np.uint64)
    k[:, 0] = s | ((s * np.uint64(3) & np.uint64(0xFFFFFFFF)) << np.uint64(32))                             # limbs 0, 1 shared
    k[:, 1] = (i * np.uint64(2654435761) & np.uint64(0xFFFFFFFF)) | ((s ^ np.uint64(0x5555)) << np.uint64(32))   # limb 2 varies, limb 3 shared
    k[:, 2] = (i >> np.uint64(3)) | ((i & np.uint64(7)) << np.uint64(32))                                   # limbs 4, 5 vary
    k[:, 3] = (s + np.uint64(9)) | ((i % np.uint64(1 << 28)) << np.uint64(32))                              # limb 6 shared, limb 7 varies
    return k


@gpu_test
def test_multiplicities_colliding_keys(gpu):
    rng = np.random.default_rng(5200)
    # ~2000 distinct keys in one probe chain, each present 8 times in the table (the smallest row takes the count)
    pool = colliding_keys(2000, 0x1234567)
    t_ids = rng.permutation(np.repeat(np.arange(256), 8))                                # 2048 rows, 256 values x 8
    got_m, got_missing, exp_m, exp_missing = run_lookup(pool, t_ids, [rng.integers(0, 256, 5000), rng.integers(0, 2000, 5000)], 5000)
    assert_same(got_m, exp_m, "256 colliding keys x 8 rows each", tile=256, chunk=32)
    assert got_missing == exp_missing > 0
    t_ids = rng.permutation(2000)
    t_ids = np.concatenate([t_ids, t_ids[:48]])                                          # 2048 rows, one chain of 2000 distinct keys
    got_m, got_missing, exp_m, exp_missing = run_lookup(pool, t_ids, [rng.integers(0, 2000, 20000)], 20000)
    assert_same(got_m, exp_m, "2000 colliding keys in one chain", tile=256, chunk=32)
    assert got_missing == exp_missing == 0
    # 32-row tables (64 slots): one chain of 32 per table, starting wherever the shared limbs hash to, so some chains wrap past slot 63
    for shared in range(1, 25):
        pool = colliding_keys(40, shared * 0x01010101 & 0x0FFFFFFF)
        got_m, got_missing, exp_m, exp_missing = run_lookup(pool, rng.permutation(32), [rng.integers(0, 40, 500)], 500)
        assert_same(got_m, exp_m, "32 colliding keys, 64 slots, shared limbs #%d" % shared, tile=256, chunk=32)
        assert got_missing == exp_missing


# ---- 8-9. the evaluate_h interpreter: the instruction set of include/ezkl_b200.h ----------------------------------------------------------------
SLOT, CONST, LOAD, PREV = 0, 1, 2, 3
ADD, SUB, MUL, NEG, DOUBLE, SQUARE, MOV, MULADD = range(8)
NOSTORE = 1 << 31
N_COLS = 3


def src(kind, index=0):
    return (kind << 30) | index


def ins(op, dst, a, b=0, c=0, store=True):
    return [op | (dst << 8) | (0 if store else NOSTORE), a, b, c]


def fold(prog, slots):
    """appends a Horner chain over the given slots, so that the row result depends on every one of them, in order"""
    prog.append(ins(MOV, 0, src(SLOT, slots[0]), store=False))
    for s in slots[1:]:
        prog.append(ins(MULADD, 0, src(PREV), src(CONST, 0), src(SLOT, s), store=False))
    return prog


def bigint_interpreter(columns, k, ext_k, loads, consts, prog, rows):
    """The instruction set as include/ezkl_b200.h describes it, on Python integers.  columns[c](j) -> int; returns {row: value}."""
    n_ext, step, out = 1 << ext_k, 1 << (ext_k - k), {}
    for idx in rows:
        slots, prev = {}, 0

        def operand(s):
            kind, index = s >> 30, s & 0x3FFFFFFF
            if kind == SLOT:
                return slots[index]
            if kind == CONST:
                return consts[index]
            if kind == LOAD:
                column, rotation = loads[index]
                return columns[column]((idx + rotation * step) % n_ext)
            return prev
        for op_dst, a, b, c in prog:
            op, dst = op_dst & 0xFF, (op_dst >> 8) & 0xFFFF
            x = operand(a)
            if op == ADD:
                r = x + operand(b)
            elif op == SUB:
                r = x - operand(b)
            elif op == MUL:
                r = x * operand(b)
            elif op == NEG:
                r = -x
            elif op == DOUBLE:
                r = 2 * x
            elif op == SQUARE:
                r = x * x
            elif op == MOV:
                r = x
            else:
                assert op == MULADD
                r = x * operand(b) + operand(c)
            prev = r % R
            if not op_dst & NOSTORE:
                slots[dst] = prev
        out[idx] = prev
    return out


def rotations(k):
    n = 1 << k
    return [0, 1, -1, n - 1, -(n - 1), n, -n, n + 1, -(n + 1), (1 << 31) - 1, -(1 << 31)]


def hand_programs(k, ext_k):
    """(name, loads, constants, program): every opcode with every operand kind in every position, PREV / no-store chains, every slot-file
    size and its edges, wrapping rotations.  Loads 0..3 and constants 0..5 are shared by all of them."""
    loads = [(0, 0), (1, 1), (2, -1), (0, 2)]
    consts = orc.gen_scalars(6, seed=8000)
    kinds = (SLOT, CONST, LOAD, PREV)
    operand = {SLOT: src(SLOT, 1), CONST: src(CONST, 2), LOAD: src(LOAD, 1), PREV: src(PREV)}
    preamble = [ins(MOV, 0, src(LOAD, 0)), ins(MOV, 1, src(CONST, 1))]
    out = [("empty", loads, consts, []), ("one instruction, not stored", loads, consts, [ins(DOUBLE, 0, src(LOAD, 1), store=False)]),
           ("one instruction, stored", loads, consts, [ins(MOV, 0, src(CONST, 0))])]
    for op, name in ((ADD, "add"), (SUB, "sub"), (MUL, "mul")):
        prog = list(preamble)
        for i, (ka, kb) in enumerate((ka, kb) for ka in kinds for kb in kinds):
            prog.append(ins(op, 2 + i, operand[ka] if ka != SLOT else src(SLOT, 0), operand[kb]))
        out.append((name + " x operand kinds", loads, consts, fold(prog, list(range(2, 18)))))
    prog = list(preamble)
    for i, (ka, kb, kc) in enumerate((ka, kb, kc) for ka in kinds for kb in kinds for kc in kinds):
        prog.append(ins(MULADD, 2 + i, operand[ka] if ka != SLOT else src(SLOT, 0), operand[kb], operand[kc] if kc != LOAD else src(LOAD, 3)))
    out.append(("muladd x operand kinds", loads, consts, fold(prog, list(range(2, 66)))))
    for op, name in ((NEG, "neg"), (DOUBLE, "double"), (SQUARE, "square"), (MOV, "mov")):
        prog = list(preamble)
        for i, ka in enumerate(kinds):
            prog.append(ins(op, 2 + i, operand[ka]))
        out.append((name + " x operand kinds", loads, consts, fold(prog, [2, 3, 4, 5])))
    out.append(("previous-result chains", loads, consts, [
        ins(MOV, 3, src(LOAD, 0)),
        ins(MUL, 3, src(LOAD, 1), src(CONST, 0), store=False),             # not stored: slot 3 keeps the load although dst says 3
        ins(ADD, 4, src(PREV), src(SLOT, 3)),                              # PREV consumed by a stored instruction
        ins(SQUARE, 5, src(PREV)),                                         # a stored result that is also read as PREV
        ins(SUB, 6, src(SLOT, 4), src(PREV)),
        ins(DOUBLE, 0, src(PREV), store=False),
        ins(MULADD, 7, src(PREV), src(PREV), src(PREV)),
        ins(NEG, 0, src(SLOT, 3), store=False),
        ins(MULADD, 0, src(PREV), src(SLOT, 7), src(SLOT, 5), store=False),
        ins(SUB, 0, src(PREV), src(SLOT, 6), store=False)]))
    for top in (31, 32, 63, 64, 127, 128, 255):
        regs = []
        for s in (top, top & 127, top & 63, top & 31, 0):                # registers a smaller slot file would fold onto one another
            if s not in regs:
                regs.append(s)
        prog = [ins(MUL, s, src(LOAD, i % 4), src(CONST, 1 + i)) for i, s in enumerate(regs)]
        out.append(("highest slot %d" % top, loads, consts, fold(prog, regs)))
        out.append(("highest slot %d written before slot 0" % top, loads, consts,
                    [ins(MOV, top, src(LOAD, 1)), ins(MOV, 0, src(LOAD, 2)), ins(ADD, 0, src(SLOT, 0), src(CONST, 1), store=False),
                     ins(MULADD, 0, src(PREV), src(SLOT, top), src(SLOT, 0), store=False)]))
    rot_loads = [(c, r) for r in rotations(k) for c in (0, 1)]
    prog = [ins(MOV, 0, src(LOAD, 0), store=False)] + [ins(MULADD, 0, src(PREV), src(CONST, 0), src(LOAD, i), store=False) for i in range(1, len(rot_loads))]
    out.append(("one column at every rotation", rot_loads, consts, prog))
    return out


def random_program(rng: random.Random, k, max_instr=300, n_instr=None):
    """A random program at the instruction level (not from an expression tree): any opcode, any operand kind that is defined at that point."""
    n_loads, n_consts = rng.randint(1, 12), rng.randint(1, 8)
    loads = [(rng.randrange(N_COLS), rng.choice(rotations(k) + list(range(-3, 4)))) for _ in range(n_loads)]
    top = rng.choice([5, 31, 32, 63, 64, 127, 128, 255])
    written, prog = [], []
    for pc in range(n_instr or rng.randint(1, max_instr)):
        def operand():
            kind = rng.choice([CONST, LOAD] + ([SLOT] * 2 if written else []) + ([PREV] * 2 if pc else []))
            return src(kind, {SLOT: lambda: rng.choice(written), CONST: lambda: rng.randrange(n_consts), LOAD: lambda: rng.randrange(n_loads), PREV: lambda: 0}[kind]())
        a, b, c = operand(), operand(), operand()
        store, dst = rng.random() < 0.7, rng.randint(0, top)
        prog.append(ins(rng.randrange(8), dst, a, b, c, store))
        if store and dst not in written:
            written.append(dst)
    return loads, orc.gen_scalars(n_consts, seed=rng.randrange(1 << 30)), prog


GEOMETRIES = [(3, 3), (3, 5), (4, 6), (10, 13)]


def programs_for(k, ext_k, n_random=50):
    rng = random.Random(8100 + 100 * k + ext_k)
    return hand_programs(k, ext_k) + [("random #%d" % i,) + random_program(rng, k) for i in range(n_random)]


def test_program_catalogue_covers_the_instruction_set():
    """The hand-assembled programs use every opcode with every operand kind in every position it has."""
    seen = set()
    for _, _, _, prog in hand_programs(3, 5):
        for op_dst, a, b, c in prog:
            op = op_dst & 0xFF
            for pos, s in enumerate((a, b, c)[:3 if op == MULADD else (2 if op <= MUL else 1)]):
                seen.add((op, pos, s >> 30))
    want = {(op, pos, kind) for op in range(8) for pos in range(3 if op == MULADD else (2 if op <= MUL else 1)) for kind in range(4)}
    assert want <= seen, sorted(want - seen)


@pytest.mark.parametrize("k,ext_k", GEOMETRIES)
def test_instruction_set_oracle_vs_bigint(k, ext_k):
    """The C oracle's interpreter against the big-integer one written from the header, on every hand-assembled and random program: the
    oracle is then a valid reference for opcodes and operand kinds the Python compiler never emits."""
    n_ext = 1 << ext_k
    cols = [orc.gen_scalars(n_ext, seed=8200 + c) for c in range(N_COLS)]
    rows = list(range(n_ext)) if n_ext <= 64 else [0, 1, 2, n_ext // 2 - 1, n_ext // 2, n_ext - 3, n_ext - 2, n_ext - 1]
    memo = [{} for _ in cols]

    def column(c):
        def at(j):
            if j not in memo[c]:
                memo[c][j] = H.fr_unwire(cols[c][j])
            return memo[c][j]
        return at
    for name, loads, consts, prog in programs_for(k, ext_k):
        l_, c_, p_ = _program_arrays(loads, consts, prog)
        got = orc.quotient_eval(cols, k, ext_k, l_, c_, p_, threads=THREADS)
        exp = bigint_interpreter([column(c) for c in range(N_COLS)], k, ext_k, loads, H.fr_list(consts), prog, rows)
        for idx in rows:
            assert H.fr_unwire(got[idx]) == exp[idx], "%s at (k, ext_k) = (%d, %d), row %d" % (name, k, ext_k, idx)


@gpu_test
@pytest.mark.parametrize("k,ext_k", GEOMETRIES)
def test_interpreter_instruction_set(gpu, k, ext_k):
    n_ext = 1 << ext_k
    cols = [orc.gen_scalars(n_ext, seed=8200 + c) for c in range(N_COLS)]
    t_cols = [up(c) for c in cols]
    for name, loads, consts, prog in programs_for(k, ext_k):
        rc, t_out = g_quotient(t_cols, k, ext_k, loads, consts, prog)
        nat.check(rc)
        l_, c_, p_ = _program_arrays(loads, consts, prog)
        assert_same(down(t_out), orc.quotient_eval(cols, k, ext_k, l_, c_, p_, threads=THREADS), "%s at (k, ext_k) = (%d, %d)" % (name, k, ext_k), tile=128, chunk=1)


@gpu_test
@pytest.mark.parametrize("k,ext_k", [(3, 5), (10, 13)])
def test_interpreter_host_pointers(gpu, k, ext_k):
    n_ext = 1 << ext_k
    cols = [orc.gen_scalars(n_ext, seed=8200 + c) for c in range(N_COLS)]
    for name, loads, consts, prog in hand_programs(k, ext_k)[:6]:
        l_, c_, p_ = _program_arrays(loads, consts, prog)
        out = np.full((n_ext, 4), 7, np.uint64)
        nat.check(nat.lib().b200_quotient_eval(nat.ptr_array(cols), C.c_size_t(N_COLS), C.c_uint32(k), C.c_uint32(ext_k), l_.ctypes.data_as(C.c_void_p), C.c_size_t(l_.shape[0]),
                                               nat.ptr(c_), C.c_size_t(c_.shape[0]), p_.ctypes.data_as(C.c_void_p), C.c_size_t(p_.shape[0]), nat.ptr(out)))
        assert_same(out, orc.quotient_eval(cols, k, ext_k, l_, c_, p_, threads=THREADS), "b200_quotient_eval: %s" % name, tile=128, chunk=1)


@gpu_test
def test_interpreter_large_grid(gpu):
    k, ext_k = 20, 22
    cols = [orc.gen_scalars(1 << ext_k, seed=8300 + c) for c in range(N_COLS)]
    loads, consts, prog = random_program(random.Random(8301), k, n_instr=40)
    rc, t_out = g_quotient([up(c) for c in cols], k, ext_k, loads, consts, prog)
    nat.check(rc)
    l_, c_, p_ = _program_arrays(loads, consts, prog)
    assert_same(down(t_out), orc.quotient_eval(cols, k, ext_k, l_, c_, p_, threads=THREADS), "40 instructions at ext_k = 22", tile=128, chunk=1)


def _horner_program(n_instr, n_loads, n_consts):
    prog = [ins(MOV, 0, src(LOAD, 0), store=False)]
    for i in range(1, n_instr):
        prog.append(ins(MULADD, 0, src(PREV), src(LOAD, i % n_loads), src(CONST, (i * 7) % n_consts if i < n_instr - 1 else n_consts - 1), store=False))
    return prog


@gpu_test
def test_interpreter_program_limits(gpu):
    """The staged program (16 B per instruction and per load, 32 B per constant, 16 B of padding) may take 160 KB: the largest one evaluates
    correctly, one instruction more is refused with a message that says what to do; every validation failure returns -1, launches nothing
    and leaves the output alone."""
    k, ext_k, limit = 6, 8, 160 * 1024
    n_ext = 1 << ext_k
    cols = [orc.gen_scalars(n_ext, seed=8400 + c) for c in range(N_COLS)]
    t_cols = [up(c) for c in cols]
    loads = [(0, 0), (1, -1), (2, 5)]
    for n_consts in (2, 2560):                                      # instruction-heavy, and with the constants reaching the end of the stage
        consts = orc.gen_scalars(n_consts, seed=8410)
        n_instr = (limit - 16 - 16 * len(loads) - 32 * n_consts) // 16
        assert 16 * n_instr + 16 * len(loads) + 32 * n_consts + 16 == limit
        prog = _horner_program(n_instr, len(loads), n_consts)
        rc, t_out = g_quotient(t_cols, k, ext_k, loads, consts, prog)
        nat.check(rc)
        l_, c_, p_ = _program_arrays(loads, consts, prog)
        assert_same(down(t_out), orc.quotient_eval(cols, k, ext_k, l_, c_, p_, threads=THREADS), "largest program, %d constants" % n_consts, tile=128, chunk=1)
        sentinel = orc.gen_scalars(n_ext, seed=8420)
        before = nat.launch_count()
        rc, t_out = g_quotient(t_cols, k, ext_k, loads, consts, prog + [ins(MOV, 0, src(PREV), store=False)], t_out=up(sentinel))
        msg = nat.lib().b200_last_error().decode()
        assert rc == -1 and "split" in msg, (rc, msg)
        assert nat.launch_count() == before and np.array_equal(down(t_out), sentinel)

    consts = orc.gen_scalars(2, seed=8430)
    ok = [ins(MOV, 0, src(LOAD, 0)), ins(ADD, 1, src(SLOT, 0), src(CONST, 1))]
    bad = {
        "opcode 8": dict(prog=ok + [ins(8, 0, src(SLOT, 0))]),
        "opcode 255": dict(prog=ok + [ins(255, 0, src(SLOT, 0))]),
        "destination slot 256": dict(prog=ok + [ins(ADD, 256, src(SLOT, 0), src(SLOT, 1))]),
        "destination slot 256, not stored": dict(prog=ok + [ins(ADD, 256, src(SLOT, 0), src(SLOT, 1), store=False)]),
        "operand slot 256": dict(prog=ok + [ins(ADD, 2, src(SLOT, 256), src(SLOT, 1))]),
        "constant index == n_constants": dict(prog=ok + [ins(ADD, 2, src(SLOT, 0), src(CONST, 2))]),
        "load index == n_loads": dict(prog=ok + [ins(MUL, 2, src(LOAD, 3), src(SLOT, 1))]),
        "third operand of muladd out of range": dict(prog=ok + [ins(MULADD, 2, src(SLOT, 0), src(SLOT, 1), src(CONST, 9))]),
        "PREV in the first instruction": dict(prog=[ins(NEG, 0, src(PREV))] + ok),
        "load column == n_columns": dict(loads=loads + [(N_COLS, 0)]),
        "load column beyond the columns passed": dict(n_columns=2),
        "ext_k < k": dict(k=ext_k + 1),
        "ext_k 29": dict(ext_k=29, k=29),
        "ext_k 0": dict(ext_k=0, k=0),
    }
    sentinel = orc.gen_scalars(n_ext, seed=8440)
    for name, change in bad.items():
        args = dict(k=k, ext_k=ext_k, loads=loads, consts=consts, prog=ok, n_columns=None)
        args.update(change)
        t_out = up(sentinel)
        before = nat.launch_count()
        rc, _ = g_quotient(t_cols, args["k"], args["ext_k"], args["loads"], args["consts"], args["prog"], t_out=t_out, n_columns=args["n_columns"])
        msg = nat.lib().b200_last_error().decode()
        assert rc == -1 and "quotient_eval" in msg, (name, rc, msg)
        assert nat.launch_count() == before, name
        assert np.array_equal(down(t_out), sentinel), name
    rc, t_out = g_quotient(t_cols, k, ext_k, loads, consts, ok)      # ... and the program they were all derived from is accepted
    nat.check(rc)
    l_, c_, p_ = _program_arrays(loads, consts, ok)
    assert_same(down(t_out), orc.quotient_eval(cols, k, ext_k, l_, c_, p_), "the valid base program", tile=128, chunk=1)


# ---- 10. argument checks: -1 on the host, nothing launched, nothing written ------------------------------------------------------------------------
class _Env:
    """Small valid buffers: a call that got past a missing check would compute something and change `out`, not touch memory it does not own."""

    def __init__(self):
        import torch
        self.h_a, self.h_b, self.h_out = orc.gen_scalars(16, seed=9001), orc.gen_scalars(16, seed=9002), orc.gen_scalars(16, seed=9003)
        self.a, self.b, self.out = up(self.h_a), up(self.h_b), up(self.h_out)
        self.big_in = torch.zeros((65536, 4), dtype=torch.int64, device="cuda")
        self.big_out = torch.zeros((65536, 4), dtype=torch.int64, device="cuda")
        self.s = orc.gen_scalars(1, seed=9004)
        self.many = orc.gen_scalars(65536, seed=9005)
        self.ptrs1 = (C.c_void_p * 1)(self.a.data_ptr())
        self.ptrs2 = (C.c_void_p * 2)(self.a.data_ptr(), self.b.data_ptr())
        self.ptrs_many = (C.c_void_p * 65536)(*([self.a.data_ptr()] * 65536))
        self.missing = C.c_uint64(0)
        self.host_q = np.zeros((16, 4), np.uint64)
        self.st = _dev()._stream()


def _sz(v):
    return C.c_size_t(v)


BAD_CALLS = {
    "poly_op_5": lambda L, e: L.b200_poly_op_dev(5, _p(e.a), _p(e.b), nat.ptr(e.s), _p(e.out), _sz(16), e.st),
    "poly_op_negative": lambda L, e: L.b200_poly_op_dev(-1, _p(e.a), _p(e.b), nat.ptr(e.s), _p(e.out), _sz(16), e.st),
    "poly_op_null_a": lambda L, e: L.b200_poly_op_dev(0, None, _p(e.b), None, _p(e.out), _sz(16), e.st),
    "poly_op_null_out": lambda L, e: L.b200_poly_op_dev(0, _p(e.a), _p(e.b), None, None, _sz(16), e.st),
    "poly_op_add_null_b": lambda L, e: L.b200_poly_op_dev(0, _p(e.a), None, None, _p(e.out), _sz(16), e.st),
    "poly_op_scale_null_s": lambda L, e: L.b200_poly_op_dev(3, _p(e.a), None, None, _p(e.out), _sz(16), e.st),
    "poly_op_axpy_null_s": lambda L, e: L.b200_poly_op_dev(4, _p(e.a), _p(e.b), None, _p(e.out), _sz(16), e.st),
    "lincomb_null_out": lambda L, e: L.b200_poly_lincomb_dev(e.ptrs2, nat.ptr(e.many), _sz(2), _sz(16), None, e.st),
    "lincomb_null_polys": lambda L, e: L.b200_poly_lincomb_dev(None, nat.ptr(e.many), _sz(2), _sz(16), _p(e.out), e.st),
    "lincomb_null_scalars": lambda L, e: L.b200_poly_lincomb_dev(e.ptrs2, None, _sz(2), _sz(16), _p(e.out), e.st),
    "scale_cycle_period_0": lambda L, e: L.b200_poly_scale_cycle_dev(_p(e.out), _sz(16), nat.ptr(e.many), C.c_uint32(0), e.st),
    "scale_cycle_period_1025": lambda L, e: L.b200_poly_scale_cycle_dev(_p(e.out), _sz(16), nat.ptr(e.many), C.c_uint32(1025), e.st),
    "scale_cycle_null_consts": lambda L, e: L.b200_poly_scale_cycle_dev(_p(e.out), _sz(16), None, C.c_uint32(2), e.st),
    "eval_batch_65536": lambda L, e: L.b200_poly_eval_batch_dev(_p(e.big_in), _sz(1), _sz(1), nat.ptr(e.many), _sz(65536), _p(e.big_out), e.st),
    "eval_null_x": lambda L, e: L.b200_poly_eval_batch_dev(_p(e.a), _sz(16), _sz(16), None, _sz(1), _p(e.out), e.st),
    "eval_null_out": lambda L, e: L.b200_poly_eval_batch_dev(_p(e.a), _sz(16), _sz(16), nat.ptr(e.many), _sz(1), None, e.st),
    "batch_invert_null": lambda L, e: L.b200_batch_invert_dev(None, _sz(16), e.st),
    "scan_batch_65536": lambda L, e: L.b200_prefix_scan_batch_dev(1, _p(e.big_in), _sz(1), _sz(1), _sz(65536), nat.ptr(e.many), _p(e.big_out), _sz(1), e.st),
    "scan_a_stride_below_n": lambda L, e: L.b200_prefix_scan_batch_dev(0, _p(e.a), _sz(7), _sz(8), _sz(2), nat.ptr(e.many), _p(e.out), _sz(8), e.st),
    "scan_out_stride_below_n": lambda L, e: L.b200_prefix_scan_batch_dev(0, _p(e.a), _sz(8), _sz(8), _sz(2), nat.ptr(e.many), _p(e.out), _sz(7), e.st),
    "scan_null_init": lambda L, e: L.b200_prefix_scan_dev(0, _p(e.a), _sz(16), None, _p(e.out), e.st),
    "scan_null_out": lambda L, e: L.b200_prefix_scan_dev(0, _p(e.a), _sz(16), nat.ptr(e.s), None, e.st),
    "kate_n_0": lambda L, e: L.b200_kate_division_dev(_p(e.a), _sz(0), nat.ptr(e.s), _p(e.out), e.st),
    "kate_null_b": lambda L, e: L.b200_kate_division_dev(_p(e.a), _sz(16), None, _p(e.out), e.st),
    "kate_in_place": lambda L, e: L.b200_kate_division_dev(_p(e.out), _sz(16), nat.ptr(e.s), _p(e.out), e.st),
    "lookup_n_table_0": lambda L, e: L.b200_lookup_multiplicities_dev(_p(e.b), _sz(0), e.ptrs1, _sz(1), _sz(16), _p(e.out), C.byref(e.missing), e.st),
    "lookup_n_inputs_0": lambda L, e: L.b200_lookup_multiplicities_dev(_p(e.b), _sz(16), e.ptrs1, _sz(0), _sz(16), _p(e.out), C.byref(e.missing), e.st),
    "lookup_n_inputs_65536": lambda L, e: L.b200_lookup_multiplicities_dev(_p(e.b), _sz(16), e.ptrs_many, _sz(65536), _sz(16), _p(e.out), C.byref(e.missing), e.st),
    "lookup_null_table": lambda L, e: L.b200_lookup_multiplicities_dev(None, _sz(16), e.ptrs1, _sz(1), _sz(16), _p(e.out), C.byref(e.missing), e.st),
    "lookup_null_inputs": lambda L, e: L.b200_lookup_multiplicities_dev(_p(e.b), _sz(16), None, _sz(1), _sz(16), _p(e.out), C.byref(e.missing), e.st),
    "lookup_null_m": lambda L, e: L.b200_lookup_multiplicities_dev(_p(e.b), _sz(16), e.ptrs1, _sz(1), _sz(16), None, C.byref(e.missing), e.st),
    "host_poly_op_null_a": lambda L, e: L.b200_poly_op(0, None, nat.ptr(e.h_b), None, nat.ptr(e.host_q), _sz(16)),
    "host_poly_op_5": lambda L, e: L.b200_poly_op(5, nat.ptr(e.h_a), nat.ptr(e.h_b), nat.ptr(e.s), nat.ptr(e.host_q), _sz(16)),
    "host_scale_cycle_period_1025": lambda L, e: L.b200_poly_scale_cycle(nat.ptr(e.host_q), _sz(16), nat.ptr(e.many), C.c_uint32(1025)),
    "host_kate_n_0": lambda L, e: L.b200_kate_division(nat.ptr(e.h_a), _sz(0), nat.ptr(e.s), nat.ptr(e.host_q)),
    "host_lookup_n_table_0": lambda L, e: L.b200_lookup_multiplicities(nat.ptr(e.h_b), _sz(0), nat.ptr_array([e.h_a]), _sz(1), _sz(16), nat.ptr(e.host_q), C.byref(e.missing)),
    "host_lookup_n_inputs_0": lambda L, e: L.b200_lookup_multiplicities(nat.ptr(e.h_b), _sz(16), nat.ptr_array([e.h_a]), _sz(0), _sz(16), nat.ptr(e.host_q), C.byref(e.missing)),
}


@pytest.fixture(scope="module")
def env(gpu):
    return _Env()


@gpu_test
@pytest.mark.parametrize("case", list(BAD_CALLS))
def test_argument_errors(env, case):
    import torch
    before = nat.launch_count()
    rc = BAD_CALLS[case](nat.lib(), env)
    msg = nat.lib().b200_last_error().decode()
    assert rc == -1 and msg, (case, rc, msg)
    torch.cuda.synchronize()
    assert nat.launch_count() == before, "%s launched a kernel" % case
    assert np.array_equal(down(env.a), env.h_a) and np.array_equal(down(env.b), env.h_b) and np.array_equal(down(env.out), env.h_out), case
    assert not env.host_q.any() and not down(env.big_out).any(), case


@gpu_test
def test_argument_boundaries(env):
    """The limits themselves are accepted: period 1024, 65535 columns of one element, strides with one column, kate division of a constant."""
    L = nat.lib()
    consts = orc.gen_scalars(1024, seed=9100)
    t = up(env.h_a)
    nat.check(L.b200_poly_scale_cycle_dev(_p(t), _sz(16), nat.ptr(consts), C.c_uint32(1024), env.st))
    assert np.array_equal(down(t), orc.poly_op("mul", env.h_a, consts[:16]))
    col = orc.gen_scalars(65535, seed=9101)
    t_col, t_out = up(col), up(np.zeros((65535, 4), np.uint64))
    nat.check(L.b200_prefix_scan_batch_dev(1, _p(t_col), _sz(1), _sz(1), _sz(65535), nat.ptr(env.many), _p(t_out), _sz(1), env.st))
    assert np.array_equal(down(t_out), env.many[:65535])                                 # one-element columns: the result is the initial value
    assert np.array_equal(g_eval(t_col, 1, 1, env.many[:65535], 65535), col)             # ... and a constant polynomial evaluates to itself
    t_out = up(env.h_out)
    nat.check(L.b200_prefix_scan_batch_dev(0, _p(env.a), _sz(0), _sz(16), _sz(1), nat.ptr(env.s), _p(t_out), _sz(0), env.st))    # strides are unused with one column
    assert np.array_equal(down(t_out), orc.prefix_scan(env.h_a, env.s[0], False))
