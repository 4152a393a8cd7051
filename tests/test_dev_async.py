"""The _dev entry points with many calls in flight, against the C oracle.

include/ezkl_b200.h promises that a _dev call does not synchronise, that its host parameters are read only during the call, that one
thread's scratch is ordered across the streams it alternates between, and that a thread's scratch is released when it exits.  Each
test here queues work behind a bounded torch.cuda._sleep on a stream (a "hold", about 200 ms), issues its calls while the stream is
still held, asserts that the hold was still running after the last call (so the calls really queued; the scratch-growth test can
assert it only for its first call, see there), and then compares every output with the oracle, bit for bit:

  ring wrap            more than three laps of the 96-slot staging ring with value-only parameter blobs, every host parameter
                       array overwritten with random words as soon as its call returns;
  staging, queued      every entry point that stages a blob, mixed, on one held stream; then blobs larger than a ring slot
                       (the overflow path) between ring calls on two streams;
  MSM                  a column stride larger than the column on both recoding paths and on a reduced table, and scratch
                       that grows while earlier MSMs are still queued;
  stream switching     one thread round-robin over three gated torch streams and the library stream; b200_sync;
  two threads          the bench's two-stream pattern, a new transform size first used by two threads at once, and a thread
                       that exits with work queued;
  bench schedule       bench.py's two-stream and one-stream schedules write the same outputs.

The CPU-tier catalogue test keeps this list complete: every _dev prototype of the header is exercised here or excluded
with a reason.
"""
import ctypes as C
import glob
import json
import os
import random
import re
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np
import pytest

from ezkl_b200 import _native as nat
from oracle import oracle as orc
from oracle import pyref
from tests import helpers as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = pyref.R
THREADS = orc.host_threads()
gpu = pytest.mark.gpu

# ---- the catalogue: which test exercises each device-pointer entry point, and why the others are not here --------------------------
EXERCISED = {
    "b200_poly_scale_cycle_dev": "test_ring_wrap_value_blobs",
    "b200_prefix_scan_dev": "test_ring_wrap_value_blobs",
    "b200_prefix_scan_batch_dev": "test_ring_wrap_value_blobs",
    "b200_kate_division_dev": "test_ring_wrap_value_blobs",
    "b200_poly_lincomb_dev": "test_every_staging_entry_point_queued",
    "b200_poly_eval_batch_dev": "test_every_staging_entry_point_queued",
    "b200_quotient_eval_dev": "test_every_staging_entry_point_queued",
    "b200_evaluate_h_dev": "test_every_staging_entry_point_queued",
    "b200_lookup_multiplicities_dev": "test_every_staging_entry_point_queued",
    "b200_ntt_dev": "test_every_staging_entry_point_queued",
    "b200_poly_op_dev": "test_every_staging_entry_point_queued",
    "b200_batch_invert_dev": "test_every_staging_entry_point_queued",
    "b200_g1_fft_dev": "test_every_staging_entry_point_queued",
    "b200_dev_upload_async": "test_every_staging_entry_point_queued",
    "b200_msm_batch_dev": "test_msm_column_stride",
}
EXCLUDED = {
    "b200_msm_sharded_dev": "needs two or more devices (tests/test_multi_device.py)",
    "b200_ntt_sharded_dev": "needs two or more devices (tests/test_multi_device.py)",
    "b200_bases_register_dev": "synchronises: the table is built before the call returns",
    "b200_bases_register_ex_dev": "synchronises: the table is built before the call returns",
    "b200_g1_sum_dev": "stages no parameters and uses no per-thread scratch: it reads only its arguments (tests/test_field_curve_layer.py)",
    "b200_g1_fixed_base_mul_dev": "stages no parameters and uses no per-thread scratch: it reads only its arguments (tests/test_field_curve_layer.py)",
    "b200_g1_generate_dev": "stages no parameters and uses no per-thread scratch: it writes only its output (tests/test_field_curve_layer.py)",
    "b200_permutation_sigmas_dev": "key generation, run once per key and not among a proof's queued calls; its one launch on the caller's stream "
                                   "is checked in tests/test_permutation_keygen.py",
    "b200_dev_alloc": "allocation, nothing is queued",
    "b200_dev_alloc_on": "allocation on a device slot of a multi-device process",
    "b200_dev_free": "release, nothing is queued",
    "b200_dev_upload": "synchronous: the bytes are on the device when it returns",
    "b200_dev_download": "synchronous: the bytes are on the host when it returns",
}


def test_dev_catalogue_is_complete():
    """Every prototype of include/ezkl_b200.h named b200_*_dev or b200_dev_* is exercised by a test of this module or excluded above
    with a reason, so a new device-pointer entry point cannot skip this file."""
    names = {n for n in nat.declarations(nat.HEADER) if re.search(r"_dev$|^b200_dev_", n)}
    assert names, "no _dev prototypes read from the header"
    missing = sorted(names - set(EXERCISED) - set(EXCLUDED))
    assert not missing, "device-pointer entry points neither exercised nor excluded here: %s" % missing
    assert not set(EXERCISED) & set(EXCLUDED)
    stale = sorted((set(EXERCISED) | set(EXCLUDED)) - names)
    assert not stale, "listed but not declared by the header: %s" % stale
    assert all(reason.strip() for reason in EXCLUDED.values())
    src = open(os.path.abspath(__file__)).read()
    for name, test in EXERCISED.items():
        assert callable(globals().get(test)), (name, test)
        # the name is called somewhere below the catalogue, not only listed in it
        assert len(re.findall(r"\b%s\(" % name, src)) >= 1, "%s is listed as exercised by %s but never called" % (name, test)


# ---- holding a stream ----------------------------------------------------------------------------------------------------------------
_CYCLES_PER_MS = None
HOLD_MS = 200


def cycles_per_ms():
    """torch.cuda._sleep cycles per millisecond, measured once with CUDA events.  An idle GPU runs at a lower clock until it has been
    busy for a while, so the rate is measured five times and the highest is kept: a hold is then at least as long as asked for."""
    global _CYCLES_PER_MS
    if _CYCLES_PER_MS is None:
        import torch
        s = torch.cuda.Stream()
        probe, rates = 20_000_000, []
        with torch.cuda.stream(s):
            torch.cuda._sleep(probe // 10)                   # warm the sleep kernel
            for _ in range(5):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(s)
                torch.cuda._sleep(probe)
                e1.record(s)
                e1.synchronize()
                rates.append(probe / max(e0.elapsed_time(e1), 1e-3))
        _CYCLES_PER_MS = max(rates)
    return _CYCLES_PER_MS


def hold(stream, ms=HOLD_MS):
    """Queue a bounded spin of about `ms` milliseconds on `stream`; returns the event recorded after it."""
    import torch
    ev = torch.cuda.Event()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(cycles_per_ms() * ms))
        ev.record(stream)
    return ev


def sptr(stream):
    return stream.cuda_stream or 1 if stream is not None else None


@pytest.fixture(scope="module")
def dev_ctx():
    import torch
    nat.init(-1)
    cycles_per_ms()
    yield
    torch.cuda.synchronize()


# ---- small helpers ---------------------------------------------------------------------------------------------------------------------
def up(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64)).cuda()


def down(t):
    return t.cpu().numpy().view(np.uint64)


def scribble(*arrays):
    """Overwrite host parameter arrays with random words: the caller may reuse them as soon as the call returns."""
    g = np.random.default_rng()
    for a in arrays:
        a.view(np.uint64)[...] = g.integers(0, 2**64, size=a.view(np.uint64).shape, dtype=np.uint64)


def rand_fr(count, rng):
    return H.fr_array([rng.randrange(R) for _ in range(count)])


def fr_small(v):
    return H.fr_wire(v)


def lincomb_ref(cols, scalars):
    acc = np.zeros_like(cols[0])
    for c, s in zip(cols, scalars):
        acc = orc.poly_op("axpy", acc, c, s, threads=THREADS)
    return acc


def scale_cycle_ref(a, consts):
    reps = -(-a.shape[0] // consts.shape[0])
    return orc.poly_op("mul", a, np.ascontiguousarray(np.tile(consts, (reps, 1))[: a.shape[0]]), threads=THREADS)


def ntt_ref(src, log_n, omega, pre, post):
    """dst[j] = post * sum_i pre[i mod 3] src[i] omega^(ij) (pre mode 3, post mode 1), src of 2^log_n elements."""
    return orc.poly_op("scale", orc.best_fft(scale_cycle_ref(src, pre), log_n, omega, threads=THREADS), s=post, threads=THREADS)


def assert_eq(got, want, what):
    got, want = np.asarray(got, np.uint64), np.asarray(want, np.uint64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if not np.array_equal(got, want):
        bad = np.flatnonzero((got.reshape(got.shape[0], -1) != want.reshape(want.shape[0], -1)).any(axis=1))
        pytest.fail("%s: %d of %d rows differ, first at %d" % (what, bad.size, got.shape[0], bad[0]))


# ---- 1. ring wrap with value-only blobs -----------------------------------------------------------------------------------------------
RING_SLOTS = 96
CYCLE_PERIOD = 7
SCAN_BATCH = 4


@gpu
def test_ring_wrap_value_blobs(dev_ctx):
    """On one held stream, 400 calls whose blobs are plain field values (scale_cycle with period 7, prefix scans, a batched scan of 4
    columns, Kate division) at n = 2^12, each with its own output and constants: more than four laps of the staging ring while
    the kernels that read earlier laps' slots are still queued.  Each host parameter array is overwritten with random words as soon
    as its call returns."""
    import torch
    lib = nat.lib()
    n = 1 << 12
    rng = random.Random(11)
    srcs = [orc.gen_scalars(n, seed=100 + i) for i in range(SCAN_BATCH)]
    d_srcs = [up(a) for a in srcs]
    d_batch = up(np.concatenate(srcs))
    calls = 4 * 100
    assert calls >= 3 * RING_SLOTS
    s = torch.cuda.Stream()
    # warm: scratch and the ring reach their sizes before the hold
    with torch.cuda.stream(s):
        w = torch.empty_like(d_batch)
        nat.check(lib.b200_prefix_scan_batch_dev(1, d_batch.data_ptr(), n, n, SCAN_BATCH, nat.ptr(rand_fr(SCAN_BATCH, rng)), w.data_ptr(), n, sptr(s)))
        nat.check(lib.b200_kate_division_dev(d_srcs[0].data_ptr(), n, nat.ptr(rand_fr(1, rng)), w.data_ptr(), sptr(s)))
    s.synchronize()
    outs = [torch.empty_like(d_srcs[0]) for _ in range(calls)]
    for i in range(0, calls, 4):
        outs[i].copy_(d_srcs[i // 4 % SCAN_BATCH])              # scale_cycle runs in place on its own copy
    outs = [o if i % 4 != 2 else torch.empty_like(d_batch) for i, o in enumerate(outs)]
    torch.cuda.synchronize()
    want, laps_queued = [], []
    for i in range(calls):
        if i % RING_SLOTS == 0:
            # a push waits for the copy that last used its slot, so each lap of the ring starts behind a fresh hold: the calls of
            # lap j are queued while the kernels of lap j - 1 that read the same slots are still waiting to run
            hold(s)
        kind, col = i % 4, i // 4 % SCAN_BATCH
        if kind == 0:
            consts = rand_fr(CYCLE_PERIOD, rng)
            want.append(("scale_cycle", lambda col=col, c=consts.copy(): scale_cycle_ref(srcs[col], c)))
            nat.check(lib.b200_poly_scale_cycle_dev(outs[i].data_ptr(), n, nat.ptr(consts), CYCLE_PERIOD, sptr(s)))
            scribble(consts)
        elif kind == 1:
            init, product = rand_fr(1, rng), bool(i % 8 == 1)
            want.append(("prefix_scan", lambda col=col, c=init[0].copy(), p=product: orc.prefix_scan(srcs[col], c, p)))
            nat.check(lib.b200_prefix_scan_dev(int(product), d_srcs[col].data_ptr(), n, nat.ptr(init), outs[i].data_ptr(), sptr(s)))
            scribble(init)
        elif kind == 2:
            inits, product = rand_fr(SCAN_BATCH, rng), bool(i % 8 == 2)
            want.append(("prefix_scan_batch", lambda c=inits.copy(), p=product: np.concatenate([orc.prefix_scan(srcs[j], c[j], p) for j in range(SCAN_BATCH)])))
            nat.check(lib.b200_prefix_scan_batch_dev(int(product), d_batch.data_ptr(), n, n, SCAN_BATCH, nat.ptr(inits), outs[i].data_ptr(), n, sptr(s)))
            scribble(inits)
        else:
            b = rand_fr(1, rng)
            want.append(("kate_division", lambda col=col, c=b[0].copy(): orc.kate_division(srcs[col], c)))
            nat.check(lib.b200_kate_division_dev(d_srcs[col].data_ptr(), n, nat.ptr(b), outs[i].data_ptr(), sptr(s)))
            scribble(b)
        if i % RING_SLOTS == RING_SLOTS - 1 or i == calls - 1:
            laps_queued.append(not s.query())
    assert all(laps_queued), "a lap's hold ended before its last call was issued (%s): lengthen it" % laps_queued
    s.synchronize()
    for i, (what, fn) in enumerate(want):
        w_ = fn()
        got = down(outs[i])[: w_.shape[0]]
        assert_eq(got, w_, "%s, call %d" % (what, i))


# ---- 2. every staging entry point, queued ---------------------------------------------------------------------------------------------
def _dom(k, ext_k):
    from ezkl_b200 import halo2 as h2
    d = h2.EvaluationDomain((1 << (ext_k - k)) + 1, k)
    assert d.extended_k == ext_k
    return d


def _quotient_dev(lib, cols, k, ext_k, loads, consts, instrs, out, st):
    ptrs = (C.c_void_p * len(cols))(*[c.data_ptr() for c in cols])
    return lib.b200_quotient_eval_dev(ptrs, len(cols), k, ext_k, loads.ctypes.data_as(C.c_void_p), loads.shape[0], nat.ptr(consts) if consts.size else None,
                                      consts.shape[0], instrs.ctypes.data_as(C.c_void_p), instrs.shape[0], out.data_ptr(), st)


def _evaluate_h_dev(lib, prog_arrays, cols, dom, t, out, st):
    loads, consts, instrs = prog_arrays
    lens = (C.c_size_t * len(cols))(*[c.shape[0] for c in cols])
    ptrs = (C.c_void_p * len(cols))(*[c.data_ptr() for c in cols])
    return lib.b200_evaluate_h_dev(ptrs, lens, len(cols), dom.k, dom.extended_k, nat.ptr(dom.extended_omega), nat.ptr(dom.g_coset),
                                   loads.ctypes.data_as(C.c_void_p), loads.shape[0], nat.ptr(consts) if consts.size else None, consts.shape[0],
                                   instrs.ctypes.data_as(C.c_void_p), instrs.shape[0], None if t is None else nat.ptr(t), 0 if t is None else t.shape[0],
                                   nat.ptr(dom.extended_omega_inv) if t is not None else None, nat.ptr(dom.extended_ifft_divisor) if t is not None else None,
                                   out.data_ptr(), st)


def _mults(table_n, ptr_cols, input_ids, n_rows):
    """multiplicities of a table of distinct values: input column j holds table indices input_ids[j][:n_rows]"""
    counts = np.zeros(table_n, np.int64)
    for j in ptr_cols:
        np.add.at(counts, input_ids[j][:n_rows], 1)
    return H.fr_array([int(c) for c in counts])


class Staging:
    """Inputs and the per-kind call makers of the queued staging test; each maker issues one call on `st`, overwrites its host parameters
    and returns (label, output tensor, expected)."""

    def __init__(self, rng):
        import torch
        from ezkl_b200 import evaluation as ev
        from tests.evaluate_h_parts_check import program, system
        self.torch, self.lib, self.rng = torch, nat.lib(), rng
        self.keep = []          # device scratch of queued calls: torch must not hand it out again before the stream reaches them
        self.n = n = 1 << 12
        self.pool = [orc.gen_scalars(n, seed=300 + i) for i in range(40)]
        self.d_pool = [up(a) for a in self.pool]
        self.decoy = up(orc.gen_scalars(n, seed=399))
        # eval batch with stride > n
        self.ev_n, self.ev_stride, self.ev_batch = 1000, 1037, 5
        self.ev_polys = orc.gen_scalars(self.ev_stride * self.ev_batch, seed=401).reshape(self.ev_batch, self.ev_stride, 4)
        self.d_ev = up(self.ev_polys.reshape(-1, 4))
        # quotient programs at (k, ext_k) = (8, 10) and evaluate_h at (9, 12)
        self.qk, self.qext = 8, 10
        self.q_cols = [orc.gen_scalars(1 << self.qext, seed=410 + i) for i in range(4)]
        self.d_q = [up(c) for c in self.q_cols]
        self.q_progs = [program(rng, 4, 1 << self.qk, 3).arrays() for _ in range(12)]
        self.dom = _dom(9, 12)
        self.h_polys = system(self.dom, 4242)
        self.d_h = [up(p) for p in self.h_polys]
        self.h_progs = [program(rng, len(self.h_polys), self.dom.n, 3) for _ in range(3)]
        self.h_want = {}
        for i, p in enumerate(self.h_progs):
            for fin in (False, True):
                self.h_want[i, fin] = ev.evaluate_h_from_polys(p, self.h_polys, self.dom, finish=fin)
        # lookup: a table of distinct values and inputs that are table entries
        self.tab_n, self.lk_rows = 512, 300
        self.table = orc.gen_scalars(self.tab_n, seed=420)
        self.d_table = up(self.table)
        self.lk_ids = [np.array([rng.randrange(self.tab_n) for _ in range(self.lk_rows)]) for _ in range(6)]
        self.d_lk = [up(self.table[ids]) for ids in self.lk_ids]
        # ntt
        self.omega = orc.omega(12)
        # pinned upload source
        self.pinned = C.c_void_p()
        nat.check(self.lib.b200_host_alloc(C.byref(self.pinned), 32 * n * 8))
        self.pinned_arr = np.ctypeslib.as_array((C.c_uint64 * (4 * n * 8)).from_address(self.pinned.value)).reshape(8, n, 4)
        self.pinned_next = 0
        # the input pointer table of the overflow lookup, pinned so that the library's copy of it is a real asynchronous DMA
        self.lk_wide = 32769
        self.ptr_pin = C.c_void_p()
        nat.check(self.lib.b200_host_alloc(C.byref(self.ptr_pin), 8 * self.lk_wide))
        self.ptr_arr = np.ctypeslib.as_array((C.c_uint64 * self.lk_wide).from_address(self.ptr_pin.value))
        # g1 fft: [s_i] G in, [scale * DFT(s)_j] G out
        self.g1_log = 7
        g1n = 1 << self.g1_log
        self.g1_s = orc.gen_scalars(g1n, seed=430)
        gen = np.tile(np.concatenate([H.fq_wire(1), H.fq_wire(2)]), (g1n, 1))
        self.g1_gen = gen
        self.d_g1_in = up(orc.g1_scalar_mul(gen, self.g1_s))

    def call(self, make, ts):
        """make(st) on torch stream ts, with every tensor it allocates or fills ordered on ts as well"""
        with self.torch.cuda.stream(ts):
            return make(sptr(ts))

    def out(self, rows):
        return self.torch.full((rows, 4), 3, dtype=self.torch.int64, device="cuda")

    def lincomb_overflow(self, st):
        """7000 terms: the pointer and scalar blob is larger than one ring slot"""
        count = 7000
        idx = [self.rng.randrange(40) for _ in range(count)]
        sc = rand_fr(count, self.rng)
        coef = {}
        for i, v in zip(idx, H.fr_list(sc)):
            coef[i] = (coef.get(i, 0) + v) % R
        want = lambda: lincomb_ref([self.pool[i] for i in coef], H.fr_array(list(coef.values())))
        ptrs = (C.c_void_p * count)(*[self.d_pool[i].data_ptr() for i in idx])
        o = self.out(self.n)
        nat.check(self.lib.b200_poly_lincomb_dev(ptrs, nat.ptr(sc), count, self.n, o.data_ptr(), st))
        scribble(sc)
        for j in range(count):
            ptrs[j] = self.decoy.data_ptr()
        return "lincomb of 7000 (overflow)", o, want

    def lookup_overflow(self, st):
        """32769 input pointers from pinned host memory: the table is larger than one ring slot.  As soon as the call returns the
        pointers are overwritten with pointers to another valid column, so a copy that ran later would count the wrong cells."""
        rows = 64
        cols = [self.rng.randrange(len(self.d_lk)) for _ in range(self.lk_wide)]
        want = lambda: _mults(self.tab_n, cols, self.lk_ids, rows)
        self.ptr_arr[:] = [self.d_lk[j].data_ptr() for j in cols]
        o = self.out(self.tab_n)
        nat.check(self.lib.b200_lookup_multiplicities_dev(self.d_table.data_ptr(), self.tab_n, self.ptr_pin, self.lk_wide, rows, o.data_ptr(), None, st))
        self.ptr_arr[:] = self.d_lk[0].data_ptr()
        return "lookup of %d inputs (overflow)" % self.lk_wide, o, want

    def lincomb(self, st):
        count = self.rng.randint(1, 40)
        idx = [self.rng.randrange(40) for _ in range(count)]
        sc = rand_fr(count, self.rng)
        want = lambda idx=idx, sc=sc.copy(): lincomb_ref([self.pool[i] for i in idx], sc)
        ptrs = (C.c_void_p * count)(*[self.d_pool[i].data_ptr() for i in idx])
        o = self.out(self.n)
        nat.check(self.lib.b200_poly_lincomb_dev(ptrs, nat.ptr(sc), count, self.n, o.data_ptr(), st))
        scribble(sc)
        for j in range(count):
            ptrs[j] = self.decoy.data_ptr()
        return "lincomb of %d" % count, o, want

    def eval_batch(self, st):
        xs = rand_fr(self.ev_batch, self.rng)
        want = lambda xs=xs.copy(): np.stack([orc.eval_polynomial(self.ev_polys[b, : self.ev_n], xs[b]) for b in range(self.ev_batch)])
        o = self.out(self.ev_batch)
        nat.check(self.lib.b200_poly_eval_batch_dev(self.d_ev.data_ptr(), self.ev_stride, self.ev_n, nat.ptr(xs), self.ev_batch, o.data_ptr(), st))
        scribble(xs)
        return "eval_batch stride %d" % self.ev_stride, o, want

    def quotient(self, st):
        loads, consts, instrs = (a.copy() for a in self.rng.choice(self.q_progs))
        consts = rand_fr(consts.shape[0], self.rng)
        want = lambda a=(loads.copy(), consts.copy(), instrs.copy()): orc.quotient_eval(self.q_cols, self.qk, self.qext, *a, threads=THREADS)
        o = self.out(1 << self.qext)
        nat.check(_quotient_dev(self.lib, self.d_q, self.qk, self.qext, loads, consts, instrs, o, st))
        scribble(consts)
        loads[:, 0] = self.rng.randrange(4)              # still valid column references: a mis-read stays in bounds
        instrs[...] = instrs[::-1]
        return "quotient_eval", o, want

    def evaluate_h(self, st):
        i, fin = self.rng.randrange(len(self.h_progs)), self.rng.random() < 0.5
        loads, consts, instrs = (a.copy() for a in self.h_progs[i].arrays())
        t = self.dom.t_evaluations.copy() if fin else None
        o = self.out(1 << self.dom.extended_k)
        nat.check(_evaluate_h_dev(self.lib, (loads, consts, instrs), self.d_h, self.dom, t, o, st))
        scribble(consts, *([t] if fin else []))
        return "evaluate_h_dev%s" % (" finished" if fin else ""), o, lambda: self.h_want[i, fin]

    def lookup(self, st):
        cols = [self.rng.randrange(len(self.d_lk)) for _ in range(self.rng.randint(1, 6))]
        rows = self.rng.randint(1, self.lk_rows)
        want = lambda: _mults(self.tab_n, cols, self.lk_ids, rows)
        ptrs = (C.c_void_p * len(cols))(*[self.d_lk[j].data_ptr() for j in cols])
        o = self.out(self.tab_n)
        nat.check(self.lib.b200_lookup_multiplicities_dev(self.d_table.data_ptr(), self.tab_n, ptrs, len(cols), rows, o.data_ptr(), None, st))
        for j in range(len(cols)):
            ptrs[j] = self.d_lk[0].data_ptr()
        return "lookup of %d inputs" % len(cols), o, want

    def ntt(self, st):
        j = self.rng.randrange(40)
        pre, post = rand_fr(3, self.rng), rand_fr(1, self.rng)
        want = lambda a=(pre.copy(), post[0].copy()): ntt_ref(self.pool[j], 12, self.omega, *a)
        o, tmp = self.out(self.n), self.out(self.n)
        self.keep.append(tmp)
        nat.check(self.lib.b200_ntt_dev(self.d_pool[j].data_ptr(), self.n, self.n, tmp.data_ptr(), o.data_ptr(), self.n, 12, nat.ptr(self.omega),
                                        3, nat.ptr(pre), 1, nat.ptr(post), 1, st))
        scribble(pre, post)
        return "ntt pre 3 post 1", o, want

    def poly_op(self, st):
        a, b = self.rng.randrange(40), self.rng.randrange(40)
        s = rand_fr(1, self.rng)
        o = self.out(self.n)
        if self.rng.random() < 0.5:
            want = lambda s=s[0].copy(): orc.poly_op("scale", self.pool[a], s=s, threads=THREADS)
            nat.check(self.lib.b200_poly_op_dev(3, self.d_pool[a].data_ptr(), None, nat.ptr(s), o.data_ptr(), self.n, st))
            what = "scale"
        else:
            want = lambda s=s[0].copy(): orc.poly_op("axpy", self.pool[a], self.pool[b], s, threads=THREADS)
            nat.check(self.lib.b200_poly_op_dev(4, self.d_pool[a].data_ptr(), self.d_pool[b].data_ptr(), nat.ptr(s), o.data_ptr(), self.n, st))
            what = "axpy"
        scribble(s)
        return what, o, want

    def invert(self, st):
        j = self.rng.randrange(40)
        o = self.d_pool[j].clone()
        nat.check(self.lib.b200_batch_invert_dev(o.data_ptr(), self.n, st))
        return "batch_invert", o, lambda: orc.batch_invert(self.pool[j])

    def g1_fft(self, st):
        g1n = 1 << self.g1_log
        w = orc.omega(self.g1_log)
        scale = rand_fr(1, self.rng)
        want = lambda sc=scale[0].copy(): orc.g1_scalar_mul(self.g1_gen, orc.poly_op("scale", orc.best_fft(self.g1_s, self.g1_log, w), s=sc))
        o = self.torch.zeros((g1n, 8), dtype=self.torch.int64, device="cuda")
        nat.check(self.lib.b200_g1_fft_dev(self.d_g1_in.data_ptr(), self.g1_log, nat.ptr(w), nat.ptr(scale), o.data_ptr(), st))
        scribble(scale)
        return "g1_fft", o, want

    def upload_then_scan(self, st):
        """b200_dev_upload_async from a b200_host_alloc buffer, read by the next call of the same queue"""
        slot = self.pinned_next % 8
        self.pinned_next += 1
        src = orc.gen_scalars(self.n, seed=500 + self.pinned_next)
        self.pinned_arr[slot] = src
        d = self.torch.empty((self.n, 4), dtype=self.torch.int64, device="cuda")
        self.keep.append(d)
        nat.check(self.lib.b200_dev_upload_async(d.data_ptr(), C.c_void_p(self.pinned.value + slot * 32 * self.n), 32 * self.n, st))
        init = rand_fr(1, self.rng)
        want = lambda init=init[0].copy(): orc.prefix_scan(src, init, True)
        o = self.out(self.n)
        nat.check(self.lib.b200_prefix_scan_dev(1, d.data_ptr(), self.n, nat.ptr(init), o.data_ptr(), st))
        scribble(init)
        return "upload_async -> prefix_scan", o, want

    def kinds(self):
        return [self.lincomb, self.eval_batch, self.quotient, self.evaluate_h, self.lookup, self.ntt, self.poly_op, self.invert, self.g1_fft]

    def free(self):
        self.torch.cuda.synchronize()           # nothing queued may still read the pinned buffers
        nat.check(self.lib.b200_host_free(self.pinned))
        nat.check(self.lib.b200_host_free(self.ptr_pin))


@gpu
def test_every_staging_entry_point_queued(dev_ctx):
    """Part one: 210 calls on one held stream, a random mix of lincomb (1 to 40 terms), eval_batch with stride > n, quotient_eval with
    distinct random programs and constants, evaluate_h_dev at (9, 12) (numerator and finished quotient), lookup multiplicities with
    missing = NULL, ntt_dev with pre mode 3 and post mode 1, poly_op scale and axpy, batch_invert, g1_fft, and uploads from pinned host
    memory (at most 8 in flight, each read by the next call).  Host parameters are overwritten after each call, pointer tables with
    pointers to other valid columns.  Part two: blobs larger than one ring slot (a lincomb of 7000 terms, a lookup with 32769 input
    pointers) between ring calls, alternating between a held stream and a second one."""
    import torch
    rng = random.Random(2024)
    stg = Staging(rng)
    try:
        s = torch.cuda.Stream()
        # warm every kind once: transform plans are built and scratch reaches its size before the hold
        for make in stg.kinds() + [stg.upload_then_scan, stg.lincomb_overflow, stg.lookup_overflow]:
            stg.call(make, s)
        s.synchronize()
        kinds = stg.kinds()
        plan = [kinds[i % len(kinds)] for i in range(len(kinds) * 22)] + [stg.upload_then_scan] * 8 + [stg.evaluate_h] * 4
        rng.shuffle(plan)
        assert len(plan) >= 200
        results = []
        hold(s, 5 * HOLD_MS)
        for make in plan:
            results.append(stg.call(make, s))
        assert not s.query(), "the hold ended before the last call was issued: lengthen it"
        s.synchronize()
        for i, (what, o, want) in enumerate(results):
            assert_eq(down(o), want(), "%s (call %d)" % (what, i))

        # ---- part two: overflow blobs between ring calls on two streams.  Each overflow lookup is issued on s behind a fresh hold, so
        # its pinned pointer table is overwritten while the stream has not reached the copy, unless the push waits for it.
        s2 = torch.cuda.Stream()
        results = []
        for r in range(6):
            ts = s if r % 2 == 0 else s2
            if ts is s:
                hold(s)
            results.append(stg.call(stg.lincomb, ts))
            results.append(stg.call(stg.lookup_overflow if ts is s else stg.lincomb_overflow, ts))
            results.append(stg.call(stg.ntt, ts))
            results.append(stg.call(stg.quotient, ts))
        torch.cuda.synchronize()
        for i, (what, o, want) in enumerate(results):
            assert_eq(down(o), want(), "%s (overflow part, call %d)" % (what, i))
    finally:
        stg.free()


# ---- 3. MSM: column stride, and scratch that grows while queued ----------------------------------------------------------------------------
def _bases(n, c, levels=None):
    from ezkl_b200 import device as dev
    pts = orc.gen_bases(n, seed=600 + n)
    b = dev.DeviceBases(up(pts), window_bits=c, max_table_bytes=0 if levels is None else levels * n * 64)
    return pts, b


def _table(b):
    L, s, nbytes = C.c_int(), C.c_int(), C.c_size_t()
    nat.check(nat.lib().b200_bases_table(b.handle, C.byref(L), C.byref(s), C.byref(nbytes)))
    return L.value, s.value


def _normalized(out):
    from ezkl_b200 import device as dev
    return dev.normalize(out)[:, :8]


@gpu
@pytest.mark.parametrize("c,levels", [(12, None), (16, None), (17, None), (13, 4)], ids=["c12-tile", "c16-tile", "c17-atomic", "c13-reduced"])
def test_msm_column_stride(dev_ctx, c, levels):
    """b200_msm_batch_dev with stride = n + 37 and the padding between columns set to r - 1 (reading it would change the sum): the
    shared-counter recoding (c <= 16), the global-atomic one (c = 17), and a reduced table (s > 1 windows per level)."""
    import torch
    n, batch = 3000, 3
    stride = n + 37
    pts, b = _bases(n, c, levels)
    L, s_ = _table(b)
    if levels is not None:
        assert s_ > 1, (L, s_)
    cols = [orc.gen_scalars(n, seed=610 + j) for j in range(batch)]
    buf = np.tile(H.fr_wire(R - 1), (stride * batch, 1))
    for j in range(batch):
        buf[j * stride: j * stride + n] = cols[j]
    d = up(buf)
    out = torch.zeros((batch, 16), dtype=torch.int64, device="cuda")
    nat.check(nat.lib().b200_msm_batch_dev(b.handle, d.data_ptr(), n, stride, batch, out.data_ptr(), torch.cuda.current_stream().cuda_stream or 1))
    got = _normalized(out)
    for j in range(batch):
        assert np.array_equal(got[j], orc.msm(cols[j], pts, THREADS)), (c, levels, j)
    b.release()


@gpu
def test_msm_scratch_grows_while_queued(dev_ctx):
    """On a fresh thread (empty scratch) and a held stream, MSMs of increasing n x batch on one handle, so that every MSM scratch buffer
    grows while earlier MSMs are queued.  A buffer that grows frees its old allocation, which waits for the device, so the hold ends at
    the first growth: the test asserts that the first MSM was queued and that every result equals the oracle."""
    import torch
    N = 1 << 14
    pts, b = _bases(N, 0)
    shapes = [(1 << 9, 1), (1 << 11, 2), (1 << 12, 3), (1 << 13, 4), (N, 6)]
    cols = {sh: [orc.gen_scalars(sh[0], seed=700 + 10 * i + j) for j in range(sh[1])] for i, sh in enumerate(shapes)}
    d_cols = {sh: up(np.concatenate(v)) for sh, v in cols.items()}
    outs = {sh: torch.zeros((sh[1], 16), dtype=torch.int64, device="cuda") for sh in shapes}
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    box = {}

    def worker():
        try:
            hold(s)
            for i, (n, batch) in enumerate(shapes):
                nat.check(nat.lib().b200_msm_batch_dev(b.handle, d_cols[n, batch].data_ptr(), n, n, batch, outs[n, batch].data_ptr(), sptr(s)))
                if i == 0:
                    box["queued"] = not s.query()
        except BaseException as e:       # re-raised on the main thread
            box["err"] = e

    t = threading.Thread(target=worker)
    t.start()
    t.join()
    if "err" in box:
        raise box["err"]
    assert box["queued"], "the hold ended before the first MSM was issued: lengthen it"
    s.synchronize()
    for sh in shapes:
        got = _normalized(outs[sh])
        for j in range(sh[1]):
            assert np.array_equal(got[j], orc.msm(cols[sh][j], pts[: sh[0]], THREADS)), (sh, j)
    b.release()


# ---- 4. stream switching in one thread -----------------------------------------------------------------------------------------------------
def _gated_streams(count, ms=HOLD_MS):
    """`count` torch streams that start together: the first is held, the others wait for an event recorded after its hold."""
    import torch
    streams = [torch.cuda.Stream() for _ in range(count)]
    ev = hold(streams[0], ms)
    for st in streams[1:]:
        st.wait_event(ev)
    return streams


@gpu
def test_stream_switching_scan_kate_eval(dev_ctx):
    """One thread round-robin over three gated torch streams and the library stream (NULL), with calls that pass values through the
    thread's scratch and overlap if unordered: prefix scans and Kate division at 2^22, eval_batch on 64 columns of 2^20.  Each call
    reads inputs that were ready before the gate and writes its own output."""
    import torch
    lib = nat.lib()
    n, en, eb = 1 << 22, 1 << 20, 64
    rng = random.Random(44)
    a = orc.gen_scalars(n, seed=801)
    polys = orc.gen_scalars(en * eb, seed=802)
    d_a, d_polys = up(a), up(polys)
    # warm at full size: the scratch does not grow while the gate holds
    nat.check(lib.b200_prefix_scan_dev(1, d_a.data_ptr(), n, nat.ptr(H.fr_wire(1)), torch.empty_like(d_a).data_ptr(), sptr(torch.cuda.current_stream())))
    nat.check(lib.b200_kate_division_dev(d_a.data_ptr(), n, nat.ptr(H.fr_wire(3)), torch.empty_like(d_a).data_ptr(), sptr(torch.cuda.current_stream())))
    g_eval_x = rand_fr(eb, rng)
    nat.check(lib.b200_poly_eval_batch_dev(d_polys.data_ptr(), en, en, nat.ptr(g_eval_x), eb, torch.empty((eb, 4), dtype=torch.int64, device="cuda").data_ptr(),
                                           sptr(torch.cuda.current_stream())))
    torch.cuda.synchronize()
    streams = _gated_streams(3) + [None]
    calls = []
    for i in range(12):
        st = streams[i % 4]
        kind = (i // 4 + i) % 3
        if kind == 0:
            init, product = rand_fr(1, rng), i % 2 == 0
            o = torch.empty_like(d_a)
            nat.check(lib.b200_prefix_scan_dev(int(product), d_a.data_ptr(), n, nat.ptr(init), o.data_ptr(), sptr(st)))
            calls.append(("prefix_scan", o, lambda init=init, product=product: orc.prefix_scan(a, init[0], product)))
        elif kind == 1:
            bb = rand_fr(1, rng)
            o = torch.empty((n - 1, 4), dtype=torch.int64, device="cuda")
            nat.check(lib.b200_kate_division_dev(d_a.data_ptr(), n, nat.ptr(bb), o.data_ptr(), sptr(st)))
            calls.append(("kate_division", o, lambda bb=bb: orc.kate_division(a, bb[0])))
        else:
            xs = rand_fr(eb, rng)
            o = torch.empty((eb, 4), dtype=torch.int64, device="cuda")
            nat.check(lib.b200_poly_eval_batch_dev(d_polys.data_ptr(), en, en, nat.ptr(xs), eb, o.data_ptr(), sptr(st)))
            calls.append(("eval_batch", o, lambda xs=xs: np.stack([orc.eval_polynomial(polys[p * en:(p + 1) * en], xs[p]) for p in range(eb)])))
    assert not streams[0].query(), "the gate opened before the last call was issued: lengthen the hold"
    torch.cuda.synchronize()
    nat.check(lib.b200_sync())
    for i, (what, o, want) in enumerate(calls):
        assert_eq(down(o), want(), "%s on stream %d (call %d)" % (what, i % 4, i))


@gpu
def test_stream_switching_msm_evaluate_h(dev_ctx):
    """The same round-robin with evaluate_h_dev at (16, 19) and MSM batches of 8 columns at 2^16, whose per-thread scratch (the coset
    parts, the part tables, the MSM workspace) every call reuses."""
    import torch
    from ezkl_b200 import evaluation as ev
    from tests.evaluate_h_parts_check import program
    lib = nat.lib()
    rng = random.Random(45)
    k, ext_k = 16, 19
    dom = _dom(k, ext_k)
    n, N = dom.n, 1 << ext_k
    polys = [orc.gen_scalars(n, seed=901), orc.gen_scalars(n - 5, seed=902), orc.gen_scalars(N, seed=903), orc.gen_scalars(2 * n + 1, seed=904)]
    d_polys = [up(p) for p in polys]
    progs = [program(rng, len(polys), n, 3) for _ in range(3)]
    mn, mb = 1 << 16, 8
    pts, b = _bases(mn, 0)
    scal = orc.gen_scalars(mn * mb, seed=905)
    d_scal = up(scal)
    cur = sptr(torch.cuda.current_stream())
    warm = torch.empty((N, 4), dtype=torch.int64, device="cuda")
    nat.check(_evaluate_h_dev(lib, progs[0].arrays(), d_polys, dom, dom.t_evaluations, warm, cur))
    nat.check(lib.b200_msm_batch_dev(b.handle, d_scal.data_ptr(), mn, mn, mb, torch.empty((mb, 16), dtype=torch.int64, device="cuda").data_ptr(), cur))
    torch.cuda.synchronize()
    streams = _gated_streams(3) + [None]
    calls = []
    for i in range(8):
        st = streams[i % 4]
        if (i // 4 + i) % 2 == 0:
            j, fin = i % 3, i % 3 == 1
            o = torch.empty((N, 4), dtype=torch.int64, device="cuda")
            arrays = tuple(a.copy() for a in progs[j].arrays())
            nat.check(_evaluate_h_dev(lib, arrays, d_polys, dom, dom.t_evaluations if fin else None, o, sptr(st)))
            calls.append(("evaluate_h_dev", o, (j, fin)))
        else:
            o = torch.empty((mb, 16), dtype=torch.int64, device="cuda")
            nat.check(lib.b200_msm_batch_dev(b.handle, d_scal.data_ptr(), mn, mn, mb, o.data_ptr(), sptr(st)))
            calls.append(("msm", o, None))
    assert not streams[0].query(), "the gate opened before the last call was issued: lengthen the hold"
    torch.cuda.synchronize()
    nat.check(lib.b200_sync())
    msm_want = np.stack([orc.msm(scal[c * mn:(c + 1) * mn], pts, THREADS) for c in range(mb)])
    h_want = {}
    for i, (what, o, key) in enumerate(calls):
        if what == "msm":
            assert_eq(_normalized(o), msm_want, "msm on stream %d (call %d)" % (i % 4, i))
        else:
            if key not in h_want:
                h_want[key] = ev.evaluate_h_from_polys(progs[key[0]], polys, dom, finish=key[1])
            assert_eq(down(o), h_want[key], "evaluate_h_dev on stream %d (call %d)" % (i % 4, i))
    b.release()


@gpu
def test_b200_sync_waits_for_the_library_stream(dev_ctx):
    """Calls queued on the library stream (NULL) behind a call on a held torch stream; after b200_sync() the outputs read with
    tensor.cpu(), without any torch synchronisation, are final (the library stream does not block torch's)."""
    import torch
    lib = nat.lib()
    n = 1 << 20
    rng = random.Random(46)
    a = orc.gen_scalars(n, seed=950)
    d_a = up(a)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    hold(s)
    first = torch.empty_like(d_a)
    nat.check(lib.b200_poly_op_dev(3, d_a.data_ptr(), None, nat.ptr(H.fr_wire(5)), first.data_ptr(), n, sptr(s)))
    outs, inits = [], []
    for i in range(6):
        init = rand_fr(1, rng)
        o = torch.empty_like(d_a)
        nat.check(lib.b200_prefix_scan_dev(i % 2, first.data_ptr(), n, nat.ptr(init), o.data_ptr(), None))
        outs.append(o)
        inits.append(init)
    assert not s.query(), "the hold ended before the last call was issued: lengthen it"
    nat.check(lib.b200_sync())
    got = [o.cpu().numpy().view(np.uint64).copy() for o in outs]
    scaled = orc.poly_op("scale", a, s=H.fr_wire(5), threads=THREADS)
    for i, g in enumerate(got):
        assert_eq(g, orc.prefix_scan(scaled, inits[i][0], i % 2 == 1), "prefix scan %d on the library stream" % i)


# ---- 5. two host threads ----------------------------------------------------------------------------------------------------------------
def _run_threads(*fns):
    errs = []

    def wrap(fn):
        def run():
            try:
                fn()
            except BaseException as e:
                errs.append(e)
        return run

    ts = [threading.Thread(target=wrap(f)) for f in fns]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errs:
        raise errs[0]


@gpu
def test_two_threads_bench_pattern(dev_ctx):
    """The bench's two-stream schedule, restated: thread B enqueues the iNTT and coset NTT of eight 2^14 columns on a low-priority stream
    and commits the coefficients; thread A commits the Lagrange columns on a high-priority stream with the same bases handle, joins B's
    stream with an event and evaluates the quotient numerator on B's cosets."""
    import torch
    from ezkl_b200 import device as dev
    from ezkl_b200 import evaluation as ev
    from tests.evaluate_h_parts_check import program
    k, ext_k, cols = 14, 16, 8
    dom = _dom(k, ext_k)
    n, N = dom.n, 1 << ext_k
    vals = [orc.gen_scalars(n, seed=1000 + j) for j in range(cols)]
    d_vals = up(np.stack(vals))
    pts, b = _bases(n, 0)
    prog = program(random.Random(47), cols, n, 3)
    lo, hi = torch.cuda.Stream.priority_range()
    s_side, s_main = torch.cuda.Stream(priority=lo), torch.cuda.Stream(priority=hi)
    one, zeta = H.fr_wire(1), dom.g_coset
    zeta2 = H.fr_wire(H.fr_unwire(zeta) ** 2)
    coeffs = torch.empty((cols, n, 4), dtype=torch.int64, device="cuda")
    cosets = torch.empty((cols, N, 4), dtype=torch.int64, device="cuda")
    tmp_n, tmp_N = torch.empty_like(coeffs), torch.empty_like(cosets)
    coeff_commit = torch.zeros((cols, 16), dtype=torch.int64, device="cuda")
    lag_commit = torch.zeros((cols, 16), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    start, done = torch.cuda.Event(), torch.cuda.Event()
    recorded = threading.Event()
    box = {}
    start.record(s_main)

    def thread_b():
        try:
            with torch.cuda.stream(s_side):
                s_side.wait_event(start)
                dev.ntt(d_vals, k, dom.omega_inv, post=[dom.ifft_divisor], out=coeffs, tmp=tmp_n)
                dev.ntt(coeffs, ext_k, dom.extended_omega, n_in=n, pre=[one, zeta, zeta2], out=cosets, tmp=tmp_N)
                done.record(s_side)
                dev.msm_batch(b, coeffs, out=coeff_commit)
        finally:
            recorded.set()

    def thread_a():
        with torch.cuda.stream(s_main):
            dev.msm_batch(b, d_vals, out=lag_commit)
            recorded.wait(60)
            s_main.wait_event(done)
            box["h"] = ev.evaluate_h_device(prog, [cosets[j] for j in range(cols)], k, ext_k)

    _run_threads(thread_b, thread_a)
    torch.cuda.synchronize()
    coeff_want = [orc.lagrange_to_coeff(v, k, THREADS) for v in vals]
    coset_want = [orc.coeff_to_extended(c, ext_k, THREADS) for c in coeff_want]
    for j in range(cols):
        assert_eq(down(cosets[j]), coset_want[j], "coset %d" % j)
    assert_eq(_normalized(lag_commit), np.stack([orc.msm(v, pts, THREADS) for v in vals]), "Lagrange commitments (thread A)")
    assert_eq(_normalized(coeff_commit), np.stack([orc.msm(c, pts, THREADS) for c in coeff_want]), "coefficient commitments (thread B)")
    loads, consts, instrs = prog.arrays()
    assert_eq(down(box["h"]), orc.quotient_eval(coset_want, k, ext_k, loads, consts, instrs, threads=THREADS), "numerator (thread A)")
    b.release()


@gpu
@pytest.mark.parametrize("log_n", [13, 16])
def test_two_threads_build_a_new_transform_plan(dev_ctx, log_n):
    """A transform size (log_n with a fresh root of unity) first used by two threads at once, A on a held stream: A builds the plan's
    tables on its held stream, B must not use them before they are complete.  Both transforms equal the oracle.  B asks 20 ms after A
    has entered the call, while A's hold still runs; that A built the plan is asserted: only the thread that builds a plan waits for its
    stream, so A's call lasts until its hold ends, and a call that built nothing returns at once."""
    import torch
    lib = nat.lib()
    n = 1 << log_n
    # omega^e for an odd e is another primitive 2^log_n-th root: a plan no other test has built
    e = 7
    w = orc.fr_pow(orc.omega(log_n), e)
    srcs = [orc.gen_scalars(n, seed=1100 + log_n + j) for j in range(2)]
    d_src = [up(a) for a in srcs]
    outs = [torch.zeros_like(d) for d in d_src]
    tmps = [torch.empty_like(d) for d in d_src]
    s_a, s_b = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    barrier = threading.Barrier(2)
    box = {}

    def run(j, st):
        nat.check(lib.b200_ntt_dev(d_src[j].data_ptr(), n, n, tmps[j].data_ptr(), outs[j].data_ptr(), n, log_n, nat.ptr(w), 0, None, 0, None, 1, sptr(st)))

    a_calling = threading.Event()

    def thread_a():
        hold(s_a)
        barrier.wait()
        t0 = time.monotonic()
        a_calling.set()
        run(0, s_a)
        box["a_call_ms"] = (time.monotonic() - t0) * 1e3

    def thread_b():
        barrier.wait()
        a_calling.wait(10)
        time.sleep(0.02)            # A asks first, so the tables are built on A's held stream
        box["b_during_hold"] = not s_a.query()
        run(1, s_b)

    _run_threads(thread_a, thread_b)
    torch.cuda.synchronize()
    for j in range(2):
        assert_eq(down(outs[j]), orc.best_fft(srcs[j], log_n, w, THREADS), "thread %s's transform" % "AB"[j])
    assert box["b_during_hold"], "B asked for the plan after A's hold had ended: lengthen it"
    assert box["a_call_ms"] > HOLD_MS / 2, "A's call returned after %.1f ms: the plan was not built on A's held stream" % box["a_call_ms"]


@gpu
def test_thread_exits_with_work_queued(dev_ctx):
    """A thread issues ten _dev calls on a held user stream and returns without synchronising, so its scratch is released while they are
    queued.  The outputs equal the oracle."""
    import torch
    lib = nat.lib()
    n = 1 << 16
    rng = random.Random(48)
    a, bcol = orc.gen_scalars(n, seed=1200), orc.gen_scalars(n, seed=1201)
    d_a, d_b = up(a), up(bcol)
    s = torch.cuda.Stream()
    want, box = [], {}

    inputs = [torch.zeros_like(d_a) if i % 5 in (0, 1, 3) else d_b.clone() for i in range(10)]
    outs = [torch.zeros_like(d_a) if i % 5 != 1 else torch.zeros((n - 1, 4), dtype=torch.int64, device="cuda") for i in range(10)]
    torch.cuda.synchronize()

    def issue(i, st):
        kind = i % 5
        if kind == 0:
            init = rand_fr(1, rng)
            nat.check(lib.b200_prefix_scan_dev(1, d_a.data_ptr(), n, nat.ptr(init), outs[i].data_ptr(), sptr(st)))
            return lambda: orc.prefix_scan(a, init[0], True)
        if kind == 1:
            bb = rand_fr(1, rng)
            nat.check(lib.b200_kate_division_dev(d_a.data_ptr(), n, nat.ptr(bb), outs[i].data_ptr(), sptr(st)))
            return lambda: orc.kate_division(a, bb[0])
        if kind == 2:
            consts = rand_fr(CYCLE_PERIOD, rng)
            outs[i] = inputs[i]
            nat.check(lib.b200_poly_scale_cycle_dev(outs[i].data_ptr(), n, nat.ptr(consts), CYCLE_PERIOD, sptr(st)))
            return lambda: scale_cycle_ref(bcol, consts)
        if kind == 3:
            sc = rand_fr(2, rng)
            ptrs = (C.c_void_p * 2)(d_a.data_ptr(), d_b.data_ptr())
            nat.check(lib.b200_poly_lincomb_dev(ptrs, nat.ptr(sc), 2, n, outs[i].data_ptr(), sptr(st)))
            return lambda: lincomb_ref([a, bcol], sc)
        outs[i] = inputs[i]
        nat.check(lib.b200_batch_invert_dev(outs[i].data_ptr(), n, sptr(st)))
        return lambda: orc.batch_invert(bcol)

    def worker():
        # the thread's scratch reaches its size first: a buffer that grows frees its old allocation, which waits for the device
        warm = torch.cuda.Stream()
        scratch = [torch.empty_like(d_a) for _ in range(3)]
        torch.cuda.synchronize()
        nat.check(lib.b200_kate_division_dev(d_a.data_ptr(), n, nat.ptr(rand_fr(1, rng)), scratch[0].data_ptr(), sptr(warm)))
        nat.check(lib.b200_prefix_scan_dev(0, d_a.data_ptr(), n, nat.ptr(rand_fr(1, rng)), scratch[1].data_ptr(), sptr(warm)))
        nat.check(lib.b200_batch_invert_dev(scratch[2].data_ptr(), n, sptr(warm)))
        warm.synchronize()
        hold(s)
        for i in range(10):
            want.append(issue(i, s))
        box["queued"] = not s.query()

    _run_threads(worker)
    assert box["queued"], "the hold ended before the thread's last call was issued: lengthen it"
    s.synchronize()
    for i, (o, w_) in enumerate(zip(outs, want)):
        assert_eq(down(o), w_(), "call %d of the exited thread" % i)


# ---- 6. the bench's timed schedule -------------------------------------------------------------------------------------------------------
def _bench(k, out_dir, overlap):
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--k", str(k), "--steps", "1", "--warmup", "1", "--no-cpu-baseline",
           "--no-host-pointer-e2e", "--dump-outputs", out_dir] + ([] if overlap else ["--no-overlap"])
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, (cmd, p.stdout[-3000:], p.stderr[-3000:])
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
    assert lines, p.stdout[-3000:]
    arrays = {os.path.basename(f): np.load(f) for f in sorted(glob.glob(os.path.join(out_dir, "*.npy")))}
    assert arrays, "bench.py --dump-outputs wrote nothing"
    return json.loads(lines[-1]), arrays


@gpu
@pytest.mark.parametrize("k", [9, 17])
def test_bench_two_stream_schedule_matches_one_stream(k):
    """bench.py's timed step in the two-stream schedule (a second host thread enqueues the witness transforms on a low-priority stream)
    writes the same outputs as the one-stream schedule; each schedule is deterministic across two runs."""
    runs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for overlap in (True, False):
            for rep in range(2):
                runs[overlap, rep] = _bench(k, os.path.join(tmp, "%s%d" % ("two" if overlap else "one", rep)), overlap)
    for overlap in (True, False):
        a, b = runs[overlap, 0][1], runs[overlap, 1][1]
        assert a.keys() == b.keys() and all(np.array_equal(a[f], b[f]) for f in a), ("not deterministic", overlap)
    line = runs[True, 0][0]
    assert line["parity_checked"] is True, line
    assert line["schedule"].startswith("two streams"), line["schedule"]
    assert runs[False, 0][0]["schedule"] == "one stream, trace order"
    two, one = runs[True, 0][1], runs[False, 0][1]
    assert two.keys() == one.keys()
    for f in two:
        assert np.array_equal(two[f], one[f]), "%s differs between the two-stream and the one-stream schedule (k = %d)" % (f, k)
