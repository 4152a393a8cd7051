"""Run by tests/test_evaluate_h_dev.py in a subprocess, because B200_WS_BUDGET_MB (which selects b200_evaluate_h's path) is read once, at
b200_init.  b200_evaluate_h_dev always evaluates by parts on the device; these checks hold it to the host entry point.  Modes:
  identity  at the budget the parent sets (default: b200_evaluate_h keeps every coset resident; 1 MiB: it evaluates by parts): five (k, ext_k)
            geometries, the systems and programs of tests/evaluate_h_parts_check.py, numerator and finished quotient (t periods 1, 3, d, 1024):
            the _dev result equals b200_evaluate_h and the composition coeff_to_extended -> quotient_eval -> scale_cycle -> extended_to_coeff
            byte for byte, and the oracle at (9, 12); every _dev call makes exactly d evaluate_h launches;
  k22       an ezkl-sized quotient at k = 22, ext_k = 25 (tools/bench_quotient.ezkl_system(8), every column in coefficient form except l0, l_last
            and l_active) whose extended cosets do not fit the card: 64 rows over all 8 parts against the program's integer semantics, the
            finished quotient against b200_evaluate_h on the same host columns, and the device memory the library holds against the stated
            scratch."""
import ctypes as C
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402

from ezkl_b200 import _native as nat  # noqa: E402
from ezkl_b200 import evaluation as ev  # noqa: E402
from ezkl_b200 import fields as F  # noqa: E402
from ezkl_b200 import halo2 as h2  # noqa: E402
from oracle import oracle as orc  # noqa: E402
from tests import helpers as H  # noqa: E402
from tests.evaluate_h_parts_check import coset, evaluate_h, finish, program, quotient_launches, system  # noqa: E402

R = F.FR_MODULUS


def evaluate_h_dev(prog, cols, dom, t=None, out=None, stream=None):
    """b200_evaluate_h_dev on torch CUDA columns with an explicit finishing table t (None: numerator only); returns the rc and `out`."""
    import torch
    N = 1 << dom.extended_k
    if out is None:
        out = torch.zeros((N, 4), dtype=torch.int64, device="cuda")
    lens = (C.c_size_t * max(1, len(cols)))(*[c.shape[0] for c in cols])
    ptrs = (C.c_void_p * max(1, len(cols)))(*[c.data_ptr() for c in cols])
    loads, consts, instrs = prog.arrays()
    rc = nat.lib().b200_evaluate_h_dev(ptrs, lens, len(cols), dom.k, dom.extended_k, nat.ptr(dom.extended_omega), nat.ptr(dom.g_coset),
                                       loads.ctypes.data_as(C.c_void_p), loads.shape[0], nat.ptr(consts) if consts.size else None, consts.shape[0],
                                       instrs.ctypes.data_as(C.c_void_p), instrs.shape[0], None if t is None else nat.ptr(t), 0 if t is None else t.shape[0],
                                       nat.ptr(dom.extended_omega_inv) if t is not None else None, nat.ptr(dom.extended_ifft_divisor) if t is not None else None,
                                       out.data_ptr(), stream if stream is not None else torch.cuda.current_stream().cuda_stream or 1)
    return rc, out


def to_device(polys):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(p).view(np.int64)).cuda() for p in polys]


def to_host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint64)


def check_identity():
    budget = os.environ.get("B200_WS_BUDGET_MB")
    rng = random.Random(2027)
    for (k, ext_k) in ((13, 13), (12, 13), (12, 14), (9, 12), (10, 13)):
        d = 1 << (ext_k - k)
        dom = h2.EvaluationDomain(d + 1, k)
        assert dom.extended_k == ext_k
        polys = system(dom, 1000 * k + ext_k + 7, extra_run=d + 1)
        dpolys = to_device(polys)
        cosets = [coset(dom, p) for p in polys]
        for trial in range(2):
            prog = program(rng, len(polys), dom.n, 5)
            loads, consts, instrs = prog.arrays()
            num = ev.evaluate_h(prog, cosets, k, ext_k)
            host, host_launches = quotient_launches(lambda: evaluate_h(prog, polys, dom))
            assert host_launches == (d if budget == "1" else 1), (k, ext_k, host_launches)
            (rc, out), launches = quotient_launches(lambda: evaluate_h_dev(prog, dpolys, dom))
            nat.check(rc)
            assert launches == d, (k, ext_k, launches)
            got = to_host(out)
            assert np.array_equal(got, host) and np.array_equal(got, num), (k, ext_k, trial)
            if (k, ext_k) == (9, 12):
                assert np.array_equal(got, orc.quotient_eval(cosets, k, ext_k, loads, consts, instrs, threads=orc.host_threads()))
            if trial:
                continue
            for period in (1, 3, d, 1024):
                t = dom.t_evaluations if period == d else H.fr_array([rng.randrange(R) for _ in range(period)])
                rc, out = evaluate_h_dev(prog, dpolys, dom, t)
                nat.check(rc)
                got = to_host(out)
                assert np.array_equal(got, evaluate_h(prog, polys, dom, t)) and np.array_equal(got, finish(dom, num, t)), (k, ext_k, period)
        print("identity (%d, %d): %d columns, %d parts OK" % (k, ext_k, len(polys), d), flush=True)


def check_k22():
    import torch
    from bench_evaluate_h_dev import l_columns
    from bench_quotient import ezkl_system
    k, ext_k = 22, 25
    dom = h2.EvaluationDomain(9, k)
    n, N, d = dom.n, 1 << ext_k, 8
    prog, ncols, _ = ezkl_system(8)
    lcols = l_columns(8)
    n_coeff = ncols - len(lcols)
    free, total = torch.cuda.mem_get_info()
    assert ncols * N * 32 > total, "the extended cosets must exceed the card's memory"
    # the caller's columns (coefficient columns as overlapping views of one allocation: they are read-only), the output, and the stated
    # scratch with DevBuf headroom (1/8) and the size-n and size-N transform plans
    lo_bits = (ext_k + 1) // 2
    stated = n_coeff * n * 32 + N * 32 + (3 + (1 << lo_bits) + (N >> lo_bits)) * 32 + 16 * n_coeff
    need = (n + ncols) * 32 + 3 * N * 32 + N * 32 + int(stated * 1.125) + 2 * N * 32
    # then b200_evaluate_h on the host columns, by parts: every column's part, the coefficient columns, h and its transform scratch
    need = max(need, int(((ncols + n_coeff) * n * 32 + 2 * N * 32) * 1.125) + 2 * N * 32)
    if free < need:
        print("SKIP: %.1f GiB free on the device, the call needs about %.1f GiB" % (free / 2**30, need / 2**30), flush=True)
        return
    g = np.random.default_rng(2225)

    def rand(rows):
        a = g.integers(0, 2**64, size=(rows, 4), dtype=np.uint64)
        a[:, 3] &= (1 << 60) - 1
        return a

    base = rand(n + ncols)
    exts = {c: rand(N) for c in sorted(lcols)}
    polys = [exts[i] if i in lcols else base[i:i + n] for i in range(ncols)]
    dbase = torch.from_numpy(base.view(np.int64)).cuda()
    dexts = {c: torch.from_numpy(e.view(np.int64)).cuda() for c, e in exts.items()}
    dpolys = [dexts[i] if i in lcols else dbase[i:i + n] for i in range(ncols)]
    assert all(p.is_contiguous() for p in dpolys)
    out = torch.empty((N, 4), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.time()
    rc, out = evaluate_h_dev(prog, dpolys, dom, out=out)
    nat.check(rc)
    torch.cuda.synchronize()
    t1 = time.time()
    held = free0 - torch.cuda.mem_get_info()[0]
    print("k22: numerator of %d columns (%d in coefficient form) at 2^%d in %.2f s; the library holds %.2f GiB, stated scratch %.2f GiB" %
          (ncols, n_coeff, ext_k, t1 - t0, held / 2**30, stated / 2**30), flush=True)
    # the stated scratch with DevBuf headroom, plus the transform plans (twiddles of the size-n and size-N transforms) and the staging ring
    assert held <= stated * 1.125 + 2 * N * 32 + (64 << 20), (held, stated)
    # 64 sampled rows, 8 per part; column values at those points from b200_poly_eval_batch_dev on the coefficients
    srng = random.Random(6)
    rows = [c + d * srng.randrange(n) for c in range(d) for _ in range(8)]
    num = to_host(out)[rows]
    zeta, w = F.FR_ZETA, pow(F.FR_ROOT_OF_UNITY, 1 << (F.FR_S - ext_k), R)
    pts = sorted({(r + rot * d) % N for r in rows for (_, rot) in prog.loads})
    xs = H.fr_array([zeta * pow(w, j, R) % R for j in pts])
    vals = []
    for p, dp in zip(polys, dpolys):
        if p.shape[0] == N:
            vals.append({j: H.fr_unwire(p[j]) for j in pts})
            continue
        ev_out = torch.empty((len(pts), 4), dtype=torch.int64, device="cuda")
        nat.check(nat.lib().b200_poly_eval_batch_dev(dp.data_ptr(), 0, n, nat.ptr(xs), len(pts), ev_out.data_ptr(), torch.cuda.current_stream().cuda_stream or 1))
        vals.append(dict(zip(pts, H.fr_list(to_host(ev_out)))))
    got = H.fr_list(num)
    for i, r in enumerate(rows):
        assert got[i] == prog.evaluate_ints(vals, r, N, d), r
    t2 = time.time()
    rc, out = evaluate_h_dev(prog, dpolys, dom, dom.t_evaluations, out=out)
    nat.check(rc)
    fin = to_host(out)
    t3 = time.time()
    del dbase, dexts, dpolys, out
    torch.cuda.empty_cache()
    nat.shutdown()                       # gives the _dev call's scratch back before the host entry point takes its own
    nat.init(-1)
    host = evaluate_h(prog, polys, dom, dom.t_evaluations)
    assert np.array_equal(fin, host)
    print("k22: OK (64 rows over %d parts against the program's integer semantics; finished in %.2f s, equal to b200_evaluate_h)" % (d, t3 - t2), flush=True)


if __name__ == "__main__":
    nat.init(-1)
    mode = sys.argv[1]
    if mode == "identity":
        check_identity()
    elif mode == "k22":
        check_k22()
    print("evaluate_h_dev %s OK" % mode)
