"""Run by tests/test_evaluate_h_parts.py in a subprocess with a small B200_WS_BUDGET_MB, so that b200_evaluate_h evaluates the quotient
numerator one n-point coset part at a time.  Modes:
  identity   (budget 1 MiB) every system exceeds the budget: the parts path against the composition coeff_to_extended -> quotient_eval ->
             scale_cycle -> extended_to_coeff, byte for byte, at five (k, ext_k) geometries, both finish modes and four t periods;
  select     systems whose extended cosets take exactly the budget and one column more: one evaluate_h launch, then d of them;
  k22        (default budget) an ezkl-sized quotient at k = 22, ext_k = 25 whose extended cosets exceed the card's memory;
  prove OUT  the tests/test_prover_mirror.py system at k = 9, proof bytes written to OUT."""
import ctypes as C
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from ezkl_b200 import _native as nat  # noqa: E402
from ezkl_b200 import evaluation as ev  # noqa: E402
from ezkl_b200 import fields as F  # noqa: E402
from ezkl_b200 import halo2 as h2  # noqa: E402
from oracle import oracle as orc  # noqa: E402
from tests import helpers as H  # noqa: E402
from tests.test_evaluation import random_expr  # noqa: E402

R = F.FR_MODULUS


def evaluate_h(prog, polys, dom, t=None):
    """b200_evaluate_h with an explicit finishing table t (None: numerator only)."""
    cols = [nat.as_u64(c, 4) for c in polys]
    N = 1 << dom.extended_k
    lens = (C.c_size_t * max(1, len(cols)))(*[c.shape[0] for c in cols])
    loads, consts, instrs = prog.arrays()
    out = np.zeros((N, 4), np.uint64)
    nat.check(nat.lib().b200_evaluate_h(nat.ptr_array(cols), lens, len(cols), dom.k, dom.extended_k, nat.ptr(dom.extended_omega), nat.ptr(dom.g_coset),
                                        loads.ctypes.data_as(C.c_void_p), loads.shape[0], nat.ptr(consts) if consts.size else None, consts.shape[0],
                                        instrs.ctypes.data_as(C.c_void_p), instrs.shape[0], None if t is None else nat.ptr(t), 0 if t is None else t.shape[0],
                                        nat.ptr(dom.extended_omega_inv) if t is not None else None, nat.ptr(dom.extended_ifft_divisor) if t is not None else None,
                                        nat.ptr(out)))
    return out


def coset(dom, p):
    """coeff_to_extended of a coefficient vector of any length below 2^ext_k (an extended column is returned as it is)."""
    N = 1 << dom.extended_k
    if p.shape[0] == N:
        return p
    out = np.zeros((N, 4), np.uint64)
    nat.check(nat.lib().b200_coeff_to_extended(nat.ptr(p), p.shape[0], dom.extended_k, nat.ptr(dom.extended_omega), nat.ptr(dom.g_coset), nat.ptr(out)))
    return out


def finish(dom, num, t):
    a = num.copy()
    nat.check(nat.lib().b200_poly_scale_cycle(nat.ptr(a), a.shape[0], nat.ptr(t), t.shape[0]))
    nat.check(nat.lib().b200_extended_to_coeff(nat.ptr(a), dom.extended_k, nat.ptr(dom.extended_omega_inv), nat.ptr(dom.extended_ifft_divisor), nat.ptr(dom.g_coset)))
    return a


def quotient_launches(fn):
    """(result of fn(), evaluate_h kernel launches it made: profile class 6)."""
    nat.check(nat.lib().b200_profile_enable(1))
    r = fn()
    ms, cnt = C.c_double(), C.c_uint64()
    nat.check(nat.lib().b200_profile_read(6, C.byref(ms), C.byref(cnt)))
    nat.check(nat.lib().b200_profile_enable(0))
    return r, cnt.value


def system(dom, seed, extra_run=0):
    """Coefficient columns of lengths 1, n/2, n, n+1, 3n+5, 2^ext_k - 1 (those below 2^ext_k), interleaved with extended columns, twice,
    plus a run of `extra_run` equal-length coefficient columns (more than one transform batch of the parts path)."""
    n, N = dom.n, 1 << dom.extended_k
    lens = [L for L in (1, n // 2, n, n + 1, 3 * n + 5, N - 1) if L < N]
    cols, s = [], seed
    for _ in range(2):
        for i, L in enumerate(lens):
            cols.append(orc.gen_scalars(L, seed=s)); s += 1
            if i % 2:
                cols.append(orc.gen_scalars(N, seed=s)); s += 1
    L = n if n < N else n // 2
    cols += [orc.gen_scalars(L, seed=s + i) for i in range(extra_run)]
    return cols


def program(rng, ncols, n, blinding):
    """A random program plus rotations that wrap both ways: -(blinding + 1), +-(n - 1), +-1."""
    e = random_expr(rng, ncols, 6)
    for j, rot in enumerate((-(blinding + 1), n - 1, -(n - 1), 1, -1)):
        e = e * ev.Constant(rng.randrange(R)) + ev.Query((3 * j + 1) % ncols, rot) * ev.Query((5 * j + 2) % ncols, 0)
    return ev.QuotientProgram(e)


def check_identity():
    rng = random.Random(2026)
    for (k, ext_k) in ((13, 13), (12, 13), (12, 14), (9, 12), (10, 13)):
        d = 1 << (ext_k - k)
        dom = h2.EvaluationDomain(d + 1, k)
        assert dom.extended_k == ext_k
        N = 1 << ext_k
        polys = system(dom, 1000 * k + ext_k, extra_run=d + 1)
        assert len(polys) * N * 32 > 1 << 20, (k, ext_k, len(polys))
        cosets = [coset(dom, p) for p in polys]
        for trial in range(2):
            prog = program(rng, len(polys), dom.n, 5)
            loads, consts, instrs = prog.arrays()
            num = ev.evaluate_h(prog, cosets, k, ext_k)
            if (k, ext_k) == (9, 12):
                assert np.array_equal(num, orc.quotient_eval(cosets, k, ext_k, loads, consts, instrs, threads=orc.host_threads()))
                assert np.array_equal(cosets[0], orc.coeff_to_extended(np.concatenate([polys[0], np.zeros((dom.n - 1, 4), np.uint64)]), ext_k, orc.host_threads()))
            got, launches = quotient_launches(lambda: evaluate_h(prog, polys, dom))
            assert launches == d, (k, ext_k, launches)
            assert np.array_equal(got, num), (k, ext_k, trial)
            if trial:
                continue
            for period in (1, 3, d, 1024):
                t = dom.t_evaluations if period == d else H.fr_array([rng.randrange(R) for _ in range(period)])
                assert np.array_equal(evaluate_h(prog, polys, dom, t), finish(dom, num, t)), (k, ext_k, period)
        print("identity (%d, %d): %d columns OK" % (k, ext_k, len(polys)), flush=True)


def check_select():
    budget = int(os.environ["B200_WS_BUDGET_MB"]) << 20
    rng = random.Random(7)
    k, ext_k = 9, 12
    dom = h2.EvaluationDomain(9, k)
    N, d = 1 << ext_k, 8
    at = budget // (N * 32)
    assert at * N * 32 == budget
    base = [orc.gen_scalars(dom.n if i % 3 else N, seed=500 + i) for i in range(at + 1)]
    for ncols, want in ((at, 1), (at + 1, d)):
        polys = base[:ncols]
        prog = program(rng, ncols, dom.n, 3)
        num = ev.evaluate_h(prog, [coset(dom, p) for p in polys], k, ext_k)
        got, launches = quotient_launches(lambda: evaluate_h(prog, polys, dom))
        assert launches == want, (ncols, launches)
        assert np.array_equal(got, num)
        got, launches = quotient_launches(lambda: evaluate_h(prog, polys, dom, dom.t_evaluations))
        assert launches == want and np.array_equal(got, finish(dom, num, dom.t_evaluations))
        print("select: %d columns x 2^%d x 32 B %s the %d MiB budget -> %d evaluate_h launch(es)" % (ncols, ext_k, "<=" if want == 1 else ">", budget >> 20, launches), flush=True)


def check_k22():
    import torch
    k, ext_k, n_coeff, n_ext = 22, 25, 100, 2
    dom = h2.EvaluationDomain(9, k)
    n, N, d = dom.n, 1 << ext_k, 8
    free, total = torch.cuda.mem_get_info()
    assert (n_coeff + n_ext) * N * 32 > total, "the extended cosets must exceed the card's memory"
    # parts (n each), coefficient columns, h + scratch, the size-n plan and the inverse extended plan, with DevBuf headroom (1/8)
    need = int(((n_coeff + n_ext) * n * 32 + n_coeff * n * 32 + 2 * N * 32) * 1.125) + 2 * N * 32
    if free < need:
        print("SKIP: %.1f GiB free on the device, the call needs about %.1f GiB" % (free / 2**30, need / 2**30), flush=True)
        return
    g = np.random.default_rng(22)
    base = g.integers(0, 2**64, size=(n + n_coeff, 4), dtype=np.uint64)
    base[:, 3] &= (1 << 60) - 1
    coeffs = [base[i:i + n] for i in range(n_coeff)]              # distinct columns, one host buffer
    exts = []
    for _ in range(n_ext):
        e = g.integers(0, 2**64, size=(N, 4), dtype=np.uint64)
        e[:, 3] &= (1 << 60) - 1
        exts.append(e)
    polys = coeffs[:50] + [exts[0]] + coeffs[50:] + [exts[1]]
    ncols = len(polys)
    # every column read, at rotations 0 / 1 / -1 / -(n - 1), folded with y
    e = ev.Constant(0)
    for c in range(ncols):
        e = e * ev.Constant(99) + ev.Query(c, (0, 1, -1, -(n - 1))[c % 4]) * ev.Query((c + 1) % ncols, 0)
    prog = ev.QuotientProgram(e)
    t0 = time.time()
    num = evaluate_h(prog, polys, dom)
    t1 = time.time()
    print("k22: numerator of %d columns at 2^%d in %.2f s" % (ncols, ext_k, t1 - t0), flush=True)
    # 64 sampled rows, 8 per part; column values at those points from b200_poly_eval_batch_dev on the coefficients (one upload each)
    srng = random.Random(5)
    rows = [c + d * srng.randrange(n) for c in range(d) for _ in range(8)]
    zeta, w = F.FR_ZETA, pow(F.FR_ROOT_OF_UNITY, 1 << (F.FR_S - ext_k), R)
    pts = sorted({(r + rot * d) % N for r in rows for (_, rot) in prog.loads})
    xs = H.fr_array([zeta * pow(w, j, R) % R for j in pts])
    vals = []
    for p in polys:
        if p.shape[0] == N:
            vals.append({j: H.fr_unwire(p[j]) for j in pts})
            continue
        dp = torch.from_numpy(p.view(np.int64)).cuda()
        out = torch.empty((len(pts), 4), dtype=torch.int64, device="cuda")
        nat.check(nat.lib().b200_poly_eval_batch_dev(dp.data_ptr(), 0, n, nat.ptr(xs), len(pts), out.data_ptr(), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        vals.append(dict(zip(pts, H.fr_list(out.cpu().numpy().view(np.uint64)))))
    got = H.fr_list(num[rows])
    for i, r in enumerate(rows):
        assert got[i] == prog.evaluate_ints(vals, r, N, d), r
    t2 = time.time()
    fin = evaluate_h(prog, polys, dom, dom.t_evaluations)
    t3 = time.time()
    assert np.array_equal(fin, finish(dom, num, dom.t_evaluations))
    print("k22: OK (64 rows over %d parts against the program's integer semantics; finish in %.2f s equals the composition)" % (d, t3 - t2), flush=True)


def prove(path):
    from ezkl_b200 import prover as pv
    from tests import test_prover_mirror as tpm
    rng = random.Random(909)
    k = 9
    s = rng.randrange(2, R)
    cs, fixed, sigmas, advice = tpm.build_system(rng, k)
    keys = pv.Keys(h2.ParamsKZG.setup(k, s), cs, fixed, sigmas, vk_repr=0x909)
    if os.environ.get("B200_WS_BUDGET_MB") == "1":
        assert cs.column_layout()["count"] * (1 << keys.domain.extended_k) * 32 > 1 << 20, "the system must exceed the 1 MiB budget"
    proof, launches = quotient_launches(lambda: pv.create_proof(keys, advice, rng=pv.ChaCha12Rng(bytes(32))))
    with open(path, "wb") as f:
        f.write(proof)
    print("prove: %d bytes, %d evaluate_h launches, trapdoor %d" % (len(proof), launches, s), flush=True)


if __name__ == "__main__":
    nat.init(-1)
    mode = sys.argv[1]
    if mode == "identity":
        assert os.environ.get("B200_WS_BUDGET_MB") == "1"
        check_identity()
    elif mode == "select":
        check_select()
    elif mode == "k22":
        check_k22()
    elif mode == "prove":
        prove(sys.argv[2])
    print("evaluate_h parts %s OK" % mode)
