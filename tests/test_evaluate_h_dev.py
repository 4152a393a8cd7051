"""b200_evaluate_h_dev: the quotient from device-resident columns, one n-point coset part at a time, with the
extended columns read in place.  Its result must be b200_evaluate_h's, byte for byte, on the same columns (DESIGN.md §4.4).  The checks that
need a scratch budget run tests/evaluate_h_dev_check.py in a child process, because B200_WS_BUDGET_MB is read once, at b200_init."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from ezkl_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHECK = os.path.join(ROOT, "tests", "evaluate_h_dev_check.py")
P, S, Z, U32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32


def run_check(budget_mb, *args):
    env = dict(os.environ)
    env.pop("B200_WS_BUDGET_MB", None)
    if budget_mb is not None:
        env["B200_WS_BUDGET_MB"] = str(budget_mb)
    r = subprocess.run([sys.executable, CHECK, *args], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    return r.stdout


# ---- CPU: the entry point is exported and typed ---------------------------------------------------------------------------------
def test_evaluate_h_dev_is_exported_and_typed():
    """include/ezkl_b200.h declares b200_evaluate_h_dev, which libezkl_b200.so exports with the argtypes / restype read from that header."""
    decls = nat.declarations(nat.HEADER)
    fn = nat.lib().b200_evaluate_h_dev
    assert (fn.argtypes, fn.restype) == decls["b200_evaluate_h_dev"]
    assert decls["b200_evaluate_h_dev"] == ([P, P, S, U32, U32, P, P, P, S, P, S, P, S, P, U32, P, P, P, P], Z)


# ---- GPU -------------------------------------------------------------------------------------------------------------------------
def _dom(k, ext_k):
    from ezkl_b200 import halo2 as h2
    d = h2.EvaluationDomain((1 << (ext_k - k)) + 1, k)
    assert d.extended_k == ext_k
    return d


@pytest.mark.gpu
@pytest.mark.parametrize("budget_mb", [None, 1], ids=["resident", "parts"])
def test_dev_is_byte_identical_to_evaluate_h(budget_mb):
    """(k, ext_k) = (13, 13), (12, 13), (12, 14), (9, 12), (10, 13); coefficient columns of lengths 1, n/2, n, n+1, 3n+5, 2^ext_k - 1 mixed with
    extended columns and a run of more equal-length columns than one transform batch; random programs with wrapping rotations; numerator and
    finished quotient (t periods 1, 3, d, 1024).  The _dev result equals b200_evaluate_h at the default budget (every coset resident) and at
    1 MiB (by parts), and the composition coeff_to_extended -> quotient_eval -> scale_cycle -> extended_to_coeff; the oracle at (9, 12)."""
    out = run_check(budget_mb, "identity")
    assert out.count("parts OK") == 5, out


@pytest.mark.gpu
def test_dev_launches_one_evaluate_h_kernel_per_part():
    import torch
    from ezkl_b200 import evaluation as ev
    from tests.evaluate_h_parts_check import program, quotient_launches, system
    nat.init(-1)
    for k, ext_k in ((9, 12), (10, 12), (11, 11)):
        dom = _dom(k, ext_k)
        polys = system(dom, 31 + k, extra_run=3)
        dpolys = [torch.from_numpy(p.view(np.int64)).cuda() for p in polys]
        prog = program(random.Random(k), len(polys), dom.n, 3)
        for fin in (False, True):
            got, launches = quotient_launches(lambda: ev.evaluate_h_from_polys_device(prog, dpolys, dom, finish=fin))
            assert launches == 1 << (ext_k - k), (k, ext_k, fin, launches)
            assert np.array_equal(got.cpu().numpy().view(np.uint64), ev.evaluate_h_from_polys(prog, polys, dom, finish=fin)), (k, ext_k, fin)


@pytest.mark.gpu
def test_dev_is_ordered_on_the_callers_stream():
    """On a non-default torch stream a column is written by b200_ntt_dev immediately before the call, with no synchronisation between them:
    the call sees the transform's result."""
    import torch
    from ezkl_b200 import evaluation as ev
    from oracle import oracle as orc
    from tests.evaluate_h_parts_check import program
    nat.init(-1)
    k, ext_k = 12, 15
    dom = _dom(k, ext_k)
    n, N = dom.n, 1 << ext_k
    src = orc.gen_scalars(n, seed=71)
    other = [orc.gen_scalars(n, seed=72), orc.gen_scalars(N, seed=73)]
    col = src.copy()
    nat.check(nat.lib().b200_ifft(nat.ptr(col), k, nat.ptr(dom.omega_inv), nat.ptr(dom.ifft_divisor)))
    prog = program(random.Random(3), 3, n, 3)
    want = ev.evaluate_h_from_polys(prog, [col] + other, dom, finish=True)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_src = torch.from_numpy(src.view(np.int64)).to("cuda", non_blocking=False)
        d_other = [torch.from_numpy(p.view(np.int64)).cuda() for p in other]
        d_col = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
        d_tmp = torch.empty((n, 4), dtype=torch.int64, device="cuda")
        s.synchronize()
        nat.check(nat.lib().b200_ntt_dev(d_src.data_ptr(), n, n, d_tmp.data_ptr(), d_col.data_ptr(), n, k, nat.ptr(dom.omega_inv), 0, None, 1,
                                         nat.ptr(dom.ifft_divisor), 1, s.cuda_stream))
        out = ev.evaluate_h_from_polys_device(prog, [d_col] + d_other, dom, finish=True)
    s.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint64), want)


@pytest.mark.gpu
def test_dev_aliasing_and_argument_errors():
    import torch
    from ezkl_b200 import evaluation as ev
    from oracle import oracle as orc
    from tests.evaluate_h_dev_check import evaluate_h_dev
    from tests.evaluate_h_parts_check import program
    nat.init(-1)
    k, ext_k = 9, 12
    dom = _dom(k, ext_k)
    n, N = dom.n, 1 << ext_k
    lib = nat.lib()
    # one tensor as two columns, one of them through a shorter view
    base = orc.gen_scalars(n, seed=81)
    ext = orc.gen_scalars(N, seed=82)
    d_base, d_ext = torch.from_numpy(base.view(np.int64)).cuda(), torch.from_numpy(ext.view(np.int64)).cuda()
    prog = program(random.Random(4), 3, n, 3)
    for fin in (False, True):
        got = ev.evaluate_h_from_polys_device(prog, [d_base, d_base[: n // 2], d_ext], dom, finish=fin)
        assert np.array_equal(got.cpu().numpy().view(np.uint64), ev.evaluate_h_from_polys(prog, [base, base[: n // 2], ext], dom, finish=fin))
    # n_columns = 0 yields zeros (the empty program's value), with or without finishing
    empty = ev.QuotientProgram(ev.Constant(0) * ev.Constant(0))
    for t in (None, dom.t_evaluations):
        rc, out = evaluate_h_dev(empty, [], dom, t, out=torch.full((N, 4), 7, dtype=torch.int64, device="cuda"))
        nat.check(rc)
        assert not out.cpu().numpy().any()
    # argument errors: -1, a message, and d_out keeps its bytes
    lens = (C.c_size_t * 2)(n, N)
    ptrs = (C.c_void_p * 2)(d_base.data_ptr(), d_ext.data_ptr())
    prog = program(random.Random(5), 2, n, 3)
    loads, consts, instrs = prog.arrays()
    out = torch.full((N, 4), 5, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream or 1
    t = dom.t_evaluations
    good = dict(d_polys=ptrs, lengths=lens, n_columns=2, k=k, ext_k=ext_k, ext_omega=nat.ptr(dom.extended_omega), zeta=nat.ptr(dom.g_coset),
                loads=loads.ctypes.data_as(C.c_void_p), n_loads=loads.shape[0], constants=nat.ptr(consts), n_constants=consts.shape[0],
                program=instrs.ctypes.data_as(C.c_void_p), n_instr=instrs.shape[0], t_evaluations=nat.ptr(t), t_period=t.shape[0],
                ext_omega_inv=nat.ptr(dom.extended_omega_inv), ext_ifft_divisor=nat.ptr(dom.extended_ifft_divisor), d_out=out.data_ptr(), stream=st)

    def call(**kw):
        a = dict(good, **kw)
        return lib.b200_evaluate_h_dev(*a.values())

    bad_instrs = instrs.copy()
    bad_instrs[0, 0] = (bad_instrs[0, 0] & ~np.uint32(0xFF)) | np.uint32(9)       # op 9 does not exist
    bad_operand = instrs.copy()
    bad_operand[0, 1] = (1 << 30) | 10**6                                         # constant index out of range
    null_col = (C.c_void_p * 2)(None, d_ext.data_ptr())
    over = (C.c_void_p * 2)(out.data_ptr() + 32 * 5, d_ext.data_ptr())            # a column starting inside d_out
    under = (C.c_void_p * 2)(out.data_ptr() - 32 * 4, d_ext.data_ptr())           # a column ending inside d_out
    cases = {
        "null d_polys": dict(d_polys=None), "null lengths": dict(lengths=None), "null column": dict(d_polys=null_col), "null ext_omega": dict(ext_omega=None),
        "null zeta": dict(zeta=None), "null loads": dict(loads=None), "null constants": dict(constants=None), "null program": dict(program=None),
        "length 0": dict(lengths=(C.c_size_t * 2)(0, N)), "length above 2^ext_k": dict(lengths=(C.c_size_t * 2)(N + 1, N)),
        "k = 0": dict(k=0), "k > ext_k": dict(k=ext_k + 1), "ext_k > 28": dict(k=25, ext_k=29),
        "finish without ext_omega_inv": dict(ext_omega_inv=None), "finish without the divisor": dict(ext_ifft_divisor=None),
        "t_period 0": dict(t_period=0), "t_period 1025": dict(t_period=1025),
        "d_out inside a column": dict(d_polys=over), "a column ending in d_out": dict(d_polys=under, lengths=(C.c_size_t * 2)(8, N)),
        "d_out is a column": dict(d_polys=(C.c_void_p * 2)(d_base.data_ptr(), out.data_ptr())),
        "load column out of range": dict(n_columns=1, lengths=(C.c_size_t * 1)(n), d_polys=(C.c_void_p * 1)(d_base.data_ptr())),
        "bad op": dict(program=bad_instrs.ctypes.data_as(C.c_void_p)), "bad operand": dict(program=bad_operand.ctypes.data_as(C.c_void_p)),
    }
    torch.cuda.synchronize()
    before = out.cpu().numpy().copy()
    for name, kw in cases.items():
        assert call(**kw) == -1, name
        assert lib.b200_last_error().decode(), name
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), before)
    assert call() == 0
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint64), ev.evaluate_h_from_polys(prog, [base, ext], dom, finish=True))


@pytest.mark.gpu
def test_prover_mirror_proof_through_the_dev_call(monkeypatch):
    """The golden case of tests/test_prover_mirror.py with the prover's evaluate_h_from_polys replaced by an upload of its columns and
    b200_evaluate_h_dev: the proof is tests/golden/mirror_proof_k6.bin and verifies at the trapdoor."""
    import torch
    from ezkl_b200 import evaluation as ev
    from ezkl_b200 import halo2 as h2
    from ezkl_b200 import prover as pv
    from tests import test_prover_mirror as tpm
    nat.init(-1)
    calls = []

    def through_dev(program, polys, domain, finish=False):
        cols = [torch.from_numpy(np.ascontiguousarray(nat.as_u64(p, 4)).view(np.int64)).cuda() for p in polys]
        calls.append(len(cols))
        out = ev.evaluate_h_from_polys_device(program, cols, domain, finish=finish)
        torch.cuda.current_stream().synchronize()
        return out.cpu().numpy().view(np.uint64).copy()

    monkeypatch.setattr(ev, "evaluate_h_from_polys", through_dev)
    k, s, cs, fixed, sigmas, advice = tpm.golden_case()
    keys = pv.Keys(h2.ParamsKZG.setup(k, s), cs, fixed, sigmas, vk_repr=0x5EED)
    proof = pv.create_proof(keys, advice, rng=pv.ChaCha12Rng(bytes(32)))
    assert calls, "the prover did not reach evaluate_h_from_polys"
    assert proof == open(tpm.GOLDEN_PROOF, "rb").read()
    assert pv.verify_proof_with_trapdoor(keys, proof, s)


@pytest.mark.gpu
def test_ezkl_sized_quotient_from_resident_columns():
    """k = 22, ext_k = 25, tools/bench_quotient.ezkl_system(8) (132 columns) with every column in coefficient form except l0, l_last and
    l_active: 132 GiB of extended cosets, more than the card holds.  64 rows over all 8 parts against the program's integer semantics, the
    finished quotient against b200_evaluate_h on the same host columns, and the library's device memory after the call within the stated
    scratch.  Skips (with the numbers) when the shared device has too little free memory."""
    out = run_check(None, "k22")
    if "SKIP" in out:
        pytest.skip(out.strip().splitlines()[0])
    assert "k22: OK" in out, out
