#!/usr/bin/env python
"""evaluate_h on an ezkl-sized constraint system (run on the GPU box; `ncu -k regex:k_quotient_eval` around it gives DRAM bytes per row):
`blocks` BaseConfig blocks (5 advice + 5 selector columns each, 5 gates), a permutation over 3 advice columns per block in chunks of 3,
and one mv-lookup per two blocks, folded with y as evaluate_h does, at k = 17 on the 2^20 extended domain with random columns
(performance only: parity of this kernel is tests/test_constraint_system.py and tests/test_evaluation.py)."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from ezkl_b200 import _native as nat  # noqa: E402
from ezkl_b200 import device as dev  # noqa: E402
from ezkl_b200 import evaluation as ev  # noqa: E402


def ezkl_system(blocks):
    """(program, number of columns, the columns a prover holds in coefficient form: advice, z, m, phi)."""
    col = 0

    def new(cnt):
        nonlocal col
        r = list(range(col, col + cnt))
        col += cnt
        return r

    terms, perm_cols, coeff = [], [], []
    blks = []
    for _ in range(blocks):
        adv, sel = new(5), new(5)
        blks.append((adv, sel))
        coeff += adv
        terms += ev.base_op_gates(dict(zip(["ADD", "MULT", "DOTINIT", "DOT", "SUM"], sel)), adv[0:2], adv[2:4], adv[4])
        perm_cols += [adv[0], adv[2], adv[4]]
    sig = new(len(perm_cols))
    nz = (len(perm_cols) + 2) // 3
    zs = new(nz)
    coeff += zs
    l0, l_last, l_active, xcol = new(4)
    terms += ev.permutation_terms(perm_cols, sig, zs, l0, l_last, l_active, xcol, 11, 13, 3, 5)
    for b in range(0, blocks, 2):
        table, sel_l, m, phi = new(4)
        coeff += [m, phi]
        f = ev.Query(sel_l) * ev.Query(blks[b][0][1]) + (ev.Constant(1) - ev.Query(sel_l)) * ev.Constant(7)
        terms += ev.mv_lookup_terms([f], ev.Query(table), m, phi, l0, l_last, l_active, 17)
    return ev.QuotientProgram(ev.fold_y(terms, 99)), col, set(coeff)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=8)
    ap.add_argument("--k", type=int, default=17)
    ap.add_argument("--ext-bits", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    nat.init(0)
    k, ext_k = a.k, a.k + a.ext_bits
    N = 1 << ext_k
    prog, ncols, _ = ezkl_system(a.blocks)
    distinct = len(prog.loads)
    print("columns %d, instructions %d (muladd %d), slots %d, distinct (column, rotation) loads %d, constants %d" %
          (ncols, len(prog.instrs), sum(1 for i in prog.instrs if i[0] == ev.OP_MULADD), prog.n_slots, distinct, len(prog.consts)), flush=True)
    pool = dev.random_scalars(N, batch=ncols, seed=3)                        # every column its own buffer (132 x 32 MB at the defaults)
    columns = [pool[i % pool.shape[0]] for i in range(ncols)]
    out = torch.empty((N, 4), dtype=torch.int64, device="cuda")
    for _ in range(2):
        ev.evaluate_h_device(prog, columns, k, ext_k, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.reps):
        ev.evaluate_h_device(prog, columns, k, ext_k, out=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.reps
    muls = sum(1 for i in prog.instrs if i[0] in (ev.OP_MUL, ev.OP_MULADD, ev.OP_SQUARE))
    print("2^%d rows: %.3f ms, %.2f G rows/s, %d multiplications/row -> %.1f G mulmod/s; algorithmic bytes/row = %d distinct columns x 32 + 32 = %d B (distinct (column, rotation) x 32 + 32 = %d B)" %
          (ext_k, ms, N / ms / 1e6, muls, N * muls / ms / 1e6, len({c for c, _ in prog.loads}), 32 * len({c for c, _ in prog.loads}) + 32, 32 * distinct + 32), flush=True)


if __name__ == "__main__":
    main()
