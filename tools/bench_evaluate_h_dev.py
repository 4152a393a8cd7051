#!/usr/bin/env python
"""b200_evaluate_h_dev on the ezkl-sized system of tools/bench_quotient.py (132 columns), d = 8, finish=True, from device-resident columns.

Two column arrangements:
  A  the prover's arrangement of tools/bench_evaluate_h.py: advice, z, m and phi in coefficient form (56 columns, n each), the other 76 on
     the extended domain (cycling through 4 device buffers: extended columns are read-only and may alias), at k = 16 ... 20;
  B  every column in coefficient form except the l-cosets l0, l_last and l_active (129 columns, n each), at k = 16 ... 22.
Where the extended cosets of the coefficient columns fit the free device memory (with room to spare), the same process also times today's
resident composition: b200_ntt_dev coset transforms of the coefficient columns, b200_quotient_eval_dev, b200_poly_scale_cycle_dev and the
extended inverse transform, the two alternating call by call.  A point is a host clock around the call plus a stream synchronise, one
warm-up, then the median of --reps calls; one extra call with the library's CUDA-event profile on gives the NTT and evaluate_h kernel
classes.  "device_gib" is the device memory the library holds after the _dev calls (its scratch never shrinks, so that is the call's peak,
before the composition allocates anything).  Each point runs in its own child process; the card's name, power limit and maximum SM clock
are read in the same run.  One JSON line per point on stdout (and in --out, when given)."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def l_columns(blocks):
    """Column indices of l0, l_last and l_active in tools/bench_quotient.ezkl_system(blocks): after 10 columns per block, the permutation's
    sigmas (3 per block) and its z columns (one per 3 sigmas)."""
    perm = 3 * blocks
    first = 10 * blocks + perm + (perm + 2) // 3
    return {first, first + 1, first + 2}


def child(k, arrangement, reps):
    import numpy as np
    import torch
    from bench_quotient import ezkl_system
    from ezkl_b200 import _native as nat
    from ezkl_b200 import device as dev
    from ezkl_b200 import evaluation as ev
    from ezkl_b200 import fields as F
    from ezkl_b200 import halo2 as h2
    nat.init(0)
    torch.cuda.init()
    L = nat.lib()
    dom = h2.EvaluationDomain(9, k)
    n, ext_k = dom.n, dom.extended_k
    N = 1 << ext_k
    prog, ncols, coeff = ezkl_system(8)
    if arrangement == "B":
        coeff = set(range(ncols)) - l_columns(8)
    coeff_idx = sorted(coeff)
    pool = dev.random_scalars(n, batch=len(coeff_idx), seed=k)                     # distinct coefficient columns, contiguous
    n_ext_bufs = 4 if arrangement == "A" else ncols - len(coeff_idx)
    exts = dev.random_scalars(N, batch=n_ext_bufs, seed=100 + k)
    cols, e = [], 0
    for i in range(ncols):
        if i in coeff:
            cols.append(pool[coeff_idx.index(i)])
        else:
            cols.append(exts[e % n_ext_bufs])
            e += 1
    out = torch.empty((N, 4), dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]

    def dev_call():
        ev.evaluate_h_from_polys_device(prog, cols, dom, finish=True, out=out)

    def timed(fn):
        t0 = time.perf_counter()
        fn()
        st.synchronize()
        return time.perf_counter() - t0

    timed(dev_call)
    held = free0 - torch.cuda.mem_get_info()[0]

    def profiled(fn):
        nat.check(L.b200_profile_enable(1))
        fn()
        prof = {}
        for cls, name in ((2, "ntt"), (6, "evaluate_h")):
            ms, cnt = C.c_double(), C.c_uint64()
            nat.check(L.b200_profile_read(cls, C.byref(ms), C.byref(cnt)))
            prof[name] = {"ms": round(ms.value, 2), "launches": cnt.value}
        nat.check(L.b200_profile_enable(0))
        return prof

    # the resident composition, where the coefficient columns' cosets fit with room to spare
    comp = None
    free = torch.cuda.mem_get_info()[0]
    batch = 8
    if len(coeff_idx) * N * 32 + (batch + 2) * N * 32 < free * 0.8:
        cosets = torch.empty((len(coeff_idx), N, 4), dtype=torch.int64, device="cuda")
        tmp = torch.empty((batch, N, 4), dtype=torch.int64, device="cuda")
        comp_out = torch.empty((N, 4), dtype=torch.int64, device="cuda")
        ext_cols = [cosets[coeff_idx.index(i)] if i in coeff else cols[i] for i in range(ncols)]
        ptrs = (C.c_void_p * ncols)(*[c.data_ptr() for c in ext_cols])
        loads, consts, instrs = prog.arrays()
        z = F.FR_ZETA
        pre = np.stack([F.fr_to_limbs(1), F.fr_to_limbs(z), F.fr_to_limbs(z * z % F.FR_MODULUS)])
        dv = F.fr_inv(N)
        post = np.stack([F.fr_to_limbs(dv), F.fr_to_limbs(dv * z * z % F.FR_MODULUS), F.fr_to_limbs(dv * z % F.FR_MODULUS)])
        h = st.cuda_stream or 1

        def comp_call():
            for b0 in range(0, len(coeff_idx), batch):
                nb = min(batch, len(coeff_idx) - b0)
                nat.check(L.b200_ntt_dev(pool[b0].data_ptr(), n, n, tmp.data_ptr(), cosets[b0].data_ptr(), N, ext_k, nat.ptr(dom.extended_omega),
                                         3, nat.ptr(pre), 0, None, nb, h))
            nat.check(L.b200_quotient_eval_dev(ptrs, ncols, k, ext_k, loads.ctypes.data_as(C.c_void_p), loads.shape[0], nat.ptr(consts), consts.shape[0],
                                               instrs.ctypes.data_as(C.c_void_p), instrs.shape[0], comp_out.data_ptr(), h))
            nat.check(L.b200_poly_scale_cycle_dev(comp_out.data_ptr(), N, nat.ptr(dom.t_evaluations), dom.t_evaluations.shape[0], h))
            nat.check(L.b200_ntt_dev(comp_out.data_ptr(), N, N, tmp.data_ptr(), comp_out.data_ptr(), N, ext_k, nat.ptr(dom.extended_omega_inv),
                                     0, None, 3, nat.ptr(post), 1, h))

        timed(comp_call)
        st.synchronize()
        assert torch.equal(comp_out, out), "the composition and the _dev call disagree"
        comp = []
    dev_times = []
    for _ in range(reps):
        dev_times.append(timed(dev_call))
        if comp is not None:
            comp.append(timed(comp_call))
    rec = {"k": k, "ext_k": ext_k, "arrangement": arrangement, "columns": ncols, "coefficient_columns": len(coeff_idx),
           "dev_s": [round(t, 4) for t in dev_times], "dev_median_s": round(statistics.median(dev_times), 4),
           "dev_spread_s": round(max(dev_times) - min(dev_times), 4), "device_gib": round(held / 2**30, 2),
           "dev_classes_one_call": profiled(dev_call)}
    if comp is not None:
        rec.update({"composition_s": [round(t, 4) for t in comp], "composition_median_s": round(statistics.median(comp), 4),
                    "composition_classes_one_call": profiled(comp_call)})
    else:
        rec["composition"] = "does not fit: %.1f GiB of cosets, %.1f GiB free" % (len(coeff_idx) * N * 32 / 2**30, free / 2**30)
    print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", default="16,17,18,19,20", help="k values of arrangement A")
    ap.add_argument("--b", default="16,17,18,19,20,21,22", help="k values of arrangement B")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    ap.add_argument("--child", default=None, help="internal: K,ARRANGEMENT")
    a = ap.parse_args()
    if a.child is not None:
        k, arr = a.child.split(",")
        child(int(k), arr, a.reps)
        return
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    lines = [json.dumps({"card": card})]
    print(lines[0], flush=True)
    points = [(int(k), "A") for k in a.a.split(",") if k] + [(int(k), "B") for k in a.b.split(",") if k]
    for k, arr in points:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "%d,%s" % (k, arr), "--reps", str(a.reps)], capture_output=True, text=True)
        line = r.stdout.strip().splitlines()[-1] if r.returncode == 0 and r.stdout.strip() else json.dumps({"k": k, "arrangement": arr, "error": (r.stdout + r.stderr)[-1500:]})
        print(line, flush=True)
        lines.append(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
