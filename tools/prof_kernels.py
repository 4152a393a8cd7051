#!/usr/bin/env python
"""Profiling helper (run on the GPU box): mulmod / group-add throughput microbenchmarks, or a minimal MSM + NTT
workload for `ncu --set full -k regex:k_accumulate|k_ntt_pass`."""
import argparse
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from ezkl_b200 import _native as nat  # noqa: E402
from ezkl_b200 import device as dev  # noqa: E402
from ezkl_b200 import fields as F  # noqa: E402
from ezkl_b200 import halo2 as h2  # noqa: E402
import gpu_peaks  # noqa: E402


def microbench():
    L = nat.lib()
    names = {0: "fq mul chain (PTX)", 1: "fq mul 2 chains (PTX)", 2: "fq mul portable", 3: "xyzz mixed add", 4: "fq add+sub pair", 5: "fq mul 9x30-bit carry-less"}
    for variant in (0, 5, 1, 2, 3, 4):
        for threads, blocks_per_sm in ((128, 4), (256, 2), (256, 4), (256, 8)):
            if variant == 3 and threads * blocks_per_sm > 512:
                continue
            iters = 2000 if variant != 3 else 200
            blocks = gpu_peaks.sm_count() * blocks_per_sm
            ms = C.c_float(0)
            nat.check(nat.dbg_lib().b200_debug_bench(variant, iters, blocks, threads, C.byref(ms)))
            ops = blocks * threads * iters
            print("%-24s threads/SM=%5d  %8.3f ms  %8.2f G op/s" % (names[variant], threads * blocks_per_sm, ms.value, ops / ms.value / 1e6), flush=True)


def pipebench():
    L = nat.lib()
    names = {0: "mad.wide.u32 (IMAD.WIDE, no carry)", 1: "mad.lo.cc/madc.hi.cc pairs (IMAD.WIDE.X)", 2: "mad.lo.u32 (IMAD)", 3: "fma.f64 (DFMA)"}
    sms, clock_hz = gpu_peaks.sm_count(), gpu_peaks.max_sm_clock_hz()
    for variant in (0, 1, 2, 3):
        for threads, bps in ((256, 2), (256, 4), (256, 8)):
            iters, blocks = 4000, sms * bps
            ms = C.c_float(0)
            nat.check(nat.dbg_lib().b200_debug_bench_pipe(variant, iters, blocks, threads, C.byref(ms)))
            per_iter = 16 if variant == 1 else 8          # PTX ops per thread per iteration (v1: 8 lo/hi pairs = 8 fused wide ops)
            ops = blocks * threads * iters * per_iter
            clk = ms.value * 1e-3 * clock_hz         # at the maximum SM clock: a power-capped card that runs slower shows fewer ops / clk
            print("%-44s threads/SM=%5d  %8.3f ms  %8.1f PTX-ops/clk/SM  (%6.2f T ops/s)" % (names[variant], threads * bps, ms.value, ops / clk / sms, ops / ms.value / 1e9), flush=True)


def workload(k, batch, c):
    n = 1 << k
    bases = dev.DeviceBases(dev.generate_bases(n, seed=1), window_bits=c)
    cols = dev.random_scalars(n, batch=batch, seed=2)
    out = dev.msm_batch(bases, cols)
    torch.cuda.synchronize()
    dom = h2.EvaluationDomain(9, k)
    one = F.fr_to_limbs(1)
    zeta, zeta2 = F.fr_to_limbs(F.FR_ZETA), F.fr_to_limbs(F.FR_ZETA * F.FR_ZETA % F.FR_MODULUS)
    ext = dev.ntt(cols[:4], dom.extended_k, dom.extended_omega, n_in=n, pre=[one, zeta, zeta2])
    torch.cuda.synchronize()
    return out, ext


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--micro", action="store_true")
    ap.add_argument("--pipe", action="store_true")
    ap.add_argument("--k", type=int, default=17)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--c", type=int, default=0)
    a = ap.parse_args()
    nat.init(0)
    if a.pipe:
        pipebench()
    elif a.micro:
        microbench()
    else:
        workload(a.k, a.batch, a.c)
        print("workload done")
