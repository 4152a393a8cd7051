#!/usr/bin/env python
"""Permutation keygen on the device (b200_permutation_sigmas_dev), and the permutation half of create_keys built on it.

1. The sigma kernel alone: k = 20, 22, 24, 26 x P = 8, 32, 128 columns, where the mapping and the result (40 B per cell) fit in 24 GiB.
   The mapping is a random permutation of all cells.  Two warm-up calls, then CUDA events around --reps calls on one stream.  bytes/s
   counts the 8 B read and 32 B written per cell; the share is of the H100 SXM data-sheet HBM3 bandwidth, 3.35 TB/s (a data-sheet figure,
   not a measured peak).  Each cell also costs two Montgomery multiplications, so the point states its multiplication rate against the
   integer-multiply ceiling of DESIGN.md section 4 (SMs x 64 product words per clock x maximum SM clock / 264 words per multiplication),
   computed from the SM count and maximum clock of the card it ran on.
2. The permutation half of keygen at k = 22, P = 32 (extended domain 2^25, the quotient degree of the reference key): sigmas ->
   inverse NTT (Lagrange -> coefficients) -> coset NTT onto the extended domain -> commitments of the sigma columns against a 2^22-point
   base table (commit_lagrange).  The coset transforms run in batches of 8 columns into one reused 8-column buffer (all 32 cosets and the
   transform scratch would not fit beside the rest).  The base table is built before the clock starts.  Each stage is timed with CUDA
   events, one warm-up pass first.  The CPU arm is the oracle on the host cores: halo2's sigma algorithm for all 32 columns, and the
   inverse NTT, coset NTT and MSM of ONE column (per-column time; the 32-column figure is 32 x that, labelled as such).
The card's name, power limit and maximum SM clock are read in the same run.  One JSON line per point on stdout (and in --out)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_DATASHEET = 3.35e12          # B/s, H100 SXM data sheet


def random_mapping(P, k, seed=0):
    import torch
    n = 1 << k
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    perm = torch.randperm(P * n, device="cuda", generator=g)
    m = torch.stack([(perm >> k).to(torch.int32), (perm & (n - 1)).to(torch.int32)], dim=-1).reshape(P, n, 2).contiguous()
    del perm
    return m


def kernel_point(k, P, reps, mul_ceiling):
    import torch
    from ezkl_b200 import device as dv
    m = random_mapping(P, k)
    out = torch.empty((P, 1 << k, 4), dtype=torch.int64, device="cuda")
    for _ in range(2):
        dv.permutation_sigmas(m, k, out=out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        dv.permutation_sigmas(m, k, out=out)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / reps
    cells = P << k
    bps = 40 * cells / (ms * 1e-3)
    del m, out
    torch.cuda.empty_cache()
    return {"bench": "perm_sigmas_kernel", "k": k, "P": P, "cells": cells, "reps": reps, "ms": round(ms, 4), "GB_per_s": round(bps / 1e9, 1), "share_of_datasheet_hbm": round(bps / HBM_DATASHEET, 3),
            "G_mulmod_per_s": round(2 * cells / (ms * 1e-3) / 1e9, 1), "share_of_multiply_ceiling": round(2 * cells / (ms * 1e-3) / mul_ceiling, 3)}


def keygen_half(k, P):
    import numpy as np
    import torch
    from ezkl_b200 import device as dv
    from ezkl_b200 import fields as F
    from ezkl_b200 import halo2 as h2
    from oracle import oracle as orc
    from tests import perm_keygen_ref as ref
    dom = h2.EvaluationDomain(9, k)
    n, N, ext_k = 1 << k, 1 << dom.extended_k, dom.extended_k
    bases_d = dv.generate_bases(n, seed=7)
    bases = dv.DeviceBases(bases_d)
    m = random_mapping(P, k, seed=1)
    sig = torch.empty((P, n, 4), dtype=torch.int64, device="cuda")
    polys = torch.empty_like(sig)
    tmp = torch.empty_like(sig)
    B = 8
    coset = torch.empty((B, N, 4), dtype=torch.int64, device="cuda")
    ctmp = torch.empty((B, N, 4), dtype=torch.int64, device="cuda")
    one, zeta = F.fr_to_limbs(1), dom.g_coset
    zeta2 = F.fr_to_limbs(F.FR_ZETA * F.FR_ZETA % F.FR_MODULUS)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]

    def run():
        ev[0].record()
        dv.permutation_sigmas(m, k, out=sig)
        ev[1].record()
        dv.ntt(sig, k, dom.omega_inv, post=[dom.ifft_divisor], out=polys, tmp=tmp)
        ev[2].record()
        for b0 in range(0, P, B):
            dv.ntt(polys[b0:b0 + B], ext_k, dom.extended_omega, n_in=n, pre=[one, zeta, zeta2], out=coset, tmp=ctmp)
        ev[3].record()
        xyzz = dv.msm_batch(bases, sig)
        ev[4].record()
        ev[4].synchronize()
        return xyzz

    run()
    xyzz = run()
    t = [ev[i].elapsed_time(ev[i + 1]) for i in range(4)]
    gpu = {"sigmas_ms": round(t[0], 3), "intt_ms": round(t[1], 3), "coset_ntt_ms": round(t[2], 3), "commit_ms": round(t[3], 3), "total_ms": round(sum(t), 3)}
    # CPU arm: the oracle on the host cores
    threads = orc.host_threads()
    m_h = m.cpu().numpy().view(np.uint32)
    t0 = time.perf_counter()
    sig_h = ref.perm_sigmas(m_h, k)
    t_sig = time.perf_counter() - t0
    assert np.array_equal(sig_h, dv.to_host(sig)), "device sigmas differ from halo2's algorithm"
    j = P - B                                      # the first column of the last coset batch, which `coset` still holds
    col = np.ascontiguousarray(sig_h[j])
    del sig_h
    t0 = time.perf_counter()
    p0 = orc.lagrange_to_coeff(col, k, threads)
    t_intt = time.perf_counter() - t0
    t0 = time.perf_counter()
    c0 = orc.coeff_to_extended(p0, ext_k, threads)
    t_coset = time.perf_counter() - t0
    bh = dv.to_host(bases_d)
    t0 = time.perf_counter()
    pt = orc.msm(col, bh, threads)
    t_msm = time.perf_counter() - t0
    assert np.array_equal(p0, dv.to_host(polys[j])) and np.array_equal(c0, dv.to_host(coset[0])), "transforms differ from the oracle"
    assert np.array_equal(pt, dv.normalize(xyzz[j:j + 1])[0, :8]), "commitment differs from the oracle"
    per_col = (t_intt + t_coset + t_msm) * 1e3
    cpu = {"threads": threads, "sigmas_ms_all_columns": round(t_sig * 1e3, 1), "intt_ms_one_column": round(t_intt * 1e3, 1),
           "coset_ntt_ms_one_column": round(t_coset * 1e3, 1), "commit_ms_one_column": round(t_msm * 1e3, 1),
           "total_ms_32x_one_column_plus_sigmas": round(t_sig * 1e3 + P * per_col, 1)}
    bases.release()
    return {"bench": "perm_keygen_half", "k": k, "ext_k": ext_k, "P": P, "gpu": gpu, "cpu_oracle": cpu,
            "speedup_total": round(cpu["total_ms_32x_one_column_plus_sigmas"] / gpu["total_ms"], 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="20,22,24,26")
    ap.add_argument("--ps", default="8,32,128")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--max-gib", type=float, default=24.0, help="skip kernel points whose mapping + result exceed this")
    ap.add_argument("--keygen-k", type=int, default=22)
    ap.add_argument("--keygen-p", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from ezkl_b200 import _native as nat
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    nat.init(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    sms, clock_mhz = torch.cuda.get_device_properties(0).multi_processor_count, float(card.split(",")[-1].split()[0])
    mul_ceiling = sms * 64 * clock_mhz * 1e6 / 264
    lines = [json.dumps({"card": card, "sms": sms, "multiply_ceiling_G_mulmod_per_s": round(mul_ceiling / 1e9, 1), "torch": torch.__version__})]
    print(lines[-1], flush=True)
    for k in [int(x) for x in a.ks.split(",") if x]:
        for P in [int(x) for x in a.ps.split(",") if x]:
            if 40 * (P << k) > a.max_gib * (1 << 30):
                lines.append(json.dumps({"bench": "perm_sigmas_kernel", "k": k, "P": P, "skipped": "mapping + result > %.0f GiB" % a.max_gib}))
            else:
                lines.append(json.dumps(kernel_point(k, P, a.reps, mul_ceiling)))
            print(lines[-1], flush=True)
    if a.keygen_k:
        lines.append(json.dumps(keygen_half(a.keygen_k, a.keygen_p)))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
