#!/usr/bin/env python
"""b200_evaluate_h on the ezkl-sized system of tools/bench_quotient.py (132 columns: advice, z, m and phi in coefficient form, n each;
selectors, tables, sigmas and the l-polynomials on the extended domain), d = 8, the way a prover calls it (finish=True).

Each point runs in its own child process, because B200_WS_BUDGET_MB is read once, at b200_init: 1 MiB forces the parts path, a budget
above n_columns * 2^ext_k * 32 B the full-coset path.  Both paths at k = 16 ... 20, the parts path alone at k = 21 and 22.  A point is a
host clock around the synchronous call (it returns after its download), --reps times after one warm-up call, plus one extra call with
the library's CUDA-event profile on (NTT and evaluate_h kernel classes).  "device_gib" is the device memory the library holds
after the calls: its scratch never shrinks, so that is the call's peak.  Extended columns cycle through 4 host buffers (a k = 22
column is 1 GiB); each is still gathered and uploaded per column.  One JSON line per point on stdout (and in --out, when given)."""
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


def child(k, reps):
    import numpy as np
    import torch
    from bench_quotient import ezkl_system
    from ezkl_b200 import _native as nat
    from ezkl_b200 import evaluation as ev
    from ezkl_b200 import halo2 as h2
    nat.init(0)
    torch.cuda.init()
    dom = h2.EvaluationDomain(9, k)
    n, N = dom.n, 1 << dom.extended_k
    prog, ncols, coeff = ezkl_system(8)
    g = np.random.default_rng(k)

    def rand(rows):
        a = g.integers(0, 2**64, size=(rows, 4), dtype=np.uint64)
        a[:, 3] &= (1 << 60) - 1
        return a

    base, exts = rand(n + ncols), [rand(N) for _ in range(4)]
    polys = [base[i:i + n] if i in coeff else exts[i % 4] for i in range(ncols)]
    free0 = torch.cuda.mem_get_info()[0]
    ev.evaluate_h_from_polys(prog, polys, dom, finish=True)
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        ev.evaluate_h_from_polys(prog, polys, dom, finish=True)
        times.append(time.perf_counter() - t0)
    held = free0 - torch.cuda.mem_get_info()[0]
    L = nat.lib()
    nat.check(L.b200_profile_enable(1))
    ev.evaluate_h_from_polys(prog, polys, dom, finish=True)
    prof = {}
    for cls, name in ((2, "ntt"), (6, "evaluate_h")):
        ms, cnt = C.c_double(), C.c_uint64()
        nat.check(L.b200_profile_read(cls, C.byref(ms), C.byref(cnt)))
        prof[name] = {"ms": round(ms.value, 2), "launches": cnt.value}
    nat.check(L.b200_profile_enable(0))
    print(json.dumps({"k": k, "ext_k": dom.extended_k, "columns": ncols, "coefficient_columns": len(coeff),
                      "path": "parts" if prof["evaluate_h"]["launches"] > 1 else "full", "budget_mb": int(os.environ.get("B200_WS_BUDGET_MB", "0")),
                      "s": [round(t, 4) for t in times], "median_s": round(statistics.median(times), 4), "spread_s": round(max(times) - min(times), 4),
                      "device_gib": round(held / 2**30, 2), "device_classes_one_call": prof}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--both", default="16,17,18,19,20", help="k values timed on both paths")
    ap.add_argument("--parts-only", default="21,22", help="k values timed on the parts path alone")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    ap.add_argument("--child", type=int, default=None)
    a = ap.parse_args()
    if a.child is not None:
        child(a.child, a.reps)
        return
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = open(a.out, "w") if a.out else None
    lines = [json.dumps({"card": card})]
    print(lines[0], flush=True)
    points = [(k, p) for k in [int(x) for x in a.both.split(",") if x] for p in ("full", "parts")]
    points += [(k, "parts") for k in [int(x) for x in a.parts_only.split(",") if x]]
    for k, path in points:
        env = dict(os.environ)
        full_bytes = 132 * (1 << (k + 3)) * 32
        env["B200_WS_BUDGET_MB"] = "1" if path == "parts" else str((full_bytes >> 20) + 1024)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", str(k), "--reps", str(a.reps)], env=env, capture_output=True, text=True)
        line = r.stdout.strip().splitlines()[-1] if r.returncode == 0 and r.stdout.strip() else json.dumps({"k": k, "path": path, "error": (r.stdout + r.stderr)[-1500:]})
        print(line, flush=True)
        lines.append(line)
    if out:
        out.write("\n".join(lines) + "\n")
        out.close()


if __name__ == "__main__":
    main()
