#!/usr/bin/env python
"""MSM cost of the base-table level count (memory-bounded tables, ezkl_b200.h): for each k and every level count L that fits on
the card, the registration time, the table bytes, the MSM time and pairs/s at batch 1 and 8 (CUDA events after a warm-up), and
the device time of the bucket scan, the bucket reduction and the sub-window fold from the library's profile classes.

One JSON line per configuration, each carrying the card name and power limit read in the same run.
Usage: python tools/bench_msm_levels.py [k ...]      (default 20 22 24 25 26)
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from ezkl_b200 import _native as nat  # noqa: E402
from ezkl_b200 import device as dev  # noqa: E402

PROF = {"accumulate": 0, "total": 1, "recode": 4, "tail": 5, "scan": 7, "reduce": 8, "fold": 9}


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, float(power)


def level_counts(W):
    """(s, L) for every distinct level count: the smallest s giving each L = ceil(W / s)."""
    seen = {}
    for s in range(1, W + 1):
        seen.setdefault(-(-W // s), s)
    return sorted(((s, L) for L, s in seen.items()), key=lambda t: t[1], reverse=True)


def time_msm(bases, sc, reps):
    dev.msm_batch(bases, sc)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        dev.msm_batch(bases, sc)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def profile_msm(bases, sc):
    """Device time per class of one MSM call (a separate run: the events cost host time)."""
    L = nat.lib()
    nat.check(L.b200_profile_enable(1))
    dev.msm_batch(bases, sc)
    torch.cuda.synchronize()
    res = {}
    for name, cls in PROF.items():
        ms, cnt = C.c_double(0), C.c_uint64(0)
        nat.check(L.b200_profile_read(cls, C.byref(ms), C.byref(cnt)))
        res[name + "_ms"] = round(ms.value, 3)
    nat.check(L.b200_profile_enable(0))
    return res


def main(ks):
    nat.init(0)
    name, power = card()
    for k in ks:
        n = 1 << k
        pts = dev.generate_bases(n, seed=3)
        sc8 = dev.random_scalars(n, batch=8, seed=5)
        torch.cuda.synchronize()
        c = 20 if k >= 22 else (18 if k >= 20 else 17)          # msm_default_window for these k
        W = (255 + c - 1) // c
        for s, L in level_counts(W):
            rec = {"card": name, "power_limit_w": power, "k": k, "window_bits": c, "levels": L, "windows_per_level": s}
            torch.cuda.empty_cache()
            try:
                t0 = time.perf_counter()
                bases = dev.DeviceBases(pts, max_table_bytes=L * n * 64)
                torch.cuda.synchronize()
                rec["register_s"] = round(time.perf_counter() - t0, 4)
            except nat.B200Error as e:
                rec["skipped"] = "table does not fit: %s" % e
                print(json.dumps(rec), flush=True)
                continue
            info = bases.info()
            assert (info["levels"], info["windows_per_level"]) == (L, s), info
            rec["table_bytes"] = info["table_bytes"]
            try:
                for batch in (1, 8):
                    sc = sc8[:batch]
                    ms = time_msm(bases, sc, reps=2 if k >= 25 else 3)
                    rec["b%d_ms" % batch] = round(ms, 3)
                    rec["b%d_pairs_per_s" % batch] = round(batch * n / ms * 1e3, 1)
                    rec["b%d_profile" % batch] = profile_msm(bases, sc)
            except nat.B200Error as e:
                rec["error"] = str(e)
            bases.release()
            print(json.dumps(rec), flush=True)
        del pts, sc8
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main([int(x) for x in sys.argv[1:]] or [20, 22, 24, 25, 26])
