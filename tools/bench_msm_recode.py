#!/usr/bin/env python
"""Per-kernel times of one MSM call at the call shapes of bench.py (run on the GPU box).

Each shape is timed twice: the whole call with CUDA events, then every kernel of the call with torch.profiler in a run of its
own (nothing else profiled).  For the recoding kernels the line also gives entries/s, where entries = batch x n x W (one per
window digit; the few zero digits are counted too).  `--equal` adds the same shapes with every scalar of a column equal, so
that all digits of a window land in one bucket.

  python tools/bench_msm_recode.py [--reps 10] [--equal] [--json OUT]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from ezkl_b200 import _native as nat  # noqa: E402
from ezkl_b200 import device as dev  # noqa: E402

# (k, window bits, batch): the six MSM batches of one bench.py --k 17 step, then the k = 20 batch-8 commitment
SHAPES = [(17, 16, 60), (17, 16, 20), (17, 16, 26), (17, 16, 1), (17, 16, 7), (17, 16, 2), (20, 18, 8)]
RECODE = ("k_digits", "k_scan_buckets", "k_fill_chunks", "k_len_offsets", "k_order_chunks", "Memset")


def short_name(name):
    """'void b200::k_digits<true, false>(...)' -> 'k_digits<true, false>' (template flags kept: they tell the passes apart)."""
    s = name.split("(")[0]
    s = s.replace("void ", "").replace("b200::", "")
    return s.strip()


def time_call(bases, sc, reps):
    dev.msm_batch(bases, sc)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        dev.msm_batch(bases, sc)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def profile_call(bases, sc, reps):
    dev.msm_batch(bases, sc)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            dev.msm_batch(bases, sc)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        key = short_name(ev.name)
        t, c = per.get(key, (0.0, 0))
        per[key] = (t + ev.device_time / 1e3, c + 1)      # device_time is in us
    return {k: (t / reps, c / reps) for k, (t, c) in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--equal", action="store_true", help="also time columns whose scalars are all equal")
    ap.add_argument("--json", default=None, help="write the rows to this file as JSON lines")
    a = ap.parse_args()
    nat.init(0)
    props = torch.cuda.get_device_properties(0)
    try:
        card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        card = props.name
    print("# %s (%d SMs)" % (card, props.multi_processor_count), flush=True)
    rows, tables = [], {}
    for k, c, batch in SHAPES:
        n = 1 << k
        if (k, c) not in tables:
            tables[(k, c)] = dev.DeviceBases(dev.generate_bases(n, seed=3), window_bits=c)
        bases = tables[(k, c)]
        W = (255 + c - 1) // c
        for dist in (("uniform", "equal") if a.equal else ("uniform",)):
            sc = dev.random_scalars(n, batch=batch, seed=5)
            if dist == "equal":
                sc[:] = sc[:, :1].clone()
            call_ms = time_call(bases, sc, a.reps)
            per = profile_call(bases, sc, a.reps)
            entries = batch * n * W
            recode = {kname: v for kname, v in per.items() if kname.startswith(RECODE)}
            recode_ms = sum(t for t, _ in recode.values())
            row = {"k": k, "c": c, "batch": batch, "scalars": dist, "call_ms": round(call_ms, 4), "entries": entries,
                   "recode_ms": round(recode_ms, 4), "kernels": {kname: {"ms": round(t, 4), "launches": cnt, "G_entries_per_s": round(entries / (t * 1e6), 2) if t > 0 else None}
                                                            for kname, (t, cnt) in sorted(per.items())}}
            rows.append(row)
            print("k=%d c=%d batch=%2d %-7s call %8.3f ms  recode kernels %7.3f ms (%5.1f G entries/s)" % (k, c, batch, dist, call_ms, recode_ms, entries / (recode_ms * 1e6)), flush=True)
            for kname, (t, cnt) in sorted(per.items(), key=lambda kv: -kv[1][0]):
                print("    %-34s %8.4f ms  %4.1f launches  %7.1f G entries/s" % (kname, t, cnt, entries / (t * 1e6) if t > 0 else 0.0), flush=True)
            del sc
    if a.json:
        with open(a.json, "w") as f:
            for r in rows:
                f.write(json.dumps(dict(r, card=card)) + "\n")


if __name__ == "__main__":
    main()
