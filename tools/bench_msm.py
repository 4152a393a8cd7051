#!/usr/bin/env python
"""MSM throughput sweep on the GPU box (device-resident, CUDA events): M pairs/s per (k, batch, window bits)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from ezkl_b200 import _native as nat  # noqa: E402
from ezkl_b200 import device as dev  # noqa: E402
import gpu_peaks  # noqa: E402


def run(bases, sc, reps=3):
    dev.msm_batch(bases, sc)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        dev.msm_batch(bases, sc)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def sweep():
    """BASELINE configs[3]: standalone MSM sweep 2^16 .. 2^26 on one GPU (default window), batch 1 and 4."""
    import json
    peak, peak_src = gpu_peaks.hbm_peak_gbs()
    print("# hbm_frac against %.0f GB/s (%s)" % (peak, peak_src), flush=True)
    res = []
    for k in range(16, 27, 2):
        n = 1 << k
        pts = dev.generate_bases(n, seed=3)
        bases = dev.DeviceBases(pts)
        del pts
        torch.cuda.empty_cache()
        for batch in (1, 4):
            if k >= 26 and batch > 1:
                continue
            sc = dev.random_scalars(n, batch=batch, seed=5)
            ms = run(bases, sc, reps=2 if k >= 24 else 3)
            res.append({"k": k, "batch": batch, "ms": round(ms, 3), "pairs_per_s": round(batch * n / ms * 1e3, 1), "hbm_frac": round(batch * n * (32 + 64 / batch) / (ms * 1e-3) / (peak * 1e9), 5)})
            print(res[-1], flush=True)
            del sc
        bases.release()
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    nat.init(0)
    if len(sys.argv) > 1 and sys.argv[1] == "one":          # one k=17, c=16, batch-60 call after a warm-up (for ncu launch lists)
        n = 1 << 17
        bases = dev.DeviceBases(dev.generate_bases(n, seed=3), window_bits=16)
        batches = [int(x) for x in sys.argv[2].split(",")] if len(sys.argv) > 2 else [60]
        for b in batches:
            sc = dev.random_scalars(n, batch=b, seed=5)
            ms = run(bases, sc, reps=3)
            print("k=17 c=16 batch=%d: %.3f ms  (%.1f M pairs/s, accumulate path: B200_MSM_AFFINE=%s)" % (b, ms, b * n / ms / 1e3, os.environ.get("B200_MSM_AFFINE", "default")), flush=True)
            del sc
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "sweep":
        sweep()
        sys.exit(0)
    ks = [int(x) for x in (sys.argv[1] if len(sys.argv) > 1 else "17,20").split(",")]
    for k in ks:
        n = 1 << k
        pts = dev.generate_bases(n, seed=3)
        for c in ([14, 15, 16, 17] if k == 17 else ([16, 17, 18, 19] if k <= 20 else [18, 19, 20, 21])):
            bases = dev.DeviceBases(pts, window_bits=c)
            for batch, small in ((1, None), (8, None), (60, None), (60, 16)) if k <= 17 else ((1, None), (8, None), (8, 16)):
                sc = dev.random_scalars(n, batch=batch, seed=5, small_bits=small)
                ms = run(bases, sc)
                print("k=%2d c=%2d batch=%3d %-10s %9.3f ms  %8.1f M pairs/s" % (k, c, batch, "small16" if small else "uniform", ms, batch * n / ms / 1e3), flush=True)
                del sc
            bases.release()
