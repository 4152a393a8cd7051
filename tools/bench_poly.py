#!/usr/bin/env python
"""Column-polynomial kernels against the HBM roofline (run on an H100): the only genuinely bandwidth-bound kernels on the path.
For each op and size, CUDA-event time over buffers larger than L2 (batch of columns back to back), algorithmic bytes per element
(BASELINE.md §3: add/sub/mul/axpy 96 B, scale / scale_cycle / batch_invert 64 B, eval 32 B, scans / kate_division 64 B) and the
fraction of the measured copy bandwidth (MEASURED_PEAKS.json)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from ezkl_b200 import _native as nat  # noqa: E402
from ezkl_b200 import device as dev  # noqa: E402
from ezkl_b200 import fields as F  # noqa: E402
import gpu_peaks  # noqa: E402


def timeit(fn, reps=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    nat.init(0)
    peak, peak_src = gpu_peaks.hbm_peak_gbs()
    one = F.fr_to_limbs(1)
    s = F.fr_to_limbs(0x1234567)
    print("# op, log2(n), columns, ms, G elts/s, algorithmic GB/s, fraction of the HBM peak (%.0f GB/s, %s)" % (peak, peak_src))
    for k, batch in ((17, 96), (20, 12), (22, 3)):
        n = 1 << k
        a = dev.random_scalars(n, batch=batch, seed=1)
        b = dev.random_scalars(n, batch=batch, seed=2)
        out = torch.empty_like(a)
        flat_a, flat_b, flat_o = a.view(-1, 4), b.view(-1, 4), out.view(-1, 4)
        tot = n * batch
        xs = dev.to_host(dev.random_scalars(batch, seed=3))
        cyc = np.ascontiguousarray(np.stack([one, s, one, s, s, one, s, s]))
        rows = [
            ("add", 96, tot, lambda: dev.poly_op("add", flat_a, flat_b, out=flat_o)),
            ("mul", 96, tot, lambda: dev.poly_op("mul", flat_a, flat_b, out=flat_o)),
            ("scale", 64, tot, lambda: dev.poly_op("scale", flat_a, s=s, out=flat_o)),
            ("axpy", 96, tot, lambda: dev.poly_op("axpy", flat_a, flat_b, s=s, out=flat_o)),
            ("scale_cycle(8)", 64, tot, lambda: dev.scale_cycle(flat_o, cyc)),
            ("lincomb(%d)" % batch, 32 * (batch + 1) / batch, tot, lambda: dev.lincomb([a[i] for i in range(batch)], np.tile(s, (batch, 1)), out=out[0])),
            ("eval_batch", 32, tot, lambda: dev.eval_batch(a, xs)),
            ("batch_invert", 64, tot, lambda: dev.batch_invert(flat_o)),
            ("prefix_product", 64, n, lambda: dev.prefix_scan(a[0], one, True, out=out[0])),
            ("prefix_sum", 64, n, lambda: dev.prefix_scan(a[0], one, False, out=out[0])),
            ("kate_division", 64, n, lambda: dev.kate_division(a[0], xs[0], out=out[0][: n - 1])),
        ]
        out.copy_(a)
        for name, bpe, elts, fn in rows:
            ms = timeit(fn)
            gbs = elts * bpe / (ms * 1e-3) / 1e9
            print("%-16s %2d %3d %9.4f ms %8.2f G elts/s %8.1f GB/s  %5.1f %%" % (name, k, batch if elts == tot else 1, ms, elts / (ms * 1e-3) / 1e9, gbs, 100 * gbs / peak), flush=True)


if __name__ == "__main__":
    main()
