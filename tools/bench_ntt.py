#!/usr/bin/env python
"""NTT throughput sweep on the GPU box (device-resident, CUDA events): G elts/s per (log_n, batch)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from ezkl_b200 import _native as nat  # noqa: E402
from ezkl_b200 import device as dev  # noqa: E402
from ezkl_b200 import fields as F  # noqa: E402


def omega(k):
    return F.fr_to_limbs(pow(F.FR_ROOT_OF_UNITY, 1 << (F.FR_S - k), F.FR_MODULUS))


def run(log_n, batch, reps=5):
    n = 1 << log_n
    src = dev.random_scalars(n, batch=batch, seed=log_n)
    out = torch.empty_like(src)
    tmp = torch.empty_like(src)
    w = omega(log_n)
    for _ in range(2):
        dev.ntt(src, log_n, w, out=out, tmp=tmp)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        dev.ntt(src, log_n, w, out=out, tmp=tmp)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    return batch * n / ms / 1e6, ms


if __name__ == "__main__":
    nat.init(0)
    for log_n, batch in ((17, 32), (19, 16), (20, 8), (20, 32), (22, 2), (23, 2), (25, 1)):
        g, ms = run(log_n, batch)
        print("log_n=%2d batch=%3d  %8.3f ms  %7.3f G elts/s  (%5.1f GB/s algorithmic)" % (log_n, batch, ms, g, g * 64), flush=True)
