#!/usr/bin/env python
"""Hybrid-multiplier experiment (run on the GPU box): checks the FP64-pipe multiplier (csrc/fd.cuh) on the device against
bigints and measures multiply throughput when r of every 8 warps use it while the others use the integer-pipe multiplier."""
import ctypes as C
import os
import random
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezkl_b200 import _native as nat  # noqa: E402
import gpu_peaks  # noqa: E402

P = 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47
R = 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001


def limbs(x):
    return np.array([(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def main():
    nat.init(0)
    D = nat.dbg_lib()
    rng = random.Random(5)
    for fid, N in ((0, R), (1, P)):
        xs = [rng.getrandbits(256) for _ in range(4096)] + [0, 1, N - 1, (1 << 256) - 1]
        ys = [rng.getrandbits(256) for _ in range(4096)] + [N - 1, (1 << 256) - 1, N - 1, (1 << 256) - 1]
        a, b = np.stack([limbs(x) for x in xs]), np.stack([limbs(y) for y in ys])
        out = np.zeros_like(a)
        nat.check(D.b200_debug_fd_mul(C.c_int(fid), nat.ptr(a), nat.ptr(b), nat.ptr(out), C.c_size_t(len(xs))))
        rinv = pow(1 << 260, -1, N)
        bad = 0
        for i, (x, y) in enumerate(zip(xs, ys)):
            v = sum(int(out[i, j]) << (64 * j) for j in range(4))
            if v % N != x * y * rinv % N or v >= 2 * N:
                bad += 1
        print("fd_mul on device, field %d: %d cases, %d mismatches" % (fid, len(xs), bad), flush=True)
    for threads, bps in ((256, 2), (256, 4), (256, 8)):
        for r in range(9):
            iters, blocks = 2000, gpu_peaks.sm_count() * bps
            ms = C.c_float(0)
            nat.check(D.b200_debug_bench(10 + r, iters, blocks, threads, C.byref(ms)))
            ops = blocks * threads * iters
            print("hybrid mul chain: %d/8 warps on the FP64 pipe  threads/SM=%5d  %8.3f ms  %8.2f G mul/s" % (r, threads * bps, ms.value, ops / ms.value / 1e6), flush=True)


if __name__ == "__main__":
    main()
