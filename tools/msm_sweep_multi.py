#!/usr/bin/env python
"""python tools/msm_sweep_multi.py N : BASELINE configs[3], MSM 2^16..2^26 through b200_msm_sharded_dev on N = 1, 2, 4 or 8 devices of one
process, host-clocked, oracle-checked at k <= 18; at N >= 2 also b200_ntt_sharded_dev against b200_ntt_dev on device 0 (byte-equal)."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from ezkl_b200 import _native as nat  # noqa: E402
from oracle import oracle as orc  # noqa: E402


def timed(fn, reps):
    fn()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return round((time.perf_counter() - t0) / reps * 1e3, 3)


def main():
    nd, L, top = int(sys.argv[1]), nat.lib(), 1 << 26
    nat.check(L.b200_init_multi(nd))
    cards = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).splitlines()[:nd]

    def alloc(slot, nbytes):
        p = C.c_void_p(0)
        nat.check(L.b200_dev_alloc_on(slot, C.byref(p), nbytes))
        return p
    arr, d_bases, bases = C.c_void_p * nd, alloc(0, top * 64), np.zeros((1 << 18, 8), np.uint64)
    nat.check(L.b200_g1_generate_dev(3, top, d_bases, None))       # point i depends on (seed, i) only: each k registers a prefix
    nat.check(L.b200_dev_download(nat.ptr(bases), d_bases, bases.nbytes))
    slices = [alloc(s, top // nd * 32) for s in range(nd)]
    if nd > 1:      # NTT scratch and output slices; source, scratch and output of the one-device transform on device 0
        tmps, dsts, one = [alloc(s, top // nd * 32) for s in range(nd)], [alloc(s, top // nd * 32) for s in range(nd)], [alloc(0, top * 32) for _ in range(3)]
    for k in range(16, 27, 2):
        n, sl, reps, handle, out = 1 << k, (1 << k) // nd, 2 if k >= 24 else 3, C.c_uint64(0), np.zeros((1, 12), np.uint64)
        sc = np.random.default_rng(5).integers(0, 1 << 64, (n, 4), dtype=np.uint64) & np.array([2**64 - 1] * 3 + [2**60 - 1], np.uint64)
        nat.check(L.b200_bases_register_ex_dev(d_bases, n, 0, 0, C.byref(handle)))
        for s in range(nd):
            nat.check(L.b200_dev_upload(slices[s], nat.ptr(sc[s * sl:(s + 1) * sl]), sl * 32))
        ms = timed(lambda: nat.check(L.b200_msm_sharded_dev(handle, arr(*slices), n, 1, nat.ptr(out))), reps)
        nat.check(L.b200_bases_release(handle))
        assert k > 18 or np.array_equal(out[0, :8], orc.msm(sc, bases[:n], orc.host_threads())), "sharded MSM != oracle at k=%d" % k
        rec = {"k": k, "n_gpus": nd, "ms": ms, "pairs_per_s": round(n / ms * 1e3, 1), "oracle_checked": k <= 18, "gpus": cards}
        if nd > 1:
            w, got, ref = orc.omega(k), np.zeros((n, 4), np.uint64), np.zeros((n, 4), np.uint64)
            nat.check(L.b200_dev_upload(one[0], nat.ptr(sc), n * 32))
            rec["ntt_ms_sharded"] = timed(lambda: (nat.check(L.b200_ntt_sharded_dev(arr(*slices), arr(*tmps), arr(*dsts), k, n, nat.ptr(w), 0, None, 0, None)), nat.check(L.b200_sync_all())), reps)
            rec["ntt_ms_single_gpu"] = timed(lambda: (nat.check(L.b200_ntt_dev(one[0], n, n, one[1], one[2], n, k, nat.ptr(w), 0, None, 0, None, 1, None)), nat.check(L.b200_sync())), reps)
            for s in range(nd):
                nat.check(L.b200_dev_download(nat.ptr(got[s * sl:(s + 1) * sl]), dsts[s], sl * 32))
            nat.check(L.b200_dev_download(nat.ptr(ref), one[2], n * 32))
            assert np.array_equal(got, ref), "sharded NTT != one-device NTT at k=%d" % k
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
