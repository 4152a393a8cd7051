#!/usr/bin/env python
"""Proving-key loading: a RawBytes key file straight to the device (device.load_proving_key -> b200_pk_load: only the value columns are read,
checked on the device, and the polys and l-cosets derived there) against the host route's lower bound (every byte of the file read in order,
as ProvingKey::read reads it, through a bounded buffer, then values, polys and l-vectors uploaded with b200_dev_upload; halo2's per-element
checks are not part of it).

Cases k:fixed:permutation:ext_k, default 17:38:32:20 (the bench trace's shape at k = 17), 20:38:32:23 and 22:8:8:25 (about 23 GiB each).  The
keys are real RawBytes files written with ProvingKey.write: random canonical values, the derived sections made by the device keygen
(ProvingKey.keygen_pk_polys), a vk prefix of zero commitments and no selectors.  Each is written to a temporary directory deleted at the end,
after free disk and host memory are checked (a case that does not fit prints a "skipped" line with the reason), and read once before timing
so that the page cache is warm; cold-cache reads are not measured (dropping the page cache needs privileges this tool does not use).  Both
arms are synchronous and timed with a host clock, alternated call by call: one warm-up pair, then --reps pairs; the line reports the median
and max - min of each, the bytes of the file each arm reads, and whether both arms' device outputs are equal.

--profile adds a pass of its own under torch.profiler: k_fr_validate's device time per call (one call per column) against the data-sheet
HBM bound of 32 B per element at 3.35 TB/s.

The card's name, power limit and maximum SM clock are read in the same run.  One JSON line per point on stdout (and in --out)."""
import argparse
import json
import os
import shutil
import statistics
import struct
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_DATASHEET = 3.35e12          # B/s, H100 SXM data sheet
CASES = [(17, 38, 32, 20), (20, 38, 32, 23), (22, 8, 8, 25)]
BLINDING = 5
READ_BUF = 64 << 20
GIB = 1 << 30


def file_bytes(k, nf, npc, ext_k):
    n, N, c = 1 << k, 1 << ext_k, nf + npc
    vk = 7 + 64 * c
    return vk + 3 * (4 + 32 * N) + 6 * 4 + 3 * 4 * c + c * (2 * (4 + 32 * n) + 4 + 32 * N)


def j_for(k, ext_k):
    return (1 << (ext_k - k)) + 1


def write_key(path, k, nf, npc, ext_k):
    import torch
    from ezkl_b200 import device as dev
    from ezkl_b200 import halo2 as h2
    n = 1 << k
    pk = h2.ProvingKey()
    pk.k = k
    pk.vk_bytes = bytes([3, k, 1]) + struct.pack("<I", nf) + bytes(64 * (nf + npc))
    cols = [dev.to_host(dev.random_scalars(n, seed=1000 * k + j)).copy() for j in range(nf + npc)]
    pk.fixed_values, pk.permutations = cols[:nf], cols[nf:]
    der = pk.keygen_pk_polys(j_for(k, ext_k), BLINDING)
    for name, v in der.items():
        setattr(pk, name, v)
    pk.write(path)
    del pk, der, cols
    torch.cuda.empty_cache()
    assert os.path.getsize(path) == file_bytes(k, nf, npc, ext_k)


def warm_page_cache(path):
    with open(path, "rb") as f:
        while f.read(READ_BUF):
            pass


def host_available_bytes():
    try:
        return os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    except (ValueError, OSError):
        return 0


def new_arm(path, npc, ext_k):
    import torch
    from ezkl_b200 import device as dev
    t0 = time.perf_counter()
    key = dev.load_proving_key(path, npc, 0, ext_k, BLINDING)
    dt = time.perf_counter() - t0
    torch.cuda.synchronize()
    return dt, (key.values, key.polys, torch.stack([key.l0, key.l_last, key.l_active_row]))


def old_arm(path, npc, ext_k):
    """Every byte of the file in order, as ProvingKey::read reads it; each values / polys / l-vector column is read into one reused host
    buffer and uploaded (b200_dev_upload) before the next is read, and the cosets are read through the same bounded buffer and dropped."""
    import numpy as np
    import torch
    from ezkl_b200 import _native as nat
    t0 = time.perf_counter()
    with open(path, "rb") as f:
        head = f.read(7)
        k, nf = head[1], struct.unpack("<I", head[3:7])[0]
        n, N, c = 1 << k, 1 << ext_k, nf + npc
        f.read(64 * c)
        values = torch.empty((c, n, 4), dtype=torch.int64, device="cuda")
        polys = torch.empty_like(values)
        l = torch.empty((3, N, 4), dtype=torch.int64, device="cuda")
        buf = np.empty(32 * max(N, READ_BUF // 32), np.uint8)
        view = memoryview(buf)
        read_bytes = 7 + 64 * c

        def column(dst):
            nonlocal read_bytes
            (ln,) = struct.unpack(">I", f.read(4))
            nb = 32 * ln
            got = f.readinto(view[:nb])
            assert got == nb
            read_bytes += 4 + nb
            if dst is not None:
                nat.check(nat.lib().b200_dev_upload(dst.data_ptr(), buf.ctypes.data, nb))

        def slice_(dsts, cnt):
            nonlocal read_bytes
            (got,) = struct.unpack(">I", f.read(4))
            assert got == cnt
            f.read(4 * cnt)
            read_bytes += 4 + 4 * cnt
            for j in range(cnt):
                column(None if dsts is None else dsts[j])
        for i in range(3):
            column(l[i])
        slice_(values[:nf], nf)
        slice_(polys[:nf], nf)
        slice_(None, nf)
        slice_(values[nf:], npc)
        slice_(polys[nf:], npc)
        slice_(None, npc)
        assert f.read(1) == b""
    torch.cuda.synchronize()
    return time.perf_counter() - t0, (values, polys, l), read_bytes


def timed_case(path, k, nf, npc, ext_k, reps):
    import torch
    new_t, old_t = [], []
    equal = None
    old_read = None
    for rep in range(1 + reps):
        dt_new, a = new_arm(path, npc, ext_k)
        dt_old, b, old_read = old_arm(path, npc, ext_k)
        if rep == 0:
            equal = all(torch.equal(x, y) for x, y in zip(a, b))
        else:
            new_t.append(dt_new)
            old_t.append(dt_old)
        del a, b
        torch.cuda.empty_cache()
    n, c = 1 << k, nf + npc
    med_new, med_old = statistics.median(new_t), statistics.median(old_t)
    return {"bench": "pk_load", "k": k, "ext_k": ext_k, "fixed": nf, "permutation": npc, "blinding_factors": BLINDING, "reps": reps,
            "file_bytes": os.path.getsize(path),
            "load_proving_key_s": round(med_new, 4), "load_proving_key_spread_s": round(max(new_t) - min(new_t), 4),
            "read_all_upload_s": round(med_old, 4), "read_all_upload_spread_s": round(max(old_t) - min(old_t), 4),
            "speedup": round(med_old / med_new, 2),
            "file_bytes_read_load_proving_key": 32 * n * c, "file_bytes_read_read_all": old_read,
            "page_cache": "warm", "same_device_outputs": equal}


def profile_case(path, k, nf, npc, ext_k):
    import torch
    from torch.profiler import ProfilerActivity, profile
    new_arm(path, npc, ext_k)                      # warm-up outside the trace
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        new_arm(path, npc, ext_k)
        torch.cuda.synchronize()
    evs = [e for e in prof.key_averages() if "k_fr_validate" in e.key]
    if not evs:
        return {"bench": "pk_load_validate_kernel", "k": k, "error": "k_fr_validate not found in the trace"}
    ev = evs[0]
    total_us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
    ms = total_us / 1e3 / ev.count
    n = 1 << k
    hbm_bound_ms = 32 * n / HBM_DATASHEET * 1e3
    return {"bench": "pk_load_validate_kernel", "k": k, "elements_per_call": n, "calls": ev.count, "ms_per_call": round(ms, 4),
            "hbm_bound_ms": round(hbm_bound_ms, 4), "bound": "data-sheet HBM (32 B read per element)", "share_of_bound": round(hbm_bound_ms / ms, 3),
            "GB_per_s": round(32 * n / (ms * 1e-3) / 1e9, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default=",".join("%d:%d:%d:%d" % c for c in CASES), help="k:fixed:permutation:ext_k")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--tmpdir", default=None, help="where the key files are written (default: the system's temporary directory)")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from ezkl_b200 import _native as nat
    nat.ensure_init()
    cases = [tuple(int(v) for v in c.split(":")) for c in args.cases.split(",")]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    card = card.splitlines()[0] if card else "unknown"
    lines = [{"card": card, "torch": torch.__version__}]
    print(json.dumps(lines[0]), flush=True)

    def emit(rec):
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    tmp = tempfile.mkdtemp(prefix="pk_bench_", dir=args.tmpdir)
    try:
        for k, nf, npc, ext_k in cases:
            size = file_bytes(k, nf, npc, ext_k)
            need_disk, need_host = size + GIB, 2 * size + 4 * GIB        # the key object while it is written, then the page cache
            free_disk, avail = shutil.disk_usage(tmp).free, host_available_bytes()
            if free_disk < need_disk or avail < need_host:
                emit({"bench": "pk_load", "k": k, "ext_k": ext_k, "fixed": nf, "permutation": npc, "file_bytes": size,
                      "skipped": "%.1f GiB free in the temporary directory (need %.1f), %.1f GiB of host memory available (need %.1f)" % (
                          free_disk / GIB, need_disk / GIB, avail / GIB, need_host / GIB)})
                continue
            path = os.path.join(tmp, "pk_k%d.key" % k)
            write_key(path, k, nf, npc, ext_k)
            warm_page_cache(path)
            emit(timed_case(path, k, nf, npc, ext_k, args.reps))
            if args.profile:
                emit(profile_case(path, k, nf, npc, ext_k))
            os.remove(path)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
