#!/usr/bin/env python
"""SRS loading: a KZG parameter file straight into two registered base tables (halo2.srs_bases -> b200_srs_register) against the path a
prover takes without it (ParamsKZG.read of the whole file, ParamsKZG.downsize with the host-pointer group FFT, then one Bases per vector).

Cases k_file -> k: 20->20, 22->22, 24->24, 22->20, 24->20, 24->22, and 26->26 / 26->20 when the temporary directory and the host memory have
room (a case that does not fit prints a "skipped" line).  The files are made with device.setup_srs (G2 tail zero), written to a temporary
directory that is deleted at the end, and read once before timing so that the page cache is warm; cold-cache reads are not measured.
Both paths are synchronous calls timed with a host clock, alternated call by call in one process: one warm-up pair, then --reps pairs;
the line reports the median and max - min of each.  It also states the bytes of the file each path reads (computed from the layout), both
handles' bases_info, and that one commitment of random scalars agrees between the two paths' tables.  halo2's own Rust read is not timed
(no Rust toolchain here).

--profile adds a pass of its own under torch.profiler: k_g1_validate's device time per call against the two computed bounds of one point
check (3 Montgomery multiplications at the integer-multiply ceiling of DESIGN.md section 4, and 64 B at the data-sheet 3.35 TB/s of HBM3),
naming the larger one as the bound that applies.

The card's name, power limit and maximum SM clock are read in the same run.  One JSON line per point on stdout (and in --out)."""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_DATASHEET = 3.35e12          # B/s, H100 SXM data sheet
CASES = [(20, 20), (22, 22), (24, 24), (22, 20), (24, 20), (24, 22), (26, 26), (26, 20)]
TRAPDOOR = 0x1D3C_5A17_9E37_79B9_7F4A_7C15_0BAD_CAFE
GIB = 1 << 30


def file_bytes(kf):
    return 4 + 128 * (1 << kf) + 256


def write_srs(path, kf):
    """ParamsKZG::write layout of setup_srs(kf, TRAPDOOR); the G2 tail is zero bytes (never read by the library)."""
    import numpy as np
    import torch
    from ezkl_b200 import device as dev
    g_d, gl_d = dev.setup_srs(kf, TRAPDOOR)
    with open(path, "wb") as f:
        f.write(np.uint32(kf).tobytes())
        for d in (g_d, gl_d):
            dev.to_host(d).tofile(f)
        f.write(bytes(256))
    del g_d, gl_d
    torch.cuda.empty_cache()


def warm_page_cache(path):
    with open(path, "rb") as f:
        while f.read(64 << 20):
            pass


def host_available_bytes():
    try:
        return os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    except (ValueError, OSError):
        return 0


def new_path(path, k):
    from ezkl_b200 import halo2 as h2
    t0 = time.perf_counter()
    bg, bl = h2.srs_bases(path, k)
    return time.perf_counter() - t0, (bg, bl)


def old_path(path, k):
    from ezkl_b200 import halo2 as h2
    t0 = time.perf_counter()
    params = h2.ParamsKZG.read(path)
    params.downsize(k)
    bg, bl = h2.Bases(params.g), h2.Bases(params.g_lagrange)
    dt = time.perf_counter() - t0
    del params
    return dt, (bg, bl)


def release(pair):
    for b in pair:
        b.release()


def timed_case(path, kf, k, reps):
    import numpy as np
    from ezkl_b200 import device as dev
    from ezkl_b200 import halo2 as h2
    new_t, old_t = [], []
    parity = None
    for rep in range(1 + reps):
        dt_new, nb = new_path(path, k)
        dt_old, ob = old_path(path, k)
        if rep == 0:
            r = dev.to_host(dev.random_scalars(1 << k, seed=k))
            parity = all(np.array_equal(h2.best_multiexp(r, a), h2.best_multiexp(r, b)) for a, b in zip(nb, ob))
            infos = [b.info() for b in nb]
            same_info = infos == [b.info() for b in ob]
        else:
            new_t.append(dt_new)
            old_t.append(dt_old)
        release(nb)
        release(ob)
    n = 1 << k
    med_new, med_old = statistics.median(new_t), statistics.median(old_t)
    return {"bench": "srs_register", "k_file": kf, "k": k, "reps": reps,
            "srs_bases_s": round(med_new, 4), "srs_bases_spread_s": round(max(new_t) - min(new_t), 4),
            "read_downsize_bases_s": round(med_old, 4), "read_downsize_bases_spread_s": round(max(old_t) - min(old_t), 4),
            "speedup": round(med_old / med_new, 2),
            "file_bytes_read_srs_bases": 4 + 64 * n * (2 if k == kf else 1), "file_bytes_read_params_read": file_bytes(kf),
            "g_lagrange": "file" if k == kf else "device group FFT (srs_bases) / host-pointer group FFT (downsize)",
            "bases_info_g": infos[0], "bases_info_g_lagrange": infos[1], "same_bases_info": same_info, "same_commitments": parity}


def profile_case(path, kf, k, mul_ceiling):
    import torch
    from torch.profiler import ProfilerActivity, profile
    _, pair = new_path(path, k)                      # warm-up outside the trace
    release(pair)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _, pair = new_path(path, k)
        torch.cuda.synchronize()
    release(pair)
    evs = [e for e in prof.key_averages() if "k_g1_validate" in e.key]
    if not evs:
        return {"bench": "srs_register_validate_kernel", "k_file": kf, "k": k, "error": "k_g1_validate not found in the trace"}
    ev = evs[0]
    total_us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
    calls = ev.count
    ms = total_us / 1e3 / calls
    n = 1 << k
    mul_bound_ms = 3 * n / mul_ceiling * 1e3
    hbm_bound_ms = 64 * n / HBM_DATASHEET * 1e3
    bound, bound_ms = ("multiply ceiling", mul_bound_ms) if mul_bound_ms >= hbm_bound_ms else ("data-sheet HBM", hbm_bound_ms)
    return {"bench": "srs_register_validate_kernel", "k_file": kf, "k": k, "points_per_call": n, "calls": calls, "ms_per_call": round(ms, 4),
            "multiply_bound_ms": round(mul_bound_ms, 4), "hbm_bound_ms": round(hbm_bound_ms, 4), "bound": bound,
            "share_of_bound": round(bound_ms / ms, 3), "G_points_per_s": round(n / (ms * 1e-3) / 1e9, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default=",".join("%d:%d" % c for c in CASES), help="k_file:k pairs")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--tmpdir", default=None, help="where the SRS files are written (default: the system's temporary directory)")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from ezkl_b200 import _native as nat
    nat.ensure_init()
    cases = [tuple(int(v) for v in c.split(":")) for c in args.cases.split(",")]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    card = card.splitlines()[0] if card else "unknown"
    props = torch.cuda.get_device_properties(0)
    try:
        max_mhz = float(card.split(",")[-1].split()[0])
    except (ValueError, IndexError):
        max_mhz = 1980.0
    mul_ceiling = props.multi_processor_count * 64 * max_mhz * 1e6 / 264
    lines = [{"card": card, "sms": props.multi_processor_count, "multiply_ceiling_G_mulmod_per_s": round(mul_ceiling / 1e9, 1), "torch": torch.__version__}]
    print(json.dumps(lines[0]), flush=True)

    def emit(rec):
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    tmp = tempfile.mkdtemp(prefix="srs_bench_", dir=args.tmpdir)
    try:
        files = {}
        for kf, k in cases:
            path = os.path.join(tmp, "kzg%d.srs" % kf)
            if kf not in files:
                need_disk = file_bytes(kf) + GIB
                need_host = 2 * file_bytes(kf) + 2 * GIB        # ParamsKZG.read: the file's bytes, then copies of both vectors
                free_disk = shutil.disk_usage(tmp).free
                if free_disk < need_disk or host_available_bytes() < need_host:
                    files[kf] = None
                    why = "%.1f GiB free in the temporary directory (need %.1f), %.1f GiB of host memory available (need %.1f)" % (
                        free_disk / GIB, need_disk / GIB, host_available_bytes() / GIB, need_host / GIB)
                else:
                    write_srs(path, kf)
                    files[kf] = path
            if files[kf] is None:
                emit({"bench": "srs_register", "k_file": kf, "k": k, "skipped": why})
                continue
            warm_page_cache(path)
            emit(timed_case(path, kf, k, args.reps))
        if args.profile:
            for kf, k in cases:
                if files.get(kf):
                    emit(profile_case(files[kf], kf, k, mul_ceiling))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
