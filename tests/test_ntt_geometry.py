"""The NTT engine (ntt.cu) through b200_ntt_dev: every pass geometry the launch code picks (kernel, lines per CTA, inter-pass
twiddle table), the pre / post scale modes with arbitrary constants, the buffer layouts (short inputs, strided and aliased
buffers), the plan cache and the argument checks, against the CPU oracle, from 2^1 to 2^28."""
import ctypes as C
import random
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from ezkl_b200 import _native as nat
from oracle import oracle as orc
from oracle import pyref
from tests import helpers as H

THREADS = orc.host_threads()
GIB = 1 << 30
R = pyref.R
BATCHES = (1, 2, 7, 64, 300, 4096, 65535)
FIELDS = ("kernel", "logm", "log_g", "threads", "smem", "grid_x", "twiddle")      # b200_debug_ntt_plan_host, per pass
TW_NONE, TW_FULL, TW_TWO_LEVEL = 0, 1, 2
HOST_CAP = (1 << 20) * 32          # host reference work of one case, in elements: bench.py's 32 columns of 2^20


def plan(log_n, batch, sms):
    out = np.zeros(21, np.int64)
    npass = nat.dbg_lib().b200_debug_ntt_plan_host(C.c_uint32(log_n), C.c_int(batch), C.c_int(sms), out.ctypes.data_as(C.c_void_p))
    assert npass in (1, 2, 3), (log_n, batch, sms, npass)
    return [dict(zip(FIELDS, (int(v) for v in out[7 * i: 7 * i + 7]))) for i in range(npass)]


def pass_shape(logms, idx):
    """(inner count, lines) of pass idx, restated from the factorisation i = i1*N2*N3 + i2*N3 + i3 -> j = j1 + N1*j2 + N1*N2*j3."""
    n = [1 << m for m in logms] + [1] * (3 - len(logms))
    if len(logms) == 1:
        return 1, 1
    if len(logms) == 2:
        return (n[1], n[1]) if idx == 0 else (n[0], n[0])
    return [(n[1] * n[2], n[1] * n[2]), (n[2], n[0] * n[2]), (n[0], n[0] * n[1])][idx]


# ---- CPU tier ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sms", [114, 132])
def test_plan_geometry_properties(sms):
    for log_n in range(1, 29):
        for batch in BATCHES:
            passes = plan(log_n, batch, sms)
            logms = [p["logm"] for p in passes]
            assert sum(logms) == log_n and all(1 <= m <= 10 for m in logms), (log_n, logms)
            for idx, p in enumerate(passes):
                where = (sms, log_n, batch, idx, p)
                inner, lines = pass_shape(logms, idx)
                m, g = p["logm"], p["log_g"]
                assert p["kernel"] in (1, 2), where
                if p["kernel"] == 2:
                    assert 7 <= m + g <= 10 and p["threads"] == 1 << (m + g - 2) <= 256, where
                    assert p["smem"] == ((1 << (m + g)) + (1 << m)) * 32 <= 200 * 1024, where
                    assert 3 * (p["smem"] + 8 + 1024) <= 228 * 1024, where          # + the mbarrier and the 1 KB reserved per CTA
                else:
                    assert 32 <= p["threads"] <= 1024 and p["smem"] <= 200 * 1024, where
                    assert p["smem"] == ((1 << (m + g)) + (1 << m) // 2) * 32, where
                assert (1 << g) <= inner and p["grid_x"] << g == lines, where
                if g > 0:                                                           # lines per CTA only while 2 CTAs per SM remain
                    assert p["grid_x"] * batch >= 2 * sms, where
                if idx == len(passes) - 1:
                    assert p["twiddle"] == TW_NONE, where
                else:
                    full = len(passes) > 1 and log_n <= 25 and p["kernel"] == 2
                    assert p["twiddle"] == (TW_FULL if full else TW_TWO_LEVEL), where
    # the routes the scale-mode tests rely on
    assert [p["kernel"] for p in plan(11, 1, sms)] == [1, 1]
    assert [(p["kernel"], p["log_g"] > 0) for p in plan(11, 4096, sms)] == [(2, True), (2, True)]
    assert [p["twiddle"] for p in plan(26, 1, sms)] == [TW_TWO_LEVEL, TW_TWO_LEVEL, TW_NONE]


def test_plan_hook_rejects_out_of_range():
    out = np.zeros(21, np.int64)
    for log_n, batch, sms in ((0, 1, 132), (29, 1, 132), (10, 0, 132), (10, 65536, 132), (10, 1, 0)):
        assert nat.dbg_lib().b200_debug_ntt_plan_host(C.c_uint32(log_n), C.c_int(batch), C.c_int(sms), out.ctypes.data_as(C.c_void_p)) == -1


# ---- GPU tier ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu():
    nat.init(-1)
    yield


def _torch():
    import torch
    return torch


def sm_count():
    return _torch().cuda.get_device_properties(0).multi_processor_count


def omega(log_n, power=1):
    return H.fr_wire(pow(pyref.omega_for(log_n), power, R))


def empty(*shape):
    torch = _torch()
    return torch.empty(shape + (4,), dtype=torch.int64, device="cuda")


def ntt_raw(src, src_stride, n_in, tmp, dst, dst_stride, log_n, w, pre_mode=0, pre=None, post_mode=0, post=None, batch=1):
    """b200_ntt_dev on raw device pointers; returns the status code (torch's current stream, synchronised)."""
    from ezkl_b200 import device as dev
    cp = lambda cs: nat.ptr(np.ascontiguousarray(np.stack(cs))) if cs is not None else None
    rc = nat.lib().b200_ntt_dev(nat.dev(src.data_ptr()), C.c_size_t(src_stride), C.c_size_t(n_in), nat.dev(tmp.data_ptr()), nat.dev(dst.data_ptr()),
                                C.c_size_t(dst_stride), C.c_uint32(log_n), nat.ptr(np.ascontiguousarray(w)), C.c_int(pre_mode), cp(pre),
                                C.c_int(post_mode), cp(post), C.c_size_t(batch), dev._stream())
    _torch().cuda.synchronize()
    return rc


def ntt(src, log_n, w, *, n_in=None, src_stride=None, dst=None, dst_stride=None, pre_mode=0, pre=None, post_mode=0, post=None):
    """src [batch, src_stride, 4] -> dst [batch, dst_stride, 4] (fresh, [batch, 2^log_n, 4], unless given)."""
    batch, N = src.shape[0], 1 << log_n
    src_stride = src.shape[1] if src_stride is None else src_stride
    n_in = src_stride if n_in is None else n_in
    if dst is None:
        dst = empty(batch, N)
    dst_stride = dst.shape[1] if dst_stride is None else dst_stride
    tmp = empty(batch, N)
    nat.check(ntt_raw(src, src_stride, n_in, tmp, dst, dst_stride, log_n, w, pre_mode, pre, post_mode, post, batch))
    return dst


def scale_vector(mode, consts, n):
    """The per-element constants of a scale mode over indices 0..n-1 (None for mode 0)."""
    if mode == 0:
        return None
    if mode == 1:
        return np.tile(consts[0], (n, 1))
    return np.tile(np.stack(consts), (-(-n // 3), 1))[:n]


def reference(cols, log_n, w, pre_mode=0, pre=None, post_mode=0, post=None):
    """best_fft of each column (n_in <= N elements, zero-padded), with the pre-scale applied before and the post-scale after."""
    N = 1 << log_n
    out = np.zeros((len(cols), N, 4), np.uint64)
    for b, col in enumerate(cols):
        a = np.zeros((N, 4), np.uint64)
        a[: col.shape[0]] = col
        s = scale_vector(pre_mode, pre, col.shape[0])
        if s is not None and col.shape[0]:
            a[: col.shape[0]] = orc.poly_op("mul", a[: col.shape[0]].copy(), s, threads=THREADS)
        f = orc.best_fft(a, log_n, w, THREADS)
        s = scale_vector(post_mode, post, N)
        out[b] = f if s is None else orc.poly_op("mul", f, s, threads=THREADS)
    return out


def columns(batch, n, seed):
    return orc.gen_scalars(batch * n, seed=seed).reshape(batch, n, 4)


def to_dev(a):
    from ezkl_b200 import device as dev
    return dev.from_host(np.ascontiguousarray(a))


def to_host(t):
    from ezkl_b200 import device as dev
    return dev.to_host(t)


def routing_cases(sms):
    """Every (pass count, pass index, kernel, log_g, twiddle table) class for log_n <= 24 and the batch set, with the cheapest
    (log_n, batch) that produces it."""
    cheapest = {}
    for log_n in range(1, 25):
        for batch in BATCHES:
            passes = plan(log_n, batch, sms)
            for idx, p in enumerate(passes):
                cls = (len(passes), idx, p["kernel"], p["log_g"], p["twiddle"])
                cost = (1 << log_n) * batch
                if cls not in cheapest or cost < cheapest[cls][0]:
                    cheapest[cls] = (cost, log_n, batch)
    return cheapest


@pytest.mark.gpu
def test_routing_coverage(gpu):
    """One case per geometry class, picked from the hook for this device's SM count; the kernels the profiler sees launched match
    the hook's plan, every column matches the oracle, and the classes run are all the classes there are."""
    import re

    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    sms = sm_count()
    cheapest = routing_cases(sms)
    over = {cls: c for cls, c in cheapest.items() if c[0] > HOST_CAP}
    assert not over, "geometry classes with no case within the host budget: %r" % over
    cases = sorted({(log_n, batch) for _, log_n, batch in cheapest.values()}, key=lambda c: (1 << c[0]) * c[1])
    covered, expected_kernels = set(), []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for log_n, batch in cases:
            passes = plan(log_n, batch, sms)
            w = omega(log_n)
            cols = columns(batch, 1 << log_n, seed=1000 * log_n + batch)
            got = to_host(ntt(to_dev(cols), log_n, w)).reshape(batch, 1 << log_n, 4)
            want = reference(list(cols), log_n, w)
            bad = [b for b in range(batch) if not np.array_equal(got[b], want[b])]
            assert not bad, (log_n, batch, passes, bad[:8])
            covered |= {(len(passes), idx, p["kernel"], p["log_g"], p["twiddle"]) for idx, p in enumerate(passes)}
            expected_kernels += ["k_ntt_pass2" if p["kernel"] == 2 else "k_ntt_pass" for p in passes]
    launched = [re.search(r"k_ntt_pass2?\b", e.name).group(0) for e in prof.events()
                if e.device_type == DeviceType.CUDA and re.search(r"k_ntt_pass2?\b", e.name)]
    assert launched == expected_kernels
    assert covered == set(cheapest), sorted(set(cheapest) ^ covered)
    print("%d SMs: %d geometry classes in %d cases" % (sms, len(cheapest), len(cases)))


def random_consts(rng, c0_zero):
    cs = [H.fr_wire(rng.randrange(2, R)) for _ in range(3)]
    if c0_zero:
        cs[0] = np.zeros(4, np.uint64)
    return cs


# (log_n, batch) per route: one pass on k_ntt_pass, one pass on k_ntt_pass2, two passes on k_ntt_pass, two and three passes on k_ntt_pass2
SCALE_ROUTES = {"1pass_v1": (5, 3), "1pass_v2": (9, 2), "2pass_v1": (11, 1), "2pass_v2": (16, 2), "3pass_v2": (21, 1)}


@pytest.mark.gpu
@pytest.mark.parametrize("c0", ["random", "zero"])
@pytest.mark.parametrize("route", list(SCALE_ROUTES))
def test_scale_modes(gpu, route, c0):
    """All nine (pre, post) pairs of modes {0, 1, 3} with arbitrary constants: pre(i) = c[i mod 3] includes c[0]."""
    log_n, batch = SCALE_ROUTES[route]
    passes = plan(log_n, batch, sm_count())
    want_kernels = {"1pass_v1": [1], "1pass_v2": [2], "2pass_v1": [1, 1], "2pass_v2": [2, 2], "3pass_v2": [2, 2, 2]}[route]
    assert [p["kernel"] for p in passes] == want_kernels, passes
    rng = random.Random(list(SCALE_ROUTES).index(route) * 2 + (c0 == "zero"))
    N = 1 << log_n
    w = omega(log_n)
    pre, post = random_consts(rng, c0 == "zero"), random_consts(rng, c0 == "zero")
    cols = columns(batch, N, seed=7 + log_n)
    src = to_dev(cols)
    for pre_mode in (0, 1, 3):
        unscaled = reference(list(cols), log_n, w, pre_mode, pre[:pre_mode] or None)
        for post_mode in (0, 1, 3):
            got = to_host(ntt(src, log_n, w, pre_mode=pre_mode, pre=pre[:pre_mode] or None, post_mode=post_mode, post=post[:post_mode] or None))
            s = scale_vector(post_mode, post, N)
            for b in range(batch):
                want = unscaled[b] if s is None else orc.poly_op("mul", unscaled[b], s, threads=THREADS)
                assert np.array_equal(got.reshape(batch, N, 4)[b], want), (route, c0, pre_mode, post_mode, b)


@pytest.mark.gpu
@pytest.mark.parametrize("log_n,batch", [(14, 2), (21, 1)])
def test_short_inputs(gpu, log_n, batch):
    """n_in < 2^log_n (the zero-skipping first round of a padded transform), with a cyclic pre-scale, on two and three passes."""
    passes = plan(log_n, batch, sm_count())
    assert len(passes) == (2 if log_n <= 20 else 3)
    N, N2 = 1 << log_n, 1 << passes[1]["logm"]
    w = omega(log_n)
    rng = random.Random(log_n)
    pre = random_consts(rng, False)
    for n_in in (0, 1, 3, N2 - 1, N2 + 1, N // 8, N // 2 + 5, N - 1):
        cols = columns(batch, n_in, seed=n_in + 3) if n_in else np.zeros((batch, 0, 4), np.uint64)
        src = to_dev(cols) if n_in else empty(batch, 1)
        got = to_host(ntt(src, log_n, w, n_in=n_in, src_stride=n_in, pre_mode=3, pre=pre)).reshape(batch, N, 4)
        want = reference(list(cols), log_n, w, 3, pre)
        assert np.array_equal(got, want), (log_n, n_in)


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", [9, 14, 21])
def test_strided_buffers(gpu, log_n):
    """src_stride > n_in with sentinels in the gaps (never read) and dst_stride > N with sentinels in the gaps (never written)."""
    torch = _torch()
    batch, N = 3, 1 << log_n
    n_in = N - 5
    src_stride, dst_stride = n_in + 37, N + 19
    w = omega(log_n)
    cols = columns(batch, n_in, seed=log_n + 40)
    src_h = columns(batch, src_stride, seed=log_n + 41)          # nonzero sentinels
    src_h[:, :n_in] = cols
    dst_h = columns(batch, dst_stride, seed=log_n + 42)
    src, dst = to_dev(src_h), to_dev(dst_h)
    ntt(src, log_n, w, n_in=n_in, src_stride=src_stride, dst=dst, dst_stride=dst_stride)
    got = to_host(dst).reshape(batch, dst_stride, 4)
    assert np.array_equal(got[:, :N], reference(list(cols), log_n, w))
    assert np.array_equal(got[:, N:], dst_h[:, N:]), "dst gaps written"
    assert torch.equal(src, to_dev(src_h)), "src written"


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", [8, 15, 21])
def test_in_place(gpu, log_n):
    """dst == src (full-length input, equal strides) on one, two and three passes."""
    batch, N = 2, 1 << log_n
    assert len(plan(log_n, batch, sm_count())) == (1 if log_n <= 10 else 2 if log_n <= 20 else 3)
    w = omega(log_n)
    cols = columns(batch, N, seed=log_n + 60)
    buf = to_dev(cols)
    tmp = empty(batch, N)
    nat.check(ntt_raw(buf, N, N, tmp, buf, N, log_n, w, batch=batch))
    assert np.array_equal(to_host(buf).reshape(batch, N, 4), reference(list(cols), log_n, w))


@pytest.mark.gpu
def test_plan_cache_interleaved_omegas(gpu):
    """omega, omega^-1 and omega^3 for one log_n, interleaved on one thread: each call finds its own plan."""
    log_n = 16
    N = 1 << log_n
    ws = {"w": omega(log_n), "w_inv": omega(log_n, -1), "w3": omega(log_n, 3)}
    for i, name in enumerate(["w", "w_inv", "w3", "w", "w3", "w_inv", "w_inv", "w"]):
        cols = columns(2, N, seed=500 + i)
        got = to_host(ntt(to_dev(cols), log_n, ws[name])).reshape(2, N, 4)
        assert np.array_equal(got, reference(list(cols), log_n, ws[name])), (i, name)


def _free_gib():
    torch = _torch()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0] / GIB


def _need(log_n, buffers):
    need = buffers * (32 << log_n) / GIB + 1
    free = _free_gib()
    if free < need:
        pytest.skip("2^%d needs %.0f GiB of free device memory, %.1f GiB free" % (log_n, need, free))


@pytest.mark.gpu
def test_2p26_vs_oracle(gpu):
    """2^26: above the full-table limit, every inter-pass twiddle comes from the two-level tables; the whole output is compared."""
    from ezkl_b200 import device as dev
    log_n = 26
    _need(log_n, 3)
    w = omega(log_n)
    src = dev.random_scalars(1 << log_n, seed=26)
    got = to_host(ntt(src.unsqueeze(0), log_n, w))[0]
    a = to_host(src)
    del src
    assert np.array_equal(got.reshape(-1, 4), orc.best_fft(a, log_n, w, THREADS))


def _eval_chunked(src, xs, chunk=1 << 22):
    """p(x) for each x, p = the device column src [N, 4], by Horner on host chunks in parallel: p(x) = sum_c x^c0 * p_c(x)."""
    N = src.shape[0]
    starts = list(range(0, N, chunk))

    def part(c0):
        h = to_host(src[c0: c0 + chunk])
        return [orc.eval_polynomial(h, x) for x in xs]

    with ThreadPoolExecutor(max_workers=min(8, THREADS)) as ex:
        parts = list(ex.map(part, starts))
    out = []
    for k, x in enumerate(xs):
        acc = np.zeros((1, 4), np.uint64)
        for c0, vals in zip(starts, parts):
            term = orc.field_op("fr", "mul", orc.fr_pow(x, c0).reshape(1, 4), vals[k].reshape(1, 4))
            acc = orc.field_op("fr", "add", acc, term)
        out.append(acc[0])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", [27, 28])
def test_two_level_tables_large(gpu, log_n):
    """2^27 and 2^28: an impulse e_i (odd i) maps to (omega^i)^j, checked element by element in host chunks; a random column comes
    back through the forward and the N^-1-scaled inverse transform, and four of its outputs equal direct evaluations."""
    torch = _torch()
    from ezkl_b200 import device as dev
    _need(log_n, 3)
    N = 1 << log_n
    rng = random.Random(log_n)
    w = omega(log_n)
    tmp, dst = empty(1, N), empty(1, N)
    i = rng.randrange(N // 2) * 2 + 1
    imp = torch.zeros((1, i + 1, 4), dtype=torch.int64, device="cuda")
    imp[0, i] = torch.from_numpy(orc.fr_one().view(np.int64)).cuda()
    nat.check(ntt_raw(imp, i + 1, i + 1, tmp, dst, N, log_n, w))
    del imp
    wi = omega(log_n, i)
    out = dst[0]
    assert np.array_equal(to_host(out[0]), orc.fr_one()), "out[0] != 1"
    chunk = 1 << 24
    for j0 in range(0, N - 1, chunk):
        g = to_host(out[j0: min(j0 + chunk + 1, N)])
        assert np.array_equal(orc.poly_op("scale", g[:-1], s=wi, threads=THREADS), g[1:]), ("impulse", i, j0)
    del g
    src = dev.random_scalars(N, seed=log_n).unsqueeze(0)
    nat.check(ntt_raw(src, N, N, tmp, dst, N, log_n, w))
    js = [1, N // 2 + 1, N - 1, rng.randrange(N)]
    evals = _eval_chunked(src[0], [omega(log_n, j) for j in js])
    for j, e in zip(js, evals):
        assert np.array_equal(to_host(dst[0, j]), e), ("direct evaluation", j)
    nat.check(ntt_raw(dst, N, N, tmp, dst, N, log_n, omega(log_n, -1), post_mode=1, post=[H.fr_wire(pow(N, -1, R))]))
    assert torch.equal(dst, src), "inverse(forward(x)) != x"
    del src, tmp, dst
    torch.cuda.empty_cache()


ONE = [np.array([0xac96341c4ffffffb, 0x36fc76959f60cd29, 0x666ea36f7879462e, 0x0e0a77c19a07df2f], np.uint64)]     # 1, Montgomery form
BAD_CALLS = {       # 2^4-element transforms on 2 x 16-element buffers
    "batch_2p32_plus_1": dict(batch=(1 << 32) + 1),
    "batch_65536": dict(batch=65536),
    "log_n_0": dict(log_n=0),
    "log_n_29": dict(log_n=29),
    "n_in_over_N": dict(n_in=17, src_stride=17, batch=1),
    "pre_mode_2": dict(pre_mode=2, pre=ONE * 2),
    "post_mode_2": dict(post_mode=2, post=ONE * 2),
    "pre_constants_null": dict(pre_mode=1),
    "post_constants_null": dict(post_mode=3),
    "src_stride_below_n_in": dict(src_stride=15, batch=2),
    "dst_stride_below_N": dict(dst_stride=15, batch=2),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(BAD_CALLS))
def test_argument_errors(gpu, case):
    """Each bad call returns -1 with a message and leaves the output untouched; all buffers are small and valid, so a check that
    is missing shows as a changed output, not as an out-of-bounds access."""
    torch = _torch()
    log_n, N = 4, 16
    w = omega(log_n)
    src, tmp = to_dev(columns(2, N, seed=90)), empty(2, N)
    sentinel = columns(2, N, seed=91)
    dst = to_dev(sentinel)
    args = dict(src_stride=N, n_in=N, dst_stride=N, log_n=log_n, pre_mode=0, pre=None, post_mode=0, post=None, batch=1)
    args.update(BAD_CALLS[case])
    rc = ntt_raw(src, args["src_stride"], args["n_in"], tmp, dst, args["dst_stride"], args["log_n"], w, args["pre_mode"], args["pre"],
                 args["post_mode"], args["post"], args["batch"])
    msg = nat.lib().b200_last_error().decode()
    assert rc == -1 and "ntt" in msg, (case, rc, msg)
    assert torch.equal(dst, to_dev(sentinel)), case


@pytest.mark.gpu
def test_argument_boundaries(gpu):
    """The limits themselves are accepted: batch 1 with any strides, n_in == N, batch 65535, both scale modes with constants."""
    log_n, N = 4, 16
    w = omega(log_n)
    src, tmp, dst = to_dev(columns(2, N, seed=92)), empty(2, N), empty(2, N)
    nat.check(ntt_raw(src, 0, N, tmp, dst, 0, log_n, w, 1, ONE, 3, ONE * 3, batch=1))
    assert np.array_equal(to_host(dst).reshape(-1, 4)[:N], reference([to_host(src).reshape(-1, 4)[:N]], log_n, w)[0])
    cols = columns(65535, 2, seed=93)
    got = to_host(ntt(to_dev(cols), 1, omega(1)))
    assert np.array_equal(got, reference(list(cols), 1, omega(1)))
