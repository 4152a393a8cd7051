"""SRS straight to the device (b200_srs_register, halo2.srs_bases): a parameter file's g and g_lagrange vectors become two
registered base tables in one call, every point passed is checked on the device as halo2curves' G1Affine::from_raw_bytes checks it, and
a file larger than the circuit is downsized on the device with the group FFT.  Pinned by the reference's SRS fixture
(tests/golden/kzg_k6.srs), by ParamsKZG::downsize's defining relation, and at k = 20..22 by known discrete logs.

The two-device check runs this file as a script in its own process: `python tests/test_srs_register.py multi`."""
import ctypes as C
import os
import random
import struct
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from ezkl_b200 import _native as nat          # noqa: E402
from oracle import oracle as orc              # noqa: E402
from oracle import pyref                      # noqa: E402
from tests import helpers as H                # noqa: E402

P_, S, Z, U32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
SRS_FIXTURE = os.path.join(H.GOLDEN, "kzg_k6.srs")
SENTINEL = 0xDEAD_BEEF
REASONS = ("x is not below p", "y is not below p", "is not on the curve")
MIB = 1 << 20


# ---- the check rule in python ints -----------------------------------------------------------------------------------------------
def _coords(pt):
    pt = np.asarray(pt, np.uint64).reshape(8)
    return H.limbs_to_int(pt[:4]), H.limbs_to_int(pt[4:])


def check_rule(pt):
    """None for a valid point, else the reason k_g1_validate reports: x, then y, must be canonical (the 256-bit limb integer below p),
    then the point must be (0, 0) or satisfy y^2 = x^3 + 3 (Montgomery wire form)."""
    x, y = _coords(pt)
    if x >= pyref.P:
        return REASONS[0]
    if y >= pyref.P:
        return REASONS[1]
    if x == 0 and y == 0:
        return None
    xc, yc = pyref.from_mont(x, pyref.P), pyref.from_mont(y, pyref.P)
    return None if (yc * yc - xc * xc * xc - 3) % pyref.P == 0 else REASONS[2]


def with_limbs(pt, x=None, y=None):
    out = np.asarray(pt, np.uint64).reshape(8).copy()
    if x is not None:
        out[:4] = H.int_to_limbs(x)
    if y is not None:
        out[4:] = H.int_to_limbs(y)
    return out


def spoil(pt, reason):
    """A copy of the valid point pt that fails with `reason`: x or y replaced by itself + p (p when that overflows 256 bits), or y + 1 in
    Montgomery form (canonical, off the curve)."""
    x, y = _coords(pt)
    if reason == REASONS[0]:
        return with_limbs(pt, x=x + pyref.P if x + pyref.P < 1 << 256 else pyref.P)
    if reason == REASONS[1]:
        return with_limbs(pt, y=y + pyref.P if y + pyref.P < 1 << 256 else pyref.P)
    return with_limbs(pt, y=(y + 1) % pyref.P)


def srs_file_bytes(g, gl, tail=bytes(256)) -> bytes:
    k = int(g.shape[0]).bit_length() - 1
    return struct.pack("<I", k) + np.ascontiguousarray(g, "<u8").tobytes() + np.ascontiguousarray(gl, "<u8").tobytes() + tail


# ---- CPU ---------------------------------------------------------------------------------------------------------------------------
def test_srs_register_is_exported_and_typed():
    """include/ezkl_b200.h declares b200_srs_register, which libezkl_b200.so exports with the argtypes / restype read from that header."""
    decls = nat.declarations(nat.HEADER)
    fn = nat.lib().b200_srs_register
    assert (fn.argtypes, fn.restype) == decls["b200_srs_register"]
    assert decls["b200_srs_register"] == ([P_, P_, U32, Z, S, P_, P_], Z)


def test_check_rule_against_the_oracle():
    """The rule on crafted points: canonical points agree with the oracle's curve check (on-curve points, y + 1, the identity); a limb
    pattern equal to p or to x + p is rejected for the coordinate even where the oracle, which reduces, finds the point on the curve; every
    point of the fixture SRS is valid."""
    _, g, gl = H.load_srs_fixture()
    assert all(check_rule(p) is None and orc.g1_is_on_curve(p) for p in np.concatenate([g, gl]))
    ident = np.zeros(8, np.uint64)
    assert check_rule(ident) is None and orc.g1_is_on_curve(ident)
    rnd = random.Random(5)
    for p in [g[0], g[1], gl[7]] + [g[i] for i in rnd.sample(range(64), 8)]:
        x, y = _coords(p)
        bumped = with_limbs(p, y=(y + 1) % pyref.P)
        assert check_rule(bumped) == REASONS[2] and not orc.g1_is_on_curve(bumped)
        for coord, reason in ((0, REASONS[0]), (1, REASONS[1])):
            v = (x, y)[coord]
            for raw in (pyref.P, v + pyref.P):
                if raw >= 1 << 256:
                    continue
                bad = with_limbs(p, **({"x": raw} if coord == 0 else {"y": raw}))
                assert check_rule(bad) == reason
            assert check_rule(spoil(p, reason)) == reason
        # x + p reduces to x: on the curve for the oracle, rejected by the canonical check
        assert orc.g1_is_on_curve(with_limbs(p, x=x)) and check_rule(with_limbs(p, x=x + pyref.P)) == REASONS[0]
    # (0, 0) is the identity; (0, 1) and (1, 0) are not on the curve
    one = H.fq_wire(1)
    for pt in (with_limbs(ident, y=H.limbs_to_int(one)), with_limbs(ident, x=H.limbs_to_int(one))):
        assert check_rule(pt) == REASONS[2] and not orc.g1_is_on_curve(pt)
    # p exactly in both coordinates: x is named first
    assert check_rule(with_limbs(ident, x=pyref.P, y=pyref.P)) == REASONS[0]


def test_srs_bases_argument_errors_raise_before_the_library(tmp_path, monkeypatch):
    """A file whose length is not 4 + 128 * 2^k_file + 256, an empty file, and k > k_file raise B200Error before any device call."""
    from ezkl_b200 import halo2 as h2

    def no_device(*a, **kw):
        raise AssertionError("the library was called")
    monkeypatch.setattr(nat, "ensure_init", no_device)
    monkeypatch.setattr(nat, "lib", no_device)
    data = open(SRS_FIXTURE, "rb").read()
    for name, blob in (("short.srs", data[:-1]), ("long.srs", data + b"\0"), ("empty.srs", b""), ("k7.srs", struct.pack("<I", 7) + data[4:])):
        p = tmp_path / name
        p.write_bytes(blob)
        with pytest.raises(nat.B200Error, match="srs_bases"):
            h2.srs_bases(str(p), 6)
    with pytest.raises(nat.B200Error, match="k = 7 not in"):
        h2.srs_bases(SRS_FIXTURE, 7)


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------
def jac_to_affine(j):
    j = np.asarray(j, np.uint64).reshape(-1, 12)
    out = j[:, :8].copy()
    for i in range(j.shape[0]):
        if not j[i, 8:].any():
            out[i] = 0
    return out


def unit_commitments(bases, n):
    """MSM of every unit vector e_j, j < n: the table's level-0 points, back through the MSM."""
    from ezkl_b200 import halo2 as h2
    eye = np.zeros((n, n, 4), np.uint64)
    eye[np.arange(n), np.arange(n)] = orc.fr_one()
    return jac_to_affine(h2.best_multiexp_batch(list(eye), bases))


def lagrange_relation(g, k):
    """ParamsKZG::downsize's defining relation with the oracle's MSM: g_lagrange[j] = n^-1 sum_i omega^(-ij) g[i]."""
    n = 1 << k
    w_inv, n_inv = pow(pyref.omega_for(k), -1, pyref.R), pow(n, -1, pyref.R)
    return np.stack([orc.msm(H.fr_array([pow(w_inv, i * j, pyref.R) * n_inv % pyref.R for i in range(n)]), g[:n]) for j in range(n)])


def register(g, gl, k, window_bits=0, max_table_bytes=0):
    """b200_srs_register straight through ctypes -> (rc, g handle, g_lagrange handle); the handles start as SENTINEL."""
    hg, hl = C.c_uint64(SENTINEL), C.c_uint64(SENTINEL)
    rc = nat.lib().b200_srs_register(None if g is None else nat.ptr(g), None if gl is None else nat.ptr(gl), k, window_bits, max_table_bytes,
                                     C.byref(hg), C.byref(hl))
    return rc, hg.value, hl.value


def release(*handles):
    for h in handles:
        nat.check(nat.lib().b200_bases_release(h))


def free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def _fixture_pins():
    """The fixture pins of the GPU tier (also run by the two-device child): unit vectors, random scalars, the 64 known answers, NULL."""
    from ezkl_b200 import halo2 as h2
    k, g, gl = H.load_srs_fixture()
    n = 1 << k
    bg, bl = h2.srs_bases(SRS_FIXTURE, k)
    assert bg.n == bl.n == n
    assert unit_commitments(bg, n).tobytes() == g.tobytes()
    assert unit_commitments(bl, n).tobytes() == gl.tobytes()
    for seed in range(3):
        r = orc.gen_scalars(n, seed=seed)
        assert np.array_equal(jac_to_affine(h2.best_multiexp(r, bg))[0], orc.msm(r, g))
        assert np.array_equal(jac_to_affine(h2.best_multiexp(r, bl))[0], orc.msm(r, gl))
    w_inv, n_inv = pow(pyref.omega_for(k), -1, pyref.R), pow(n, -1, pyref.R)
    cols = [H.fr_array([pow(w_inv, i * j, pyref.R) * n_inv % pyref.R for i in range(n)]) for j in range(n)]
    assert np.array_equal(jac_to_affine(h2.best_multiexp_batch(cols, bg)), gl)
    # NULL g_lagrange: the device FFT of the file's g gives the file's g_lagrange
    rc, hg, hl = register(g, None, k)
    assert rc == 0, nat.lib().b200_last_error()
    ng, nl = h2.Bases.from_handle(hg), h2.Bases.from_handle(hl)
    assert unit_commitments(ng, n).tobytes() == g.tobytes() and unit_commitments(nl, n).tobytes() == gl.tobytes()
    for b in (bg, bl, ng, nl):
        b.release()


@pytest.fixture(scope="module")
def gpu():
    nat.ensure_init()
    yield


@pytest.mark.gpu
def test_reference_pin(gpu):
    """tests/golden/kzg_k6.srs with its g_lagrange passed: the unit-vector commitments return all 128 file points byte for byte, random
    commitments equal the oracle's MSM on the file's points, the 64 known answers hold; NULL instead gives the same points."""
    _fixture_pins()


@pytest.mark.gpu
def test_downsize_pin(gpu):
    """From the fixture at every k < 6: the g handle holds g[:2^k], and the g_lagrange handle's points are n^-1 sum_i omega^(-ij) g[i]
    (the oracle's MSM) and those of Bases(g_to_lagrange(g[:2^k]))."""
    from ezkl_b200 import halo2 as h2
    _, g, _ = H.load_srs_fixture()
    for k in range(1, 6):
        n = 1 << k
        bg, bl = h2.srs_bases(SRS_FIXTURE, k)
        want = lagrange_relation(g, k)
        assert unit_commitments(bg, n).tobytes() == g[:n].tobytes(), k
        got = unit_commitments(bl, n)
        assert got.tobytes() == want.tobytes(), k
        old = h2.Bases(h2.g_to_lagrange(g[:n], k))
        assert unit_commitments(old, n).tobytes() == got.tobytes(), k
        for b in (bg, bl, old):
            b.release()


@pytest.mark.gpu
def test_large_k_known_discrete_logs(gpu, tmp_path):
    """A k_file = 22 file from device.setup_srs(22, s) (G2 tail zero): at (22, file), (22, NULL), (21, NULL) and (20, NULL), commitments
    of random r with the g handle are [r(s)] G, with the g_lagrange handle [(iNTT r)(s)] G.  One reduced table (max_table_bytes below the
    full table) gives the same commitments and the same bases_info as Bases(...) with that budget."""
    from ezkl_b200 import device as dev
    from ezkl_b200 import fields as F
    from ezkl_b200 import halo2 as h2
    kf, s = 22, 0x2F1E_0D3C_4B5A_6978_8796_A5B4_C3D2_E1F0
    g_d, gl_d = dev.setup_srs(kf, s)
    g, gl = dev.to_host(g_d), dev.to_host(gl_d)
    del g_d, gl_d
    path = tmp_path / "kzg22.srs"
    path.write_bytes(srs_file_bytes(g, gl))
    gen = np.concatenate([F.fq_to_limbs(1), F.fq_to_limbs(2)]).reshape(1, 8)
    threads = orc.host_threads()
    for k, passed in ((22, True), (22, False), (21, False), (20, False)):
        n = 1 << k
        r = orc.gen_scalars(n, seed=k + 100 * passed)
        want_g = orc.g1_scalar_mul(gen, orc.eval_polynomial(r, H.fr_wire(s)).reshape(1, 4))[0]
        want_l = orc.g1_scalar_mul(gen, orc.eval_polynomial(orc.lagrange_to_coeff(r, k, threads), H.fr_wire(s)).reshape(1, 4))[0]
        if passed:
            bg, bl = h2.srs_bases(str(path), k)
        else:
            rc, hg, hl = register(np.ascontiguousarray(g[:n]), None, k)
            assert rc == 0, nat.lib().b200_last_error()
            bg, bl = h2.Bases.from_handle(hg), h2.Bases.from_handle(hl)
        got = jac_to_affine(np.stack([h2.best_multiexp(r, bg), h2.best_multiexp(r, bl)]))
        assert np.array_equal(got[0], want_g), (k, passed, "g")
        assert np.array_equal(got[1], want_l), (k, passed, "g_lagrange")
        bg.release()
        bl.release()
    # reduced table: 2 levels of 2^22 points
    budget = 2 * 64 << kf
    bg, bl = h2.srs_bases(str(path), kf, max_table_bytes=budget)
    og, ol = h2.Bases(g, max_table_bytes=budget), h2.Bases(gl, max_table_bytes=budget)
    assert bg.info() == og.info() and bl.info() == ol.info() and bg.info()["windows_per_level"] > 1, bg.info()
    r = orc.gen_scalars(1 << kf, seed=7)
    assert np.array_equal(h2.best_multiexp(r, bg), h2.best_multiexp(r, og))
    assert np.array_equal(h2.best_multiexp(r, bl), h2.best_multiexp(r, ol))
    for b in (bg, bl, og, ol):
        b.release()


def _rejection_cases(g, gl):
    """(vector, reason, index) over both vectors, every reason and indices 0, n/2, n - 1."""
    n = g.shape[0]
    return [(v, reason, i) for v in ("g", "g_lagrange") for reason in REASONS for i in (0, n // 2, n - 1)]


def _assert_rejected(g, gl, k, want_msg):
    before = free_bytes()
    rc, hg, hl = register(g, gl, k)
    err = nat.lib().b200_last_error().decode()
    assert rc == -1 and err == want_msg, (rc, err, want_msg)
    assert hg == SENTINEL and hl == SENTINEL
    assert abs(free_bytes() - before) <= MIB, (before, free_bytes())


@pytest.mark.gpu
def test_rejection(gpu, tmp_path):
    """In the fixture's points and a k = 16 file: each vector x each reason x index 0, n/2, n - 1 returns -1 naming the vector, the index
    and the reason, writes no handle and gives its device memory back; of two bad points the lower index is named, and g before
    g_lagrange.  srs_bases raises the same message."""
    from ezkl_b200 import device as dev
    from ezkl_b200 import halo2 as h2
    _, g6, gl6 = H.load_srs_fixture()
    g16_d, gl16_d = dev.setup_srs(16, 0x51_6E_A7)
    g16, gl16 = dev.to_host(g16_d), dev.to_host(gl16_d)
    del g16_d, gl16_d
    ok = register(g6, gl6, 6)                       # warm-up: the context's scratch exists before memory is compared
    assert ok[0] == 0
    release(ok[1], ok[2])
    for k, g, gl in ((6, g6, gl6), (16, g16, gl16)):
        for v, reason, i in _rejection_cases(g, gl):
            bad = {"g": g.copy(), "g_lagrange": gl.copy()}
            bad[v][i] = spoil(bad[v][i], reason)
            assert check_rule(bad[v][i]) == reason
            _assert_rejected(bad["g"], bad["g_lagrange"], k, "srs_register: %s[%d] %s" % (v, i, reason))
        n = 1 << k
        bg, bl = g.copy(), gl.copy()
        bg[n - 1] = spoil(bg[n - 1], REASONS[2])
        bg[n // 2] = spoil(bg[n // 2], REASONS[0])
        bl[0] = spoil(bl[0], REASONS[1])
        _assert_rejected(bg, bl, k, "srs_register: g[%d] %s" % (n // 2, REASONS[0]))
        _assert_rejected(g, bl, k, "srs_register: g_lagrange[0] %s" % REASONS[1])
        bl[3] = spoil(bl[3], REASONS[2])
        bl[0] = gl[0]
        bl[n - 1] = spoil(bl[n - 1], REASONS[0])
        _assert_rejected(g, bl, k, "srs_register: g_lagrange[3] %s" % REASONS[2])
        _assert_rejected(bg, None, k, "srs_register: g[%d] %s" % (n // 2, REASONS[0]))
    bad = g16.copy()
    bad[12345] = spoil(bad[12345], REASONS[1])
    path = tmp_path / "bad16.srs"
    path.write_bytes(srs_file_bytes(bad, gl16))
    with pytest.raises(nat.B200Error, match=r"srs_register: g\[12345\] y is not below p"):
        h2.srs_bases(str(path), 16)


@pytest.mark.gpu
def test_accepted_points(gpu, tmp_path):
    """(0, 0) is valid at any index; a bad point of g beyond 2^k, or in the file's g_lagrange when downsizing, is never read.  In both
    cases the commitments match the oracle on the same bases."""
    from ezkl_b200 import halo2 as h2
    k, g, gl = H.load_srs_fixture()
    n = 1 << k
    zg, zl = g.copy(), gl.copy()
    for i in (0, 31, n - 1):
        zg[i] = 0
    zl[17] = 0
    path = tmp_path / "zero.srs"
    path.write_bytes(srs_file_bytes(zg, zl))
    bg, bl = h2.srs_bases(str(path), k)
    r = orc.gen_scalars(n, seed=11)
    assert np.array_equal(jac_to_affine(h2.best_multiexp(r, bg))[0], orc.msm(r, zg))
    assert np.array_equal(jac_to_affine(h2.best_multiexp(r, bl))[0], orc.msm(r, zl))
    bg.release()
    bl.release()
    kd = 5
    nd = 1 << kd
    sg, sl = g.copy(), gl.copy()
    sg[nd] = spoil(sg[nd], REASONS[0])
    sg[n - 1] = spoil(sg[n - 1], REASONS[2])
    sl[0] = spoil(sl[0], REASONS[2])
    path = tmp_path / "skipped.srs"
    path.write_bytes(srs_file_bytes(sg, sl))
    bg, bl = h2.srs_bases(str(path), kd)
    r = orc.gen_scalars(nd, seed=12)
    assert np.array_equal(jac_to_affine(h2.best_multiexp(r, bg))[0], orc.msm(r, g[:nd]))
    assert np.array_equal(jac_to_affine(h2.best_multiexp(r, bl))[0], orc.msm(r, lagrange_relation(g, kd)))
    bg.release()
    bl.release()


@pytest.mark.gpu
def test_argument_errors(gpu):
    """Null g, null handle pointers, k > 26 and window_bits outside {0, 4..24} return -1 with a message and launch nothing."""
    _, g, gl = H.load_srs_fixture()
    L = nat.lib()
    hg, hl = C.c_uint64(SENTINEL), C.c_uint64(SENTINEL)
    before = nat.launch_count()
    cases = [((None, nat.ptr(gl), 6, 0, 0, C.byref(hg), C.byref(hl)), "null argument"),
             ((nat.ptr(g), nat.ptr(gl), 6, 0, 0, None, C.byref(hl)), "null argument"),
             ((nat.ptr(g), nat.ptr(gl), 6, 0, 0, C.byref(hg), None), "null argument"),
             ((nat.ptr(g), None, 27, 0, 0, C.byref(hg), C.byref(hl)), "k = 27 out of range"),
             ((nat.ptr(g), nat.ptr(gl), 6, 3, 0, C.byref(hg), C.byref(hl)), "window_bits 3 not in"),
             ((nat.ptr(g), nat.ptr(gl), 6, 25, 0, C.byref(hg), C.byref(hl)), "window_bits 25 not in"),
             ((nat.ptr(g), nat.ptr(gl), 6, -1, 0, C.byref(hg), C.byref(hl)), "window_bits -1 not in")]
    for args, msg in cases:
        assert L.b200_srs_register(*args) == -1, msg
        err = L.b200_last_error().decode()
        assert err.startswith("srs_register: ") and msg in err, (msg, err)
    assert nat.launch_count() == before
    assert hg.value == SENTINEL and hl.value == SENTINEL


def _device_count():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.gpu
def test_two_devices():
    """The fixture pins in a two-device process: both tables are replicated, and the host MSMs deal their columns over both devices."""
    if _device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "multi"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "multi OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


if __name__ == "__main__" and sys.argv[1:] == ["multi"]:
    nat.check(nat.lib().b200_init_multi(C.c_int(2)))
    nat._inited = True
    _fixture_pins()
    print("multi OK")
