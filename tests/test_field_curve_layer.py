"""Layer 0: BN254 field arithmetic and the G1 group law, on the device and through the host twins, against Python integers.

Every layer above (NTT, MSM, the column kernels, the quotient interpreter) is built from these operations, so each one is
checked here on its own: the generated PTX (fp_ptx.cuh: mul, sqr, the two-product mul2, add, sub), every branch of the XYZZ
formulas (ec.cuh) and of their four-lane cooperative form (ec_coop.cuh), the final-sum kernel behind b200_g1_sum_dev, the
fixed-base and synthetic-base generators of gen_srs, and the group FFT.

The reference is Python integers: oracle/pyref.py plus the Montgomery and XYZZ helpers below; the C oracle's inverse is kept as
one more reference.  The device tier (-m gpu) runs the test hooks of libezkl_b200_dbg.so and the product's entry points; the host
tier runs the same corpus and cases through the host twins, which compile the same op tables for the CPU through the portable
path that the host tail (normalize_host) runs.
"""
import ctypes as C
import functools
import random

import numpy as np
import pytest

from ezkl_b200 import _native as nat
from oracle import oracle as orc
from oracle import pyref

P, R = pyref.P, pyref.R
RM = 1 << 256
FIELDS = {"fr": (0, R), "fq": (1, P)}
OPS = {"add": 0, "sub": 1, "mul": 2, "inv": 3, "from_mont": 4, "sqr": 5, "neg": 6, "dbl": 7, "to_mont": 8}
OPS4 = {"muladd2": 0, "mulsub2": 1}
XYZZ_OPS = {"add": 0, "dbl": 1, "add_mixed": 2, "mul_small": 3, "to_affine": 4, "add_coop4": 5, "dbl_coop4": 6}
G = (1, 2)
BACKENDS = [pytest.param("device", marks=pytest.mark.gpu), "host"]
# random operands per field: the device takes about 2^20 pairs and 2^18 quads; the host twins (and the not-gpu tier) far fewer
N_RANDOM = {"device": (1 << 20, 1 << 18, 1 << 16), "host": (1 << 12, 1 << 11, 1 << 10)}      # pairs, quads, inversions


@pytest.fixture(scope="module")
def dev_ctx():
    nat.init(-1)
    yield


# ---- wire conversion ---------------------------------------------------------------------------------------------
def to_arr(words, width=4) -> np.ndarray:
    """ints < 2^256 -> uint64 [n/k, 4*k] little-endian words."""
    b = b"".join(w.to_bytes(32, "little") for w in words)
    return np.frombuffer(b, dtype="<u8").astype(np.uint64).reshape(-1, width)


def to_ints(a) -> list:
    b = np.ascontiguousarray(a, np.uint64).tobytes()
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def mont(x: int, m: int = P) -> int:
    return x * RM % m


def unmont(w: int, m: int = P) -> int:
    return w * pow(RM, -1, m) % m


def first_diff(got: list, want: list, what) -> str:
    for i, (g, w) in enumerate(zip(got, want)):
        if g != w:
            return "%s: element %d of %d: got %#x, want %#x" % (what, i, len(want), g, w)
    return "%s: lengths %d != %d" % (what, len(got), len(want))


# ---- field reference -----------------------------------------------------------------------------------------------
def ref_field(op: str, m: int, a: list, b: list) -> list:
    """Montgomery words in and out (R = 2^256), each op as the device defines it."""
    ri = pow(RM, -1, m)
    if op == "add":
        return [(x + y) % m for x, y in zip(a, b)]
    if op == "sub":
        return [(x - y) % m for x, y in zip(a, b)]
    if op == "mul":
        return [x * y * ri % m for x, y in zip(a, b)]
    if op == "sqr":
        return [x * x * ri % m for x in a]
    if op == "neg":
        return [-x % m for x in a]
    if op == "dbl":
        return [2 * x % m for x in a]
    if op == "to_mont":
        return [x * RM % m for x in a]
    if op == "from_mont":
        return [x * ri % m for x in a]
    if op == "inv":
        r2 = RM * RM % m
        return [r2 * pow(x, -1, m) % m if x % m else 0 for x in a]
    raise ValueError(op)


def ref_field4(op: str, m: int, a, b, c, d) -> list:
    ri, sg = pow(RM, -1, m), 1 if op == "muladd2" else -1
    return [(w * x + sg * y * z) * ri % m for w, x, y, z in zip(a, b, c, d)]


def redc_t(a: int, b: int, m: int) -> int:
    """The REDC value before its final conditional subtraction: t = (ab + qm) / 2^256 with q = -ab m^-1 mod 2^256 (< 2m)."""
    q = -a * b * pow(m, -1, RM) % RM
    return (a * b + q * m) >> 256


def sqrt_mod(x: int, p: int):
    """Tonelli-Shanks; None when x is not a square mod the prime p."""
    x %= p
    if x == 0:
        return 0
    if pow(x, (p - 1) // 2, p) != 1:
        return None
    q, s = p - 1, 0
    while q % 2 == 0:
        q, s = q // 2, s + 1
    z = 2
    while pow(z, (p - 1) // 2, p) != p - 1:
        z += 1
    mm, c, t, r = s, pow(z, q, p), pow(x, q, p), pow(x, (q + 1) // 2, p)
    while t != 1:
        i, t2 = 0, t
        while t2 != 1:
            t2, i = t2 * t2 % p, i + 1
        bb = pow(c, 1 << (mm - i - 1), p)
        mm, c, t, r = i, bb * bb % p, t * bb * bb % p, r * bb % p
    return r


@functools.lru_cache(maxsize=None)
def field_corpus(field: str, backend: str):
    """(a, b, quads): operand pairs and two-product quads of Montgomery words, all < M except where the generator's mul2 edge
    quads use M itself."""
    _, m = FIELDS[field]
    n_pairs, n_quads, _ = N_RANDOM[backend]
    rng = random.Random(0xF1E1D + len(field) + m % 1000)
    limb1 = [(0xFFFFFFFF << (32 * i)) % m for i in range(8)]                              # one all-ones 32-bit limb
    alt = [int("ffffffff00000000" * 4, 16) % m, int("00000000ffffffff" * 4, 16) % m]       # alternating all-ones / zero limbs
    small = sorted({0, 1, 2, m - 1, m - 2, m >> 1, RM % m, RM * RM % m} | set(limb1) | set(alt)
                   | {m - (1 << (32 * i)) for i in range(8)})                            # M with one limb decremented
    powers = sorted({v for k in range(256) for v in ((1 << k), (1 << k) - 1, m - (1 << k)) if 0 <= v < m})
    edges = sorted(set(small) | set(powers))
    a = [x for x in edges for _ in small] + [y for _ in edges for y in small]
    b = [y for _ in edges for y in small] + [x for x in edges for _ in small]
    # pairs whose Montgomery product is the word 0, 1, field one (R mod M) or field minus one
    for target in (1, RM % m, m - RM % m, m - 1):
        for _ in range(16):
            x = rng.randrange(1, m)
            a.append(x)
            b.append(target * RM * pow(x, -1, m) % m)
    a += [0, rng.randrange(m)]
    b += [rng.randrange(m), 0]
    # pairs whose REDC value t lands just below and just above M (both sides of the final subtraction); squares likewise
    below, above = [], []
    for d in [1, 2, 3] + [1 << k for k in range(2, 200, 7)]:
        for t, side in ((m - d, below), (m + d, above)):
            x = rng.randrange(1, m)
            y = t * RM * pow(x, -1, m) % m
            side.append((x, y))
            s = sqrt_mod(t * RM, m)
            if s is not None:
                s = max(s, m - s)            # the smaller root of a small square would land a multiple of M away
                side.append((s, s))
    for pairs, is_above in ((below, False), (above, True)):
        assert len(pairs) > 32
        assert all((redc_t(x, y, m) >= m) == is_above and abs(redc_t(x, y, m) - m) < (1 << 200) for x, y in pairs)
        assert any(x == y for x, y in pairs)
        a += [x for x, _ in pairs]
        b += [y for _, y in pairs]
    a += [rng.randrange(m) for _ in range(n_pairs)]
    b += [rng.randrange(m) for _ in range(n_pairs)]
    # two-product quads: fp_gen.py's 7^4 edge quads (operands up to and including M), corpus maxima, random
    e2 = [0, 1, m - 1, m, (1 << 254) % m, 0xFFFFFFFF, m >> 1]
    top = [m - 1, m - 2, limb1[7], alt[0], RM % m]
    quads = [(w, x, y, z) for w in e2 for x in e2 for y in e2 for z in e2]
    quads += [(w, x, y, z) for w in top for x in top for y in top for z in top]
    quads += [(x, y, x, y) for x, y in below[:8] + above[:8]]
    quads += [tuple(rng.randrange(m) for _ in range(4)) for _ in range(n_quads)]
    return a, b, quads


def field_call(backend, fid, op, a, b):
    out = np.zeros_like(a)
    L = nat.dbg_lib()
    fn = L.b200_debug_field_op if backend == "device" else L.b200_debug_host_field_op
    assert fn(fid, op, nat.ptr(a), nat.ptr(b), nat.ptr(out), a.shape[0]) == 0
    return out


def field_call4(backend, fid, op, arrs):
    out = np.zeros_like(arrs[0])
    L = nat.dbg_lib()
    fn = L.b200_debug_field_op4 if backend == "device" else L.b200_debug_host_field_op4
    assert fn(fid, op, *[nat.ptr(x) for x in arrs], nat.ptr(out), out.shape[0]) == 0
    return out


@pytest.mark.parametrize("field", ["fr", "fq"])
@pytest.mark.parametrize("backend", BACKENDS)
def test_field_ops_against_python_integers(backend, field, request):
    """add, sub, mul, sqr, neg, dbl, to_mont, from_mont, inv: the value Python computes, every output word vector < M,
    sqr(a) == mul(a, a) word for word, inv(a) * a == 1 and inv(0) == 0; add / sub / mul / inv also against the C oracle."""
    if backend == "device":
        request.getfixturevalue("dev_ctx")
    fid, m = FIELDS[field]
    a, b, _ = field_corpus(field, backend)
    A, B = to_arr(a), to_arr(b)
    got = {}
    for op, code in OPS.items():
        ua = a if op != "inv" else a[:len(a) - N_RANDOM[backend][0] + N_RANDOM[backend][2]]       # the corpus and part of the random pairs
        X = A[:len(ua)]
        out = field_call(backend, fid, code, X, B[:len(ua)])
        g = to_ints(out)
        want = ref_field(op, m, ua, b[:len(ua)])
        assert g == want, first_diff(g, want, (backend, field, op))
        assert max(g) < m, (field, op)
        got[op] = out
        if op in ("add", "sub", "mul"):
            assert np.array_equal(out, orc.field_op(field, op, A, B)), (field, op, "C oracle")
    assert np.array_equal(got["sqr"], field_call(backend, fid, OPS["mul"], A, A)), (field, "sqr(a) != mul(a, a) word for word")
    inv = got["inv"]
    ua = to_ints(inv)
    X = A[:inv.shape[0]]
    assert np.array_equal(inv, orc.fr_inv(X) if field == "fr" else orc.fq_inv(X)), (field, "inv vs C oracle")
    prod = to_ints(field_call(backend, fid, OPS["mul"], inv, X))
    xs = a[:inv.shape[0]]
    assert all(p == (RM % m if x else 0) for p, x in zip(prod, xs)), (field, "inv(a) * a")
    assert all(v == 0 for v, x in zip(ua, xs) if x == 0) and 0 in xs


@pytest.mark.parametrize("field", ["fr", "fq"])
@pytest.mark.parametrize("backend", BACKENDS)
def test_two_product_ops_against_python_integers(backend, field, request):
    """fp_muladd2 / fp_mulsub2 (one Montgomery reduction on the device, the composition of single products on the host)."""
    if backend == "device":
        request.getfixturevalue("dev_ctx")
    fid, m = FIELDS[field]
    quads = field_corpus(field, backend)[2]
    cols = [[q[i] for q in quads] for i in range(4)]
    arrs = [to_arr(c) for c in cols]
    for op, code in OPS4.items():
        g = to_ints(field_call4(backend, fid, code, arrs))
        want = ref_field4(op, m, *cols)
        assert g == want, first_diff(g, want, (backend, field, op))
        assert max(g) < m


# ---- G1 in XYZZ ------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def g1_mul_cached(base, s: int):
    return pyref.g1_mul(base, s)


def xyzz_words(pt, z: int = 1) -> list:
    """affine point (None = identity) -> Montgomery words of (X, Y, ZZ, ZZZ) = (x z^2, y z^3, z^2, z^3); identity is all zero."""
    if pt is None:
        return [0, 0, 0, 0]
    zz = z * z % P
    return [mont(pt[0] * zz), mont(pt[1] * zz * z), mont(zz), mont(zz * z)]


def xyzz_value(words):
    """raw XYZZ words -> the affine point they stand for (None for zz == 0), after checking the representation."""
    assert all(w < P for w in words), "XYZZ word not fully reduced: %s" % [hex(w) for w in words]
    X, Y, ZZ, ZZZ = (unmont(w) for w in words)
    if ZZ == 0:
        return None
    assert ZZZ != 0 and pow(ZZ, 3, P) == pow(ZZZ, 2, P), "ZZ^3 != ZZZ^2"
    return (X * pow(ZZ, -1, P) % P, Y * pow(ZZZ, -1, P) % P)


def rand_z(rng) -> int:
    return rng.randrange(2, P)


@functools.lru_cache(maxsize=None)
def group_cases():
    """The binary cases of the group law: (name, s_a, s_b, z_a, z_b) with a = [s_a]G, b = [s_b]G (s = 0: identity), interleaved
    case by case so that the quads of one warp take different branches, and n not a multiple of 8."""
    rng = random.Random(0x6A0)
    kinds = ["generic", "generic_z1", "equal_same_z", "equal_diff_z", "negated_diff_z", "identity_left", "identity_right",
             "identity_both", "b_is_2a"]
    per = []
    for kind in kinds:
        rows = []
        for rep in range(7):
            sa, sb = rng.randrange(1, R), rng.randrange(1, R)
            za, zb = 1 if rep == 0 else rand_z(rng), rand_z(rng)     # one element of every case with a Z = 1 left operand
            if kind == "generic_z1":
                za = zb = 1
            elif kind == "equal_same_z":
                sb, zb = sa, za
            elif kind == "equal_diff_z":
                sb = sa
            elif kind == "negated_diff_z":
                sb = R - sa
            elif kind == "identity_left":
                sa = 0
            elif kind == "identity_right":
                sb = 0
            elif kind == "identity_both":
                sa = sb = 0
            elif kind == "b_is_2a":
                sb = 2 * sa % R
            rows.append((kind, sa, sb, za, zb))
        per.append(rows)
    cases = [rows[i] for i in range(7) for rows in per]
    assert len(cases) % 8 != 0
    return cases


def pt(s):
    return g1_mul_cached(G, s % R) if s % R else None


def xyzz_call(backend, op, a, b, k):
    out = np.zeros_like(a)
    L = nat.dbg_lib()
    fn = L.b200_debug_g1_xyzz_op if backend == "device" else L.b200_debug_host_g1_xyzz_op
    kk = np.ascontiguousarray(k, np.uint32)
    assert fn(XYZZ_OPS[op], nat.ptr(a), nat.ptr(b), kk.ctypes.data_as(C.c_void_p), nat.ptr(out), a.shape[0]) == 0
    return out


def check_xyzz_outputs(out, want, what):
    words = to_ints(out)
    for i, exp in enumerate(want):
        w = words[4 * i:4 * i + 4]
        got = xyzz_value(w)
        assert got == exp, (what, i, got, exp)
        if exp is None:
            assert w[2] == 0, (what, i, "identity with zz != 0")


@pytest.mark.parametrize("backend", BACKENDS)
def test_xyzz_group_law_every_branch(backend, request):
    """g1_add, g1_add_mixed, g1_dbl, g1_to_affine (and on the device g1_add_coop4 / g1_dbl_coop4) on generic points, a == b with
    the same and with different Z, a == -b, identity on either side and on both, and b == 2a: the affine value pyref gives,
    ZZ^3 == ZZZ^2, zz == 0 for identity, every word < P; the cooperative ops equal the plain ones word for word."""
    if backend == "device":
        request.getfixturevalue("dev_ctx")
    cases = group_cases()
    A = to_arr([w for _, sa, _, za, _ in cases for w in xyzz_words(pt(sa), za)], 16)
    B = to_arr([w for _, _, sb, _, zb in cases for w in xyzz_words(pt(sb), zb)], 16)
    Baff = to_arr([w for _, _, sb, _, _ in cases for w in xyzz_words(pt(sb), 1)], 16)   # (x, y) of b read as affine
    Baff[:, 8:] = 0
    k = np.zeros(len(cases), np.uint32)
    plain = {}
    for op, b, want in (("add", B, [pt(sa + sb) for _, sa, sb, _, _ in cases]),
                        ("add_mixed", Baff, [pt(sa + sb) for _, sa, sb, _, _ in cases]),
                        ("dbl", B, [pt(2 * sa) for _, sa, _, _, _ in cases])):
        plain[op] = xyzz_call(backend, op, A, b, k)
        for i, (kind, *_rest) in enumerate(cases):
            check_xyzz_outputs(plain[op][i:i + 1], [want[i]], (backend, op, kind))
    # g1_dbl on every operand form, b included (its Z != 1 and identity rows)
    dB = xyzz_call(backend, "dbl", B, B, k)
    check_xyzz_outputs(dB, [pt(2 * sb) for _, _, sb, _, _ in cases], (backend, "dbl of b"))
    aff = xyzz_call(backend, "to_affine", A, B, k)
    words = to_ints(aff)
    for i, (_, sa, _, _, _) in enumerate(cases):
        p = pt(sa)
        assert words[4 * i:4 * i + 4] == ([mont(p[0]), mont(p[1]), 0, 0] if p else [0, 0, 0, 0]), ("to_affine", i)
    if backend == "device":
        for op, coop in (("add", "add_coop4"), ("dbl", "dbl_coop4")):
            got = xyzz_call(backend, coop, A, B, k)
            for i, (kind, *_rest) in enumerate(cases):
                assert np.array_equal(got[i], plain[op][i]), (coop, kind, i, "differs from the plain op word for word")
        assert np.array_equal(xyzz_call(backend, "dbl_coop4", B, B, k), dB)


@pytest.mark.parametrize("backend", BACKENDS)
def test_xyzz_mul_small(backend, request):
    """g1_mul_small: k = 0..4, alternating bits, the top 2-bit windows, 2^32 - 1 and random, on Z != 1 points and on identity."""
    if backend == "device":
        request.getfixturevalue("dev_ctx")
    rng = random.Random(0x5A11)
    ks = [0, 1, 2, 3, 4, 0x55555555, 0xAAAAAAAA, 1 << 31, 3 << 30, 0xFFFFFFFF] + [rng.randrange(1 << 32) for _ in range(13)]
    rows = [(k, s) for k in ks for s in (rng.randrange(1, R), rng.randrange(1, R), 0)]
    A = to_arr([w for _, s in rows for w in xyzz_words(pt(s), rand_z(rng))], 16)
    out = xyzz_call(backend, "mul_small", A, A, np.array([k for k, _ in rows], np.uint32))
    check_xyzz_outputs(out, [pt(k * s) for k, s in rows], (backend, "mul_small"))


@pytest.mark.parametrize("backend", BACKENDS)
def test_affine_group_law_hooks(backend, request):
    """b200_debug_g1_op (affine in and out: mixed add, dbl, mul_small, the g1_dbl_affine doubling branch of g1_add, P + (-P)) on
    generic and degenerate inputs, against pyref and the C oracle."""
    if backend == "device":
        request.getfixturevalue("dev_ctx")
    rng = random.Random(6)
    n = 37
    sa, sb = [rng.randrange(1, R) for _ in range(n)], [rng.randrange(1, R) for _ in range(n)]
    sa[0] = 0                 # identity + P
    sb[1] = 0                 # P + identity
    sa[2] = sb[2]             # P + P through the mixed-add doubling branch
    sa[3] = 2 * sb[3] % R     # a == 2b through g1_add's doubling branch
    sa[4] = R - sb[4]         # P + (-P)
    A = to_arr([w for s in sa for w in xyzz_words(pt(s))[:2]], 8)
    B = to_arr([w for s in sb for w in xyzz_words(pt(s))[:2]], 8)
    L = nat.dbg_lib()
    fn = L.b200_debug_g1_op if backend == "device" else L.b200_debug_host_g1_op

    def run(op, b):
        out = np.zeros_like(A)
        assert fn(op, nat.ptr(A), nat.ptr(b), nat.ptr(out), n) == 0
        return out

    def affine(out):
        w = to_ints(out)
        return [None if not (w[2 * i] or w[2 * i + 1]) else (unmont(w[2 * i]), unmont(w[2 * i + 1])) for i in range(n)]

    out = run(0, B)
    assert affine(out) == [pt(x + y) for x, y in zip(sa, sb)] and np.array_equal(out, orc.g1_add_affine(A, B))
    out = run(1, B)
    assert affine(out) == [pt(2 * x) for x in sa] and np.array_equal(out, orc.g1_add_affine(A, A))
    ks = [rng.randrange(1 << 20) for _ in range(n)]
    ks[5:16] = [0, 1, 2, 3, 4, 0xFFFFF, 0x55555, 0xAAAAA, 0xFFFFFFFF, 0x80000000, 0x30003]
    K = B.copy()
    K[:, 0] = ks
    assert affine(run(2, K)) == [pt(k * x) for k, x in zip(ks, sa)]
    assert affine(run(3, B)) == [pt(x + 2 * y) for x, y in zip(sa, sb)]
    out = run(4, B)
    assert not out.any()


# ---- the product's G1 entry points -----------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def point_pool():
    """16 points [s]G, each under 4 Z (the first Z = 1), and the same for the negated points: (scalars, words [16, 4, 2, 4])."""
    rng = random.Random(0x5E7)
    ss = [rng.randrange(1, R) for _ in range(16)]
    words = np.zeros((16, 4, 2, 16), np.uint64)
    for i, s in enumerate(ss):
        p = pt(s)
        for j in range(4):
            z = 1 if j == 0 else rand_z(rng)
            words[i, j, 0] = to_arr(xyzz_words(p, z), 16)[0]
            words[i, j, 1] = to_arr(xyzz_words(pyref.g1_neg(p), z), 16)[0]
    return ss, words


def sum_column(kind: str, count: int, rng: random.Random):
    """One column of `count` XYZZ points of the given kind: (words [count, 16], sum of their scalars mod r)."""
    ss, words = point_pool()
    idx, zi, neg = [], [], []
    if kind == "random":
        idx = [rng.randrange(16) for _ in range(count)]
        zi, neg = [rng.randrange(4) for _ in range(count)], [0] * count
    elif kind == "repeated":                 # one point under different Z: the tree doubles at every level
        p = rng.randrange(16)
        idx, zi, neg = [p] * count, [j % 4 for j in range(count)], [0] * count
    elif kind == "cancelling":               # +-P pairs half a column apart: identity partials in lanes and in the tree
        h = count // 2
        idx = [rng.randrange(16) for _ in range(h)]
        idx = idx + idx + [rng.randrange(16) for _ in range(count - 2 * h)]
        zi = [rng.randrange(4) for _ in range(count)]
        neg = [0] * h + [1] * h + [0] * (count - 2 * h)
    elif kind == "identity":
        idx = [-1] * count
    else:                                    # mixed: random, identity, a repeat and the negation of the previous point
        for j in range(count):
            c = rng.randrange(4)
            if c == 0 or not idx or idx[-1] < 0:
                idx.append(rng.randrange(16)); neg.append(0)
            elif c == 1:
                idx.append(-1); neg.append(0)
            elif c == 2:
                idx.append(idx[-1]); neg.append(neg[-1])
            else:
                idx.append(idx[-1]); neg.append(1 - neg[-1])
            zi.append(rng.randrange(4))
    if kind == "identity":
        return np.zeros((count, 16), np.uint64), 0
    out = np.zeros((count, 16), np.uint64)
    total = 0
    for j, (i, z, ng) in enumerate(zip(idx, zi, neg)):
        if i >= 0:
            out[j] = words[i, z, ng]
            total += -ss[i] if ng else ss[i]
    return out, total % R


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["random", "repeated", "cancelling", "identity", "mixed"])
def test_g1_sum_dev(kind, dev_ctx):
    """b200_g1_sum_dev (k_final_coop: the COOP_LT-strided partials loop, then the four-lane tree), read back through
    b200_g1_normalize (identity as (0, 1, 0)), against the Python sum, for groups {1, 2, 5, 33} x count {0 .. 1000}."""
    import torch
    from ezkl_b200 import device as D
    rng = random.Random(hash(kind) & 0xFFFF)
    one = mont(1)
    for groups in (1, 2, 5, 33):
        for count in (0, 1, 2, 3, 63, 64, 65, 127, 128, 129, 1000):
            cols = [sum_column(kind, count, rng) for _ in range(groups)]
            host = np.concatenate([c for c, _ in cols]) if count else np.zeros((1, 16), np.uint64)
            d_in = torch.from_numpy(host.view(np.int64)).cuda()
            d_out = torch.full((groups, 16), -1, dtype=torch.int64, device="cuda")
            nat.check(nat.lib().b200_g1_sum_dev(d_in.data_ptr(), groups, count, d_out.data_ptr(), D._stream()))
            jac = to_ints(D.normalize(d_out).reshape(-1, 4))
            for g, (_, s) in enumerate(cols):
                x, y, z = jac[3 * g:3 * g + 3]
                p = pt(s)
                want = (0, one, 0) if p is None else (mont(p[0]), mont(p[1]), one)
                assert (x, y, z) == want, (kind, groups, count, g)


@pytest.mark.gpu
def test_g1_fixed_base_mul_dev(dev_ctx):
    """k_g1_fixed_base_mul: scalars 0, 1, 2, r - 1, r - 2, (r - 1) / 2, 2^k for k = 0..253 and random, on G, a random point and
    the identity, in calls of n = 1, 127, 128 and 129, against pyref.g1_mul."""
    import torch
    from ezkl_b200 import device as D
    rng = random.Random(0xF1B)
    scalars = [0, 1, 2, R - 1, R - 2, (R - 1) // 2] + [1 << k for k in range(254)] + [rng.randrange(R) for _ in range(40)]
    rnd = pt(rng.randrange(1, R))
    for base in (G, rnd, None):
        bw = to_arr(xyzz_words(base)[:2], 8)[0]
        want_all = [g1_mul_cached(base, s % R) if base and s % R else None for s in scalars]
        for n in (1, 127, 128, 129):
            for lo in range(0, len(scalars), n):
                chunk = scalars[lo:lo + n]
                d_s = torch.from_numpy(to_arr([mont(s % R, R) for s in chunk]).view(np.int64)).cuda()
                out = D.to_host(D.fixed_base_mul(d_s, bw))
                w = to_ints(out)
                got = [None if not (w[2 * i] or w[2 * i + 1]) else (unmont(w[2 * i]), unmont(w[2 * i + 1])) for i in range(len(chunk))]
                assert got == want_all[lo:lo + n], (base is G, base is None, n, lo)


def splitmix_scalar(seed: int, i: int) -> int:
    """k_g1_generate's scalar for index i: four splitmix64 outputs from seed + golden * (i + 1), top 4 bits cleared (< 2^252)."""
    gold, m64 = 0x9E3779B97F4A7C15, (1 << 64) - 1
    z, s = (seed + gold * (i + 1)) & m64, 0
    for w in range(4):
        z = (z + gold) & m64
        x = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m64
        x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & m64
        s |= (x ^ (x >> 31)) << (64 * w)
    return s & ((1 << 252) - 1)


@pytest.mark.gpu
def test_g1_generate_dev(dev_ctx):
    """b200_g1_generate_dev: exact points [splitmix(seed, i)]G at indices {0, 1, 127, 128, n - 1}, and every point on the curve."""
    from ezkl_b200 import device as D
    for seed in (0xE2C1B200, 0x0123456789ABCDEF):
        for n in (1, 129, 5000):
            w = to_ints(D.to_host(D.generate_bases(n, seed=seed)).reshape(-1, 4))
            pts = [(unmont(w[2 * i]), unmont(w[2 * i + 1])) for i in range(n)]
            assert all(pyref.g1_is_on_curve(p) and p != (0, 0) for p in pts), (seed, n)
            for i in sorted({0, 1, 127, 128, n - 1}):
                if i < n:
                    assert pts[i] == pt(splitmix_scalar(seed, i)), (seed, n, i)


def fft_scalars(log_n: int, rng: random.Random) -> list:
    """Random scalars with zeros (identity inputs), and equal and opposite values at bit-reversed neighbours (i, i + n/2), whose
    first-stage butterfly doubles (u + t) and cancels (u - t), or the reverse."""
    n = 1 << log_n
    s = [rng.randrange(R) for _ in range(n)]
    if n >= 4:
        s[0] = 0
        s[n // 2 + 1] = s[1]
    if n >= 8:
        s[n // 2 + 2] = R - s[2]
        s[3] = s[n // 2 + 3] = 0
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", [0, 1, 2, 3, 4, 5, 6, 8, 10, 12, 14])
def test_g1_fft_exact(log_n, dev_ctx):
    """b200_g1_fft and b200_g1_fft_dev on inputs [s_i]G: the outputs are [scale * s^_j]G with s^ the scalar DFT, with and without
    scale.  Up to 2^6 the DFT and the points come from Python; above, the C oracle's scalar NTT and the device's fixed-base
    multiplication (checked exactly above) give them."""
    import torch
    from ezkl_b200 import device as D
    rng = random.Random(0xECF + log_n)
    n = 1 << log_n
    s = fft_scalars(log_n, rng)
    w = pyref.omega_for(log_n)
    sc = rng.randrange(1, R)
    small = log_n <= 6
    if small:
        hat = pyref.dft_naive(s, w)
        to_pts = lambda xs: to_arr([v for x in xs for v in xyzz_words(pt(x))[:2]], 8)
    else:
        hat = to_ints(orc.best_fft(to_arr([mont(x, R) for x in s]), log_n, to_arr([mont(w, R)])[0]))
        hat = [unmont(x, R) for x in hat]

        def to_pts(xs):
            d_s = torch.from_numpy(to_arr([mont(x, R) for x in xs]).view(np.int64)).cuda()
            return D.to_host(D.fixed_base_mul(d_s)).astype(np.uint64)
    pin = np.ascontiguousarray(to_pts(s))
    omega = to_arr([mont(w, R)])[0]
    for scale in (None, sc):
        want = to_pts([x * (scale or 1) % R for x in hat])
        scale_w = to_arr([mont(scale, R)])[0] if scale else None
        out = np.zeros_like(pin)
        nat.check(nat.lib().b200_g1_fft(nat.ptr(pin), log_n, nat.ptr(omega), nat.ptr(scale_w) if scale else None, nat.ptr(out)))
        assert np.array_equal(out, want), (log_n, scale is not None, "b200_g1_fft")
        d_in = torch.from_numpy(pin.view(np.int64)).cuda()
        d_out = torch.empty_like(d_in)
        nat.check(nat.lib().b200_g1_fft_dev(d_in.data_ptr(), log_n, nat.ptr(omega), nat.ptr(scale_w) if scale else None, d_out.data_ptr(),
                                            D._stream()))
        assert np.array_equal(D.to_host(d_out).astype(np.uint64), want), (log_n, scale is not None, "b200_g1_fft_dev")
    assert n == pin.shape[0]
