"""Proving key straight to the device (b200_pk_load, device.load_proving_key): the key's fixed_values and permutations columns are
staged into device memory and checked there as halo2curves' Fr::from_raw_bytes checks them, and the key's coefficient columns and l-cosets are
derived on the device instead of read.  Pinned by the reference proving key: its sections are rebuilt from tests/golden (the fixture's
values, the fixture mapping's sigma columns, the derived sections) into a file whose sha256 is the manifest's, and the device's outputs equal
that file's sections byte for byte.

The small-budget check needs its own process (the budget is read once, at b200_init) and runs this file as a script:
`python tests/test_pk_load.py budget`."""
import ctypes as C
import hashlib
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
from oracle import pyref                      # noqa: E402
from tests import helpers as H                # noqa: E402
from tests import perm_keygen_ref as ref      # noqa: E402
from tests import test_permutation_keygen as tpk  # noqa: E402

P_, S, Z, U32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
K6, EXT6, BF6, NPERM6, NSEL6 = 6, 9, 5, 32, 80          # the reference key: k = 6, ext_k = 9, 5 blinding rows, 32 permutation columns, 80 selectors
SENTINEL = -0x2152411021524111                           # 0xDEADBEEFDEADBEEF as int64
MIB = 1 << 20


def reference_key():
    """The reference pk.key as a ProvingKey: vk and fixed values from the fixture, the fixture mapping's sigma columns as the permutations and
    the derived sections from keygen_pk_polys (on the device, or on whatever backend the caller patched in)."""
    from ezkl_b200 import halo2 as h2
    prim = np.load(os.path.join(H.GOLDEN, "pk_k6_primary.npz"))
    sig = ref.perm_sigmas(tpk.fixture_mapping(), K6)
    der = tpk.keygen_derived(sig)
    pk = h2.ProvingKey()
    pk.k, pk.vk_bytes = K6, prim["vk"].tobytes()
    pk.l0, pk.l_last, pk.l_active_row = der["l0"], der["l_last"], der["l_active_row"]
    pk.fixed_values, pk.fixed_polys, pk.fixed_cosets = list(prim["fixed_values"]), der["fixed_polys"], der["fixed_cosets"]
    pk.permutations, pk.permutation_polys, pk.permutation_cosets = list(sig), der["permutation_polys"], der["permutation_cosets"]
    return pk


def below_r(limbs) -> bool:
    """The check rule: the four little-endian u64 limbs, read as one 256-bit integer, are below r."""
    return H.limbs_to_int(np.asarray(limbs, np.uint64).reshape(4)) < pyref.R


# ---- CPU ---------------------------------------------------------------------------------------------------------------------------
def test_pk_load_is_exported_and_typed():
    """include/ezkl_b200.h declares b200_pk_load, exported with the argtypes / restype read from that header."""
    decls = nat.declarations(nat.HEADER)
    fn = nat.lib().b200_pk_load
    assert (fn.argtypes, fn.restype) == decls["b200_pk_load"]
    assert decls["b200_pk_load"] == ([P_, S, P_, S, U32, U32, U32, P_, P_, S, P_], Z)


@pytest.fixture(scope="module")
def cpu_key_bytes():
    from tests import cpu_backend as cb
    with pytest.MonkeyPatch.context() as mp:
        cb.patch_backend(mp)
        return reference_key().to_bytes()


def test_writer_reproduces_the_reference_key(cpu_key_bytes, tmp_path):
    """ProvingKey.write of the rebuilt reference key (derived sections on the CPU oracle) has the manifest's sha256, and ProvingKey.read of the
    written file gives back every section."""
    from ezkl_b200 import halo2 as h2
    from tests import cpu_backend as cb
    assert hashlib.sha256(cpu_key_bytes).hexdigest() == tpk.reference_sha256()
    with pytest.MonkeyPatch.context() as mp:
        cb.patch_backend(mp)
        pk = reference_key()
    path = tmp_path / "pk.key"
    pk.write(str(path))
    assert path.read_bytes() == cpu_key_bytes
    back = h2.ProvingKey.read(str(path), NPERM6, NSEL6)
    assert back.k == K6 and back.vk_bytes == pk.vk_bytes
    for name in ("l0", "l_last", "l_active_row"):
        assert np.array_equal(getattr(back, name), getattr(pk, name)), name
    for name in h2.ProvingKey.SECTIONS[3:]:
        got, want = getattr(back, name), getattr(pk, name)
        assert len(got) == len(want) and all(np.array_equal(a, b) for a, b in zip(got, want)), name


def test_layout_matches_read(cpu_key_bytes, tmp_path):
    """The header walker's offsets point at the columns ProvingKey.read finds, section by section."""
    from ezkl_b200 import halo2 as h2
    path = tmp_path / "pk.key"
    path.write_bytes(cpu_key_bytes)
    pk = h2.ProvingKey.read(str(path), NPERM6, NSEL6)
    lay = h2.ProvingKey.layout(cpu_key_bytes, NPERM6, NSEL6, EXT6)
    assert lay["k"] == K6 and lay["vk_len"] == 5127 == len(pk.vk_bytes)
    for name in h2.ProvingKey.SECTIONS:
        want = [getattr(pk, name)] if name.startswith("l") else getattr(pk, name)
        assert len(lay[name]) == len(want), name
        for off, col in zip(lay[name], want):
            assert np.frombuffer(cpu_key_bytes, "<u8", count=4 * col.shape[0], offset=off).reshape(-1, 4).tobytes() == col.tobytes(), name


def _malformed(data):
    """(name, bytes, num_permutation_columns, num_selectors, ext_k, message) of every malformed variant of the reference key."""
    from ezkl_b200 import halo2 as h2
    lay = h2.ProvingKey.layout(data, NPERM6, NSEL6, EXT6)
    fv = lay["fixed_values"][0] - 4 - 4 - 4 * 38                # the fixed_values slice header: count, length table
    poly0 = lay["permutation_polys"][0] - 4                     # the first permutation poly's length
    return [("truncated", data[:-1], NPERM6, NSEL6, EXT6, "truncated"),
           ("vk only", data[:5127], NPERM6, NSEL6, EXT6, "truncated"),
           ("empty header", data[:5], NPERM6, NSEL6, EXT6, "no vk header"),
           ("trailing", data + b"\0", NPERM6, NSEL6, EXT6, "trailing"),
           ("version 2", b"\x02" + data[1:], NPERM6, NSEL6, EXT6, "version 2"),
           ("count", data[:fv] + struct.pack(">I", 37) + data[fv + 4:], NPERM6, NSEL6, EXT6, "fixed_values has 37 columns, expected 38"),
           ("length table", data[:fv + 4] + struct.pack(">I", 63) + data[fv + 8:], NPERM6, NSEL6, EXT6, "length table"),
           ("length", data[:poly0] + struct.pack(">I", 65) + data[poly0 + 4:], NPERM6, NSEL6, EXT6, "permutation_polys has a column of length 65"),
           ("ext_k", data, NPERM6, NSEL6, EXT6 + 1, "l0 has a column of length 512, expected 1024"),
           ("ext_k < k", data, NPERM6, NSEL6, K6 - 1, "need 1 <= k"),
           ("fewer permutation columns", data, NPERM6 - 1, NSEL6, EXT6, "pk layout"),
           ("more permutation columns", data, NPERM6 + 1, NSEL6, EXT6, "pk layout"),
           ("fewer selectors", data, NPERM6, NSEL6 - 1, EXT6, "pk layout"),
           ("more selectors", data, NPERM6, NSEL6 + 1, EXT6, "pk layout")]


def test_layout_rejects_malformed_keys_before_the_library(cpu_key_bytes, tmp_path, monkeypatch):
    """Truncation, trailing bytes, a wrong version, a wrong count, length or length-table entry, a wrong ext_k and wrong permutation column or
    selector counts each raise B200Error from the walker, and load_proving_key raises it before the library is called."""
    from ezkl_b200 import device as dv
    from ezkl_b200 import halo2 as h2

    def no_device(*a, **kw):
        raise AssertionError("the library was called")
    monkeypatch.setattr(nat, "ensure_init", no_device)
    monkeypatch.setattr(nat, "lib", no_device)
    for name, blob, npc, nsel, ext_k, msg in _malformed(cpu_key_bytes):
        with pytest.raises(nat.B200Error, match=msg):
            h2.ProvingKey.layout(blob, npc, nsel, ext_k)
        p = tmp_path / ("%s.key" % name.replace(" ", "_"))
        p.write_bytes(blob)
        with pytest.raises(nat.B200Error, match=msg):
            dv.load_proving_key(str(p), npc, nsel, ext_k, BF6)
    empty = tmp_path / "empty.key"
    empty.write_bytes(b"")
    with pytest.raises(nat.B200Error, match="empty"):
        dv.load_proving_key(str(empty), NPERM6, NSEL6, EXT6, BF6)


def test_check_rule_in_python_ints():
    """r - 1 passes; r, r + 1 and 2^256 - 1 fail; a value above r only through its top limb fails, and one below r in its top limb passes
    whatever its lower limbs; the reference key's value columns all pass."""
    r = pyref.R
    top = r >> 192
    assert below_r(H.int_to_limbs(r - 1)) and below_r(H.int_to_limbs(0))
    for v in (r, r + 1, (1 << 256) - 1):
        assert not below_r(H.int_to_limbs(v)), hex(v)
    low = r & ((1 << 192) - 1)
    for lo in (0, low, low - 1, (1 << 192) - 1):
        assert not below_r(H.int_to_limbs(((top + 1) << 192) | lo)), hex(lo)
        assert below_r(H.int_to_limbs(((top - 1) << 192) | lo)), hex(lo)
    assert below_r(H.int_to_limbs((top << 192) | (low - 1))) and not below_r(H.int_to_limbs((top << 192) | low))
    prim = np.load(os.path.join(H.GOLDEN, "pk_k6_primary.npz"))
    cols = np.concatenate([prim["fixed_values"], ref.perm_sigmas(tpk.fixture_mapping(), K6)])
    assert all(below_r(e) for e in cols.reshape(-1, 4))


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu():
    nat.ensure_init()
    yield


def free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def host_columns(cols, offsets=None):
    """Each column copied to its own host buffer at a byte offset (odd by default: the library must read them as bytes) -> (pointers, keep)."""
    keep, ptrs = [], []
    for j, c in enumerate(cols):
        off = (2 * j + 1) % 7 if offsets is None else offsets
        b = np.zeros(c.nbytes + off, np.uint8)
        b[off:] = np.ascontiguousarray(c, np.uint64).view(np.uint8).reshape(-1)
        keep.append(b)
        ptrs.append(b.ctypes.data + off)
    return ptrs, keep


def pk_load(fixed, perm, k, ext_k, bf, values, polys, stride, l):
    """b200_pk_load through ctypes; fixed / perm are lists of host addresses, values / polys / l device addresses (or None)."""
    arr = lambda ps: (C.c_void_p * len(ps))(*ps) if ps else None
    return nat.lib().b200_pk_load(arr(fixed), len(fixed), arr(perm), len(perm), k, ext_k, bf, values, polys, stride, l)


def outputs(ncols, n, N, stride=None):
    import torch
    stride = stride or n
    v = torch.full((max(ncols, 1), stride, 4), SENTINEL, dtype=torch.int64, device="cuda")
    p = torch.full_like(v, SENTINEL)
    l = torch.full((3, N, 4), SENTINEL, dtype=torch.int64, device="cuda")
    return v, p, l


def host(t):
    from ezkl_b200 import device as dv
    return dv.to_host(t)


@pytest.mark.gpu
def test_reference_pin(gpu, tmp_path):
    """The rebuilt reference key (derived sections on the device, sha256 checked) written to a file and loaded: values, polys and the three
    l-vectors equal the file's own sections byte for byte, and the vk bytes are the file's prefix."""
    from ezkl_b200 import device as dv
    pk = reference_key()
    data = pk.to_bytes()
    assert hashlib.sha256(data).hexdigest() == tpk.reference_sha256()
    path = tmp_path / "pk.key"
    pk.write(str(path))
    got = dv.load_proving_key(str(path), NPERM6, NSEL6, EXT6, BF6)
    _assert_equals_key(got, pk)


def _assert_equals_key(got, pk):
    assert got.k == K6 and got.ext_k == EXT6 and got.num_fixed == 38 and got.vk_bytes == pk.vk_bytes
    assert host(got.values).tobytes() == np.stack(pk.fixed_values + pk.permutations).tobytes()
    assert host(got.polys).tobytes() == np.stack(list(pk.fixed_polys) + list(pk.permutation_polys)).tobytes()
    for name in ("l0", "l_last", "l_active_row"):
        assert host(getattr(got, name)).tobytes() == np.ascontiguousarray(getattr(pk, name)).tobytes(), name


@pytest.mark.gpu
def test_unread_sections_stay_unread(gpu, tmp_path):
    """Every element byte of the file's polys, cosets and l-vectors overwritten with 0xff (not below r): the key still loads, with the same
    bytes, because those sections are never read."""
    from ezkl_b200 import device as dv
    from ezkl_b200 import halo2 as h2
    pk = reference_key()
    data = bytearray(pk.to_bytes())
    lay = h2.ProvingKey.layout(bytes(data), NPERM6, NSEL6, EXT6)
    for name in ("l0", "l_last", "l_active_row", "fixed_polys", "fixed_cosets", "permutation_polys", "permutation_cosets"):
        length = 32 * ((1 << EXT6) if name.startswith("l") or name.endswith("cosets") else (1 << K6))
        for off in lay[name]:
            data[off:off + length] = b"\xff" * length
    path = tmp_path / "spoiled.key"
    path.write_bytes(bytes(data))
    _assert_equals_key(dv.load_proving_key(str(path), NPERM6, NSEL6, EXT6, BF6), pk)


def random_columns(count, n, seed):
    rng = np.random.default_rng(seed)
    cols = rng.integers(0, 1 << 64, size=(count, n, 4), dtype=np.uint64)
    cols[..., 3] &= np.uint64(0x0FFFFFFFFFFFFFFF)            # below 2^252 < r
    return cols


J_OF_D = {0: 2, 1: 3, 2: 5, 3: 9}                            # EvaluationDomain(j, k) with extended_k = k + d
# (k, ext_k - k, blinding_factors, fixed, permutation, stride - 2^k)
LARGE = ([(k, k % 4, [0, 1, 5, (1 << k) - 1, (1 << k) // 2][k % 5] % (1 << k), 1 + k % 3, k % 2 + 1, [0, 3][k % 2]) for k in range(1, 13)]
         + [(20, 3, 5, 2, 2, 0), (22, 3, 5, 1, 1, 0), (24, 1, 6, 1, 1, 0)])


@pytest.mark.gpu
@pytest.mark.parametrize("k,d,bf,nf,npc,extra", LARGE, ids=["k%d-d%d-bf%d-%d+%d-s%d" % c for c in LARGE])
def test_random_values_from_host_memory(gpu, k, d, bf, nf, npc, extra):
    """Random canonical columns passed from host memory at odd byte offsets (no file): values are the columns, polys equal
    EvaluationDomain.lagrange_to_coeff_batch, the l-vectors equal keygen_l_polys (both pinned at k = 6); rows between 2^k and the stride
    keep their fill."""
    from ezkl_b200 import halo2 as h2
    n = 1 << k
    dom = h2.EvaluationDomain(J_OF_D[d], k)
    assert dom.extended_k == k + d
    N = 1 << dom.extended_k
    cols = random_columns(nf + npc, n, seed=k * 7 + d)
    ptrs, keep = host_columns(cols)
    v, p, l = outputs(nf + npc, n, N, n + extra)
    rc = pk_load(ptrs[:nf], ptrs[nf:], k, k + d, bf, v.data_ptr(), p.data_ptr(), n + extra, l.data_ptr())
    assert rc == 0, nat.lib().b200_last_error()
    hv, hp = host(v), host(p)
    assert hv[:, :n].tobytes() == cols.tobytes()
    assert hp[:, :n].tobytes() == np.stack(dom.lagrange_to_coeff_batch(list(cols))).tobytes()
    if extra:
        assert (hv[:, n:] == np.uint64(SENTINEL & (2**64 - 1))).all() and (hp[:, n:] == np.uint64(SENTINEL & (2**64 - 1))).all()
    assert host(l).tobytes() == np.stack(dom.keygen_l_polys(bf)).tobytes()
    del keep


def _spoil(col, row, how, rng):
    """A non-canonical element in place of col[row]: r, r + a small value, or 2^256 - 1."""
    col[row] = H.int_to_limbs({"r": pyref.R, "r+": pyref.R + rng.randrange(1, 1 << 20), "max": (1 << 256) - 1}[how])
    assert not below_r(col[row])


def _assert_rejected(fixed, perm, k, ext_k, msg):
    n, N = 1 << k, 1 << ext_k
    cols = fixed + perm
    ptrs, keep = host_columns(cols)
    v, p, l = outputs(len(cols), n, N)
    before, launches = free_bytes(), nat.launch_count()
    rc = pk_load(ptrs[:len(fixed)], ptrs[len(fixed):], k, ext_k, 3, v.data_ptr(), p.data_ptr(), n, l.data_ptr())
    err = nat.lib().b200_last_error().decode()
    assert rc == -1 and err == msg, (rc, err, msg)
    assert nat.launch_count() - launches == len(cols)          # the checks and nothing else
    assert (host(p) == np.uint64(SENTINEL & (2**64 - 1))).all() and (host(l) == np.uint64(SENTINEL & (2**64 - 1))).all()
    assert abs(free_bytes() - before) <= MIB, (before, free_bytes())
    del keep


@pytest.mark.gpu
def test_rejection(gpu):
    """Each section x first / middle / last column x first / middle / last row: -1 naming the section, column and row; d_polys and d_l keep
    their fill, only the check kernels ran and no device memory is kept.  With several bad elements the lowest (section, column, row) is named,
    fixed_values before permutations.  One case at k = 20, whose columns take the pinned copy path."""
    rng = random.Random(9)
    k, ext_k, nf, npc = 10, 12, 5, 4
    n = 1 << k
    base = random_columns(nf + npc, n, seed=1)
    v, p, l = outputs(nf + npc, n, 1 << ext_k)                    # warm-up: the context and its check word exist before memory is compared
    ptrs, keep = host_columns(base)
    assert pk_load(ptrs[:nf], ptrs[nf:], k, ext_k, 3, v.data_ptr(), p.data_ptr(), n, l.data_ptr()) == 0
    del v, p, l, keep
    for section, count in (("fixed_values", nf), ("permutations", npc)):
        for j in (0, count // 2, count - 1):
            for row in (0, n // 2 + 1, n - 1):
                cols = [c.copy() for c in base]
                _spoil(cols[j if section == "fixed_values" else nf + j], row, rng.choice(["r", "r+", "max"]), rng)
                _assert_rejected(cols[:nf], cols[nf:], k, ext_k, "pk_load: %s[%d][%d] is not below r" % (section, j, row))
    cols = [c.copy() for c in base]
    _spoil(cols[nf + 0], 0, "r", rng)
    _spoil(cols[3], 700, "max", rng)
    _spoil(cols[3], 9, "r+", rng)
    _spoil(cols[4], 1, "r", rng)
    _assert_rejected(cols[:nf], cols[nf:], k, ext_k, "pk_load: fixed_values[3][9] is not below r")
    _assert_rejected([], cols[nf:], k, ext_k, "pk_load: permutations[0][0] is not below r")
    big = random_columns(2, 1 << 20, seed=2)
    _spoil(big[1], (1 << 20) - 2, "r", rng)
    _spoil(big[1], 123457, "max", rng)
    _assert_rejected([big[0]], [big[1]], 20, 21, "pk_load: permutations[0][123457] is not below r")


@pytest.mark.gpu
def test_argument_errors_and_no_columns(gpu):
    """Every argument error returns -1 with a message, launches nothing and writes nothing; with no columns (NULL d_values / d_polys and column
    arrays) only the l-cosets are written, equal to keygen_l_polys."""
    import torch
    from ezkl_b200 import halo2 as h2
    k, ext_k, n, N = 5, 7, 32, 128
    cols = random_columns(3, n, seed=3)
    ptrs, keep = host_columns(cols)
    v, p, l = outputs(3, n, N)
    V, Pp, L = v.data_ptr(), p.data_ptr(), l.data_ptr()
    hostbuf = np.zeros(3 * N * 4, np.uint64)
    cases = [(([ptrs[0]], ptrs[1:], 0, ext_k, 3, V, Pp, n, L), "need 1 <= k <= ext_k"),
             (([ptrs[0]], ptrs[1:], k, k - 1, 3, V, Pp, n, L), "need 1 <= k <= ext_k"),
             (([ptrs[0]], ptrs[1:], k, 29, 3, V, Pp, n, L), "need 1 <= k <= ext_k"),
             (([ptrs[0]], ptrs[1:], k, ext_k, n, V, Pp, n, L), "blinding_factors = 32"),
             (([ptrs[0]], ptrs[1:], k, ext_k, 3, V, Pp, n - 1, L), "stride 31 < 2^k"),
             (([ptrs[0]], ptrs[1:], k, ext_k, 3, V, Pp, n, None), "null pointer"),
             (([ptrs[0]], ptrs[1:], k, ext_k, 3, None, Pp, n, L), "null pointer"),
             (([ptrs[0]], ptrs[1:], k, ext_k, 3, V, None, n, L), "null pointer"),
             (([ptrs[0]], [ptrs[1], None], k, ext_k, 3, V, Pp, n, L), "h_permutations[1] is null"),
             (([None], ptrs[1:], k, ext_k, 3, V, Pp, n, L), "h_fixed_values[0] is null"),
             (([ptrs[0]], ptrs[1:], k, ext_k, 3, V, V + 32 * n, n, L), "d_polys overlaps d_values"),
             (([ptrs[0]], ptrs[1:], k, ext_k, 3, V, Pp, n, V + 32 * 2 * n), "d_l overlaps d_values"),
             (([ptrs[0]], ptrs[1:], k, ext_k, 3, V, Pp, n, Pp), "d_l overlaps d_polys"),
             (([ptrs[0]], ptrs[1:], k, ext_k, 3, V + 8, Pp, n, L), "d_values is not 16-byte aligned"),
             (([ptrs[0]], ptrs[1:], k, ext_k, 3, V, Pp, n, hostbuf.ctypes.data), "d_l is not device memory")]
    before = nat.launch_count()
    for args, msg in cases:
        fixed, perm = args[0], args[1]
        arr = lambda ps: (C.c_void_p * len(ps))(*ps)
        rc = nat.lib().b200_pk_load(arr(fixed), len(fixed), arr(perm), len(perm), *args[2:])
        err = nat.lib().b200_last_error().decode()
        assert rc == -1 and err.startswith("pk_load: ") and msg in err, (msg, err)
    # null column arrays with columns
    assert nat.lib().b200_pk_load(None, 1, None, 0, k, ext_k, 3, V, Pp, n, L) == -1
    assert nat.lib().b200_pk_load(None, 0, None, 2, k, ext_k, 3, V, Pp, n, L) == -1
    assert nat.launch_count() == before
    fill = np.uint64(SENTINEL & (2**64 - 1))
    assert (host(v) == fill).all() and (host(p) == fill).all() and (host(l) == fill).all() and not hostbuf.any()
    # no columns: only d_l
    for bf in (0, 3, n - 1):
        l.fill_(SENTINEL)
        assert pk_load([], [], k, ext_k, bf, None, None, n, L) == 0, nat.lib().b200_last_error()
        assert host(l).tobytes() == np.stack(h2.EvaluationDomain(5, k).keygen_l_polys(bf)).tobytes(), bf
    assert (host(v) == fill).all() and (host(p) == fill).all()
    torch.cuda.synchronize()
    del keep


def _run_self(mode, env_extra=None):
    env = dict(os.environ)
    env.pop("B200_WS_BUDGET_MB", None)
    env.update(env_extra or {})
    r = subprocess.run([sys.executable, os.path.abspath(__file__), mode], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


@pytest.mark.gpu
def test_one_column_groups_under_a_small_scratch_budget():
    """With a 1 MiB per-call budget the coefficient columns and the l-cosets go one column per transform: the same bytes as the defaults'
    host transforms, and the device memory the call adds stays within the header's statement."""
    assert "budget OK" in _run_self("budget", {"B200_WS_BUDGET_MB": "1"})


def _child(mode):
    import torch
    from ezkl_b200 import device as dv
    from ezkl_b200 import fields as F
    from ezkl_b200 import halo2 as h2
    assert mode == "budget"
    nat.init(-1)
    k, ext_k, nf, npc, bf = 17, 19, 3, 2, 5
    n, N = 1 << k, 1 << ext_k
    cols = random_columns(nf + npc, n, seed=17)
    ptrs, keep = host_columns(cols)
    # the transforms' twiddle tables exist before memory is compared (the header states them apart)
    w_inv = F.fr_to_limbs(F.fr_inv(pow(F.FR_ROOT_OF_UNITY, 1 << (F.FR_S - k), F.FR_MODULUS)))
    w_ext = F.fr_to_limbs(pow(F.FR_ROOT_OF_UNITY, 1 << (F.FR_S - ext_k), F.FR_MODULUS))
    for log_n, w in ((k, w_inv), (ext_k, w_ext)):
        dv.ntt(torch.zeros((1, 1 << log_n, 4), dtype=torch.int64, device="cuda"), log_n, w)
    v, p, l = outputs(nf + npc, n, N)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    before = free_bytes()
    assert pk_load(ptrs[:nf], ptrs[nf:], k, ext_k, bf, v.data_ptr(), p.data_ptr(), n, l.data_ptr()) == 0, nat.lib().b200_last_error()
    held = before - free_bytes()
    stated = 32 * 3 * n + 32 * max(1 * n, 1 * N) + 8
    assert held <= stated * 9 // 8 + 6 * MIB, (held, stated)
    dom = h2.EvaluationDomain(J_OF_D[ext_k - k], k)
    assert host(v).tobytes() == cols.tobytes()
    assert host(p).tobytes() == np.stack(dom.lagrange_to_coeff_batch(list(cols))).tobytes()
    assert host(l).tobytes() == np.stack(dom.keygen_l_polys(bf)).tobytes()
    print("budget OK held %d stated %d" % (held, stated))
    del keep


if __name__ == "__main__":
    _child(sys.argv[1])
