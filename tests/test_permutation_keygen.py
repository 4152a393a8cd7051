"""Permutation keygen on the device (b200_permutation_sigmas[_dev]): the sigma columns of Assembly::build_pk from the copy-constraint mapping,
against halo2's own algorithm restated on the host (tests/perm_keygen_ref.py) and pinned by the reference proving key: the device's 32 sigma
columns of tests/golden/pk_k6_primary.npz's mapping rebuild the reference pk.key byte for byte (its sha256 is in tests/golden/manifest.json).

Checks that need their own process (a small scratch budget, read once at b200_init, or a two-device process) run this file as a script:
`python tests/test_permutation_keygen.py budget` / `multi`."""
import ctypes as C
import hashlib
import json
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

P_, S, Z, U32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
KINDS = ("identity", "random", "long_cycle", "two_cycles")


def fixture_mapping():
    """The reference pk.key's mapping: 32 columns x 64 rows stored as column * 64 + row -> [32, 64, 2] uint32."""
    cells = np.load(os.path.join(H.GOLDEN, "pk_k6_primary.npz"))["permutation_cells"].astype(np.uint32)
    return np.stack([cells >> 6, cells & 63], axis=-1)


def pk_key_bytes(sigmas, der) -> bytes:
    """ProvingKey::write (RawBytes) of the reference key: the vk bytes and fixed values from the fixture, `sigmas` as build_pk's
    permutations, the rest from keygen_pk_polys (`der`): a poly is a u32 BE length and its limbs, a slice a u32 BE count, a u32 BE length
    per poly, then the polys."""
    prim = np.load(os.path.join(H.GOLDEN, "pk_k6_primary.npz"))
    poly = lambda p: struct.pack(">I", len(p)) + np.ascontiguousarray(p, np.uint64).tobytes()
    slc = lambda ps: struct.pack(">I", len(ps)) + struct.pack(">%dI" % len(ps), *[len(p) for p in ps]) + b"".join(poly(p) for p in ps)
    return (prim["vk"].tobytes() + poly(der["l0"]) + poly(der["l_last"]) + poly(der["l_active_row"]) + slc(list(prim["fixed_values"]))
            + slc(der["fixed_polys"]) + slc(der["fixed_cosets"]) + slc(list(sigmas)) + slc(der["permutation_polys"]) + slc(der["permutation_cosets"]))


def reference_sha256() -> str:
    return json.load(open(os.path.join(H.GOLDEN, "manifest.json")))["pk.key"]["sha256"]


def keygen_derived(sigmas):
    from ezkl_b200 import halo2 as h2
    key = h2.ProvingKey()
    key.k = 6
    key.fixed_values = list(np.load(os.path.join(H.GOLDEN, "pk_k6_primary.npz"))["fixed_values"])
    key.permutations = list(sigmas)
    return key.keygen_pk_polys(9, 5)


# ---- CPU ---------------------------------------------------------------------------------------------------------------------------
def test_permutation_sigmas_are_exported_and_typed():
    """include/ezkl_b200.h declares b200_permutation_sigmas and b200_permutation_sigmas_dev, which libezkl_b200.so exports with the argtypes /
    restype read from that header."""
    decls = nat.declarations(nat.HEADER)
    for name in ("b200_permutation_sigmas", "b200_permutation_sigmas_dev"):
        fn = getattr(nat.lib(), name)
        assert (fn.argtypes, fn.restype) == decls[name], name
    assert decls["b200_permutation_sigmas"] == ([P_, S, U32, P_, P_, P_], Z)
    assert decls["b200_permutation_sigmas_dev"] == ([P_, S, U32, P_, P_, P_, S, P_, P_], Z)


def test_host_algorithm_reproduces_the_reference_proving_key(monkeypatch):
    """halo2's algorithm on the fixture's mapping gives the sigma columns of the reference pk.key: laid out with the other sections (the
    transforms on the CPU oracle), the key's sha256 is the manifest's, and column 0 is the fixture's perm_values_0."""
    from tests import cpu_backend as cb
    sig = ref.perm_sigmas(fixture_mapping(), 6)
    assert np.array_equal(sig[0], H.load_pk_fixture()["perm_values_0"])
    cb.patch_backend(monkeypatch)
    assert hashlib.sha256(pk_key_bytes(sig, keygen_derived(sig))).hexdigest() == reference_sha256()


@pytest.mark.parametrize("seed", range(6))
def test_host_algorithm_matches_python_ints(seed):
    """The restatement against DELTA^column * omega^row in python ints, on small random mappings (any cell may map anywhere)."""
    rng = random.Random(seed)
    k, P = seed % 5, 1 + rng.randrange(5)
    n = 1 << k
    m = np.array([[[rng.randrange(P), rng.randrange(n)] for _ in range(n)] for _ in range(P)], np.uint32)
    got = ref.perm_sigmas(m, k)
    for j in range(P):
        assert H.fr_list(got[j]) == [ref.sigma_int(int(c), int(r), k) for c, r in m[j]], (k, P, j)


def test_mapping_kinds_are_permutations():
    for kind in KINDS:
        m = ref.mapping_of(kind, 3, 4, seed=1)
        flat = m[..., 0].astype(np.int64) * 16 + m[..., 1]
        assert sorted(flat.reshape(-1).tolist()) == list(range(48)), kind
    assert (ref.mapping_of("identity", 2, 3)[1, 5] == [1, 5]).all()


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------
def _dev_mapping(m):
    import torch
    return torch.from_numpy(np.ascontiguousarray(m).view(np.int32)).cuda()


@pytest.mark.gpu
def test_reference_pin_on_the_device():
    """The device's 32 sigma columns of the reference mapping: both entry points equal halo2's algorithm and perm_values_0; keygen_pk_polys
    on the device turns them into perm_polys_0 / perm_cosets_0, and the rebuilt pk.key has the reference's sha256."""
    from ezkl_b200 import device as dv
    from ezkl_b200 import halo2 as h2
    m = fixture_mapping()
    sig = h2.permutation_sigmas(m, 6)
    assert np.array_equal(sig, ref.perm_sigmas(m, 6))
    assert np.array_equal(dv.to_host(dv.permutation_sigmas(_dev_mapping(m), 6)), sig)
    fx = H.load_pk_fixture()
    assert np.array_equal(sig[0], fx["perm_values_0"])
    der = keygen_derived(sig)
    assert np.array_equal(der["permutation_polys"][0], fx["perm_polys_0"]) and np.array_equal(der["permutation_cosets"][0], fx["perm_cosets_0"])
    assert hashlib.sha256(pk_key_bytes(sig, der)).hexdigest() == reference_sha256()


# (k, P): every domain size class up to the one-column k = 26 case below, and column counts around the parameter ring's slot (256 KiB holds
# 8192 table entries, so P = 10 000 stages its delta table through the ring's larger-blob path)
SIZES = [(0, 32), (1, 32), (10, 32), (17, 32), (20, 32), (24, 4), (6, 1), (6, 3), (5, 300), (3, 10000)]


@pytest.mark.gpu
@pytest.mark.parametrize("k,P", SIZES, ids=["k%d-P%d" % s for s in SIZES])
def test_sigmas_match_the_host_algorithm(k, P):
    """Both entry points, byte for byte, on the identity, a random permutation, one long cycle through every cell and random 2-cycles; the
    _dev form also with out_stride > 2^k (the rows past 2^k stay untouched) and reports no invalid cell."""
    import torch
    from ezkl_b200 import device as dv
    from ezkl_b200 import halo2 as h2
    nat.ensure_init()
    table = ref.deltaomega(P, k)
    n = 1 << k
    for kind in KINDS:
        m = ref.mapping_of(kind, P, k, seed=k * 131 + P)
        want = ref.perm_sigmas(m, k, table)
        assert np.array_equal(h2.permutation_sigmas(m, k), want), (kind, "host")
        dm = _dev_mapping(m)
        got, invalid = dv.permutation_sigmas(dm, k, count_invalid=True)
        assert invalid == 0 and np.array_equal(dv.to_host(got), want), (kind, "dev")
        if n <= 1 << 17:
            out = torch.full((P, n + 5, 4), -1, dtype=torch.int64, device="cuda")
            dv.permutation_sigmas(dm, k, out=out)
            h = dv.to_host(out)
            assert np.array_equal(h[:, :n], want) and (h[:, n:] == np.uint64(2**64 - 1)).all(), (kind, "stride")
        del dm, got


@pytest.mark.gpu
def test_sigmas_k26_one_column():
    """k = 26 with one column (a random permutation of 2^26 rows): the two entry points agree byte for byte, and rows spread over the column
    equal DELTA^column * omega^row in python ints."""
    from ezkl_b200 import device as dv
    from ezkl_b200 import halo2 as h2
    k = 26
    m = ref.mapping_of("random", 1, k, seed=26)
    dev = dv.to_host(dv.permutation_sigmas(_dev_mapping(m), k))
    host = h2.permutation_sigmas(m, k)
    assert np.array_equal(dev, host)
    rows = sorted(set(random.Random(26).sample(range(1 << k), 2000)) | {0, 1, (1 << k) - 1})
    for i in rows:
        assert H.fr_unwire(host[0, i]) == ref.sigma_int(int(m[0, i, 0]), int(m[0, i, 1]), k), i


@pytest.mark.gpu
def test_mirror_sigmas_equal_sigma_labels():
    """The mirror's test system (tests/test_constraint_system.py: copy constraints spliced into cycles over 5 permutation columns): the mapping
    read back from its sigma columns gives, on the device, exactly prover.sigma_labels of the same cycles, which are the system's columns."""
    from ezkl_b200 import device as dv
    from ezkl_b200 import halo2 as h2
    from ezkl_b200 import prover as pv
    from tests import test_constraint_system as tcs
    k = 6
    n = 1 << k
    col, _ = tcs.build_witness(random.Random(7), k)
    where = {ref.sigma_int(c, r, k): (c, r) for c in range(len(tcs.SIG)) for r in range(n)}
    m = np.array([[where[col[s][i]] for i in range(n)] for s in tcs.SIG], np.uint32)
    cycles = {(j, i): tuple(int(x) for x in m[j, i]) for j in range(len(tcs.SIG)) for i in range(n) if tuple(m[j, i]) != (j, i)}
    assert cycles, "the system has copy constraints"
    labels = np.stack(pv.sigma_labels(k, len(tcs.SIG), cycles))
    assert np.array_equal(labels, np.stack([H.fr_array(col[s]) for s in tcs.SIG]))
    assert np.array_equal(h2.permutation_sigmas(m, k), labels)
    assert np.array_equal(dv.to_host(dv.permutation_sigmas(_dev_mapping(m), k)), labels)


@pytest.mark.gpu
def test_argument_errors():
    """The host form checks every cell first: a bad cell returns -1 and leaves out untouched.  The _dev form writes such cells as zero and
    counts them.  Both: -1 for k = 29, null pointers and out_stride < 2^k; 0 and no work for zero columns."""
    import torch
    from ezkl_b200 import device as dv
    from ezkl_b200 import fields as F
    nat.ensure_init()
    L = nat.lib()
    k, P, n = 4, 3, 16
    w, d = F.fr_to_limbs(pyref.omega_for(k)), F.fr_to_limbs(ref.DELTA)
    good = ref.mapping_of("random", P, k, seed=4)
    want = ref.perm_sigmas(good, k)
    for j, i, cell in ((1, 3, (P, 0)), (2, 15, (0, n)), (0, 0, (0xFFFFFFFF, 0xFFFFFFFF))):
        bad = good.copy()
        bad[j, i] = cell
        out = np.full((P, n, 4), 7, np.uint64)
        assert L.b200_permutation_sigmas(bad.ctypes.data, P, k, nat.ptr(w), nat.ptr(d), nat.ptr_array(list(out))) == -1
        assert (out == 7).all() and b"permutation_sigmas" in L.b200_last_error()
    out = np.zeros((P, n, 4), np.uint64)
    outs = nat.ptr_array(list(out))
    assert L.b200_permutation_sigmas(good.ctypes.data, P, 29, nat.ptr(w), nat.ptr(d), outs) == -1
    assert L.b200_permutation_sigmas(None, P, k, nat.ptr(w), nat.ptr(d), outs) == -1
    assert L.b200_permutation_sigmas(good.ctypes.data, P, k, None, nat.ptr(d), outs) == -1
    assert L.b200_permutation_sigmas(good.ctypes.data, P, k, nat.ptr(w), nat.ptr(d), None) == -1
    assert L.b200_permutation_sigmas(good.ctypes.data, P, k, nat.ptr(w), nat.ptr(d), (C.c_void_p * P)(out[0].ctypes.data, None, out[2].ctypes.data)) == -1
    assert not out.any()
    assert L.b200_permutation_sigmas(None, 0, k, None, None, None) == 0
    assert L.b200_permutation_sigmas(good.ctypes.data, P, k, nat.ptr(w), nat.ptr(d), outs) == 0 and np.array_equal(out, want)
    # device form
    bad = good.copy()
    cells = [(0, 1, (P, 2)), (1, 5, (1, n)), (2, 9, (0xFFFFFFFF, 0)), (2, 10, (0, 0xFFFFFFFF))]
    for j, i, cell in cells:
        bad[j, i] = cell
    dm = _dev_mapping(bad)
    dout = torch.full((P, n, 4), -1, dtype=torch.int64, device="cuda")
    exp = want.copy()
    for j, i, _ in cells:
        exp[j, i] = 0
    for count in (True, False):
        dout.fill_(-1)
        r = dv.permutation_sigmas(dm, k, out=dout, count_invalid=count)
        if count:
            assert r[1] == len(cells)
        assert np.array_equal(dv.to_host(dout), exp), count
    st = torch.cuda.current_stream().cuda_stream or 1
    assert L.b200_permutation_sigmas_dev(dm.data_ptr(), P, 29, nat.ptr(w), nat.ptr(d), dout.data_ptr(), 1 << 29, None, st) == -1
    assert L.b200_permutation_sigmas_dev(dm.data_ptr(), P, k, nat.ptr(w), nat.ptr(d), dout.data_ptr(), n - 1, None, st) == -1
    assert L.b200_permutation_sigmas_dev(None, P, k, nat.ptr(w), nat.ptr(d), dout.data_ptr(), n, None, st) == -1
    assert L.b200_permutation_sigmas_dev(dm.data_ptr(), P, k, nat.ptr(w), None, dout.data_ptr(), n, None, st) == -1
    assert L.b200_permutation_sigmas_dev(dm.data_ptr(), 0, k, None, None, dout.data_ptr(), n, None, st) == 0
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_dev_is_one_launch_on_the_callers_stream():
    """One kernel launch per _dev call, enqueued on torch's current stream: a side stream's result is read after that stream only."""
    import torch
    from ezkl_b200 import device as dv
    nat.ensure_init()
    k, P = 16, 8
    m = ref.mapping_of("long_cycle", P, k, seed=3)
    dm = _dev_mapping(m)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    before = nat.launch_count()
    with torch.cuda.stream(side):
        out = dv.permutation_sigmas(dm, k)
        host = out.to("cpu", non_blocking=False)
    assert nat.launch_count() - before == 1
    side.synchronize()
    assert np.array_equal(host.numpy().view(np.uint64), ref.perm_sigmas(m, k))


def _run_self(mode, env_extra=None):
    env = dict(os.environ)
    env.pop("B200_WS_BUDGET_MB", None)
    env.update(env_extra or {})
    r = subprocess.run([sys.executable, os.path.abspath(__file__), mode], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


@pytest.mark.gpu
def test_host_column_groups_under_a_small_scratch_budget():
    """With a 1 MiB per-call budget every column is its own group (5 MiB per column at k = 17): one launch per column, same bytes."""
    assert "budget OK 8 launches" in _run_self("budget", {"B200_WS_BUDGET_MB": "1"})


def _device_count():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.gpu
def test_two_devices_deal_the_columns():
    """A two-device process deals the host call's columns over both devices; the _dev call runs on the device that owns d_out."""
    if _device_count() < 2:
        pytest.skip("needs 2 GPUs")
    assert "multi OK" in _run_self("multi")


def _child(mode):
    import torch
    from ezkl_b200 import device as dv
    from ezkl_b200 import halo2 as h2
    k, P = 17, 8
    m = ref.mapping_of("random", P, k, seed=17)
    want = ref.perm_sigmas(m, k)
    if mode == "budget":
        nat.init(-1)
        before = nat.launch_count()
        assert np.array_equal(h2.permutation_sigmas(m, k), want)
        print("budget OK %d launches" % (nat.launch_count() - before))
    elif mode == "multi":
        nat.check(nat.lib().b200_init_multi(C.c_int(2)))
        nat._inited = True
        assert np.array_equal(h2.permutation_sigmas(m, k), want)
        with torch.cuda.device(1):
            got = dv.permutation_sigmas(_dev_mapping(m).to("cuda:1"), k)
            assert got.device.index == 1 and np.array_equal(dv.to_host(got), want)
        print("multi OK")


if __name__ == "__main__":
    _child(sys.argv[1])
