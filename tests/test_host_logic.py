"""CPU-side checks of the product: C-ABI surface, loud failure without a device, and the host-compiled (portable-path)
field / group-law / digit-recoding code that the CUDA kernels share with the host, against the oracle."""
import ctypes as C
import os
import random

import numpy as np
import pytest

from ezkl_b200 import _native as nat
from ezkl_b200 import fields as F
from oracle import oracle as orc
from oracle import pyref
from tests import helpers as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cabi_exports_every_declared_symbol():
    """Every prototype of include/ezkl_b200.h (and of the test hooks' csrc/debug.h) is exported, with the argtypes / restype read from it."""
    for load, header in ((nat.lib, nat.HEADER), (nat.dbg_lib, nat.DBG_HEADER)):
        lib, decls = load(), nat.declarations(header)
        assert len(decls) >= 13
        for name, (argtypes, restype) in decls.items():
            assert hasattr(lib, name), "%s does not export %s" % (lib._name, name)
            fn = getattr(lib, name)
            assert fn.argtypes == argtypes and fn.restype is restype, name


def test_cabi_signatures_and_hook_counts_follow_the_headers():
    """Pointers are c_void_p; int, uint32_t, uint64_t and size_t keep their C width; every declared function is typed.  The
    headers declare 71 product entry points and 18 test hooks."""
    prod, dbg = nat.declarations(nat.HEADER), nat.declarations(nat.DBG_HEADER)
    assert (len(prod), len(dbg)) == (71, 18)
    for decls in (prod, dbg):
        for name, (argtypes, restype) in decls.items():
            assert set(argtypes) <= {C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_size_t}, name
            assert restype in (C.c_int, C.c_uint64, C.c_char_p, None), name
    assert prod["b200_last_error"] == ([], C.c_char_p) and prod["b200_launch_count"] == ([], C.c_uint64)
    assert prod["b200_shutdown"] == ([], None) and prod["b200_init"] == ([C.c_int], C.c_int)
    assert prod["b200_msm"] == ([C.c_uint64, C.c_void_p, C.c_size_t, C.c_void_p], C.c_int)
    assert prod["b200_fft"] == ([C.c_void_p, C.c_uint32, C.c_void_p], C.c_int)
    assert prod["b200_ntt_dev"] == ([C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_int, C.c_void_p,
                                     C.c_int, C.c_void_p, C.c_size_t, C.c_void_p], C.c_int)
    assert dbg["b200_debug_msm_pick_levels"] == ([C.c_size_t, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p], C.c_int)
    assert dbg["b200_debug_ntt_plan_host"] == ([C.c_uint32, C.c_int, C.c_int, C.c_void_p], C.c_int)
    assert dbg["b200_debug_msm_plan"] == ([C.c_size_t] + [C.c_int] * 6 + [C.c_void_p], C.c_int)
    assert dbg["b200_debug_g1_xyzz_op"] == dbg["b200_debug_host_g1_xyzz_op"] == ([C.c_int] + [C.c_void_p] * 4 + [C.c_size_t], C.c_int)
    assert dbg["b200_debug_field_op4"] == dbg["b200_debug_host_field_op4"] == ([C.c_int, C.c_int] + [C.c_void_p] * 5 + [C.c_size_t], C.c_int)


def test_cabi_rejects_untyped_declarations(tmp_path):
    """A parameter or return type outside the mapping, or a missing header, is an error at load, never an unchecked call."""
    h = tmp_path / "h.h"
    h.write_text("#include <stdint.h>\n/* int b200_commented(double d); */\nint b200_ok(size_t n, const void* p); // void b200_x(float f);\n")
    assert nat.declarations(str(h)) == {"b200_ok": ([C.c_size_t, C.c_void_p], C.c_int)}
    for decl in ("int b200_x(float f);", "float b200_x(int a);", "int b200_x(struct s v);", "int b200_x(int);"):
        h.write_text("#include <stdint.h>\n" + decl + "\n")
        with pytest.raises(nat.B200Error):
            nat.declarations(str(h))
    with pytest.raises(nat.B200Error):
        nat.declarations(str(tmp_path / "missing.h"))


def test_cabi_call_with_a_missing_argument_raises_before_the_library():
    with pytest.raises(TypeError):
        nat.lib().b200_poly_op(0, None)


def test_no_cpu_fallback_without_device():
    """Without a usable CUDA device the product must fail loudly (never compute on the CPU)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    lib = nat.lib()
    assert lib.b200_init(C.c_int(-1)) != 0
    assert b"no CUDA device" in lib.b200_last_error()
    a = np.zeros((4, 4), np.uint64)
    w = np.zeros(4, np.uint64)
    assert lib.b200_fft(nat.ptr(a), C.c_uint32(2), nat.ptr(w)) == -3
    out = np.zeros(12, np.uint64)
    assert lib.b200_msm(C.c_uint64(1), nat.ptr(a), C.c_size_t(4), nat.ptr(out)) == -3
    with pytest.raises(nat.B200Error):
        nat.init(-1)


def test_product_does_not_import_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "ezkl_b200")):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h", ".hpp")):
                src = open(os.path.join(dirpath, fn)).read()
                assert "oracle" not in src.replace("# oracle-free", ""), "%s mentions the oracle" % fn


def test_host_constants_match_oracle():
    assert F.FR_MODULUS == pyref.R and F.FQ_MODULUS == pyref.P
    assert F.FR_ROOT_OF_UNITY == pyref.FR_ROOT_OF_UNITY and F.FR_ZETA == pyref.FR_ZETA
    assert np.array_equal(F.fr_to_limbs(1), orc.fr_one())
    assert F.fr_from_limbs(orc.omega(17)) == pyref.omega_for(17)


def test_portable_field_ops_vs_oracle():
    L = nat.lib()
    rng = random.Random(5)
    for fid, (field, mod) in enumerate((("fr", pyref.R), ("fq", pyref.P))):
        xs = [rng.randrange(mod) for _ in range(300)] + [0, 1, mod - 1]
        ys = [rng.randrange(mod) for _ in range(300)] + [mod - 1, 0, mod - 1]
        a = np.stack([H.int_to_limbs(pyref.to_mont(x, mod)) for x in xs])
        b = np.stack([H.int_to_limbs(pyref.to_mont(y, mod)) for y in ys])
        for opi, op in enumerate(("add", "sub", "mul")):
            out = np.zeros_like(a)
            assert nat.dbg_lib().b200_debug_host_field_op(fid, opi, nat.ptr(a), nat.ptr(b), nat.ptr(out), C.c_size_t(len(xs))) == 0
            assert np.array_equal(out, orc.field_op(field, op, a, b)), (field, op)
        out = np.zeros_like(a)
        nat.dbg_lib().b200_debug_host_field_op(fid, 3, nat.ptr(a), nat.ptr(b), nat.ptr(out), C.c_size_t(len(xs)))
        assert np.array_equal(out, orc.fr_inv(a) if field == "fr" else orc.fq_inv(a))


def test_group_law_vs_oracle_including_degenerate_inputs():
    L = nat.lib()
    rng = random.Random(6)
    bases = orc.gen_bases(64, seed=9, threads=2)
    A, B = bases[:32].copy(), bases[32:].copy()
    A[0] = 0          # identity + P
    B[1] = 0          # P + identity
    A[2] = B[2]       # P + P through the mixed-add doubling branch
    n = C.c_size_t(32)
    out = np.zeros_like(A)
    nat.dbg_lib().b200_debug_host_g1_op(0, nat.ptr(A), nat.ptr(B), nat.ptr(out), n)
    assert np.array_equal(out, orc.g1_add_affine(A, B))
    nat.dbg_lib().b200_debug_host_g1_op(1, nat.ptr(A), nat.ptr(B), nat.ptr(out), n)
    assert np.array_equal(out, orc.g1_add_affine(A, A))
    K = B.copy()
    ks = [rng.randrange(1 << 20) for _ in range(32)]
    ks[3], ks[4] = 0, 1
    ks[5:16] = [2, 3, 4, 0xFFFFF, 0x55555, 0xAAAAA, 0xFFFFFFFF, 0x80000000, 0x40000000, 12, 0x30003]      # every 2-bit window digit, top windows, max
    for i, k in enumerate(ks):
        K[i, 0] = k
    nat.dbg_lib().b200_debug_host_g1_op(2, nat.ptr(A), nat.ptr(K), nat.ptr(out), n)
    assert np.array_equal(out, orc.g1_scalar_mul(A, H.fr_array(ks)))
    nat.dbg_lib().b200_debug_host_g1_op(3, nat.ptr(A), nat.ptr(B), nat.ptr(out), n)
    assert np.array_equal(out, orc.g1_add_affine(A, orc.g1_add_affine(B, B)))
    out[:] = 1
    nat.dbg_lib().b200_debug_host_g1_op(4, nat.ptr(A), nat.ptr(B), nat.ptr(out), n)
    assert not out.any()      # P + (-P) = identity = (0,0)


@pytest.mark.parametrize("c", [4, 7, 8, 13, 15, 16, 17, 20, 22, 24])
def test_signed_window_recoding(c):
    L = nat.lib()
    rng = random.Random(c)
    xs = [rng.randrange(pyref.R) for _ in range(200)] + [0, 1, pyref.R - 1, 1 << 253, (1 << c) - 1, 1 << (c - 1), (1 << (c - 1)) + 1]
    can = np.stack([H.int_to_limbs(x) for x in xs])
    W = (255 + c - 1) // c
    out = np.zeros((len(xs), W), np.int32)
    nat.dbg_lib().b200_debug_digits_host(nat.ptr(can), C.c_size_t(len(xs)), C.c_int(c), out.ctypes.data_as(C.c_void_p))
    for i, x in enumerate(xs):
        assert sum(int(out[i, w]) << (c * w) for w in range(W)) == x
        assert all(-(1 << (c - 1)) <= int(d) <= (1 << (c - 1)) for d in out[i])


def reference_pk_key(monkeypatch, path):
    """Rebuilds the reference's own tests/assets/pk.key at `path`, byte for byte (its sha256 is in tests/golden/manifest.json):
    the sections keygen does not derive come from tests/golden/pk_k6_primary.npz, the others are recomputed on the CPU backend
    and laid out as ProvingKey::write (RawBytes) does: a poly is a u32 BE length and its limbs, a slice of polys is a u32 BE
    count and a u32 BE length per poly, then the polys."""
    import hashlib
    import json
    import struct
    from ezkl_b200 import halo2 as h2
    from tests import cpu_backend as cb
    cb.patch_backend(monkeypatch)
    prim = np.load(os.path.join(H.GOLDEN, "pk_k6_primary.npz"))
    key = h2.ProvingKey()
    key.k = 6
    delta, w = pow(7, 1 << 28, pyref.R), pyref.omega_for(6)           # permutation values are delta^c * omega^r, stored as c * 64 + r
    key.fixed_values = list(prim["fixed_values"])
    key.permutations = [np.stack([H.fr_wire(pow(delta, int(x) >> 6, pyref.R) * pow(w, int(x) & 63, pyref.R)) for x in col]) for col in prim["permutation_cells"]]
    der = key.keygen_pk_polys(9, 5)
    poly = lambda p: struct.pack(">I", len(p)) + np.ascontiguousarray(p, np.uint64).tobytes()
    slc = lambda ps: struct.pack(">I", len(ps)) + struct.pack(">%dI" % len(ps), *[len(p) for p in ps]) + b"".join(poly(p) for p in ps)
    data = (prim["vk"].tobytes() + poly(der["l0"]) + poly(der["l_last"]) + poly(der["l_active_row"]) + slc(key.fixed_values)
            + slc(der["fixed_polys"]) + slc(der["fixed_cosets"]) + slc(key.permutations) + slc(der["permutation_polys"]) + slc(der["permutation_cosets"]))
    assert hashlib.sha256(data).hexdigest() == json.load(open(os.path.join(H.GOLDEN, "manifest.json")))["pk.key"]["sha256"]
    with open(path, "wb") as f:
        f.write(data)
    monkeypatch.undo()
    return path


def test_proving_key_reader_on_reference_fixture(monkeypatch, tmp_path):
    """ProvingKey::read mirror against the reference's own tests/assets/pk.key."""
    path = reference_pk_key(monkeypatch, str(tmp_path / "pk.key"))
    from ezkl_b200 import halo2 as h2
    pk = h2.ProvingKey.read(path, num_permutation_columns=32, num_selectors=80)
    g = H.load_pk_fixture()
    assert pk.k == 6 and len(pk.fixed_values) == 38 and len(pk.permutations) == 32
    assert pk.l0.shape == (512, 4) and pk.fixed_cosets[0].shape == (512, 4) and pk.fixed_polys[0].shape == (64, 4)
    for c in (0, 1, 5, 37):
        assert np.array_equal(pk.fixed_values[c], g["fixed_values_%d" % c])
        assert np.array_equal(pk.fixed_polys[c], g["fixed_polys_%d" % c])
        assert np.array_equal(pk.fixed_cosets[c], g["fixed_cosets_%d" % c])
    assert np.array_equal(pk.permutation_cosets[0], g["perm_cosets_0"]) and np.array_equal(pk.l_active_row, g["l_active_row"])
    with pytest.raises(nat.B200Error):
        h2.ProvingKey.read(path, num_permutation_columns=31, num_selectors=80)      # wrong layout is detected, not mis-parsed


def test_bench_reference_arm_prints_contract_json():
    """`bench.py --impl reference` (the CPU port arm the driver runs first) prints one JSON line with the contract's keys."""
    import json
    import subprocess
    import sys
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--k", "8", "--steps", "1", "--warmup", "0", "--cpu-budget", "1"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data",
                "config", "cpu_baseline", "e2e"):
        assert key in line, key
    assert line["impl"] == "reference" and line["higher_is_better"] is False and line["cpu_baseline"]["kind"] == "port"
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and "workload" in line["config"]


def test_generated_field_arithmetic_is_verified_and_current(tmp_path):
    """fp_gen.py executes every emitted PTX instruction list (multiply, add, sub, two-product multiply, squaring) in its own
    interpreter against bigints; the committed fp_ptx.cuh must be exactly what the generator emits today."""
    import importlib.util
    gen_path = os.path.join(ROOT, "ezkl_b200", "csrc", "fp_gen.py")
    spec = importlib.util.spec_from_file_location("fp_gen", gen_path)
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    for name, mod in gen.FIELDS.items():
        counts = gen.check(name, mod, trials=300)
        assert counts[0] == 312 and counts[3] < 2 * counts[0] and counts[4] < counts[0]
    committed = open(os.path.join(ROOT, "ezkl_b200", "csrc", "fp_ptx.cuh")).read()
    for name, mod in gen.FIELDS.items():
        for fn, ins, n_in in (("mul", gen.gen_mul(mod), 2), ("mul2", gen.gen_mul2(mod), 4), ("sqr", gen.gen_sqr(mod), 1)):
            assert gen.emit_fn("%s_%s_ptx" % (name, fn), ins, n_in) in committed, "%s_%s_ptx is stale: run fp_gen.py" % (name, fn)


def test_keygen_host_logic_reproduces_reference_proving_key_bytes_on_the_cpu_backend(monkeypatch):
    """create_keys' derived vectors (src/pfsys/mod.rs:376-400) through the SAME host code the GPU test drives (ProvingKey.keygen_pk_polys,
    EvaluationDomain.keygen_l_polys: which rows l_last / the blinding rows sit on, how l_active_row is formed, which columns are
    transformed how), with the transforms redirected to the CPU oracle: byte for byte the reference pk.key's polys, extended cosets, l0,
    l_last and l_active_row (tests/golden/pk_k6_subset.npz)."""
    from ezkl_b200 import halo2 as h2
    from tests import cpu_backend as cb
    cb.patch_backend(monkeypatch)
    pk = H.load_pk_fixture()
    key = h2.ProvingKey()
    key.k = 6
    cols = (0, 1, 5, 37)
    key.fixed_values = [pk["fixed_values_%d" % c] for c in cols]
    key.permutations = [pk["perm_values_0"]]
    out = key.keygen_pk_polys(9, 5)
    for i, c in enumerate(cols):
        assert np.array_equal(out["fixed_polys"][i], pk["fixed_polys_%d" % c])
        assert np.array_equal(out["fixed_cosets"][i], pk["fixed_cosets_%d" % c])
    assert np.array_equal(out["permutation_polys"][0], pk["perm_polys_0"])
    assert np.array_equal(out["permutation_cosets"][0], pk["perm_cosets_0"])
    assert np.array_equal(out["l0"], pk["l0"]) and np.array_equal(out["l_last"], pk["l_last"]) and np.array_equal(out["l_active_row"], pk["l_active_row"])


def test_bench_trace_shape_matches_the_reference_fixture_proof():
    """bench.py's default op trace is shaped like the reference's own fixture proof (tests/assets/proof.json, SURVEY.md Appendix B/D4):
    114 commitments + 2 SHPLONK points, 231 evaluations; config dicts of the two bench arms are the same object shape."""
    import sys
    sys.path.insert(0, ROOT)
    import bench
    tr = bench.TRACES["conv2d_mnist"]
    ops = bench.trace_ops(tr)
    msm_cols = [c for kind, c in ops if kind.startswith("msm")]
    assert sum(msm_cols) == 114 + 2 and msm_cols[-1] == 2
    assert dict(ops)["eval"] == 231
    assert bench.n_coset_columns(tr) == tr["advice"] + tr["instance"] + tr["perm_z"] + 2 * tr["lookups"] == 107
    pairs, ntt_elts = bench.count_units(ops, 1 << 17, tr)
    assert pairs == 116 << 17 and ntt_elts == (107 << 17) + (108 << 20)
    cfg = bench.make_config(17, "conv2d_mnist")
    assert cfg["k"] == 17 and cfg["msm_pairs_per_step"] == pairs and "workload" in cfg
