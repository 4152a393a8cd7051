"""The create_proof mirror at realistic sizes: proofs made through the CUDA library (ezkl_b200/prover.py driving the host-pointer entry
points) are byte-identical to the proofs made with every primitive on the CPU oracle (tests/cpu_backend.py), at k = 10, 12, 14 and 16, on
an ezkl-shaped circuit that the k = 6 system of tests/test_prover_mirror.py does not reach:

  * eight advice columns, all in the permutation, so the columns do not divide by chunk_len = 5: the last grand product covers a partial
    chunk, and copy-constraint cycles run across both chunks;
  * two mv-lookups, one of them with two inputs, so the degree is 7, the quotient has 6 pieces and the extended domain is 8n (not 4n);
    tables padded with their last entry, as ezkl pads them;
  * an all-zero fixed column (the selector of an op the circuit never uses) and two fixed columns with equal contents (two lookups enabled
    on the same rows), whose commitments are equal;
  * quantised witnesses: signed integers below 2^12 in magnitude (negatives as r - |v|), about a third zeros, long runs of one value; one
    advice column stays uniform.  These are the scalars that reach the MSM's zero-digit and heavy-bucket branches.

At k = 14 a child process proves the same circuit with a 4 MiB scratch budget, which sends b200_evaluate_h down its coset-part path and makes
the host NTT and MSM calls run in sub-batches; the bytes must not move.  The child runs this file as a script:
`python tests/test_proof_scale.py budget <k> <proof path>`.

Which calls cross the 24 MiB pinned-bounce threshold and which split into sub-batches at each k is derived by `host_call_plan` from the
library's rules (ezkl_b200/csrc/capi.cu: call_budget, DIRECT_MAX_BYTES, ntt_host_on, msm_host_on, b200_evaluate_h) and pinned by
test_host_call_plan_of_the_scale_cases.

CPU tier: the plan, the circuit's shape, and the verifier's grouping of openings (two equal fixed columns on the k = 6 system)."""
import ctypes as C
import functools
import os
import random
import subprocess
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from ezkl_b200 import evaluation as ev        # noqa: E402
from ezkl_b200 import prover as pv            # noqa: E402
from oracle import pyref                      # noqa: E402
from tests import test_constraint_system as tcs   # noqa: E402
from tests import test_prover_mirror as tpm   # noqa: E402

R = pyref.R
BLIND = 5
MIB = 1 << 20


# ---- the ezkl-shaped circuit ---------------------------------------------------------------------------------------------------------
class Layout:
    """Flat column indices: advice [a0, a1, b0, b1, out, e0, e1, e2, ...], then the fixed columns.  e0 and e1 feed the two-input range
    lookup; e2 onwards only sit in the permutation.  b1 is the uniform advice column."""

    OPS = ("ADD", "SUB", "MULT", "DOTINIT", "DOT", "SUM")
    FIXED = OPS + ("SEL_L1", "SEL_L2", "T1", "T2")

    def __init__(self, num_advice: int):
        assert num_advice >= 7
        self.num_advice = num_advice
        self.A0, self.A1, self.B0, self.B1, self.OUT = range(5)
        self.E = list(range(5, num_advice))
        self.fixed = {name: num_advice + i for i, name in enumerate(self.FIXED)}
        self.num_fixed = len(self.FIXED)


def quantised(rng, count: int, bound: int) -> list:
    """ezkl-like quantised cells: runs (mean length about 7) of one value, a third of the runs zero, the others signed integers in
    [-bound, bound], negatives stored as r - |v|."""
    out = []
    while len(out) < count:
        v = 0 if rng.random() < 1 / 3 else rng.randint(-bound, bound)
        out += [v % R] * (1 + int(rng.expovariate(1 / 6.0)))
    return out[:count]


def build_scale_system(rng, k: int, num_advice: int = 8):
    """A satisfying ezkl-shaped system at 2^k rows -> (cs, fixed wire columns, sigma wire columns, advice int columns, the copy cycles as
    {(permutation column, row): successor}).  Rows 0 .. u-1 are
    active (u = n - BLIND - 1); every gate, copy constraint and lookup holds there.  Rows from u on hold random values with every selector
    off; the prover overwrites the last BLIND of them with blinding values drawn from its own rng."""
    lay = Layout(num_advice)
    n = 1 << k
    u = n - BLIND - 1
    A0, A1, B0, B1, OUT, E = lay.A0, lay.A1, lay.B0, lay.B1, lay.OUT, lay.E
    fx = {name: [0] * n for name in lay.FIXED}
    # tables: T1 holds 40 distinct quantised values, T2 the signed range [-L, L]; both padded with their last entry up to row u
    t1 = rng.sample(range(-(1 << 12) + 1, 1 << 12), 40)
    L = min((1 << 12) - 1, (u - 1) // 2)
    t2 = list(range(-L, L + 1))
    for i in range(u):
        fx["T1"][i] = t1[min(i, len(t1) - 1)] % R
        fx["T2"][i] = t2[min(i, len(t2) - 1)] % R
    adv = [quantised(rng, n, (1 << 12) - 1) for _ in range(5)] + [quantised(rng, n, L) for _ in E]
    adv[B1] = [rng.randrange(R) for _ in range(n)]
    # copy constraints: groups of cells forced equal; sources (out, a1, e1) are never targets (a0, b0, e0, e2), so a group is one cycle
    groups, group_of = [], {}

    def copy(src, dst):
        if src not in group_of:
            group_of[src] = len(groups)
            groups.append([src])
        groups[group_of[src]].append(dst)
        adv[dst[0]][dst[1]] = adv[src[0]][src[1]]

    heavy = t1[:4]                                                  # most lookup rows hit a few table rows: heavy multiplicities
    for i in range(u):
        if rng.random() < 0.5:                                      # a lookup row of both lookups (their selectors are equal columns)
            fx["SEL_L1"][i] = fx["SEL_L2"][i] = 1
            adv[A1][i] = (rng.choice(heavy) if rng.random() < 0.7 else rng.choice(t1)) % R
        if i > 2:
            if rng.random() < 0.3:
                copy((OUT, rng.randrange(i)), (A0, i))
            if rng.random() < 0.3:
                copy((E[1], rng.randrange(i)), (B0, i))             # chunk 1 -> chunk 0
            if rng.random() < 0.2:
                copy((E[1], rng.randrange(i)), (E[0], i))
            if len(E) > 2 and rng.random() < 0.2:
                copy((A1, rng.randrange(i)), (E[2], i))             # chunk 0 -> chunk 1
        op = rng.choice(["ADD", "MULT", "DOTINIT"] + (["DOT", "SUM"] if i > 0 else []))
        fx[op][i] = 1
        a0, a1, b0, b1 = adv[A0][i], adv[A1][i], adv[B0][i], adv[B1][i]
        prev = adv[OUT][i - 1]
        adv[OUT][i] = {"ADD": a0 + b0, "MULT": a0 * b0, "DOTINIT": a0 * b0 + a1 * b1, "DOT": prev + a0 * b0 + a1 * b1, "SUM": prev + b0 + b1}[op] % R
    for c in range(num_advice):
        for i in range(u, n):
            adv[c][i] = rng.randrange(R)
    perm = list(range(num_advice))
    cycles_next = {}
    for g in groups:
        for a, b in zip(g, g[1:] + g[:1]):
            cycles_next[(perm.index(a[0]), a[1])] = (perm.index(b[0]), b[1])
    f = lay.fixed
    gates = ev.base_op_gates({op: f[op] for op in lay.OPS}, [A0, A1], [B0, B1], OUT)
    sel1, sel2 = ev.Query(f["SEL_L1"]), ev.Query(f["SEL_L2"])
    d1, d2 = ev.Constant(fx["T1"][0]), ev.Constant(fx["T2"][0])
    lookups = [([sel1 * ev.Query(A1) + (ev.Constant(1) - sel1) * d1], ev.Query(f["T1"])),
               ([sel2 * ev.Query(E[0]) + (ev.Constant(1) - sel2) * d2, sel2 * ev.Query(E[1]) + (ev.Constant(1) - sel2) * d2], ev.Query(f["T2"]))]
    cs = pv.ConstraintSystem(num_advice, lay.num_fixed, gates, perm, lookups, blinding_factors=BLIND)
    fixed = [pv._wire(fx[name]) for name in lay.FIXED]
    sigmas = pv.sigma_labels(k, len(perm), cycles_next)
    return cs, fixed, sigmas, adv, cycles_next


@functools.lru_cache(maxsize=None)
def scale_case(k: int):
    """One trapdoor and one system per k (seeded by k): (s, cs, fixed, sigmas, advice, cycles)."""
    rng = random.Random(0x5CA1E000 + k)
    s = rng.randrange(2, R)
    return (s,) + build_scale_system(rng, k)


def commitment_count(cs, quotient_poly_degree: int) -> int:
    """Points before the evaluations: advice, m, z, phi, the random polynomial, the quotient pieces."""
    return cs.num_advice + len(cs.lookups) + cs.num_z + len(cs.lookups) + 1 + quotient_poly_degree


# ---- which host calls bounce and which split ----------------------------------------------------------------------------------------
DIRECT_MAX_BYTES = 24 * MIB           # capi.cu: a host <-> device copy of at least this many bytes goes through the pinned bounce slots
DEFAULT_CALL_BUDGET = 12 << 30        # capi.cu call_budget(): 24 GiB over the calling threads of a device, clamped to [256 MiB, 12 GiB]
SMALL_BUDGET_MB = 4                   # B200_WS_BUDGET_MB of the k = 14 child


def scale_shape_cs():
    """The scale system's constraint system alone (its shape does not depend on k): built at k = 10."""
    return scale_case(10)[1]


def host_call_plan(cs, k: int, ext_k: int, budget: int = DEFAULT_CALL_BUDGET) -> dict:
    """The batched host-pointer calls of Keys + create_proof on this constraint system, with the library's rules applied:
    ntt_host_on takes budget / (32 B * 2^log_n * 3) transforms per sub-batch, msm_host_on budget / (32 B * n * 2) columns, b200_evaluate_h
    evaluates 2^(ext_k - k) coset parts when 32 B * 2^ext_k * columns exceeds the budget; a sub-batch's upload or download of at least
    DIRECT_MAX_BYTES takes the bounce path, as does every strided upload (the extended columns' parts).
    Returns {"bounce": sorted names of calls with a bounced copy, "split": {name: sub-batches} for calls of more than one,
    "evaluate_h_parts": number of coset parts}."""
    n, N, fr = 1 << k, 1 << ext_k, 32
    nf, npc, na, nz, nl = cs.num_fixed, len(cs.permutation_columns), cs.num_advice, cs.num_z, len(cs.lookups)
    # (name, kind, columns, elements up per column, elements down per column)
    calls = [("keys.lagrange_to_coeff_batch", "ntt", nf + npc, n, n), ("keys.coeff_to_extended_batch", "ext", nf + npc, n, N),
             ("keys.commit_lagrange_batch", "msm", nf + npc, n, 0), ("keygen_l_polys.lagrange_to_coeff_batch", "ntt", 3, n, n),
             ("keygen_l_polys.coeff_to_extended_batch", "ext", 3, n, N), ("advice.commit_lagrange_batch", "msm", na, n, 0),
             ("m.commit_lagrange_batch", "msm", nl, n, 0), ("z.commit_lagrange_batch", "msm", nz, n, 0), ("phi.commit_lagrange_batch", "msm", nl, n, 0),
             ("quotient.lagrange_to_coeff_batch", "ntt", na + nz + 2 * nl, n, n), ("h.commit_batch", "msm", cs.degree - 1, n, 0),
             ("shplonk.poly_lincomb", "whole", max(rotation_set_sizes(cs)), n, 0)]
    bounce, split = set(), {}
    for name, kind, count, up, down in calls:
        size = N if kind == "ext" else n
        per = fr * size * (3 if kind in ("ntt", "ext") else 2)
        sub = count if kind == "whole" else max(1, min(count, budget // per))
        batches = -(-count // sub)
        if batches > 1:
            split[name] = batches
        if fr * up * sub >= DIRECT_MAX_BYTES or fr * down * sub >= DIRECT_MAX_BYTES:
            bounce.add(name)
    n_coeff, n_ext = na + nz + 2 * nl, nf + npc + 4
    parts = 1 << (ext_k - k) if fr * N * (n_coeff + n_ext) > budget else 1
    if fr * n * n_coeff >= DIRECT_MAX_BYTES or parts > 1 or fr * N * n_ext >= DIRECT_MAX_BYTES:
        bounce.add("evaluate_h")
    return {"bounce": sorted(bounce), "split": split, "evaluate_h_parts": parts}


def rotation_set_sizes(cs) -> list:
    """Polynomials per SHPLONK rotation set (the prover's grouping: one polynomial per source, grouped by its set of rotations); b200_poly_lincomb
    uploads one set's polynomials in one copy."""
    rots = {}
    for c, rot in cs.advice_queries + cs.fixed_queries:
        rots.setdefault(c, set()).add(rot)
    last = -(cs.blinding_factors + 1)
    sets = [frozenset(r) for r in rots.values()] + [frozenset({0})] * len(cs.permutation_columns)
    sets += [frozenset({0, 1, last} if i + 1 < cs.num_z else {0, 1}) for i in range(cs.num_z)]
    sets += [frozenset({0, 1}), frozenset({0})] * len(cs.lookups) + [frozenset({0})] * 2          # phi, m; h and the random polynomial
    return [sets.count(s) for s in set(sets)]


def test_scale_system_shape():
    """Degree 7 (the two-input lookup), chunk_len 5 with eight permutation columns (a partial last chunk), quotient of 6 pieces on an 8n
    extended domain; the fixed columns hold one all-zero column and two equal ones; the quantised columns are a third zeros."""
    from ezkl_b200 import halo2 as h2
    from tests import cpu_backend as cb
    _, cs, fixed, sigmas, advice, cycles = scale_case(10)
    with pytest.MonkeyPatch.context() as mp:
        cb.patch_backend(mp)
        dom = h2.EvaluationDomain(cs.degree, 10)
    assert cs.degree == 7 and cs.chunk_len == 5 and len(cs.permutation_columns) == 8 and cs.num_z == 2
    assert dom.quotient_poly_degree == 6 and dom.extended_k == 13
    lay = Layout(8)
    f = {name: fixed[i] for i, name in enumerate(Layout.FIXED)}
    assert not f["SUB"].any() and np.array_equal(f["SEL_L1"], f["SEL_L2"]) and f["SEL_L1"].any()
    q = set(cs.fixed_queries)
    assert {(lay.fixed[c], 0) for c in ("SUB", "SEL_L1", "SEL_L2")} <= q          # the equal columns are opened, so the verifier groups them
    u = (1 << 10) - BLIND - 1
    for c in (lay.A1, lay.E[0], lay.E[1], lay.E[2]):                 # a0 and b0 also receive copies of other cells
        zeros = sum(1 for v in advice[c][:u] if v == 0) / u
        assert 0.15 < zeros < 0.6, (c, zeros)
        assert all(v < 1 << 12 or R - v < 1 << 12 for v in advice[c][:u])
    # copy-constraint cycles cross the chunk boundary in both directions (chunk 0 = permutation columns 0 .. 4)
    assert any(j < 5 <= tj for (j, _), (tj, _) in cycles.items()) and any(tj < 5 <= j for (j, _), (tj, _) in cycles.items())


def test_host_call_plan_of_the_scale_cases():
    """The bounce / sub-batch facts each parity case's docstring states, derived from the library's rules and the column counts."""
    got = {k: host_call_plan(scale_shape_cs(), k, k + 3) for k in (10, 12, 14, 16)}
    assert got[10] == {"bounce": [], "split": {}, "evaluate_h_parts": 1}
    assert got[12] == {"bounce": [], "split": {}, "evaluate_h_parts": 1}
    assert got[14] == {"bounce": ["evaluate_h", "keys.coeff_to_extended_batch"], "split": {}, "evaluate_h_parts": 1}
    assert got[16] == {"bounce": ["evaluate_h", "keygen_l_polys.coeff_to_extended_batch", "keys.coeff_to_extended_batch", "keys.commit_lagrange_batch",
                                  "keys.lagrange_to_coeff_batch", "quotient.lagrange_to_coeff_batch", "shplonk.poly_lincomb"], "split": {}, "evaluate_h_parts": 1}
    small = host_call_plan(scale_shape_cs(), 14, 17, budget=SMALL_BUDGET_MB * MIB)
    assert small == {"bounce": ["evaluate_h"], "split": {"keys.lagrange_to_coeff_batch": 9, "keys.coeff_to_extended_batch": 18, "keys.commit_lagrange_batch": 5,
                                                        "keygen_l_polys.lagrange_to_coeff_batch": 2, "keygen_l_polys.coeff_to_extended_batch": 3,
                                                        "advice.commit_lagrange_batch": 2, "quotient.lagrange_to_coeff_batch": 7, "h.commit_batch": 2},
                     "evaluate_h_parts": 8}


# ---- the verifier groups openings by source --------------------------------------------------------------------------------------------
def system_with_equal_fixed_columns(rng, k: int, variant: str):
    """The k = 6 system of tests/test_prover_mirror.py with two more fixed columns of equal contents, each gating a constraint that holds:
    "zero" — the selectors of two ops the circuit never uses (SUB and SUMINIT), both all zero, so both commit to the identity;
    "copy" — two copies of the ADD selector, each gating the ADD constraint again."""
    cs0, fixed, sigmas, advice = tpm.build_system(rng, k)
    n = 1 << k
    c1, c2 = cs0.num_advice + cs0.num_fixed, cs0.num_advice + cs0.num_fixed + 1
    if variant == "zero":
        extra = [np.zeros((n, 4), np.uint64)] * 2
        gates = ev.base_op_gates({"SUB": c1, "SUMINIT": c2}, [tcs.A0, tcs.A1], [tcs.B0, tcs.B1], tcs.OUT)
    else:
        extra = [fixed[tcs.SEL["ADD"] - cs0.num_advice].copy() for _ in range(2)]
        gates = ev.base_op_gates({"ADD": c1}, [tcs.A0, tcs.A1], [tcs.B0, tcs.B1], tcs.OUT) + \
            ev.base_op_gates({"ADD": c2}, [tcs.A0, tcs.A1], [tcs.B0, tcs.B1], tcs.OUT)
    cs = pv.ConstraintSystem(cs0.num_advice, cs0.num_fixed + 2, cs0.gates + gates, cs0.permutation_columns, cs0.lookups, blinding_factors=cs0.blinding_factors)
    assert (c1, 0) in cs.fixed_queries and (c2, 0) in cs.fixed_queries
    return cs, list(fixed) + extra, sigmas, advice


@pytest.mark.parametrize("variant", ["zero", "copy"])
def test_equal_fixed_columns_verify_on_the_cpu_backend(monkeypatch, variant):
    """Two fixed columns with equal contents have equal commitments.  The prover opens them as two polynomials of one rotation set; the
    verifier must do the same (openings keyed by their source column, not by the commitment's value), or it rejects an honest proof."""
    from tests import cpu_backend as cb
    cb.patch_backend(monkeypatch)
    rng = random.Random(0xE0 + (variant == "copy"))
    k = 6
    s = rng.randrange(2, R)
    cs, fixed, sigmas, advice = system_with_equal_fixed_columns(rng, k, variant)
    keys = pv.Keys(cb.FullTrapdoorParams(k, s), cs, fixed, sigmas, vk_repr=0xE0)
    nf = cs.num_fixed
    assert np.array_equal(keys.fixed_commitments[nf - 1], keys.fixed_commitments[nf - 2])
    proof = pv.create_proof(keys, advice, rng=pv.ChaCha12Rng(bytes(32)))
    assert pv.verify_proof_with_trapdoor(keys, proof, s)
    n_pts = commitment_count(cs, keys.domain.quotient_poly_degree)
    bad = bytearray(proof)
    bad[64 * n_pts + 32 * (len(cs.advice_queries) + nf - 1) + 31] ^= 1          # the evaluation of the last equal column
    assert not pv.verify_proof_with_trapdoor(keys, bytes(bad), s)


# ---- parity at scale: device bytes == CPU-oracle bytes -------------------------------------------------------------------------------
STAGES = ("theta", "m", "beta", "gamma", "z", "phi", "y", "x")


def _stage(trace, name):
    if name == "m" or name == "phi":
        return [x[name] for x in trace["lookups"]]
    return trace[name]


def first_differing_stage(a: dict, b: dict):
    """The first stage, in transcript order, at which two create_proof traces differ (None when they agree): the challenges and the m, z and
    phi columns each come right after the commitments they depend on."""
    for name in STAGES:
        if _stage(a, name) != _stage(b, name):
            return name
    return None


def cpu_proof(k: int):
    from tests import cpu_backend as cb
    s, cs, fixed, sigmas, advice, _ = scale_case(k)
    trace = {}
    with pytest.MonkeyPatch.context() as mp:
        cb.patch_backend(mp)
        keys = pv.Keys(cb.FullTrapdoorParams(k, s), cs, fixed, sigmas, vk_repr=0x5CA1E)
        proof = pv.create_proof(keys, advice, rng=pv.ChaCha12Rng(bytes(32)), trace=trace)
    return proof, trace


@functools.lru_cache(maxsize=None)
def device_proof(k: int):
    from ezkl_b200 import _native as nat
    from ezkl_b200 import halo2 as h2
    nat.init(-1)
    s, cs, fixed, sigmas, advice, _ = scale_case(k)
    keys = pv.Keys(h2.ParamsKZG.setup(k, s), cs, fixed, sigmas, vk_repr=0x5CA1E)
    trace = {}
    proof = pv.create_proof(keys, advice, rng=pv.ChaCha12Rng(bytes(32)), trace=trace)
    return proof, trace, keys


def _parity(k: int):
    t0 = time.time()
    want, want_trace = cpu_proof(k)
    t1 = time.time()
    got, got_trace, keys = device_proof(k)
    t2 = time.time()
    print("k=%d: CPU-oracle proof %.1f s, device proof %.1f s" % (k, t1 - t0, t2 - t1))
    assert first_differing_stage(got_trace, want_trace) is None, "first differing stage: %s" % first_differing_stage(got_trace, want_trace)
    assert got == want
    s = scale_case(k)[0]
    assert pv.verify_proof_with_trapdoor(keys, got, s)
    bad = bytearray(got)
    bad[64 * commitment_count(keys.cs, keys.domain.quotient_poly_degree) + 31] ^= 1
    assert not pv.verify_proof_with_trapdoor(keys, bytes(bad), s)


@pytest.mark.gpu
def test_device_proof_equals_the_cpu_oracle_proof_k10():
    """k = 10, ext_k = 13.  Every host transfer stays below 24 MiB (the largest is the quotient's 22 extended columns, 5.5 MiB) and no
    host call splits into sub-batches."""
    _parity(10)


@pytest.mark.gpu
def test_device_proof_equals_the_cpu_oracle_proof_k12():
    """k = 12, ext_k = 15.  Still no bounced transfer: the quotient's 22 extended columns are 22 MiB, the key's 18 extended cosets 18 MiB;
    no host call splits into sub-batches."""
    _parity(12)


@pytest.mark.gpu
def test_device_proof_equals_the_cpu_oracle_proof_k14():
    """k = 14, ext_k = 17 (4 MiB per extended column).  Bounced: the key's coeff_to_extended_batch download (18 cosets, 72 MiB) and the
    quotient's extended-column upload in b200_evaluate_h (22 columns, 88 MiB).  No host call splits into sub-batches at the default budget."""
    _parity(14)


@pytest.mark.gpu
def test_device_proof_equals_the_cpu_oracle_proof_k16():
    """k = 16, ext_k = 19 (2 MiB per column, 16 MiB per extended column).  Bounced: the key's lagrange_to_coeff_batch (18 columns, 36 MiB
    each way), coeff_to_extended_batch (36 MiB up, 288 MiB down) and commit_lagrange_batch (36 MiB); the l-polynomials'
    coeff_to_extended_batch download (48 MiB); the quotient's lagrange_to_coeff_batch (14 columns, 28 MiB each way); b200_evaluate_h's
    coefficient upload (28 MiB) and extended upload (352 MiB); SHPLONK's poly_lincomb over the largest rotation set (29 polynomials, 58 MiB).
    No host call splits into sub-batches at the default 12 GiB budget."""
    _parity(16)


def _run_budget_child(k: int, path: str):
    env = dict(os.environ)
    env["B200_WS_BUDGET_MB"] = str(SMALL_BUDGET_MB)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "budget", str(k), path], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


@pytest.mark.gpu
def test_small_scratch_budget_proof_equals_the_default_k14(tmp_path):
    """k = 14 with a 4 MiB per-call scratch budget, in a child process (the budget is read once, at b200_init): b200_evaluate_h takes its
    coset-part path (the 36 columns' extended cosets take 144 MiB, more than 4 MiB: 8 parts, one evaluate_h launch each), and the host calls split: the key's
    lagrange_to_coeff_batch into 9 sub-batches, its coeff_to_extended_batch into 18 and its commit_lagrange_batch into 5, the l-polynomials'
    transforms into 2 and 3, the advice commitments into 2, the quotient's lagrange_to_coeff_batch into 7 and the quotient pieces'
    commit_batch into 2.  The proof bytes equal the in-process device proof at the default budget."""
    path = str(tmp_path / "proof_k14_budget.bin")
    out = _run_budget_child(14, path)
    with open(path, "rb") as f:
        small = f.read()
    got, _, keys = device_proof(14)
    launches = [int(line.split()[-1]) for line in out.splitlines() if line.startswith("evaluate_h launches")]
    print(out.strip())
    assert launches == [1 << (keys.domain.extended_k - 14)], out
    assert small == got


def _budget_child(k: int, path: str):
    """Child of test_small_scratch_budget_proof_equals_the_default_k14: the device proof under B200_WS_BUDGET_MB, with the number of
    evaluate_h kernel launches (profile class 6) of the quotient call reported."""
    from ezkl_b200 import _native as nat
    assert os.environ.get("B200_WS_BUDGET_MB") == str(SMALL_BUDGET_MB)
    nat.init(-1)
    inner = ev.evaluate_h_from_polys

    def counted(*args, **kw):
        nat.check(nat.lib().b200_profile_enable(1))
        out = inner(*args, **kw)
        ms, cnt = C.c_double(), C.c_uint64()
        nat.check(nat.lib().b200_profile_read(6, C.byref(ms), C.byref(cnt)))
        nat.check(nat.lib().b200_profile_enable(0))
        print("evaluate_h launches %d" % cnt.value)
        return out

    ev.evaluate_h_from_polys = counted
    proof, _, _ = device_proof(k)
    with open(path, "wb") as f:
        f.write(proof)


if __name__ == "__main__":
    if sys.argv[1] == "budget":
        _budget_child(int(sys.argv[2]), sys.argv[3])
