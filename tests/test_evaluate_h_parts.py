"""b200_evaluate_h when the columns' extended cosets exceed the call budget: the numerator is evaluated one n-point coset part at a time
(DESIGN.md §4.4).  Each case runs tests/evaluate_h_parts_check.py in a child process, because B200_WS_BUDGET_MB is read once, at b200_init."""
import os
import random
import subprocess
import sys

import pytest

from oracle import pyref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHECK = os.path.join(ROOT, "tests", "evaluate_h_parts_check.py")


def run_check(budget_mb, *args):
    env = dict(os.environ)
    env.pop("B200_WS_BUDGET_MB", None)
    if budget_mb is not None:
        env["B200_WS_BUDGET_MB"] = str(budget_mb)
    r = subprocess.run([sys.executable, CHECK, *args], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    return r.stdout


@pytest.mark.gpu
def test_parts_path_is_byte_identical_to_the_composition():
    """Budget 1 MiB: (k, ext_k) = (13, 13), (12, 13), (12, 14), (9, 12), (10, 13); coefficient columns of lengths 1 ... 2^ext_k - 1 mixed
    with extended columns; random programs with wrapping rotations; numerator and finished quotient (t periods 1, 3, d, 1024) equal to
    coeff_to_extended -> quotient_eval -> scale_cycle -> extended_to_coeff, and to the oracle at (9, 12)."""
    out = run_check(1, "identity")
    assert out.count("OK") == 6, out


@pytest.mark.gpu
def test_budget_selects_the_path():
    """Budget 2 MiB at ext_k = 12: columns whose cosets take exactly the budget run as one evaluate_h launch, one column more as 8 parts."""
    out = run_check(2, "select")
    assert "-> 1 evaluate_h launch" in out and "-> 8 evaluate_h launch" in out, out


@pytest.mark.gpu
def test_ezkl_sized_quotient_beyond_device_memory():
    """k = 22, ext_k = 25, 100 coefficient columns and 2 extended ones at the default budget: 102 GiB of extended cosets, more than the
    card holds.  64 rows over all 8 parts against the program's integer semantics, and the finished quotient against the composition.
    Skips (with the numbers) when the shared device has too little free memory.  About 25 s on one H100 80GB HBM3."""
    out = run_check(None, "k22")
    if "SKIP" in out:
        pytest.skip(out.strip().splitlines()[0])
    assert "k22: OK" in out, out


@pytest.mark.gpu
def test_prover_mirror_proof_is_the_same_by_parts(tmp_path):
    """The tests/test_prover_mirror.py system at k = 9 proved at the default budget (every coset resident) and with a 1 MiB budget
    (evaluate_h by parts): the same bytes, and the proof verifies at the trapdoor."""
    from ezkl_b200 import _native as nat
    from ezkl_b200 import halo2 as h2
    from ezkl_b200 import prover as pv
    from tests import test_prover_mirror as tpm
    nat.init(-1)
    rng = random.Random(909)
    k = 9
    s = rng.randrange(2, pyref.R)
    cs, fixed, sigmas, advice = tpm.build_system(rng, k)
    keys = pv.Keys(h2.ParamsKZG.setup(k, s), cs, fixed, sigmas, vk_repr=0x909)
    proof = pv.create_proof(keys, advice, rng=pv.ChaCha12Rng(bytes(32)))
    path = str(tmp_path / "proof_parts.bin")
    out = run_check(1, "prove", path)
    with open(path, "rb") as f:
        by_parts = f.read()
    assert "trapdoor %d" % s in out, out
    assert by_parts == proof
    assert pv.verify_proof_with_trapdoor(keys, by_parts, s)
