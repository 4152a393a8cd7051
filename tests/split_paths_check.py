"""Run by tests/test_gpu_parity.py::test_batch_splitting_paths in a subprocess with B200_WS_BUDGET_MB=1, which forces the
rarely-taken sub-batching loops of the host-buffer MSM and NTT entry points (one column per device call).  The kernel launches of
each call pin the group sizes that the budget gives."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from ezkl_b200 import _native as nat  # noqa: E402
from ezkl_b200 import halo2 as h2  # noqa: E402
from oracle import oracle as orc  # noqa: E402

assert os.environ.get("B200_WS_BUDGET_MB") == "1"
nat.init(-1)
n, k = 1 << 11, 11
bases_np = orc.gen_bases(n, seed=91)
bases = h2.Bases(bases_np, window_bits=9)
cols = [orc.gen_scalars(n, seed=92 + i) for i in range(5)]
launches = nat.launch_count()
got = h2.best_multiexp_batch(cols, bases)
msm_launches = nat.launch_count() - launches
for c, g in zip(cols, got):
    assert np.array_equal(g[:8], orc.msm(c, bases_np, 4))
dom = h2.EvaluationDomain(5, k)
launches = nat.launch_count()
coeffs = dom.lagrange_to_coeff_batch(cols)
intt_launches = nat.launch_count() - launches
for c, v in zip(coeffs, cols):
    assert np.array_equal(c, orc.lagrange_to_coeff(v, k, 4))
launches = nat.launch_count()
exts = dom.coeff_to_extended_batch(coeffs)
ext_launches = nat.launch_count() - launches
for e, c in zip(exts, coeffs):
    assert np.array_equal(e, orc.coeff_to_extended(c, dom.extended_k, 4))
assert (msm_launches, intt_launches, ext_launches) == (60, 9, 17), (msm_launches, intt_launches, ext_launches)
print("split paths OK")
