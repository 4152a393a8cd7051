"""ezkl_b200 — Hopper (sm_90a, H100) backend for ezkl's Halo2/KZG prover hot path: BN254 G1 MSM, Fr NTT, column
polynomial ops.  The product is libezkl_b200.so (C ABI: include/ezkl_b200.h); this package is its Python host mirror of
the halo2 interfaces (halo2.py) and the column dealing of `bench.py --gpus N` over torch.distributed (parallel.py)."""
from ._native import B200Error, init, shutdown, launch_count  # noqa: F401
