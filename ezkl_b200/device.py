"""Device-resident front end: the same operations as halo2.py, on torch CUDA tensors, with no host round trips.

Tensors are torch.int64 views of the wire format (bit-identical to uint64): Fr columns [n, 4] (or [batch, n, 4]),
G1Affine [n, 8], XYZZ partial sums [batch, 16].  Every call is enqueued on torch's current stream (so torch.cuda.Event
timing and stream ordering see the kernels) and does not synchronise.  torch is plumbing here — allocation, streams,
torch.distributed — the arithmetic is all in libezkl_b200.so.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _native as nat
from . import fields as F


def _stream():
    """torch's current stream as a cudaStream_t.  The legacy default stream has handle 0, which the C ABI reads as "use the
    library's own stream"; pass CUDA's explicit cudaStreamLegacy handle (0x1) instead so ordering and event timing hold."""
    return torch.cuda.current_stream().cuda_stream or 1


def _chk(t: torch.Tensor, last: int):
    assert t.is_cuda and t.dtype == torch.int64 and t.is_contiguous() and t.shape[-1] == last, (t.dtype, t.shape, t.device)


def _host_fr(x) -> np.ndarray:
    return nat.as_u64(x, 4)


def generate_bases(n: int, seed: int = 0xE2C1B200) -> torch.Tensor:
    nat.ensure_init()
    out = torch.empty((n, 8), dtype=torch.int64, device="cuda")
    nat.check(nat.lib().b200_g1_generate_dev(seed, n, out.data_ptr(), _stream()))
    return out


def fixed_base_mul(scalars: torch.Tensor, base=None) -> torch.Tensor:
    """scalars [n,4] (Montgomery wire) -> [n,8] affine points [scalar_i] * base (default: the G1 generator (1, 2))."""
    _chk(scalars, 4)
    n = scalars.numel() // 4
    if base is None:
        base = np.concatenate([F.fq_to_limbs(1), F.fq_to_limbs(2)])
    base = nat.as_u64(base, 8)
    out = torch.empty((n, 8), dtype=torch.int64, device="cuda")
    nat.check(nat.lib().b200_g1_fixed_base_mul_dev(scalars.data_ptr(), n, nat.ptr(base), out.data_ptr(), _stream()))
    return out


def constant_column(value_int: int, n: int) -> torch.Tensor:
    t = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    t[:] = torch.from_numpy(F.fr_to_limbs(value_int).view(np.int64)).cuda()
    return t


def setup_srs(k: int, s: int):
    """ParamsKZG::new / setup with a caller-chosen trapdoor s (gen_srs, /root/reference/src/pfsys/srs.rs:14-16), all on the device:
    g[i] = [s^i] G,  g_lagrange[i] = [L_i(s)] G with L_i(s) = omega^i (s^n - 1) / (n (s - omega^i)).  Returns (g, g_lagrange) [n,8]."""
    r = F.FR_MODULUS
    n = 1 << k
    omega = pow(F.FR_ROOT_OF_UNITY, 1 << (F.FR_S - k), r)
    one = F.fr_to_limbs(1)
    s_pows = prefix_scan(constant_column(s, n), one, True)                      # s^i
    w_pows = prefix_scan(constant_column(omega, n), one, True)                  # omega^i
    den = poly_op("sub", constant_column(s, n), w_pows)                         # s - omega^i  (s must not be an n-th root of unity)
    batch_invert(den)
    lag = poly_op("mul", w_pows, den)
    poly_op("scale", lag, s=F.fr_to_limbs((pow(s, n, r) - 1) * F.fr_inv(n) % r), out=lag)
    return fixed_base_mul(s_pows), fixed_base_mul(lag)


def random_scalars(n: int, batch: int | None = None, seed: int = 0, small_bits: int | None = None) -> torch.Tensor:
    """Uniform scalars < 2^252 (or < 2^small_bits) in Montgomery wire form, generated on the device with torch's RNG."""
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    shape = (n, 4) if batch is None else (batch, n, 4)
    t = torch.randint(-(1 << 63), (1 << 63) - 1, shape, dtype=torch.int64, device="cuda", generator=g)
    if small_bits is not None:
        assert small_bits <= 62
        t[..., 1:] = 0
        t[..., 0] &= (1 << small_bits) - 1
        # canonical small integers -> Montgomery form: multiply by R^2 via the library (x * R^2 * R^-1 = x R)
        r2 = F.fr_to_limbs(pow(2, 256, F.FR_MODULUS))     # to_limbs(R) = R*R mod r in limbs = R^2 representation
        flat = t.view(-1, 4)
        poly_op("scale", flat, s=r2, out=flat)
        return t
    t[..., 3] &= 0x0FFFFFFFFFFFFFFF
    return t


class DeviceBases:
    """Base table built from device points; max_table_bytes as in halo2.Bases (0 = the B200_MSM_TABLE_MB budget)."""

    def __init__(self, d_points: torch.Tensor, window_bits: int = 0, max_table_bytes: int = 0):
        nat.ensure_init()
        _chk(d_points, 8)
        self.n = d_points.shape[0]
        torch.cuda.current_stream().synchronize()
        h = C.c_uint64(0)
        nat.check(nat.lib().b200_bases_register_ex_dev(d_points.data_ptr(), self.n, window_bits, max_table_bytes, C.byref(h)))
        self.handle = h.value

    def info(self) -> dict:
        from .halo2 import bases_info
        return bases_info(self.handle)

    def release(self):
        if self.handle:
            nat.check(nat.lib().b200_bases_release(self.handle))
            self.handle = 0


def msm_batch(bases: DeviceBases, scalars: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """scalars [batch, n, 4] (or [n, 4]) -> un-normalised XYZZ partial sums [batch, 16] on the device."""
    if scalars.dim() == 2:
        scalars = scalars.unsqueeze(0)
    _chk(scalars, 4)
    batch, n = scalars.shape[0], scalars.shape[1]
    if out is None:
        out = torch.empty((batch, 16), dtype=torch.int64, device="cuda")
    nat.check(nat.lib().b200_msm_batch_dev(bases.handle, scalars.data_ptr(), n, n, batch, out.data_ptr(), _stream()))
    return out


def g1_sum(points: torch.Tensor) -> torch.Tensor:
    """points [groups, count, 16] -> [groups, 16]."""
    _chk(points, 16)
    groups, count = points.shape[0], points.shape[1]
    out = torch.empty((groups, 16), dtype=torch.int64, device="cuda")
    nat.check(nat.lib().b200_g1_sum_dev(points.data_ptr(), groups, count, out.data_ptr(), _stream()))
    return out


def normalize(points_xyzz: torch.Tensor) -> np.ndarray:
    """Device XYZZ [m,16] -> host normalised Jacobian wire [m,12] (synchronises)."""
    h = points_xyzz.cpu().numpy().view(np.uint64).reshape(-1, 16)
    out = np.zeros((h.shape[0], 12), np.uint64)
    nat.check(nat.lib().b200_g1_normalize(nat.ptr(np.ascontiguousarray(h)), h.shape[0], nat.ptr(out)))
    return out


def ntt(src: torch.Tensor, log_n: int, omega, *, n_in: int | None = None, pre=None, post=None, out: torch.Tensor | None = None,
        tmp: torch.Tensor | None = None) -> torch.Tensor:
    """src [batch, n_in, 4] -> out [batch, 2^log_n, 4]; pre/post = None | [c] | [c0,c1,c2] host constants (wire form)."""
    if src.dim() == 2:
        src = src.unsqueeze(0)
    _chk(src, 4)
    batch, n_src = src.shape[0], src.shape[1]
    N = 1 << log_n
    n_in = n_src if n_in is None else n_in
    if out is None:
        out = torch.empty((batch, N, 4), dtype=torch.int64, device="cuda")
    if tmp is None:
        tmp = torch.empty((batch, N, 4), dtype=torch.int64, device="cuda")
    pre_a = np.ascontiguousarray(np.stack([_host_fr(c) for c in pre])) if pre is not None else None
    post_a = np.ascontiguousarray(np.stack([_host_fr(c) for c in post])) if post is not None else None
    nat.check(nat.lib().b200_ntt_dev(src.data_ptr(), n_src, n_in, tmp.data_ptr(), out.data_ptr(), N,
                                     log_n, nat.ptr(_host_fr(omega)), 0 if pre is None else len(pre), nat.ptr(pre_a) if pre is not None else None,
                                     0 if post is None else len(post), nat.ptr(post_a) if post is not None else None, batch, _stream()))
    return out


_OPS = {"add": 0, "sub": 1, "mul": 2, "scale": 3, "axpy": 4}


def poly_op(op: str, a: torch.Tensor, b: torch.Tensor | None = None, s=None, out: torch.Tensor | None = None) -> torch.Tensor:
    _chk(a, 4)
    if out is None:
        out = torch.empty_like(a)
    n = a.numel() // 4
    sp = nat.ptr(_host_fr(s)) if s is not None else None
    nat.check(nat.lib().b200_poly_op_dev(_OPS[op], a.data_ptr(), b.data_ptr() if b is not None else None, sp, out.data_ptr(), n, _stream()))
    return out


def lincomb(polys, scalars, out: torch.Tensor | None = None) -> torch.Tensor:
    """sum_j scalars[j] * polys[j]; polys = list of [n,4] CUDA tensors (or a [count,n,4] tensor), scalars host [count,4]."""
    plist = [polys[i] for i in range(len(polys))]
    for p_ in plist:
        _chk(p_, 4)
    n = plist[0].numel() // 4
    sc = nat.as_u64(scalars, 4)
    assert sc.shape[0] == len(plist)
    if out is None:
        out = torch.empty_like(plist[0])
    ptrs = (C.c_void_p * len(plist))(*[p_.data_ptr() for p_ in plist])
    nat.check(nat.lib().b200_poly_lincomb_dev(ptrs, nat.ptr(sc), len(plist), n, out.data_ptr(), _stream()))
    return out


def scale_cycle(a: torch.Tensor, consts) -> torch.Tensor:
    _chk(a, 4)
    cs = nat.as_u64(consts, 4)
    nat.check(nat.lib().b200_poly_scale_cycle_dev(a.data_ptr(), a.numel() // 4, nat.ptr(cs), cs.shape[0], _stream()))
    return a


def eval_batch(polys: torch.Tensor, xs) -> torch.Tensor:
    """polys [batch, n, 4], xs host [batch, 4] -> device [batch, 4]."""
    _chk(polys, 4)
    batch, n = polys.shape[0], polys.shape[1]
    xs = nat.as_u64(xs, 4)
    out = torch.empty((batch, 4), dtype=torch.int64, device="cuda")
    nat.check(nat.lib().b200_poly_eval_batch_dev(polys.data_ptr(), n, n, nat.ptr(xs), batch, out.data_ptr(), _stream()))
    return out


def batch_invert(a: torch.Tensor) -> torch.Tensor:
    _chk(a, 4)
    nat.check(nat.lib().b200_batch_invert_dev(a.data_ptr(), a.numel() // 4, _stream()))
    return a


def prefix_scan(a: torch.Tensor, init, product: bool, out: torch.Tensor | None = None) -> torch.Tensor:
    _chk(a, 4)
    if out is None:
        out = torch.empty_like(a)
    nat.check(nat.lib().b200_prefix_scan_dev(1 if product else 0, a.data_ptr(), a.numel() // 4, nat.ptr(_host_fr(init)), out.data_ptr(), _stream()))
    return out


def prefix_scan_batch(a: torch.Tensor, inits, product: bool, out: torch.Tensor | None = None) -> torch.Tensor:
    """a [batch, n, 4]: one exclusive running product / sum per column in one call; inits host [batch, 4]."""
    _chk(a, 4)
    batch, n = a.shape[0], a.shape[1]
    if out is None:
        out = torch.empty_like(a)
    iv = nat.as_u64(inits, 4)
    assert iv.shape[0] == batch
    nat.check(nat.lib().b200_prefix_scan_batch_dev(1 if product else 0, a.data_ptr(), n, n, batch, nat.ptr(iv),
                                                   out.data_ptr(), n, _stream()))
    return out


def kate_division(a: torch.Tensor, b, out: torch.Tensor | None = None) -> torch.Tensor:
    _chk(a, 4)
    n = a.numel() // 4
    if out is None:
        out = torch.empty((n - 1, 4), dtype=torch.int64, device="cuda")
    nat.check(nat.lib().b200_kate_division_dev(a.data_ptr(), n, nat.ptr(_host_fr(b)), out.data_ptr(), _stream()))
    return out


def permutation_sigmas(mapping: torch.Tensor, k: int, out: torch.Tensor | None = None, count_invalid: bool = False):
    """Sigma columns from the copy-constraint mapping (int32 [P, 2^k, 2], (column, row) per cell) -> out [P, m, 4] with m >= 2^k (rows
    beyond 2^k untouched).  Cells outside P columns x 2^k rows are written as zero; with count_invalid the call synchronises and returns
    (out, number of such cells)."""
    from .evaluation import DELTA
    assert mapping.is_cuda and mapping.dtype == torch.int32 and mapping.is_contiguous() and mapping.dim() == 3 and mapping.shape[1:] == (1 << k, 2), \
        (mapping.dtype, mapping.shape)
    nat.ensure_init()
    P = mapping.shape[0]
    if out is None:
        out = torch.empty((P, 1 << k, 4), dtype=torch.int64, device=mapping.device)
    _chk(out, 4)
    assert out.dim() == 3 and out.shape[0] == P, out.shape
    omega = F.fr_to_limbs(pow(F.FR_ROOT_OF_UNITY, 1 << (F.FR_S - k), F.FR_MODULUS))
    invalid = C.c_uint64(0)
    nat.check(nat.lib().b200_permutation_sigmas_dev(mapping.data_ptr(), P, k, nat.ptr(omega), nat.ptr(F.fr_to_limbs(DELTA)), out.data_ptr(), out.shape[1],
                                                    C.byref(invalid) if count_invalid else None, _stream()))
    return (out, invalid.value) if count_invalid else out


class DeviceProvingKey:
    """What the resident prover needs of a proving key, on the device: values / polys [num_fixed + num_permutation, 2^k, 4] (fixed columns
    first), l0 / l_last / l_active_row [2^ext_k, 4], and the vk bytes of the file."""

    def __init__(self, k, ext_k, num_fixed, vk_bytes, values, polys, l):
        self.k, self.ext_k, self.num_fixed, self.vk_bytes = k, ext_k, num_fixed, vk_bytes
        self.values, self.polys = values, polys
        self.l0, self.l_last, self.l_active_row = l[0], l[1], l[2]


def load_proving_key(path: str, num_permutation_columns: int, num_selectors: int, ext_k: int, blinding_factors: int) -> DeviceProvingKey:
    """A RawBytes proving key file (ProvingKey::write) -> DeviceProvingKey, through b200_pk_load: the file is memory-mapped, its section
    headers are walked (halo2.ProvingKey.layout: only the u32 counts and lengths are read), and only the fixed_values and permutations
    columns are passed to the library, which checks every element on the device and derives the polys and l-cosets there.  The file's
    polys, cosets and l-vectors are never read.  A malformed file raises B200Error before the library is called."""
    from .halo2 import ProvingKey
    import os
    if os.path.getsize(path) == 0:
        raise nat.B200Error("load_proving_key: %s is empty" % path)
    mm = np.memmap(path, dtype=np.uint8, mode="r")
    try:
        lay = ProvingKey.layout(mm, num_permutation_columns, num_selectors, ext_k)
        k = lay["k"]
        nf, cols = len(lay["fixed_values"]), lay["fixed_values"] + lay["permutations"]
        nat.ensure_init()
        values = torch.empty((len(cols), 1 << k, 4), dtype=torch.int64, device="cuda")
        polys = torch.empty_like(values)
        l = torch.empty((3, 1 << ext_k, 4), dtype=torch.int64, device="cuda")
        base = mm.ctypes.data
        ptrs = lambda offs: (C.c_void_p * len(offs))(*[base + o for o in offs]) if offs else None
        torch.cuda.current_stream().synchronize()          # the allocations' stream work is done before the library's stream writes them
        nat.check(nat.lib().b200_pk_load(ptrs(lay["fixed_values"]), nf, ptrs(lay["permutations"]), len(cols) - nf, k, ext_k, blinding_factors,
                                         values.data_ptr() if cols else None, polys.data_ptr() if cols else None, 1 << k, l.data_ptr()))
        vk = bytes(mm[:lay["vk_len"]])
    finally:
        del mm
    return DeviceProvingKey(k, ext_k, nf, vk, values, polys, l)


def to_host(t: torch.Tensor) -> np.ndarray:
    return t.cpu().numpy().view(np.uint64)


def from_host(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()
