// ecfft.cu — FFT over G1 (best_fft with group elements): out[j] = scale * sum_i omega^(i*j) * P_i.
//
// This is what halo2's `g_to_lagrange` runs (UPSTREAM poly/kzg/commitment.rs: best_fft over projective points with omega^-1,
// then * n^-1, then batch normalisation) — the body of `ParamsKZG::downsize`, which ezkl calls whenever the SRS file is larger
// than the circuit (`load_params_prover`, /root/reference/src/execute.rs:1739-1750).  The reference's own SRS fixture pins it:
// g_lagrange == FFT_{omega^-1}(g) / n (tests/golden/kzg_k6.srs).
// Radix-2 decimation-in-time on XYZZ points in global memory, one kernel per stage; each butterfly multiplies its odd input by
// a 254-bit twiddle with a 4-bit fixed-window ladder (the table of 1..15 multiples lives in the thread's local memory).
// Bound: n/2 * log n * ~3000 field multiplications — pure multiply issue, like everything else here.
// Also here: k_g1_validate, the point check of an SRS vector read from a file (b200_srs_register, include/ezkl_b200.h).
#include "msm.cuh"

namespace b200 {

// [s] * p for a canonical 254-bit scalar (limbs little-endian), 4-bit windows, MSB first
DEV G1Xyzz g1_mul_scalar(const G1Xyzz& p, const uint32_t s[8]) {
    if (g1_is_identity(p)) return p;
    G1Xyzz tab[15];
    tab[0] = p;
    tab[1] = g1_dbl(p);
#pragma unroll 1
    for (int i = 2; i < 15; ++i) tab[i] = g1_add(tab[i - 1], p);
    G1Xyzz acc = g1_xyzz_identity();
#pragma unroll 1
    for (int w = 63; w >= 0; --w) {
        if (w != 63) { acc = g1_dbl(acc); acc = g1_dbl(acc); acc = g1_dbl(acc); acc = g1_dbl(acc); }
        const uint32_t d = (s[w >> 3] >> ((w & 7) * 4)) & 15u;
        if (d) acc = g1_add(acc, tab[d - 1]);
    }
    return acc;
}

// load in bit-reversed order, pre-scaled: work[bitrev(i)] = [scale] * P_i
__global__ void __launch_bounds__(64) k_ecfft_load(const G1Affine* __restrict__ in, uint32_t log_n, Fr scale_mont, int apply_scale, G1Xyzz* __restrict__ work) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (1u << log_n)) return;
    G1Xyzz p = g1_to_xyzz(in[i]);
    if (apply_scale) { const Fr s = fp_from_mont(scale_mont); p = g1_mul_scalar(p, s.l); }
    work[log_n ? (__brev(i) >> (32 - log_n)) : 0] = p;
}
// stage with half-size h: pairs (base + j, base + j + h), twiddle omega^(j * n / 2h) from the table tw[k] = omega^k, k < n/2
__global__ void __launch_bounds__(64) k_ecfft_stage(G1Xyzz* __restrict__ work, uint32_t log_n, uint32_t log_h, const Fr* __restrict__ tw) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= (1u << (log_n - 1))) return;
    const uint32_t h = 1u << log_h, j = b & (h - 1), base = (b >> log_h) << (log_h + 1);
    const G1Xyzz u = work[base + j];
    G1Xyzz t = work[base + j + h];
    if (j) { const Fr w = fp_from_mont(fp_load(tw + ((size_t)j << (log_n - 1 - log_h)))); t = g1_mul_scalar(t, w.l); }
    work[base + j] = g1_add(u, t);
    G1Xyzz nt = t; nt.y = fp_neg(t.y);
    work[base + j + h] = g1_add(u, nt);
}
__global__ void __launch_bounds__(128) k_ecfft_store(const G1Xyzz* __restrict__ work, size_t n, G1Affine* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = g1_to_affine(work[i]);
}
__global__ void k_powers_fr(Fr base, uint32_t count, Fr* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) fp_store(out + i, fp_pow_u64(base, (uint64_t)i));
}

// SRS point check (halo2curves G1Affine::from_raw_bytes, as ParamsKZG::read in RawBytes form applies it to every point it reads):
// both coordinates canonical (the 256-bit limb integer below p), and (x, y) = (0, 0) or y^2 = x^3 + 3 in Montgomery form.  One thread
// per point, 64 B read and 2 squarings + 1 multiplication; the first failure is kept as min(index << 2 | reason) in *first.
__global__ void __launch_bounds__(256) k_g1_validate(const G1Affine* __restrict__ pts, size_t n, unsigned long long* __restrict__ first) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    G1Affine p;
    p.x = fp_load(&pts[i].x); p.y = fp_load(&pts[i].y);
    unsigned reason = G1_VALID;
    if (!fp_is_canonical(p.x)) reason = G1_X_NOT_CANONICAL;
    else if (!fp_is_canonical(p.y)) reason = G1_Y_NOT_CANONICAL;
    else if (!g1_is_identity(p)) {
        const Fq b = fp_one<FqTag>() + fp_one<FqTag>() + fp_one<FqTag>();         // 3 R mod p
        if (!fp_eq(fp_sqr(p.y), fp_sqr(p.x) * p.x + b)) reason = G1_NOT_ON_CURVE;
    }
    if (reason != G1_VALID) atomicMin(first, ((unsigned long long)i << 2) | reason);
}
int g1_validate_run(const G1Affine* d_pts, size_t n, unsigned long long* d_first, cudaStream_t st) {
    if (n == 0) return 0;
    k_g1_validate<<<div_up(n, 256), 256, 0, st>>>(d_pts, n, d_first); count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}

int g1_fft_run(const G1Affine* d_in, uint32_t log_n, const Fr& omega, const Fr* scale /*nullable*/, G1Affine* d_out, DevBuf& scratch, cudaStream_t st) {
    B200_CHECK(log_n <= 26, -1, "g1_fft: log_n = %u out of range [0, 26]", log_n);
    const size_t n = (size_t)1 << log_n, half = n > 1 ? n / 2 : 1;
    if (scratch.ensure(sizeof(G1Xyzz) * n + sizeof(Fr) * half)) return -2;
    G1Xyzz* work = scratch.as<G1Xyzz>();
    Fr* tw = reinterpret_cast<Fr*>(work + n);
    k_powers_fr<<<div_up(half, 128), 128, 0, st>>>(omega, (uint32_t)half, tw); count_launch();
    k_ecfft_load<<<div_up(n, 64), 64, 0, st>>>(d_in, log_n, scale ? *scale : fp_one<FrTag>(), scale ? 1 : 0, work); count_launch();
    for (uint32_t log_h = 0; log_h < log_n; ++log_h) { k_ecfft_stage<<<div_up(n / 2, 64), 64, 0, st>>>(work, log_n, log_h, tw); count_launch(); }
    k_ecfft_store<<<div_up(n, 128), 128, 0, st>>>(work, n, d_out); count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace b200
