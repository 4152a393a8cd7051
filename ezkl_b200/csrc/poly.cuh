// poly.cuh — internal interface of the batched column-polynomial kernels (poly.cu).
#pragma once
#include "common.cuh"
#include "field.cuh"

namespace b200 {

enum PolyOp { POLY_ADD = 0, POLY_SUB = 1, POLY_MUL = 2, POLY_SCALE = 3, POLY_AXPY = 4 };

struct PolyWorkspace { DevBuf scratch; };

// out[i] = a[i] (+|-|*) b[i]  |  a[i]*s  |  a[i] + s*b[i]        (all device pointers; out may alias a or b)
int poly_binary(int op, const Fr* a, const Fr* b, const Fr* h_s, Fr* out, size_t n, cudaStream_t st);   // h_s: host scalar
// The host arrays (h_*) below are staged through `ring` (common.cuh: StagingRing) and may be reused when the call returns.
// out[i] = sum_j scalars[j] * polys[j][i]; h_polys = host array of device addresses, h_scalars = host scalars
int poly_lincomb(const Fr* const* h_polys, const Fr* h_scalars, size_t count, Fr* out, size_t n, StagingRing& ring, cudaStream_t st);
// out[i] = a[i] * consts[i mod period]   (distribute_powers_zeta: period 3; divide_by_vanishing_poly: period 2^(ext_k-k)); h_consts host array
int poly_scale_cycle(const Fr* a, const Fr* h_consts, uint32_t period, Fr* out, size_t n, StagingRing& ring, cudaStream_t st);
// one n-point coset part of n_cols coefficient columns before its size-n NTT; d_cols = device table, column p at d_cols[p].a with d_cols[p].len elements:
// out[p * out_stride + s] = sum_{t = s + q n < len} a[p][t] * g^t for s < n, with g^t = cyc[t mod 3] * w^(mul * t mod 2^log_w).
// d_tab = [cyc[3] | w^e for e < 2^lo_bits | w^(e << lo_bits) for e < 2^(log_w - lo_bits)], device resident.  One launch per 65535 columns.
struct FoldCol { const Fr* a; uint64_t len; };
int poly_coset_fold(const FoldCol* d_cols, size_t n_cols, const Fr* d_tab, uint32_t lo_bits, uint32_t log_w, uint64_t mul, Fr* out, size_t out_stride, size_t n,
                    cudaStream_t st);
// permutation sigma columns (halo2 permutation/keygen.rs build_pk): d_map = n_columns * 2^k (column, row) uint32 pairs, column-major;
// d_out[j * out_stride + i] = delta^column * omega^row of cell (j, i).  h_tab = [delta^c, c < n_delta | omega^e, e < 2^lo_bits |
// omega^(e << lo_bits), e < 2^(k - lo_bits)] (host, staged through `ring`).  A cell with column >= n_delta or row >= 2^k is written as zero
// and counted in *d_invalid (a device counter; may be null).
int perm_sigmas_run(const uint32_t* d_map, size_t n_columns, uint32_t k, const Fr* h_tab, size_t n_delta, uint32_t lo_bits, Fr* d_out, size_t out_stride,
                    unsigned long long* d_invalid, StagingRing& ring, cudaStream_t st);
// proving-key column check (k_fr_validate): for every element i < n of d_col that is not canonical (its limb integer not below r),
// *d_first = min(*d_first, column << 32 | i); the caller sets *d_first to ~0 first.  n <= 2^32, column < 2^32.
int fr_validate_run(const Fr* d_col, size_t n, size_t column, unsigned long long* d_first, cudaStream_t st);
// three Lagrange indicator columns of n elements at d_out (column j at d_out + j n): 1 on rows lo[j] <= i < hi[j], 0 elsewhere
int fr_indicator_run(Fr* d_out, size_t n, const uint64_t lo[3], const uint64_t hi[3], cudaStream_t st);
// out[p] = sum_i coeffs[p*stride + i] * x[p]^i   for p < batch (eval_polynomial); h_x host array, d_out device array
int poly_eval(const Fr* coeffs, size_t stride, size_t n, const Fr* h_x, Fr* d_out, int batch, PolyWorkspace& ws, StagingRing& ring, cudaStream_t st);
// in place a[i] <- a[i]^-1 (zeros stay zero)  (ff::BatchInvert)
int poly_batch_invert(Fr* a, size_t n, PolyWorkspace& ws, cudaStream_t st);
// exclusive running product / sum per column: out[p][0] = inits[p], out[p][i+1] = out[p][i] (op) a[p][i], p < batch
int poly_prefix_scan(bool product, const Fr* a, size_t a_stride, size_t n, const Fr* h_inits, Fr* out, size_t out_stride, int batch, PolyWorkspace& ws, StagingRing& ring,
                     cudaStream_t st);
// quotient of a(X) by (X - b): q has n-1 coefficients (kate_division)
int poly_kate_division(const Fr* a, size_t n, const Fr* h_b, Fr* q, PolyWorkspace& ws, StagingRing& ring, cudaStream_t st);

// mv-lookup multiplicities (lookup.cu): m[i] = number of input cells equal to table[i], counted on the first row holding each value
// h_inputs: host array of n_inputs device addresses
int lookup_multiplicities_run(const Fr* d_table, size_t n_table, const Fr* const* h_inputs, size_t n_inputs, size_t n_rows, Fr* d_m, DevBuf& scratch, StagingRing& ring,
                              unsigned long long** d_missing_out, cudaStream_t st);

}  // namespace b200
