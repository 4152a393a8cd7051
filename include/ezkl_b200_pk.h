/*
 * ezkl_b200_pk.h — proving-key loading entry point of libezkl_b200.so: the Lagrange columns of a RawBytes proving key straight into
 * device memory, checked on the device, with the key's coefficient columns and its l0 / l_last / l_active_row cosets derived there
 * instead of read.  The types and conventions are those of ezkl_b200.h, which this header includes.
 */
#ifndef EZKL_B200_PK_H
#define EZKL_B200_PK_H

#include "ezkl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- ProvingKey::read (RawBytes, with precompute-coset) for a device-resident prover, in one call -------------------------------
 * Inputs: h_fixed_values[j] (j < n_fixed) and h_permutations[j] (j < n_perm) are host pointers, each to one column of 2^k Fr in the
 * key file's raw-bytes form (4 little-endian u64 Montgomery limbs, 32 B per element): the file's fixed_values and permutations
 * sections.  They typically point into a memory-mapped key file, where they are not even 4-byte aligned (the vk prefix of the
 * reference key is 5127 B and every column follows a u32 big-endian length), so the library treats them as byte pointers and only
 * copies them (memcpy or a DMA copy); pageable memory is fine.  k and ext_k are the key's domain sizes (2^k rows, 2^ext_k extended
 * rows) and blinding_factors its number of blinding rows.
 *
 * Outputs, all device memory owned by the caller, on one device:
 *   d_values  the fixed columns, then the permutation columns: column c (c < n_fixed + n_perm) at element offset c * stride;
 *   d_polys   the same columns in coefficient form (EvaluationDomain::lagrange_to_coeff), in the same layout with the same stride;
 *   d_l       three extended columns of 2^ext_k elements back to back: l0, l_last, l_active_row.
 * Every output is fully reduced, in Montgomery form, and byte-identical to the key's own section: fixed_values / permutations,
 * fixed_polys / permutations.polys, and l0 / l_last / l_active_row.  Keygen's definitions apply: u = 2^k - blinding_factors - 1,
 * l0 = L_0, l_last = L_u and l_active_row = 1 - (l_last + l_blind), where l_blind is the sum of the Lagrange polynomials of rows
 * u + 1 ... 2^k - 1, each on the extended coset (coeff_to_extended).  The domain constants (omega, the extended omega, zeta = Fr::ZETA and
 * 2^-k) are derived inside the library from k and ext_k.  Rows of d_values / d_polys between 2^k and stride are not written.
 *
 * The check: every element passed is checked as halo2curves' Fr::from_raw_bytes checks it: the four little-endian u64 limbs, read as
 * one 256-bit integer, must be below r.  A failure returns -1 with b200_last_error() naming the section, the column and the lowest bad
 * row, e.g. "pk_load: permutations[3][1234] is not below r"; with several bad elements the lowest (section, column, row) is named,
 * fixed_values before permutations.  After a rejection d_polys and d_l are not written; d_values holds whatever was staged.
 *
 * Not read: the key's polys, cosets and l-vectors are never read, so a bad byte there is never seen.  A key whose polys disagree with
 * its values gets the polys of its values here; halo2's keygen never writes such a key.
 *
 * Argument errors return -1 before any device work and write nothing: k < 1, ext_k < k, ext_k > 28, blinding_factors >= 2^k;
 * stride < 2^k; a null pointer (d_values, d_polys and the two host arrays may be NULL when n_fixed + n_perm == 0; then only d_l is
 * written); outputs that are not 16-byte aligned device memory of the process; outputs that overlap; outputs on different devices.
 * -2 for a CUDA failure.
 *
 * Execution: on the device that owns the outputs, synchronous (the outputs are complete when the call returns), re-entrant per thread
 * like every entry point.  No replica is made on another device.  Each column is staged through the pageable copy path straight into
 * its slot of d_values (no per-thread staging buffer grows to the key's size) and checked right behind its copy; the check word is read
 * back once, after the last column.
 *
 * Device memory held beyond the caller's buffers, by the calling thread's context (kept for its later calls, as every call's scratch
 * is), with n = 2^k, N = 2^ext_k, C = n_fixed + n_perm and B the per-call scratch budget (B200_WS_BUDGET_MB, else a share of
 * B200_WS_TOTAL_MB): 3 n * 32 B (the l-vectors' coefficients) and 32 * max(g n, s N) B of transform scratch, where the coefficient
 * columns go in groups of g = min(C, max(1, floor(B / (32 n)))) columns and the l-cosets in groups of s = min(3, max(1,
 * floor(B / (32 N)))); each buffer is allocated with 1/8 headroom, plus 8 B for the check word.  The twiddle tables of the transforms of
 * sizes 2^k (omega^-1) and 2^ext_k (the extended omega) come on top and stay with the device.  A rejected call allocates only the check
 * word.  The pageable copy path's two 16 MiB pinned host buffers are per thread, as for every host-pointer entry point. */
int b200_pk_load(const void* const* h_fixed_values, size_t n_fixed, const void* const* h_permutations, size_t n_perm,
                 uint32_t k, uint32_t ext_k, uint32_t blinding_factors,
                 void* d_values, void* d_polys, size_t stride, void* d_l);

#ifdef __cplusplus
}
#endif
#endif /* EZKL_B200_PK_H */
