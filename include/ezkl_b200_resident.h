/*
 * ezkl_b200_resident.h — entry points of libezkl_b200.so for callers that keep a proof's columns resident on the device
 * (INTEGRATION.md §2b): the witness, the key's polynomials and every column derived from them stay in device memory for the
 * whole proof, and each stage is handed device pointers.  The types and conventions are those of ezkl_b200.h, which this header
 * includes; the _dev conventions there (device pointers, a cudaStream_t with NULL = the calling thread's library stream, no
 * synchronisation, per-thread scratch ordered across streams) hold for every call below.
 */
#ifndef EZKL_B200_RESIDENT_H
#define EZKL_B200_RESIDENT_H

#include "ezkl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- quotient: b200_evaluate_h on device-resident columns ----------------------------------------------------------
 * The device-pointer twin of b200_evaluate_h, with the same semantics and the same result bytes:
 *   - column i of the program is coeff_to_extended(d_polys[i]) when lengths[i] < 2^ext_k (coefficient form: the advice, lookup and
 *     permutation polynomials, ProvingKey.fixed_polys / permutation.polys), and d_polys[i] itself when lengths[i] == 2^ext_k (an
 *     extended column: the key's l0 / l_last / l_active_row cosets, a running partial sum);
 *   - the program encoding is that of b200_quotient_eval (ezkl_b200.h);
 *   - t_evaluations == NULL: d_out = the numerator on the extended domain (2^ext_k elements).  Otherwise d_out = the quotient's 2^ext_k
 *     coefficients, extended_to_coeff(numerator * t_evaluations[i mod t_period]), which needs t_period in 1 ... 1024, ext_omega_inv
 *     and ext_ifft_divisor;
 *   - the result equals b200_evaluate_h's on the same columns, byte for byte, whatever that call's scratch budget selects.
 * Pointers and streams: d_polys[i] and d_out are device pointers; every other pointer is host memory, read during the call.  The call
 * runs on the device that owns d_out, is enqueued on `stream` (NULL = the calling thread's library stream) and does not synchronise.
 * Columns are read-only and may overlap each other (views of one allocation); d_out must not overlap any column [d_polys[i],
 * d_polys[i] + 32 * lengths[i]).
 * One path: the numerator is evaluated one n-point coset part at a time, n = 2^k, for the d = 2^(ext_k - k) parts c < d (the extended
 * indices c + d i; one part when k == ext_k).  Per part, every coefficient column is folded and transformed into its n-point part;
 * extended columns are read where they are, every d-th element from d_polys[i] + c, never copied; the interpreter stores row i at
 * index c + d i of d_out.  The finishing step then runs in place in d_out.  The per-call scratch budget (B200_WS_BUDGET_MB) selects
 * nothing here, because the caller's columns are already resident.
 * Device scratch held by the calling thread: n_coeff * 2^k * 32 B (the coefficient columns' parts, n_coeff = the number of columns
 * with lengths[i] < 2^ext_k) + 2^ext_k * 32 B (transform scratch) + the power table ((3 + 2^ceil(ext_k/2) + 2^floor(ext_k/2)) * 32 B)
 * and 16 B per coefficient column; each buffer is allocated with 1/8 headroom, and the transform plans of sizes 2^k and 2^ext_k come on
 * top.  At k = 22, ext_k = 25 with 129 coefficient columns that is 17.1 GiB stated and 20.4 GiB held after a finished call (H100 80GB
 * HBM3, 700 W; DESIGN.md §4.4).
 * Argument errors return -1, with a message in b200_last_error(), and write nothing to d_out: a null pointer (d_polys and lengths may be
 * NULL when n_columns == 0), a length of 0 or above 2^ext_k, k == 0, k > ext_k or ext_k > 28, finishing without its constants or with
 * t_period outside 1 ... 1024, d_out overlapping a column, and every program check of b200_quotient_eval_dev. */
int b200_evaluate_h_dev(const void* const* d_polys, const size_t* lengths, size_t n_columns, uint32_t k, uint32_t ext_k,
                        const b200_fr* ext_omega, const b200_fr* zeta,
                        const b200_col_ref* loads, size_t n_loads, const b200_fr* constants, size_t n_constants,
                        const b200_instr* program, size_t n_instr,
                        const b200_fr* t_evaluations, uint32_t t_period, const b200_fr* ext_omega_inv, const b200_fr* ext_ifft_divisor,
                        void* d_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* EZKL_B200_RESIDENT_H */
