/*
 * ezkl_b200.h — C ABI of libezkl_b200.so, the Hopper (sm_90a, H100) proving backend for ezkl's Halo2/KZG prover.
 *
 * This is the drop-in boundary (SURVEY.md §8b): the entry points a Rust `mod b200;` inside the halo2 fork binds in place
 * of `mod icicle;` behind cfg(feature = "gpu-accelerated") (/root/reference/Cargo.toml:259), so that
 * `pfsys::create_proof_circuit` / `create_keys` (/root/reference/src/pfsys/mod.rs:404-489, 376-400), `ezkl prove`
 * (/root/reference/src/execute.rs:1575-1627) and the Python bindings stay unchanged.  INTEGRATION.md shows the shim.
 *
 * Conventions
 *   - return 0 = ok, < 0 = error (-1 bad argument, -2 CUDA failure, -3 not initialised); message via b200_last_error()
 *     (thread-local).  Nothing throws or aborts across the boundary; there is NO CPU fallback — without a usable
 *     sm_90 device every compute entry point fails with -2/-3.
 *   - the caller owns every host pointer for the duration of the call only; the library never frees caller memory.
 *   - Fr / Fq: 4 x u64 little-endian limbs in Montgomery form, exactly halo2curves' in-memory representation
 *     (zero-copy from &[Fr]).  G1 affine = {x, y} 64 B, identity = (0,0).  G1 Jacobian = {x, y, z} 96 B, identity z = 0.
 *   - every call is synchronous with respect to its host buffers and re-entrant: each calling thread gets its own CUDA
 *     stream and scratch arena per device (halo2 commits / transforms columns from Rayon worker threads).  The scratch
 *     the library holds is bounded process-wide (B200_WS_TOTAL_MB, default 24 GiB per device, divided among the calling
 *     threads), released when a calling thread exits and at b200_shutdown, which first waits for calls in flight.
 *   - a process may own 1, 2, 4 or 8 devices (b200_init_multi).  Host-pointer entry points then use all of them: columns
 *     of a batch are dealt over the devices, a single MSM is split by base range, a single transform of >= 2^22 elements is
 *     sharded; one host thread per extra device drives its own PCIe link.  Device-pointer entry points run on the device
 *     that owns the first device pointer they are given.  Environment overrides are read once, in b200_init.
 *   - MSM results are returned NORMALISED (z = 1, or (0,1,0) for the identity), so bytes are canonical and independent
 *     of accumulation order: what `best_multiexp(..).to_affine()` / `batch_normalize` yields on the CPU prover.
 *   - the *_dev entry points take device pointers (e.g. torch tensors' data_ptr) and a cudaStream_t (NULL = the
 *     calling thread's library stream); they do not synchronise.  Scratch is per calling thread: a call on a different
 *     stream than the thread's previous call first waits (cudaStreamWaitEvent) for that call's work, so one thread may
 *     alternate streams safely; calls that stage host parameters (quotient program, lincomb scalars, cycle constants)
 *     cannot be captured into a CUDA graph.
 */
#ifndef EZKL_B200_H
#define EZKL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct { uint64_t l[4]; } b200_fr;              /* halo2curves::bn256::Fr, Montgomery */
typedef struct { uint64_t l[4]; } b200_fq;              /* halo2curves::bn256::Fq, Montgomery */
typedef struct { b200_fq x, y; } b200_g1_affine;        /* halo2curves::bn256::G1Affine */
typedef struct { b200_fq x, y, z; } b200_g1_jac;        /* halo2curves::bn256::G1 */
typedef struct { b200_fq x, y, zz, zzz; } b200_g1_xyzz; /* device-side partial sums (x = X/ZZ, y = Y/ZZZ), identity zz = 0 */

/* ---- lifecycle: replaces halo2_proofs::icicle::try_load_and_set_backend_device("CUDA") + icicle_runtime::warmup
 *      (/root/reference/src/execute.rs:85-97).  device < 0 keeps the current device (e.g. the one torch selected). */
int b200_init(int device);
/* one process driving n_devices = 1, 2, 4 or 8 GPUs (devices 0 .. n-1, NVLink peer access enabled between all pairs): the
 * `b200_init(int n_devices)` of SURVEY.md §8b; what execute::set_device calls when EZKL_B200_DEVICES > 1 (INTEGRATION.md). */
int b200_init_multi(int n_devices);
int b200_device_count(void);
void b200_shutdown(void);
const char* b200_last_error(void);
int b200_version(void);
/* kernels launched by this library since load (all threads); used by bench.py's gpu_launches */
uint64_t b200_launch_count(void);

/* device-side timing of kernel classes with CUDA events on the launching stream (off by default).
 * cls: 0 = MSM bucket-accumulation kernel, 1 = whole MSM pipeline, 2 = NTT (all passes of a call), 3 = poly, 4 = MSM digit recoding +
 * bucket sort (kernels 1-6), 5 = MSM tail (combine, bucket reduction, final sum), 6 = evaluate_h kernel, 7 = MSM bucket scan
 * (k_scan_buckets), 8 = MSM bucket reduction and final sum, 9 = MSM sub-window fold (reduced tables only).
 * b200_profile_enable(1) clears earlier records; b200_profile_read synchronises the device and sums the class. */
int b200_profile_enable(int on);
int b200_profile_read(int cls, double* total_ms, uint64_t* count);

/* ---- SRS bases: ParamsKZG.g / .g_lagrange uploaded once (src/pfsys/srs.rs:30-47 loads them; every commit reuses them).
 *      Registration builds the window-precomputed table on the device.  window_bits = c (0 picks it from n) splits a scalar into
 *      W = ceil(255 / c) signed windows.  The table stores L = ceil(W / s) levels, level j = 2^(c*s*j) * P_i (affine, 64 B per
 *      point), so it takes L * n * 64 B per device.  s = 1 is the full table: every window shares one set of 2^(c-1) buckets.
 *      s > 1 (a reduced table) gives each of the s windows of a level its own bucket set and folds the s results at the end
 *      with (s-1)*c doublings: the same bucket additions per scalar, an s-fold bucket reduction.
 *      Level count: the smallest s whose table fits the budget, and never fewer than one level (the bases themselves), so a
 *      budget smaller than one level gives L = 1 rather than an error.  The budget is per registered vector and per device:
 *      max_table_bytes of b200_bases_register_ex[_dev], or, when that is 0 and for b200_bases_register[_dev], the process budget
 *      B200_MSM_TABLE_MB (MiB, a positive whole number, read in b200_init, which fails with -1 on anything else; default 16384 =
 *      16 GiB).  At the default window the default budget keeps the full table up to n = 2^24 (13 GiB) and gives s = 2, L = 7
 *      (14 GiB) at 2^25 and s = 4, L = 4 (16 GiB) at 2^26.  MSM results are normalised, so they are identical for every level count.
 *      Cost of a reduced table, measured for n = 2^20 .. 2^26 on an H100 80GB HBM3 at 700 W (DESIGN.md §4.2): 289 M pairs/s at 2^26
 *      and the default budget against 313 M with a 28 GiB table; 297 M against 318 M at 2^24 with half the full table.
 *      A handle may be used from any number of threads at once; b200_bases_release (and b200_shutdown, which releases every
 *      handle) must not run while another thread still has an MSM in flight on that handle (ParamsKZG outlives its commits). */
int b200_bases_register(const b200_g1_affine* bases, size_t n, int window_bits, uint64_t* handle);
int b200_bases_register_dev(const void* d_bases, size_t n, int window_bits, uint64_t* handle);
int b200_bases_register_ex(const b200_g1_affine* bases, size_t n, int window_bits, size_t max_table_bytes, uint64_t* handle);
int b200_bases_register_ex_dev(const void* d_bases, size_t n, int window_bits, size_t max_table_bytes, uint64_t* handle);
int b200_bases_release(uint64_t handle);
int b200_bases_info(uint64_t handle, size_t* n, int* window_bits, int* windows);
/* the table's layout: stored levels L, windows per level s, bytes per device (L * n * 64) */
int b200_bases_table(uint64_t handle, int* levels, int* windows_per_level, size_t* table_bytes);

/* ---- MSM: halo2_proofs::arithmetic::best_multiexp / ParamsKZG::{commit, commit_lagrange}
 *      (in-tree caller: /root/reference/src/circuit/modules/polycommit.rs:71).  n <= registered length. */
int b200_msm(uint64_t bases, const b200_fr* scalars, size_t n, b200_g1_jac* out);
/* batch columns sharing the bases (the advice / lookup / permutation commit loops of create_proof) */
int b200_msm_batch(uint64_t bases, const b200_fr* const* scalars, size_t n, size_t batch, b200_g1_jac* out);
/* device-resident: scalars[b*stride + i]; writes batch un-normalised XYZZ partial sums to d_out */
int b200_msm_batch_dev(uint64_t bases, const void* d_scalars, size_t n, size_t stride, size_t batch, void* d_out_xyzz, void* stream);
/* ONE MSM (or `batch` of them) whose (scalar, base) pairs are split across the devices of the process: d_scalar_slices[g] is a
 * device pointer on device g holding, per column, the pairs [lo_g, hi_g) of the contiguous n / n_devices split (remainder to
 * the low devices), columns back to back.  Every device runs its range against its table replica, the 128-byte XYZZ partial
 * sums cross NVLink to device 0 and are added there in device order (the group law has no NCCL reduction); out = normalised
 * points on the host.  Synchronises. */
int b200_msm_sharded_dev(uint64_t bases, const void* const* d_scalar_slices, size_t n, size_t batch, b200_g1_jac* out);
/* out[g] = sum_{j < count} points[g*count + j] (device XYZZ arrays): the local add after an all-gather of per-rank partials */
int b200_g1_sum_dev(const void* d_points_xyzz, size_t groups, size_t count, void* d_out_xyzz, void* stream);
/* FFT over G1: out[j] = scale * sum_i omega^(i*j) * in[i], 2^log_n affine points in and out (scale may be NULL = 1).
 * halo2's g_to_lagrange = this with omega^-1 and scale = n^-1: the body of ParamsKZG::downsize, which ezkl runs whenever the SRS
 * file is larger than the circuit (load_params_prover, /root/reference/src/execute.rs:1739-1750). */
int b200_g1_fft(const b200_g1_affine* in, uint32_t log_n, const b200_fr* omega, const b200_fr* scale, b200_g1_affine* out);
int b200_g1_fft_dev(const void* d_in_affine, uint32_t log_n, const b200_fr* omega, const b200_fr* scale, void* d_out_affine, void* stream);
/* out[i] = [scalars[i]] * base, affine: the n fixed-base multiplications behind ParamsKZG::new / gen_srs
 * (/root/reference/src/pfsys/srs.rs:14-16: g[i] = [s^i] G, g_lagrange[i] = [L_i(s)] G).  Device pointers. */
int b200_g1_fixed_base_mul_dev(const void* d_scalars, size_t n, const b200_g1_affine* base, void* d_out_affine, void* stream);
/* synthetic SRS-shaped bases for benchmarks: out[i] = [splitmix(seed, i)] * G, affine, pairwise distinct w.h.p. */
int b200_g1_generate_dev(uint64_t seed, size_t n, void* d_out_affine, void* stream);
/* host: XYZZ partials -> normalised Jacobian (one shared inversion) */
int b200_g1_normalize(const b200_g1_xyzz* points, size_t n, b200_g1_jac* out);

/* ---- NTT: halo2_proofs::arithmetic::best_fft and poly/domain.rs EvaluationDomain transforms -------------------- */
/* best_fft(a, omega, log_n): natural order in/out, a[j] <- sum_i a[i] omega^(ij) */
int b200_fft(b200_fr* a, uint32_t log_n, const b200_fr* omega);
int b200_fft_batch(b200_fr* const* a, size_t batch, uint32_t log_n, const b200_fr* omega);
/* EvaluationDomain::ifft(a, omega_inv, log_n, divisor): fft with omega_inv, then every element * divisor */
int b200_ifft(b200_fr* a, uint32_t log_n, const b200_fr* omega_inv, const b200_fr* divisor);
int b200_ifft_batch(b200_fr* const* a, size_t batch, uint32_t log_n, const b200_fr* omega_inv, const b200_fr* divisor);
/* coeff_to_extended: out[j] = p(zeta * ext_omega^j), j < 2^ext_k; coeffs has n_coeffs <= 2^ext_k entries */
int b200_coeff_to_extended(const b200_fr* coeffs, size_t n_coeffs, uint32_t ext_k, const b200_fr* ext_omega, const b200_fr* zeta, b200_fr* out);
int b200_coeff_to_extended_batch(const b200_fr* const* coeffs, size_t batch, size_t n_coeffs, uint32_t ext_k, const b200_fr* ext_omega, const b200_fr* zeta, b200_fr* const* out);
/* extended_to_coeff: ifft over the extended domain, * divisor, undo the zeta coset; caller truncates */
int b200_extended_to_coeff(b200_fr* a, uint32_t ext_k, const b200_fr* ext_omega_inv, const b200_fr* ext_ifft_divisor, const b200_fr* zeta);
/* device-resident generic transform: dst[p][j] = post(j) * sum_{i<n_in} pre(i) src[p][i] omega^(ij).
 * pre/post: mode 0 none, 1 constant c[0], 3 cycle c[i mod 3]; c points to HOST constants. tmp: 2^log_n * batch scratch.
 * batch <= 65535; with batch > 1, src_stride >= n_in and dst_stride >= 2^log_n (polynomials do not overlap). */
int b200_ntt_dev(const void* d_src, size_t src_stride, size_t n_in, void* d_tmp, void* d_dst, size_t dst_stride, uint32_t log_n,
                 const b200_fr* omega, int pre_mode, const b200_fr* pre, int post_mode, const b200_fr* post, size_t batch, void* stream);

/* ONE transform of 2^log_n elements split across the devices of the process: slice g (2^log_n / n_devices contiguous
 * natural-order elements) lives on device g, for the source, the scratch and the destination alike (dst may alias src).  All
 * passes run on all devices at once; the exchange steps of the six-step scheme are peer loads / stores over NVLink inside the
 * butterfly kernels, not separate copies or collectives.  Same pre / post scaling as b200_ntt_dev; n_in <= 2^log_n valid source
 * elements.  Enqueued on the calling thread's library stream of every device: b200_sync_all() waits for it. */
int b200_ntt_sharded_dev(const void* const* d_src_slices, void* const* d_tmp_slices, void* const* d_dst_slices, uint32_t log_n, size_t n_in,
                         const b200_fr* omega, int pre_mode, const b200_fr* pre, int post_mode, const b200_fr* post);

/* ---- column polynomial ops (halo2 `parallelize` loops; create_proof stages 2-9) ---------------------------------
 * op: 0 add, 1 sub, 2 mul (element-wise), 3 scale (out = a * s), 4 axpy (out = a + s * b).  out may alias a or b. */
int b200_poly_op(int op, const b200_fr* a, const b200_fr* b, const b200_fr* s, b200_fr* out, size_t n);
int b200_poly_op_dev(int op, const void* d_a, const void* d_b, const b200_fr* s, void* d_out, size_t n, void* stream);
/* out = sum_j scalars[j] * polys[j]  (n coefficients each): the SHPLONK / multiopen linear combinations q(X) = sum y^j p_j(X),
 * one pass over the inputs instead of count axpy calls */
int b200_poly_lincomb(const b200_fr* const* polys, const b200_fr* scalars, size_t count, size_t n, b200_fr* out);
int b200_poly_lincomb_dev(const void* const* d_polys, const b200_fr* scalars, size_t count, size_t n, void* d_out, void* stream);
/* a[i] *= consts[i mod period]: distribute_powers_zeta (period 3) / divide_by_vanishing_poly (period 2^(ext_k-k)) */
int b200_poly_scale_cycle(b200_fr* a, size_t n, const b200_fr* consts, uint32_t period);
int b200_poly_scale_cycle_dev(void* d_a, size_t n, const b200_fr* consts, uint32_t period, void* stream);
/* eval_polynomial(coeffs, x) */
int b200_poly_eval(const b200_fr* coeffs, size_t n, const b200_fr* x, b200_fr* out);
/* out[p] = polys[p](x[p]), p < batch: the evaluation round of create_proof */
int b200_poly_eval_batch(const b200_fr* const* polys, size_t n, const b200_fr* x, size_t batch, b200_fr* out);
int b200_poly_eval_batch_dev(const void* d_polys, size_t stride, size_t n, const b200_fr* x, size_t batch, void* d_out, void* stream);
/* ff::BatchInvert (zeros stay zero) */
int b200_batch_invert(b200_fr* a, size_t n);
int b200_batch_invert_dev(void* d_a, size_t n, void* stream);
/* out[0] = init, out[i+1] = out[i] (* or +) a[i]: permutation z(X) / mv-lookup phi(X) running columns.  The _dev forms may run in
 * place (d_out == d_a, and for the batch form out_stride == a_stride): every element is read by the thread that overwrites it. */
int b200_prefix_scan(int product, const b200_fr* a, size_t n, const b200_fr* init, b200_fr* out);
int b200_prefix_scan_dev(int product, const void* d_a, size_t n, const b200_fr* init, void* d_out, void* stream);
/* `batch` independent columns in one call (the mv-lookup grand sums of a proof are independent of each other; the permutation products are
 * chained through last_z and are not): column p at d_a + p * a_stride elements, its result at d_out + p * out_stride, initial value inits[p] */
int b200_prefix_scan_batch_dev(int product, const void* d_a, size_t a_stride, size_t n, size_t batch, const b200_fr* inits, void* d_out, size_t out_stride, void* stream);
/* kate_division(a, b): quotient of a(X) by (X - b), n-1 coefficients.  Not in place: q[e] depends on a[e+1 ..], so the _dev form
 * returns -1 when d_q == d_a. */
int b200_kate_division(const b200_fr* a, size_t n, const b200_fr* b, b200_fr* q);
int b200_kate_division_dev(const void* d_a, size_t n, const b200_fr* b, void* d_q, void* stream);

/* ---- mv-lookup multiplicities: halo2 plonk/mv_lookup/prover.rs (stage 2 of create_proof; every ezkl lookup, range check, dynamic
 *      lookup and shuffle: /root/reference/src/circuit/ops/chip.rs:496,662,782,870).  m[i] = number of cells inputs[j][r], j < n_inputs,
 *      r < n_rows, equal to table[i]; when a value occurs in several table rows (ezkl pads tables with a repeated entry) the FIRST
 *      row gets the whole count and the others 0.  *missing (may be NULL) = input cells whose value is not in the table (the CPU
 *      prover panics on those).  m has n_table elements, Montgomery form.  The _dev form synchronises only when missing != NULL. */
int b200_lookup_multiplicities(const b200_fr* table, size_t n_table, const b200_fr* const* inputs, size_t n_inputs, size_t n_rows, b200_fr* m, uint64_t* missing);
int b200_lookup_multiplicities_dev(const void* d_table, size_t n_table, const void* const* d_inputs, size_t n_inputs, size_t n_rows, void* d_m, uint64_t* missing, void* stream);

/* ---- quotient numerator: halo2 plonk/evaluation.rs Evaluator::evaluate_h (GraphEvaluator) -------------------------
 * A straight-line program of field operations evaluated once per row of the extended domain:
 *   out[idx] = program(columns[c][(idx + rotation * 2^(ext_k - k)) mod 2^ext_k], constants).
 * Operand encoding (b200_instr.a / .b / .c): bits 31..30 kind — 0 slot (result register, < 256), 1 constants[index],
 * 2 loads[index], 3 the result of the previous instruction — bits 29..0 index.  op_dst = op | (dst_slot << 8) | (no_store << 31);
 * op: 0 add, 1 sub, 2 mul, 3 neg(a), 4 double(a), 5 square(a), 6 mov(a), 7 muladd (a * b + c: one step of GraphEvaluator's Horner
 * calculation).  no_store marks a result that only the next instruction reads (as operand kind 3).  The row's result is the
 * result of the last instruction.  Gates, permutation and lookup terms, l0 / l_last / l_active_row, the identity coset and earlier
 * partial sums are all just columns; y, beta, gamma, theta and the phase challenges are constants.  Columns are 2^ext_k elements
 * each; the program, its loads and constants must fit 160 KB (split larger constraint systems into partial sums carried as a column). */
typedef struct { uint32_t op_dst; uint32_t a, b, c; } b200_instr;
typedef struct { uint32_t column; int32_t rotation; } b200_col_ref;
int b200_quotient_eval(const b200_fr* const* columns, size_t n_columns, uint32_t k, uint32_t ext_k, const b200_col_ref* loads, size_t n_loads,
                       const b200_fr* constants, size_t n_constants, const b200_instr* program, size_t n_instr, b200_fr* out);
int b200_quotient_eval_dev(const void* const* d_columns, size_t n_columns, uint32_t k, uint32_t ext_k, const b200_col_ref* loads, size_t n_loads,
                           const b200_fr* constants, size_t n_constants, const b200_instr* program, size_t n_instr, void* d_out, void* stream);

/* evaluate_h at the boundary the CPU evaluator has (UPSTREAM plonk/evaluation.rs builds the advice / instance cosets itself from the
 * coefficient-form polynomials; plonk/vanishing/prover.rs then divides by the vanishing polynomial and converts back): column i of the
 * program is coeff_to_extended(polys[i]) when lengths[i] < 2^ext_k (coefficient form, zeta coset, zero padded) and polys[i] itself when
 * lengths[i] == 2^ext_k (the key's fixed / permutation cosets, l0 / l_last / l_active_row, a running partial sum).  out = the numerator on
 * the extended domain, or, when t_evaluations != NULL, extended_to_coeff(numerator * t_evaluations[i mod t_period]): the quotient's
 * 2^ext_k coefficients.  A coefficient column crosses PCIe once (its n elements) instead of its coset twice.
 * Device memory: when n_columns * 2^ext_k * 32 B fits the per-call scratch budget (B200_WS_BUDGET_MB, else derived from
 * B200_WS_TOTAL_MB, as for every host-pointer entry point) all columns' cosets are resident at once, which holds
 * n_columns * 2^ext_k * 32 B + (sum of the coefficient columns' lengths) * 32 B + 2 * 2^ext_k * 32 B.  Otherwise (and k >= 1) the
 * numerator is evaluated one n-point coset part at a time (the extended indices c + d i, d = 2^(ext_k - k), for c < d), which holds
 * about n_columns * n * 32 B + (sum of the coefficient columns' lengths) * 32 B + 2 * 2^ext_k * 32 B.  The result is the same bytes
 * either way. */
int b200_evaluate_h(const b200_fr* const* polys, const size_t* lengths, size_t n_columns, uint32_t k, uint32_t ext_k, const b200_fr* ext_omega, const b200_fr* zeta,
                    const b200_col_ref* loads, size_t n_loads, const b200_fr* constants, size_t n_constants, const b200_instr* program, size_t n_instr,
                    const b200_fr* t_evaluations, uint32_t t_period, const b200_fr* ext_omega_inv, const b200_fr* ext_ifft_divisor, b200_fr* out);

/* ---- quotient from device-resident columns: b200_evaluate_h for callers that keep a proof's columns on the device -----------------
 * (INTEGRATION.md §2b): the witness, the key's polynomials and every column derived from them stay in device memory for the whole proof,
 * and each stage is handed device pointers.  The device-pointer twin of b200_evaluate_h, with the same semantics and the same result bytes:
 *   - column i of the program is coeff_to_extended(d_polys[i]) when lengths[i] < 2^ext_k (coefficient form: the advice, lookup and
 *     permutation polynomials, ProvingKey.fixed_polys / permutation.polys), and d_polys[i] itself when lengths[i] == 2^ext_k (an
 *     extended column: the key's l0 / l_last / l_active_row cosets, a running partial sum);
 *   - the program encoding is that of b200_quotient_eval;
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

/* ---- permutation keygen: the sigma columns (halo2 plonk/permutation/keygen.rs, Assembly::build_vk / build_pk) -------------------
 * A step of create_keys (keygen_vk / keygen_pk) that is not also a step of create_proof.
 * The mapping is the Assembly's after every copy constraint has been merged into its cycles: n_columns * 2^k pairs of uint32
 * (column, row), column-major, so cell (column j, row i) sits at mapping[2 * (j * 2^k + i)] (its column) and
 * mapping[2 * (j * 2^k + i) + 1] (its row).  The shim flattens halo2's `mapping: Vec<Vec<(usize, usize)>>` into this layout.
 * Sigma column j, row i = delta^c * omega^r where (c, r) is cell (j, i)'s entry: Fr in Montgomery form, fully reduced, so the bytes are
 * those of build_pk's `permutations` (halo2 computes them as a table of delta^j * omega^i followed by a gather).  omega = the domain's
 * n-th root of unity, delta = Fr::DELTA.  The library does not check that the mapping is a permutation (halo2 does not either); it only
 * needs every column < n_columns and every row < 2^k.
 * Both entry points: -1 for k > 28, and for a null pointer when n_columns > 0; 0 with no work when n_columns == 0.
 *
 * Host pointers: out[j] receives sigma column j (2^k elements).  Every cell is checked on the host before any device work: a cell
 * outside n_columns x 2^k returns -1 and writes nothing.  The mapping and the results are staged in column groups bounded by the
 * per-call scratch budget (B200_WS_BUDGET_MB, else derived from B200_WS_TOTAL_MB), which holds a group's 40 B per cell (8 B of mapping
 * and 32 B of result), so k = 26 and beyond need no more than one column at a time.  In a multi-device process the columns are dealt
 * over the devices, each staging its own columns over its own PCIe link.
 * Device pointers: sigma column j at d_out + 32 * j * out_stride bytes (out_stride >= 2^k elements, else -1); d_out must not overlap
 * d_mapping.  A cell outside n_columns x 2^k is written as zero; when `invalid` is non-NULL it receives the number of such cells and
 * the call synchronises its stream, otherwise the call only enqueues.  Runs on the device that owns d_out.
 * Device memory held beyond the caller's buffers: the table [delta^c, c < n_columns | omega^e, e < 2^ceil(k/2) | omega^(e 2^ceil(k/2)),
 * e < 2^floor(k/2)], 32 B per entry, in the thread's parameter ring (a slot up to 256 KiB, a reused device buffer above), 8 B for the
 * counter of invalid cells, and for the host-pointer form the staging of one column group. */
int b200_permutation_sigmas(const uint32_t* mapping, size_t n_columns, uint32_t k, const b200_fr* omega, const b200_fr* delta, b200_fr* const* out);
int b200_permutation_sigmas_dev(const void* d_mapping, size_t n_columns, uint32_t k, const b200_fr* omega, const b200_fr* delta, void* d_out, size_t out_stride,
                                uint64_t* invalid, void* stream);

/* ---- proving-key and SRS loading: a parameter file or a proving key straight to the device, checked there -----------------------
 *
 * b200_srs_register: ParamsKZG::read + ParamsKZG::downsize + two b200_bases_register_ex, in one call.  A KZG parameter file's two G1
 * vectors go straight into registered base tables, checked on the device, with the Lagrange-basis vector computed on the device when the
 * file is larger than the circuit.
 * g: the first 2^k points of the file's `g` vector (G1Affine wire form, as ParamsKZG::write lays them out), in host memory; pageable
 * memory and a memory-mapped file are both fine.  g_lagrange: the file's own 2^k-point Lagrange-basis vector, which the caller passes
 * when the file's k equals k; NULL computes it on the device from g with the group FFT (omega^-1, then scale n^-1), as
 * ParamsKZG::downsize does.  window_bits and max_table_bytes mean what they mean for b200_bases_register_ex and apply to both tables.
 *
 * Each given vector is staged through the pageable copy path straight into level 0 of its new table (no per-thread staging buffer grows
 * to the vector's size) and every point passed is checked on the device as halo2curves' G1Affine::from_raw_bytes checks it: x and y are
 * canonical (the 4 little-endian u64 limbs, read as a 256-bit integer, are below p) and the point is (0, 0) or satisfies y^2 = x^3 + 3.
 * Then the Lagrange-basis vector is transformed if needed, both tables are built and copied to the other devices of the process, and
 * *g_handle / *g_lagrange_handle receive two handles for b200_msm* and b200_bases_release.  Synchronous, like b200_bases_register.
 *
 * All or nothing: on any error no handle is written and no table memory is kept.  Returns -1 for bad arguments (NULL g or handle
 * pointers, k > 26, window_bits not 0 or 4..24) before any device work, and for an invalid point, with b200_last_error() naming the
 * vector, the index and the reason: "srs_register: g_lagrange[1234] is not on the curve" ("x is not below p", "y is not below p").
 * With several invalid points the lowest index of g is named, else the lowest of g_lagrange.  -2 for a CUDA failure.
 *
 * Unlike halo2's read, only the points passed are checked: a bad point of the file beyond 2^k, or in a g_lagrange vector the caller
 * skips because it downsizes, is never read and so never seen. */
int b200_srs_register(const b200_g1_affine* g, const b200_g1_affine* g_lagrange, uint32_t k, int window_bits, size_t max_table_bytes,
                      uint64_t* g_handle, uint64_t* g_lagrange_handle);

/* b200_pk_load: ProvingKey::read (RawBytes, with precompute-coset) for a device-resident prover, in one call.  The Lagrange columns of a
 * RawBytes proving key go straight into device memory, checked on the device, with the key's coefficient columns and its l0 / l_last /
 * l_active_row cosets derived there instead of read.
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
 * columns go in groups of g = min(C, 65535, max(1, floor(B / (32 n)))) columns and the l-cosets in groups of s = min(3, max(1,
 * floor(B / (32 N)))); each buffer is allocated with 1/8 headroom, plus 8 B for the check word.  The twiddle tables of the transforms of
 * sizes 2^k (omega^-1) and 2^ext_k (the extended omega) come on top and stay with the device.  A rejected call allocates only the check
 * word.  The pageable copy path's two 16 MiB pinned host buffers are per thread, as for every host-pointer entry point. */
int b200_pk_load(const void* const* h_fixed_values, size_t n_fixed, const void* const* h_permutations, size_t n_perm,
                 uint32_t k, uint32_t ext_k, uint32_t blinding_factors,
                 void* d_values, void* d_polys, size_t stride, void* d_l);

/* ---- device / pinned memory helpers for callers without their own CUDA runtime ---------------------------------- */
int b200_dev_alloc(void** d_ptr, size_t bytes);
int b200_dev_alloc_on(int device_slot, void** d_ptr, size_t bytes);   /* multi-device process: allocate on device `device_slot` */
int b200_dev_free(void* d_ptr);
/* synchronous: on return the bytes are on the device (upload) or in h_dst (download).  Pageable host memory is staged like every
 * host-pointer entry point's columns; a null pointer with bytes > 0 is an argument error (-1) */
int b200_dev_upload(void* d_dst, const void* h_src, size_t bytes);
/* enqueue-only upload on `stream` (NULL = the calling thread's library stream); the host buffer must be pinned (b200_host_alloc)
 * and stay untouched until the stream reaches the copy: lets a resident-column shim overlap witness uploads with the first commits */
int b200_dev_upload_async(void* d_dst, const void* h_src, size_t bytes, void* stream);
int b200_dev_download(void* h_dst, const void* d_src, size_t bytes);
int b200_host_alloc(void** h_ptr, size_t bytes);      /* pinned */
int b200_host_free(void* h_ptr);
int b200_sync(void);                                   /* the calling thread's library stream */
int b200_sync_all(void);                               /* ... on every device of the process */

#ifdef __cplusplus
}
#endif
#endif /* EZKL_B200_H */
