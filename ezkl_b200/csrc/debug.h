/*
 * debug.h — the test-only hooks of libezkl_b200_dbg.so (debug.cu): per-layer self tests, the host-compiled recoding, level and
 * NTT-geometry policies, and microbenchmarks.  Not part of the drop-in ABI of include/ezkl_b200.h.  ezkl_b200/_native.py reads
 * the call signatures below when it loads the library.  Every pointer is a HOST pointer.
 */
#pragma once
#include "../../include/ezkl_b200.h"

extern "C" {
/* device: stage the inputs, run one kernel, copy back */
/* field: 0 Fr, 1 Fq; op: 0 add, 1 sub, 2 mul, 3 inv, 4 from_mont, 5 sqr, 6 neg, 7 dbl, 8 to_mont (Montgomery words in and out) */
int b200_debug_field_op(int field, int op, const b200_fr* a, const b200_fr* b, b200_fr* out, size_t n);
/* op: 0 a b + c d (fp_muladd2), 1 a b - c d (fp_mulsub2) */
int b200_debug_field_op4(int field, int op, const b200_fr* a, const b200_fr* b, const b200_fr* c, const b200_fr* d, b200_fr* out, size_t n);
/* affine in and out; op: 0 a + b, 1 2a, 2 k a (k = b.x limb 0), 3 a + 2b, 4 a + (-a) */
int b200_debug_g1_op(int op, const b200_g1_affine* a, const b200_g1_affine* b, b200_g1_affine* out, size_t n);
/* XYZZ in, raw XYZZ words out; op: 0 g1_add(a, b), 1 g1_dbl(a), 2 g1_add_mixed(a, (b.x, b.y)), 3 g1_mul_small(a, k[i]),
 * 4 g1_to_affine(a) as (x, y, 0, 0), 5 g1_add_coop4(a, b), 6 g1_dbl_coop4(a) (5 and 6: one quad of lanes per element) */
int b200_debug_g1_xyzz_op(int op, const b200_g1_xyzz* a, const b200_g1_xyzz* b, const uint32_t* k, b200_g1_xyzz* out, size_t n);
int b200_debug_digits(const b200_fr* s, size_t n, int c, int32_t* out);
int b200_debug_bench(int variant, int iters, int blocks, int threads, float* ms);
int b200_debug_bench_pipe(int variant, int iters, int blocks, int threads, float* ms);
int b200_debug_msm_base_off(const b200_fr* scalars, size_t n, int batch, const b200_g1_affine* bases, size_t table_n, int c,
                            size_t max_table_bytes, size_t base_off, b200_g1_affine* out);
/* host only: no device needed */
int b200_debug_digits_host(const b200_fr* s_canonical, size_t n, int c, int32_t* out);
int b200_debug_digit_slots_host(const b200_fr* s_canonical, size_t n, int c, int wpl, int32_t* out);
int b200_debug_msm_pick_levels(size_t n, int c, size_t max_table_bytes, int* s, int* L);
int b200_debug_msm_recode_plan(size_t n, int batch, uint32_t nbuckets, int W, int sm_count, uint32_t* out);
/* msm_run's launch geometry and workspace bytes (16 values, see debug.cu); reduce_m / reduce_threads: the tuning overrides, 0 = automatic */
int b200_debug_msm_plan(size_t n, int batch, int c, int s, int sm_count, int reduce_m, int reduce_threads, uint64_t* out);
int b200_debug_ntt_plan_host(uint32_t log_n, int batch, int sm_count, int64_t* out);
int b200_debug_host_g1_op(int op, const b200_g1_affine* a, const b200_g1_affine* b, b200_g1_affine* out, size_t n);
int b200_debug_host_g1_xyzz_op(int op, const b200_g1_xyzz* a, const b200_g1_xyzz* b, const uint32_t* k, b200_g1_xyzz* out, size_t n);   /* ops 0-4 */
int b200_debug_host_field_op(int field, int op, const b200_fr* a, const b200_fr* b, b200_fr* out, size_t n);
int b200_debug_host_field_op4(int field, int op, const b200_fr* a, const b200_fr* b, const b200_fr* c, const b200_fr* d, b200_fr* out, size_t n);
}
