/*
 * debug.h — the test-only hooks of libezkl_b200_dbg.so (debug.cu): per-layer self tests, the host-compiled recoding, level and
 * NTT-geometry policies, and microbenchmarks.  Not part of the drop-in ABI of include/ezkl_b200.h.  ezkl_b200/_native.py reads
 * the call signatures below when it loads the library.  Every pointer is a HOST pointer.
 */
#pragma once
#include "../../include/ezkl_b200.h"

extern "C" {
/* device: stage the inputs, run one kernel, copy back */
int b200_debug_field_op(int field, int op, const b200_fr* a, const b200_fr* b, b200_fr* out, size_t n);
int b200_debug_g1_op(int op, const b200_g1_affine* a, const b200_g1_affine* b, b200_g1_affine* out, size_t n);
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
int b200_debug_ntt_plan_host(uint32_t log_n, int batch, int sm_count, int64_t* out);
int b200_debug_host_g1_op(int op, const b200_g1_affine* a, const b200_g1_affine* b, b200_g1_affine* out, size_t n);
int b200_debug_host_field_op(int field, int op, const b200_fr* a, const b200_fr* b, b200_fr* out, size_t n);
}
