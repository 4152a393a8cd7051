/*
 * ezkl_b200_srs.h — SRS loading entry point of libezkl_b200.so: a KZG parameter file's two G1 vectors straight into registered base
 * tables, checked on the device, with the Lagrange-basis vector computed on the device when the file is larger than the circuit.  The
 * types and conventions are those of ezkl_b200.h, which this header includes.
 */
#ifndef EZKL_B200_SRS_H
#define EZKL_B200_SRS_H

#include "ezkl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- ParamsKZG::read + ParamsKZG::downsize + two b200_bases_register_ex, in one call ---------------------------------------------
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

#ifdef __cplusplus
}
#endif
#endif /* EZKL_B200_SRS_H */
