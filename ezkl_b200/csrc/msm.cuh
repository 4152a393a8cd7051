// msm.cuh — internal interface of the BN254 G1 multi-scalar-multiplication engine (msm.cu).
#pragma once
#include "common.cuh"
#include "ec.cuh"

namespace b200 {

// Device-resident, window-precomputed base table for one SRS vector (ParamsKZG.g or .g_lagrange):
// level w holds 2^(c*w) * P_i in affine form, so every signed c-bit digit of every scalar lands in ONE shared set of
// 2^(c-1) buckets and no per-window doubling chain is left for the end.
struct MsmTable {
    G1Affine* d_table = nullptr;   // [W][n]
    size_t n = 0;
    int c = 0;
    int W = 0;
    int device = 0;
};

struct MsmWorkspace {
    DevBuf counts, offs, ents, subs, sums, misc;
};

int msm_default_window(size_t n);
// Builds the table from n affine points already on the device (copied; caller keeps ownership of d_bases).
int msm_table_build(MsmTable* t, const G1Affine* d_bases, size_t n, int c, cudaStream_t st);
void msm_table_free(MsmTable* t);
// out[b] = sum_i scalars[b*stride + i] * P_(base_off + i)   (base_off + n <= table.n), XYZZ form, one point per column, on device.
// base_off > 0 is the base-split MSM: each device takes a contiguous range of the (scalar, base) pairs against its table replica.
int msm_run(const MsmTable& t, const Fr* d_scalars, size_t n, size_t stride, int batch, G1Xyzz* d_out,
            MsmWorkspace& ws, cudaStream_t st, size_t base_off = 0);
int g1_fixed_base_mul_run(const Fr* d_scalars, size_t n, const G1Affine& base, G1Affine* d_out, cudaStream_t st);
// out[j] = scale * sum_i omega^(i j) * P_i over G1 (halo2 g_to_lagrange / ParamsKZG::downsize); affine in, affine out
int g1_fft_run(const G1Affine* d_in, uint32_t log_n, const Fr& omega, const Fr* scale, G1Affine* d_out, DevBuf& scratch, cudaStream_t st);
int g1_generate_run(uint64_t seed, size_t n, G1Affine* d_out, cudaStream_t st);
// out[g] = sum_j points[g*count + j]
int g1_sum_run(const G1Xyzz* d_points, size_t groups, size_t count, G1Xyzz* d_out, cudaStream_t st);
// bytes of workspace msm_run needs per column (upper bound, for batch splitting)
size_t msm_workspace_per_column(const MsmTable& t, size_t n);

// Signed c-bit window recoding of a canonical (non-Montgomery) scalar, one digit per call, low window first:
// consumes the low c bits of s (s is shifted right in place) and returns a digit in [-2^(c-1), 2^(c-1)].
// *carry must start at 0.  Static limb indexing only, so s stays in registers.  Requires 1 <= c <= 31.
HD int32_t msm_next_digit(uint32_t s[8], int c, uint32_t* carry) {
    uint32_t v = (s[0] & ((1u << c) - 1u)) + *carry;
#pragma unroll
    for (int j = 0; j < 7; ++j) s[j] = (s[j] >> c) | (s[j + 1] << (32 - c));
    s[7] >>= c;
    if (v > (1u << (c - 1))) { *carry = 1; return (int32_t)v - (int32_t)(1u << c); }
    *carry = 0;
    return (int32_t)v;
}

}  // namespace b200
