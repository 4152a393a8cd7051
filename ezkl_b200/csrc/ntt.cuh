// ntt.cuh — internal interface of the BN254 Fr number-theoretic-transform engine (ntt.cu).
#pragma once
#include <map>
#include <vector>
#include "common.cuh"
#include "field.cuh"

namespace b200 {

// Twiddle tables for one (log_n, omega) pair, device resident.
struct NttPlan {
    uint32_t log_n = 0;
    Fr omega;                 // Montgomery form
    int npass = 0;
    int logm[3] = {0, 0, 0};
    Fr* d_tw[3] = {nullptr, nullptr, nullptr};   // per pass: (omega^(N/M))^k, k < M/2
    uint4* d_staged[3] = {nullptr, nullptr, nullptr};   // per pass: per-stage twiddles, planar (v2 kernel)
    Fr* d_full = nullptr;     // omega^e, e < N (ntt_full_table): single-multiply inter-pass twiddles
    Fr* d_lo = nullptr;       // omega^e, e < 2^lo_bits
    Fr* d_hi = nullptr;       // omega^(e << lo_bits), e < N >> lo_bits
    uint32_t lo_bits = 0;
};

struct NttScale {             // optional per-element scaling fused into the first load / last store
    int mode = 0;             // 0 none, 1 one constant (c[0]), 3 cycle c[i % 3]
    Fr c[3];
};

struct NttContext {
    std::vector<NttPlan*> plans;
    NttPlan* get(uint32_t log_n, const Fr& omega, cudaStream_t st);
    void release();
};

// ---- pass geometry: pure host functions of (log_n, batch, SM count), shared by the launch code and the test hook ----------
// Factorisation N = M1 * M2 (* M3), every M <= 1024: one pass per factor.
inline void ntt_choose_passes(uint32_t log_n, int* npass, int logm[3]) {
    logm[0] = logm[1] = logm[2] = 0;
    if (log_n <= 10) { *npass = 1; logm[0] = (int)log_n; return; }
    if (log_n <= 20) { *npass = 2; logm[0] = (int)(log_n + 1) / 2; logm[1] = (int)log_n - logm[0]; return; }
    *npass = 3;
    logm[0] = (int)(log_n + 2) / 3; logm[1] = (int)(log_n - logm[0] + 1) / 2; logm[2] = (int)log_n - logm[0] - logm[1];
}
// whether a plan keeps the full omega^e table (N * 32 B) for single-multiply inter-pass twiddles; above 2^25 the two-level
// t_lo / t_hi tables serve alone
inline bool ntt_full_table(uint32_t log_n, int npass) { return npass > 1 && log_n <= 25; }

// Pass `idx` transforms `lines` lines of 2^logm elements; `inner_cnt` of them are adjacent (the inner index a CTA may group).
struct NttPassShape { uint32_t inner_cnt; uint64_t lines; };
inline NttPassShape ntt_pass_shape(int npass, const int logm[3], int idx) {
    const uint64_t N1 = 1ull << logm[0], N2 = 1ull << logm[1], N3 = 1ull << logm[2];
    if (npass == 1) return {1, 1};
    if (npass == 2) return idx == 0 ? NttPassShape{(uint32_t)N2, N2} : NttPassShape{(uint32_t)N1, N1};
    if (idx == 0) return {(uint32_t)(N2 * N3), N2 * N3};
    if (idx == 1) return {(uint32_t)N3, N1 * N3};
    return {(uint32_t)N1, N1 * N2};
}

// Launch geometry of one pass: kernel 2 (k_ntt_pass2) where a CTA of 2^(logm + log_g) elements holds at least 32 quads,
// else kernel 1 (k_ntt_pass).  2^log_g lines per CTA, as many as still give 2 CTAs per SM.
struct NttPassGeom { int kernel; uint32_t log_g, threads; size_t smem; uint64_t grid_x; };
inline NttPassGeom ntt_pass_geometry(uint32_t logm, uint32_t inner_cnt, uint64_t lines, int batch, int sm_count) {
    NttPassGeom g{};
    const uint64_t min_ctas = 2 * (uint64_t)sm_count;
    if (logm >= 2) {        // v2: G lines per CTA chosen so that a CTA holds 1024 elements (256 threads, one quad each; 3 CTAs per SM)
        uint32_t log_g = logm >= 10 ? 0 : 10 - logm;
        while (log_g > 0 && ((1u << log_g) > inner_cnt || (lines >> log_g) * (uint64_t)batch < min_ctas)) --log_g;
        while (log_g > 0 && (logm + log_g > 10)) --log_g;
        if (logm + log_g >= 7) {
            g.kernel = 2; g.log_g = log_g;
            g.threads = 1u << (logm + log_g - 2);
            g.smem = (((size_t)1 << (logm + log_g)) + ((size_t)1 << logm)) * 32;
            g.grid_x = lines >> log_g;
            return g;
        }
    }
    // v1: largest G in {4,2,1} that still yields >= 2 CTAs per SM (and fits shared memory)
    uint32_t log_g = 2;
    while (log_g > 0 && ((1u << log_g) > inner_cnt || (lines >> log_g) * (uint64_t)batch < min_ctas)) --log_g;
    while (log_g > 0 && (((size_t)1 << (logm + log_g)) + ((size_t)1 << logm) / 2) * 32 > 200 * 1024) --log_g;
    g.kernel = 1; g.log_g = log_g;
    g.smem = (((size_t)1 << (logm + log_g)) + (((size_t)1 << logm) >> 1)) * 32;
    const uint32_t nbf = (1u << (logm + log_g)) >> 1;
    g.threads = nbf < 32 ? 32 : (nbf > 1024 ? 1024 : nbf);
    g.grid_x = lines >> log_g;
    return g;
}

// `plan` = NttContext::get(log_n, omega) obtained by the caller under its own lock (plans are immutable once built).
// dst[p][j] = post(j) * sum_{i < n_in} pre(i) * src[p][i] * omega^(i j),  j < 2^log_n, for p < batch polynomials.
// src has n_in <= 2^log_n valid elements per polynomial (rest treated as zero), tmp and dst hold 2^log_n each;
// dst may alias src (when n_in == 2^log_n and strides match); tmp must not alias either.
int ntt_run(NttPlan* plan, const Fr* d_src, size_t src_stride, size_t n_in, Fr* d_tmp, size_t tmp_stride, Fr* d_dst, size_t dst_stride,
            uint32_t log_n, const Fr& omega, const NttScale& pre, const NttScale& post, int batch, cudaStream_t st);
// one transform split across devices in contiguous natural-order slices, exchanges fused into the passes (ntt.cu)
int ntt_run_sharded(NttPlan* const* plans, int ndev, const int* dev_ids, const Fr* const* src, Fr* const* tmp, Fr* const* dst, uint32_t log_n, const Fr& omega,
                    const NttScale& pre, const NttScale& post, uint64_t n_in, cudaStream_t* st, cudaEvent_t* ev);

}  // namespace b200
