// msm_affine.cu — EXPERIMENT, not part of libezkl_b200.so: kernels and orchestration of the fused batched-affine bucket accumulation
// (see msm_affine.cuh).  Per MSM call: one producer pass, then per round one fused consumer/producer kernel and one small inversion
// kernel, then the hand-over to the XYZZ combine / reduce tail.  Wired into msm_run at commit e30e8c9 it is bit-exact and was measured
// slower than the XYZZ chain; the host bodies stay under test through the debug library.
#include <vector>
#include "../../ezkl_b200/csrc/msm.cuh"
#include "msm_affine.cuh"

namespace b200 {

// warp-wide products of one Fq per lane: `others` = product of the other 31 lanes' values, `total` = product of all 32.
// Two Kogge-Stone scans (prefix and suffix), 12 multiplications per lane.
DEV Fq shfl_fq(const Fq& v, int delta, int mode) {
    Fq r;
#pragma unroll
    for (int i = 0; i < 8; ++i)
        r.l[i] = mode == 0 ? __shfl_up_sync(0xffffffffu, v.l[i], delta) : (mode == 1 ? __shfl_down_sync(0xffffffffu, v.l[i], delta) : __shfl_sync(0xffffffffu, v.l[i], delta));
    return r;
}
DEV void warp_products(const Fq& mine, Fq* others, Fq* total) {
    const int lane = threadIdx.x & 31;
    Fq pre = mine, suf = mine;
#pragma unroll 1
    for (int d = 1; d < 32; d <<= 1) {
        const Fq t = shfl_fq(pre, d, 0), u = shfl_fq(suf, d, 1);
        if (lane >= d) pre = pre * t;
        if (lane + d < 32) suf = suf * u;
    }
    Fq pre_ex = shfl_fq(pre, 1, 0), suf_ex = shfl_fq(suf, 1, 1);
    if (lane == 0) pre_ex = fp_one<FqTag>();
    if (lane == 31) suf_ex = fp_one<FqTag>();
    *others = pre_ex * suf_ex;
    *total = shfl_fq(pre, 31, 2);
}

__global__ void __launch_bounds__(128) k_aff_first(const AffineArgs a, uint64_t total_threads) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;          // the grid covers whole warps
    const Fq mine = g < total_threads ? aff_first_pass(a, g) : fp_one<FqTag>();
    Fq others, total;
    warp_products(mine, &others, &total);
    if (g < total_threads) a.thr_aux[g] = others;
    if ((threadIdx.x & 31) == 0 && g < total_threads) a.warp_prod[g >> 5] = total;
}
__global__ void __launch_bounds__(128) k_aff_round(const AffineArgs a, uint64_t total_threads) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    Fq mine = fp_one<FqTag>();
    if (g < total_threads) mine = aff_round(a, g, a.warp_prod[g >> 5] * a.thr_aux[g]);
    if (a.last_round) return;
    __syncwarp();
    Fq others, total;
    warp_products(mine, &others, &total);
    // the warp's inverse for THIS round has been read by every lane above (program order within the warp), so the slots are reused
    if (g < total_threads) a.thr_aux[g] = others;
    if ((threadIdx.x & 31) == 0 && g < total_threads) a.warp_prod[g >> 5] = total;
}
// one Fermat inversion per warp total; idle warps hold 1 and skip it.  32-thread CTAs spread the chains over all SMs.
__global__ void __launch_bounds__(32) k_aff_invert(Fq* vals, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fq v = vals[i];
    if (!fp_eq(v, fp_one<FqTag>())) vals[i] = fp_inv(v);
}
// chunk sums for the downstream combine / reduce kernels: XYZZ view of each chunk's final affine point
__global__ void __launch_bounds__(128) k_aff_finish(const AffineArgs a, G1Xyzz* __restrict__ chunk_sums, uint64_t total) {
    const uint64_t gidx = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gidx >= total) return;
    const uint64_t col = gidx / a.chunk_stride;
    const uint32_t t = (uint32_t)(gidx % a.chunk_stride);
    const uint32_t nchunks = a.chunk_offs[col * (a.nbuckets + 1) + a.nbuckets];
    if (t >= nchunks) return;
    const uint32_t ch = a.order[col * a.chunk_stride + t];
    const uint32_t start = a.chunk_start[col * a.chunk_stride + ch], L = a.chunk_len[col * a.chunk_stride + ch];
    const uint32_t r = aff_rounds_of(L);
    G1Affine p;
    if (r == 0) {
        const uint32_t e = a.ents[col * a.ent_stride + start];
        p = a.table[e & 0x7fffffffu];
        if (e >> 31) p = g1_neg(p);
    } else p = a.pb[(r - 1) & 1][col * a.ent_stride + start];
    chunk_sums[col * a.chunk_stride + ch] = g1_to_xyzz(p);
}

static uint32_t aff_threads_per_col(size_t chunk_stride) { return (uint32_t)(((chunk_stride + AFF_CPT - 1) / AFF_CPT + 31) & ~(size_t)31); }

size_t msm_affine_workspace_bytes(size_t batch, size_t ent_stride, size_t chunk_stride) {
    const size_t tt = batch * aff_threads_per_col(chunk_stride);
    return 2 * batch * (ent_stride + 2) * sizeof(G1Affine) + (tt + tt / 32 + 8) * sizeof(Fq);
}

int msm_accumulate_affine(const MsmTable& t, const uint32_t* ents, size_t ent_stride, const uint32_t* chunk_start, const uint32_t* chunk_len,
                          const uint32_t* order, size_t chunk_stride, const uint32_t* chunk_offs, uint32_t nbuckets, uint32_t cap, int batch,
                          G1Xyzz* chunk_sums, DevBuf& scratch, cudaStream_t st) {
    if (scratch.ensure(msm_affine_workspace_bytes(batch, ent_stride, chunk_stride))) return -2;
    AffineArgs a;
    a.table = t.d_table; a.ents = ents; a.chunk_start = chunk_start; a.chunk_len = chunk_len; a.order = order; a.chunk_offs = chunk_offs;
    a.pb[0] = scratch.as<G1Affine>();
    a.pb[1] = a.pb[0] + (size_t)batch * ent_stride + 2;          // +2: parked products may round up past the last chunk's region by one slot
    a.threads_per_col = aff_threads_per_col(chunk_stride);
    const uint64_t tt = (uint64_t)batch * a.threads_per_col;
    a.thr_aux = reinterpret_cast<Fq*>(a.pb[1] + (size_t)batch * ent_stride + 2);
    a.warp_prod = a.thr_aux + tt;
    a.ent_stride = ent_stride; a.chunk_stride = chunk_stride; a.nbuckets = nbuckets; a.batch = (uint32_t)batch;
    uint32_t rounds = 0;
    while ((1u << rounds) < cap) ++rounds;
    const unsigned blocks = div_up(tt, 128);
    a.round = 0; a.last_round = 0;
    if (rounds > 0) {
        k_aff_first<<<blocks, 128, 0, st>>>(a, tt);
        for (uint32_t r = 0; r < rounds; ++r) {
            k_aff_invert<<<div_up(tt / 32, 32), 32, 0, st>>>(a.warp_prod, tt / 32);
            a.round = r; a.last_round = r + 1 == rounds;
            k_aff_round<<<blocks, 128, 0, st>>>(a, tt);
        }
    }
    k_aff_finish<<<div_up((uint64_t)batch * chunk_stride, 128), 128, 0, st>>>(a, chunk_sums, (uint64_t)batch * chunk_stride);
    B200_CUDA(cudaGetLastError());
    return 0;
}
int msm_affine_launches(uint32_t cap) {      // kernels msm_accumulate_affine launches
    uint32_t rounds = 0;
    while ((1u << rounds) < cap) ++rounds;
    return (int)(2 * rounds + 2);
}

// ---- CPU run of the same bodies on host arrays (single column, identity order): tests/test_host_logic.py -------------
int msm_affine_host_chunks(const G1Affine* table, const uint32_t* ents, size_t n_ents, const uint32_t* chunk_start, const uint32_t* chunk_len,
                           size_t nchunks, G1Affine* out) {
    std::vector<uint32_t> order(nchunks), offs(1, (uint32_t)nchunks);
    uint32_t cap = 1;
    for (size_t i = 0; i < nchunks; ++i) { order[i] = (uint32_t)i; if (chunk_len[i] > cap) cap = chunk_len[i]; }
    std::vector<G1Affine> pba(n_ents + 2), pbb(n_ents + 2);
    AffineArgs a;
    a.table = table; a.ents = ents; a.chunk_start = chunk_start; a.chunk_len = chunk_len; a.order = order.data(); a.chunk_offs = offs.data();
    a.pb[0] = pba.data(); a.pb[1] = pbb.data();
    a.ent_stride = n_ents; a.chunk_stride = nchunks; a.nbuckets = 0; a.batch = 1;
    a.threads_per_col = aff_threads_per_col(nchunks);
    const uint64_t tt = a.threads_per_col;
    std::vector<Fq> prod(tt), inv(tt);
    uint32_t rounds = 0;
    while ((1u << rounds) < cap) ++rounds;
    a.round = 0; a.last_round = 0;
    for (uint64_t g = 0; g < tt; ++g) prod[g] = aff_first_pass(a, g);
    for (uint32_t r = 0; r < rounds; ++r) {
        // the warp scans + Fermat inversion of the device path amount to: every thread receives the inverse of its own total
        for (uint64_t g = 0; g < tt; ++g) inv[g] = fp_inv(prod[g]);
        a.round = r; a.last_round = r + 1 == rounds;
        for (uint64_t g = 0; g < tt; ++g) prod[g] = aff_round(a, g, inv[g]);
    }
    for (size_t i = 0; i < nchunks; ++i) {
        const uint32_t rr = aff_rounds_of(chunk_len[i]);
        if (rr == 0) { a.round = 0; out[i] = aff_table_point(a, 0, chunk_start[i]); }
        else out[i] = a.pb[(rr - 1) & 1][chunk_start[i]];
    }
    return 0;
}

}  // namespace b200
