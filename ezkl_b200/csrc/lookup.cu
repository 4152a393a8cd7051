// lookup.cu — mv-lookup multiplicities m(X) on the device (halo2 plonk/mv_lookup/prover.rs, stage 2 of create_proof, SURVEY.md
// §3.1 / §8 f2; ezkl's static lookups, range checks, dynamic lookups and shuffles all go through it:
// /root/reference/src/circuit/ops/chip.rs:496,662,782,870).
//
// The CPU prover builds a BTreeMap {table value -> row} and bumps one counter per input cell.  Here the map is an open-addressing
// hash table of row indices keyed by the 256-bit cell value (keys compared through the table column itself, so a slot is 4 bytes):
//   k_lk_build  inserts every table row; equal values keep the SMALLEST row (atomicMin), which makes the result deterministic,
//   k_lk_count  probes with every input cell and bumps the row's counter (warp-aggregated when a warp hits one row),
//   k_lk_finish writes the counters as Montgomery field elements.
// Which duplicate row receives the count does not affect soundness (the logUp identity only sums m / (t + beta) over equal t);
// "first row" is this library's rule (SURVEY.md Appendix F.6 lists the upstream rule as an open question).
#include "poly.cuh"

namespace b200 {

static constexpr uint32_t LK_EMPTY = 0xffffffffu;

DEV uint32_t lk_hash(const Fr& v) {
    uint32_t h = v.l[0] ^ (v.l[1] * 0x9e3779b1u) ^ (v.l[3] * 0x85ebca6bu) ^ (v.l[6] * 0xc2b2ae35u);
    h ^= h >> 16; h *= 0x7feb352du; h ^= h >> 15; h *= 0x846ca68bu; h ^= h >> 16;
    return h;
}

__global__ void __launch_bounds__(256) k_lk_build(const Fr* __restrict__ table, uint32_t n, uint32_t* __restrict__ slots, uint32_t mask) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fr key = fp_load(table + i);
    uint32_t h = lk_hash(key) & mask;
    for (;;) {
        uint32_t cur = slots[h];
        if (cur == LK_EMPTY) {
            cur = atomicCAS(&slots[h], LK_EMPTY, i);
            if (cur == LK_EMPTY) return;
        }
        if (fp_eq(fp_load(table + cur), key)) { atomicMin(&slots[h], i); return; }      // any row stored here holds this value
        h = (h + 1) & mask;
    }
}
__global__ void __launch_bounds__(256) k_lk_count(const Fr* __restrict__ table, const uint32_t* __restrict__ slots, uint32_t mask, const Fr* const* __restrict__ inputs,
                                                   uint32_t n_rows, uint32_t* __restrict__ counts, unsigned long long* __restrict__ missing) {
    const Fr* in = inputs[blockIdx.y];
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += gridDim.x * blockDim.x) {
        const Fr key = fp_load(in + r);
        uint32_t h = lk_hash(key) & mask, row = LK_EMPTY;
        for (;;) {
            const uint32_t cur = slots[h];
            if (cur == LK_EMPTY) break;
            if (fp_eq(fp_load(table + cur), key)) { row = cur; break; }
            h = (h + 1) & mask;
        }
        if (row == LK_EMPTY) { atomicAdd(missing, 1ull); continue; }
        // ezkl inputs are full of repeated values (padding rows, saturated activations): one atomic per distinct row per warp
        const unsigned act = __activemask();
        const unsigned peers = __match_any_sync(act, row);
        if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&counts[row], (uint32_t)__popc(peers));
    }
}
__global__ void __launch_bounds__(256) k_lk_finish(const uint32_t* __restrict__ counts, uint32_t n, Fr* __restrict__ m) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr c = fp_zero<FrTag>();
    c.l[0] = counts[i];
    fp_store(m + i, counts[i] ? fp_to_mont(c) : c);
}

// scratch layout: [slots 2^s][counts n_table][missing u64]
int lookup_multiplicities_run(const Fr* d_table, size_t n_table, const Fr* const* h_inputs, size_t n_inputs, size_t n_rows, Fr* d_m, DevBuf& scratch, StagingRing& ring,
                              unsigned long long** d_missing_out, cudaStream_t st) {
    B200_CHECK(n_table >= 1 && n_table < (1u << 30) && n_rows < (1u << 31) && n_inputs >= 1 && n_inputs <= 65535, -1, "lookup_multiplicities: sizes out of range");
    const void* staged;
    if (int rc = ring.push(h_inputs, sizeof(void*) * n_inputs, st, &staged)) return rc;
    const Fr* const* d_inputs = reinterpret_cast<const Fr* const*>(staged);
    uint32_t cap = 64;
    while (cap < 2 * n_table) cap <<= 1;
    const size_t bytes = sizeof(uint32_t) * ((size_t)cap + n_table) + 16;
    if (scratch.ensure(bytes)) return -2;
    uint32_t* slots = scratch.as<uint32_t>();
    uint32_t* counts = slots + cap;
    unsigned long long* missing = reinterpret_cast<unsigned long long*>(scratch.as<uint8_t>() + ((sizeof(uint32_t) * ((size_t)cap + n_table) + 7) & ~(size_t)7));
    B200_CUDA(cudaMemsetAsync(slots, 0xff, sizeof(uint32_t) * cap, st));
    B200_CUDA(cudaMemsetAsync(counts, 0, sizeof(uint32_t) * n_table + 16, st));
    k_lk_build<<<div_up(n_table, 256), 256, 0, st>>>(d_table, (uint32_t)n_table, slots, cap - 1); count_launch();
    if (n_rows) {
        const unsigned gmax = (unsigned)sm_count() * 8u;
        const unsigned gx = div_up(n_rows, 256) > gmax ? gmax : div_up(n_rows, 256);
        k_lk_count<<<dim3(gx, (unsigned)n_inputs), 256, 0, st>>>(d_table, slots, cap - 1, d_inputs, (uint32_t)n_rows, counts, missing); count_launch();
    }
    k_lk_finish<<<div_up(n_table, 256), 256, 0, st>>>(counts, (uint32_t)n_table, d_m); count_launch();
    B200_CUDA(cudaGetLastError());
    *d_missing_out = missing;
    return 0;
}

}  // namespace b200
