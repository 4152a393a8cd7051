// msm.cu — BN254 G1 multi-scalar multiplication for sm_90a (Pippenger buckets over a window-precomputed table).
//
// Replaces halo2_proofs arithmetic.rs best_multiexp / ParamsKZG::{commit, commit_lagrange} (UPSTREAM; in-tree
// callers /root/reference/src/circuit/modules/polycommit.rs:71 and create_proof at src/pfsys/mod.rs:456).
// The result is exact group arithmetic, so after normalisation it is bit-identical to the CPU prover's point.
//
// Pipeline for a batch of `batch` scalar columns sharing one base table (grid.y = column):
//   1 k_digits<false>   scalar -> canonical -> W signed c-bit digits; per-bucket histogram (warp-aggregated REDs)
//                       (<= 2^15 buckets: k_digits_tile<false> with shared counters per tile of scalars + k_tile_prefix)
//   2 k_scan_buckets    exclusive scan of bucket sizes; splits every bucket into chunks of <= cap entries
//   3 k_digits<true>    same recoding, scatters (table index | sign) into bucket-sorted order  (or k_digits_tile<true>)
//   4 k_fill_chunks     chunk table + histogram of chunk lengths;  5 k_len_offsets;  6 k_order_chunks
//                       (counting sort of chunks by length, longest first => every warp runs equal-length loops)
//   7 k_accumulate      one thread per chunk: XYZZ += affine table entry (8M+2S), next base prefetched
//   8 k_combine / 9 k_combine_heavy   chunk sums -> bucket sums
//  10 k_reduce          sum_b (b+1) * B_b by per-thread running sums + small-multiple fix-up + block tree
//  11 k_final           per-column sum of the block partials -> one XYZZ point per column
//  12 k_subwindow_fold  only for a reduced table (s > 1 windows per level): 10 and 11 run on the s bucket sets of a column as
//                       s virtual columns; this Horner chain folds their s results into the column's point
// HBM traffic per (scalar, base) pair: 32 B scalar (read twice) + W x 64 B table gathers; the kernel is bound by
// integer issue (IMAD.WIDE), not HBM — see DESIGN.md §kernels.
#include "msm.cuh"
#include "ec_coop.cuh"

namespace b200 {

int msm_default_window(size_t n) {
    int k = 0;
    while (((size_t)1 << (k + 1)) <= n) ++k;
    int c = k <= 10 ? 8 : (k <= 13 ? k - 2 : (k <= 17 ? k - 1 : (k <= 19 ? 17 : (k <= 21 ? 18 : 20))));
    if (c < 4) c = 4;
    if (c > 22) c = 22;
    return c;
}

// ---------------------------------------------------------------------------------------------------------
// table precomputation
__global__ void __launch_bounds__(128) k_table_next_level(const G1Affine* __restrict__ prev, G1Affine* __restrict__ next, size_t n, int c) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    G1Affine p = prev[i];
    G1Xyzz a = g1_dbl_affine(p);
#pragma unroll 1
    for (int j = 1; j < c; ++j) a = g1_dbl(a);
    next[i] = g1_to_affine(a);
}

int msm_table_alloc(MsmTable* t, size_t n, int c, size_t max_table_bytes) {
    B200_CHECK(n > 0, -1, "msm_table_build: empty base vector");
    if (c <= 0) c = msm_default_window(n);
    int W = (255 + c - 1) / c, s = 1, L = W;
    msm_pick_levels(n, c, max_table_bytes, &s, &L);
    B200_CHECK((size_t)L * n < ((size_t)1 << 31), -1, "msm_table_build: L*n = %zu exceeds the 31-bit entry index", (size_t)L * n);
    t->n = n; t->c = c; t->W = W; t->s = s; t->L = L;
    B200_CUDA(cudaGetDevice(&t->device));
    const cudaError_t e = cudaMalloc(&t->d_table, t->bytes());
    if (e != cudaSuccess) {
        cudaGetLastError();          // an allocation failure must not surface in a later launch check
        t->d_table = nullptr;
        set_error("msm_table_build: %zu MiB table (%d levels of %zu points): %s", t->bytes() >> 20, L, n, cudaGetErrorString(e));
        return -2;
    }
    return 0;
}

int msm_table_build(MsmTable* t, const G1Affine* d_bases, cudaStream_t st) {
    const size_t n = t->n;
    if (d_bases) B200_CUDA(cudaMemcpyAsync(t->d_table, d_bases, sizeof(G1Affine) * n, cudaMemcpyDeviceToDevice, st));
    for (int j = 1; j < t->L; ++j) {
        k_table_next_level<<<div_up(n, 128), 128, 0, st>>>(t->d_table + (size_t)(j - 1) * n, t->d_table + (size_t)j * n, n, t->c * t->s); count_launch();
    }
    B200_CUDA(cudaGetLastError());
    return 0;
}
void msm_table_free(MsmTable* t) {
    if (t->d_table) cudaFree(t->d_table);
    t->d_table = nullptr;
}

// ---------------------------------------------------------------------------------------------------------
// 1 / 3: digit extraction, histogram and scatter with global atomics, for bucket sets too large for k_digits_tile.  SUBWIN (s > 1 windows per table level): window w reads level j = w / s and
// counts into bucket set r = w % s, i.e. bucket r * 2^(c-1) + |d| - 1; without it j = w, r = 0 (the full table).
template <bool SCATTER, bool SUBWIN>
__global__ void __launch_bounds__(256) k_digits(const Fr* __restrict__ scalars, size_t stride, uint32_t n, uint32_t table_n, uint32_t base_off, int c, int W,
                                                 uint32_t nbuckets, uint32_t* __restrict__ counters /*[col][nbuckets]*/,
                                                 const uint32_t* __restrict__ offs /*[col][nbuckets+1]*/, uint32_t* __restrict__ ents, size_t ent_stride,
                                                 const uint32_t* __restrict__ skew, int wpl) {
    const uint32_t col = blockIdx.y;
    const bool aggregate = !SCATTER || skew[col] != 0;        // the counting pass cannot know yet; the scatter pass can
    const Fr* sc = scalars + (size_t)col * stride;
    uint32_t* cnt = counters + (size_t)col * nbuckets;
    const uint32_t* off = SCATTER ? offs + (size_t)col * (nbuckets + 1) : nullptr;
    uint32_t* ent = SCATTER ? ents + (size_t)col * ent_stride : nullptr;
    const unsigned lane = threadIdx.x & 31;
    const uint32_t n_up = (n + 31u) & ~31u;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_up; i += gridDim.x * blockDim.x) {
        const bool valid = i < n;
        Fr s = fp_zero<FrTag>();
        if (valid) s = fp_from_mont(fp_load(sc + i));
        uint32_t carry = 0;
        MsmWindowSlot slot;
#pragma unroll 1
        for (int w = 0; w < W; ++w) {
            int32_t d = msm_next_digit(s.l, c, &carry);
            const uint32_t j = SUBWIN ? slot.level : (uint32_t)w;
            const bool nz = d != 0;     // invalid lanes carry s = 0 -> all digits 0
            const unsigned act = __ballot_sync(0xffffffffu, nz);
            if (nz && !aggregate) {
                const uint32_t bucket = (SUBWIN ? slot.set_off : 0u) + (uint32_t)(d < 0 ? -d : d) - 1u;
                ent[off[bucket] + atomicAdd(&cnt[bucket], 1u)] = (j * table_n + base_off + i) | (d < 0 ? 0x80000000u : 0u);
            } else if (nz) {
                const uint32_t bucket = (SUBWIN ? slot.set_off : 0u) + (uint32_t)(d < 0 ? -d : d) - 1u;
                const unsigned peers = __match_any_sync(act, bucket);
                const int leader = __ffs(peers) - 1;
                uint32_t base = 0;
                if ((int)lane == leader) base = atomicAdd(&cnt[bucket], (uint32_t)__popc(peers));
                if (SCATTER) {
                    base = __shfl_sync(peers, base, leader);
                    const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
                    ent[off[bucket] + base + rank] = (j * table_n + base_off + i) | (d < 0 ? 0x80000000u : 0u);
                }
            }
            if (SUBWIN) slot.next(c, wpl);
        }
    }
}

// 1 / 3 with the counters in shared memory (msm_pick_recode: nb <= MSM_TILE_MAX_BUCKETS).  CTA (x, col) recodes its tile of `tile`
// scalars with one shared counter per bucket.  Counting pass: count, then write the tile's counts to tile_counts[col][x][.].
// Placement pass: start each counter at offs[b] + (entries of bucket b in the column's earlier tiles), which k_tile_prefix left in
// tile_counts, and place every entry at its counter's old value.  No global atomics; the entry encoding is k_digits'.
template <bool SCATTER, bool SUBWIN>
__global__ void __launch_bounds__(MSM_TILE_THREADS, 1) k_digits_tile(const Fr* __restrict__ scalars, size_t stride, uint32_t n, uint32_t table_n, uint32_t base_off,
                                                                     int c, int W, uint32_t nbuckets, uint32_t tile, uint32_t* __restrict__ tile_counts /*[col][tiles][nbuckets]*/,
                                                                     const uint32_t* __restrict__ offs /*[col][nbuckets+1]*/, uint32_t* __restrict__ ents, size_t ent_stride, int wpl) {
    extern __shared__ uint32_t sh_cnt[];    // nbuckets
    const uint32_t col = blockIdx.y;
    const Fr* sc = scalars + (size_t)col * stride;
    uint32_t* tc = tile_counts + ((size_t)col * gridDim.x + blockIdx.x) * nbuckets;
    if (SCATTER) {
        const uint32_t* off = offs + (size_t)col * (nbuckets + 1);
        for (uint32_t b = threadIdx.x; b < nbuckets; b += blockDim.x) sh_cnt[b] = off[b] + tc[b];
    } else {
        for (uint32_t b = threadIdx.x; b < nbuckets; b += blockDim.x) sh_cnt[b] = 0;
    }
    __syncthreads();
    uint32_t* ent = SCATTER ? ents + (size_t)col * ent_stride : nullptr;
    const uint32_t lo = blockIdx.x * tile, hi = min(lo + tile, n);
    for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        Fr s = fp_from_mont(fp_load(sc + i));
        uint32_t carry = 0;
        MsmWindowSlot slot;
#pragma unroll 1
        for (int w = 0; w < W; ++w) {
            const int32_t d = msm_next_digit(s.l, c, &carry);
            if (d != 0) {
                const uint32_t bucket = (SUBWIN ? slot.set_off : 0u) + (uint32_t)(d < 0 ? -d : d) - 1u;
                const uint32_t pos = atomicAdd(&sh_cnt[bucket], 1u);
                if (SCATTER) ent[pos] = ((SUBWIN ? slot.level : (uint32_t)w) * table_n + base_off + i) | (d < 0 ? 0x80000000u : 0u);
            }
            if (SUBWIN) slot.next(c, wpl);
        }
    }
    if (!SCATTER) {
        __syncthreads();
        for (uint32_t b = threadIdx.x; b < nbuckets; b += blockDim.x) tc[b] = sh_cnt[b];
    }
}

// 1b (shared-counter path): per bucket, the exclusive prefix of the tile counts over the column's tiles, in place, and the column's
// total into hist[col][b], which is what k_scan_buckets reads.  Consecutive threads take consecutive buckets (coalesced rows).
__global__ void __launch_bounds__(256) k_tile_prefix(uint32_t* __restrict__ tile_counts, uint32_t tiles, uint32_t nbuckets, uint32_t* __restrict__ hist) {
    const uint32_t col = blockIdx.y;
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nbuckets) return;
    uint32_t* tc = tile_counts + (size_t)col * tiles * nbuckets + b;
    uint32_t acc = 0;
    for (uint32_t t0 = 0; t0 < tiles; t0 += 8) {
        uint32_t v[8];              // eight loads in flight before the stores, which the compiler may not move them past
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = t0 + j < tiles ? tc[(size_t)(t0 + j) * nbuckets] : 0u;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (t0 + j < tiles) tc[(size_t)(t0 + j) * nbuckets] = acc;
            acc += v[j];
        }
    }
    hist[(size_t)col * nbuckets + b] = acc;
}

// 2: one block per column. offs = exclusive scan of counts; chunk_offs = exclusive scan of ceil(count / cap).
__global__ void __launch_bounds__(1024) k_scan_buckets(const uint32_t* __restrict__ counts, uint32_t* __restrict__ offs, uint32_t* __restrict__ chunk_offs,
                                                        uint32_t nbuckets, uint32_t cap, uint32_t* __restrict__ skew /*[col]*/) {
    __shared__ uint32_t sh_max;
    if (threadIdx.x == 0) sh_max = 0;
    __syncthreads();
    const uint32_t col = blockIdx.x;
    const uint32_t lc = 31u - (uint32_t)__clz(cap);            // cap is a power of two (msm_pick_cap)
    const uint32_t* cnt = counts + (size_t)col * nbuckets;
    uint32_t* off = offs + (size_t)col * (nbuckets + 1);
    uint32_t* coff = chunk_offs + (size_t)col * (nbuckets + 1);
    const uint32_t ipt = (nbuckets + blockDim.x - 1) / blockDim.x;
    const uint32_t lo = threadIdx.x * ipt, hi = min(lo + ipt, nbuckets);
    uint32_t s = 0, cs = 0;
    uint32_t mx = 0;
    // a thread's buckets are consecutive: 128-bit loads (independent, so they pipeline) when its run is a multiple of four
    const bool vec = (ipt & 3u) == 0 && lo + ipt <= nbuckets;
    if (vec) {
        const uint4* c4 = reinterpret_cast<const uint4*>(cnt + lo);
#pragma unroll 4
        for (uint32_t q = 0; q < (ipt >> 2); ++q) {
            const uint4 v = c4[q];
            s += v.x + v.y + v.z + v.w;
            cs += ((v.x + cap - 1) >> lc) + ((v.y + cap - 1) >> lc) + ((v.z + cap - 1) >> lc) + ((v.w + cap - 1) >> lc);
            mx = max(max(mx, v.x), max(max(v.y, v.z), v.w));
        }
    } else {
        for (uint32_t b = lo; b < hi; ++b) { uint32_t v = cnt[b]; s += v; cs += ((v + cap - 1) >> lc); mx = max(mx, v); }
    }
    if (mx) atomicMax(&sh_max, mx);
    uint32_t tot, ctot;
    uint32_t ex = block_exclusive_scan(s, &tot);
    uint32_t cex = block_exclusive_scan(cs, &ctot);
    if (vec) {
        const uint4* c4 = reinterpret_cast<const uint4*>(cnt + lo);
#pragma unroll 4
        for (uint32_t q = 0; q < (ipt >> 2); ++q) {
            const uint4 v = c4[q];
            const uint32_t b = lo + 4 * q;
            off[b] = ex; coff[b] = cex; ex += v.x; cex += ((v.x + cap - 1) >> lc);
            off[b + 1] = ex; coff[b + 1] = cex; ex += v.y; cex += ((v.y + cap - 1) >> lc);
            off[b + 2] = ex; coff[b + 2] = cex; ex += v.z; cex += ((v.z + cap - 1) >> lc);
            off[b + 3] = ex; coff[b + 3] = cex; ex += v.w; cex += ((v.w + cap - 1) >> lc);
        }
    } else {
        for (uint32_t b = lo; b < hi; ++b) { uint32_t v = cnt[b]; off[b] = ex; coff[b] = cex; ex += v; cex += ((v + cap - 1) >> lc); }
    }
    if (threadIdx.x == 0) {
        off[nbuckets] = tot; coff[nbuckets] = ctot;
        // a column is "skewed" when some bucket holds far more than its share: only then is warp-level aggregation of the
        // scatter atomics worth its MATCH / SHFL cost (uniform scalars almost never collide inside a warp)
        skew[col] = sh_max > 16u * (tot / nbuckets + 1u) ? 1u : 0u;
    }
}

// 4: chunk table (start, len) + histogram of lengths + list of heavy buckets
__global__ void __launch_bounds__(256) k_fill_chunks(const uint32_t* __restrict__ offs, const uint32_t* __restrict__ chunk_offs, uint32_t nbuckets, uint32_t cap,
                                                      uint32_t* __restrict__ chunk_start, uint32_t* __restrict__ chunk_len, size_t chunk_stride,
                                                      uint32_t* __restrict__ len_hist /*[col][cap+1]*/, uint32_t* __restrict__ heavy /*[col][1+max_heavy]*/, uint32_t heavy_stride) {
    extern __shared__ uint32_t sh_hist[];   // cap + 1
    const uint32_t col = blockIdx.y;
    for (uint32_t j = threadIdx.x; j <= cap; j += blockDim.x) sh_hist[j] = 0;
    __syncthreads();
    const uint32_t* off = offs + (size_t)col * (nbuckets + 1);
    const uint32_t* coff = chunk_offs + (size_t)col * (nbuckets + 1);
    uint32_t* cs = chunk_start + (size_t)col * chunk_stride;
    uint32_t* cl = chunk_len + (size_t)col * chunk_stride;
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < nbuckets) {
        const uint32_t start = off[b], size = off[b + 1] - start, c0 = coff[b], nch = coff[b + 1] - c0;
        for (uint32_t j = 0; j < nch; ++j) {
            const uint32_t len = min(cap, size - j * cap);
            cs[c0 + j] = start + j * cap;
            cl[c0 + j] = len;
            if (j + 1 == nch) atomicAdd(&sh_hist[len], 1u);
        }
        if (nch > 1) atomicAdd(&sh_hist[cap], nch - 1);
        if (nch > (uint32_t)HEAVY_CHUNKS) {
            uint32_t* hv = heavy + (size_t)col * heavy_stride;
            uint32_t slot = atomicAdd(&hv[0], 1u);
            if (slot + 1 < heavy_stride) hv[1 + slot] = b;
        }
    }
    __syncthreads();
    uint32_t* gh = len_hist + (size_t)col * (cap + 1);
    for (uint32_t j = threadIdx.x; j <= cap; j += blockDim.x) if (sh_hist[j]) atomicAdd(&gh[j], sh_hist[j]);
}

// 5: descending-length start offsets: len_offs[l] = #chunks with length > l
__global__ void k_len_offsets(const uint32_t* __restrict__ len_hist, uint32_t* __restrict__ len_offs, uint32_t cap) {
    const uint32_t col = blockIdx.x;
    if (threadIdx.x != 0) return;
    const uint32_t* h = len_hist + (size_t)col * (cap + 1);
    uint32_t* o = len_offs + (size_t)col * (cap + 1);
    uint32_t acc = 0;
    for (int l = (int)cap; l >= 0; --l) { o[l] = acc; acc += h[l]; }
}

// 6: order[pos] = chunk id, longest chunks first
__global__ void __launch_bounds__(256) k_order_chunks(const uint32_t* __restrict__ chunk_len, size_t chunk_stride, const uint32_t* __restrict__ chunk_offs, uint32_t nbuckets,
                                                       const uint32_t* __restrict__ len_offs, uint32_t* __restrict__ len_cursor, uint32_t cap, uint32_t* __restrict__ order) {
    const uint32_t col = blockIdx.y;
    const uint32_t nchunks = chunk_offs[(size_t)col * (nbuckets + 1) + nbuckets];
    const uint32_t* cl = chunk_len + (size_t)col * chunk_stride;
    uint32_t* ord = order + (size_t)col * chunk_stride;
    const uint32_t* lo = len_offs + (size_t)col * (cap + 1);
    uint32_t* lc = len_cursor + (size_t)col * (cap + 1);
    const unsigned lane = threadIdx.x & 31;
    const uint32_t n_up = (nchunks + 31u) & ~31u;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_up; i += gridDim.x * blockDim.x) {
        const bool valid = i < nchunks;
        const uint32_t len = valid ? cl[i] : 0;
        const unsigned act = __ballot_sync(0xffffffffu, valid);
        if (valid) {
            const unsigned peers = __match_any_sync(act, len);
            const int leader = __ffs(peers) - 1;
            uint32_t base = 0;
            if ((int)lane == leader) base = atomicAdd(&lc[len], (uint32_t)__popc(peers));
            base = __shfl_sync(peers, base, leader);
            ord[lo[len] + base + __popc(peers & ((1u << lane) - 1u))] = i;
        }
    }
}

// 7: the hot kernel. One thread per chunk (<= cap entries of one bucket).
DEV G1Affine load_base(const G1Affine* __restrict__ table, uint32_t e) {
    const uint4* q = reinterpret_cast<const uint4*>(table + (e & 0x7fffffffu));
    uint4 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2), d = __ldg(q + 3);
    G1Affine p;
    p.x.l[0] = a.x; p.x.l[1] = a.y; p.x.l[2] = a.z; p.x.l[3] = a.w; p.x.l[4] = b.x; p.x.l[5] = b.y; p.x.l[6] = b.z; p.x.l[7] = b.w;
    p.y.l[0] = c.x; p.y.l[1] = c.y; p.y.l[2] = c.z; p.y.l[3] = c.w; p.y.l[4] = d.x; p.y.l[5] = d.y; p.y.l[6] = d.z; p.y.l[7] = d.w;
    return p;
}
__global__ void __launch_bounds__(128, 4) k_accumulate(const G1Affine* __restrict__ table, const uint32_t* __restrict__ ents, size_t ent_stride,
                                                        const uint32_t* __restrict__ chunk_start, const uint32_t* __restrict__ chunk_len, const uint32_t* __restrict__ order,
                                                        size_t chunk_stride, const uint32_t* __restrict__ chunk_offs, uint32_t nbuckets, G1Xyzz* __restrict__ chunk_sums) {
    const uint32_t col = blockIdx.y;
    const uint32_t nchunks = chunk_offs[(size_t)col * (nbuckets + 1) + nbuckets];
    const uint32_t* ent = ents + (size_t)col * ent_stride;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < nchunks; t += gridDim.x * blockDim.x) {
        const uint32_t ch = order[(size_t)col * chunk_stride + t];
        const uint32_t start = chunk_start[(size_t)col * chunk_stride + ch], len = chunk_len[(size_t)col * chunk_stride + ch];
        uint32_t e = ent[start];
        G1Affine p = load_base(table, e);
        if (e >> 31) p = g1_neg(p);
        G1Xyzz acc = g1_to_xyzz(p);
        if (len > 1) {
            uint32_t e_next = ent[start + 1];
            G1Affine nx = load_base(table, e_next);
#pragma unroll 1
            for (uint32_t j = 1; j < len; ++j) {
                p = nx; e = e_next;
                if (j + 1 < len) { e_next = ent[start + j + 1]; nx = load_base(table, e_next); }
                if (e >> 31) p = g1_neg(p);
                acc = g1_add_mixed(acc, p);
            }
        }
        chunk_sums[(size_t)col * chunk_stride + ch] = acc;
    }
}

// block-wide sum of one XYZZ point per thread; result valid in thread 0. blockDim.x is a power of two <= TREE_THREADS.
DEV G1Xyzz block_sum(G1Xyzz v, G1Xyzz* sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
#pragma unroll 1
    for (unsigned s = blockDim.x / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) { v = g1_add(v, sh[threadIdx.x + s]); sh[threadIdx.x] = v; }
        __syncthreads();
    }
    return v;
}

// 8: bucket_sums[b] = sum of its chunk sums (light buckets)
__global__ void __launch_bounds__(128) k_combine(const uint32_t* __restrict__ chunk_offs, uint32_t nbuckets, const G1Xyzz* __restrict__ chunk_sums, size_t chunk_stride,
                                                  G1Xyzz* __restrict__ bucket_sums) {
    const uint32_t col = blockIdx.y;
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nbuckets) return;
    const uint32_t* coff = chunk_offs + (size_t)col * (nbuckets + 1);
    const uint32_t c0 = coff[b], nch = coff[b + 1] - c0;
    if (nch > (uint32_t)HEAVY_CHUNKS) return;
    const G1Xyzz* cs = chunk_sums + (size_t)col * chunk_stride;
    G1Xyzz acc = g1_xyzz_identity();
    if (nch > 0) acc = cs[c0];
#pragma unroll 1
    for (uint32_t j = 1; j < nch; ++j) acc = g1_add(acc, cs[c0 + j]);
    bucket_sums[(size_t)col * nbuckets + b] = acc;
}
// 9: heavy buckets: a block per bucket
__global__ void __launch_bounds__(TREE_THREADS) k_combine_heavy(const uint32_t* __restrict__ heavy, uint32_t heavy_stride, const uint32_t* __restrict__ chunk_offs, uint32_t nbuckets,
                                                                 const G1Xyzz* __restrict__ chunk_sums, size_t chunk_stride, G1Xyzz* __restrict__ bucket_sums) {
    __shared__ G1Xyzz sh[TREE_THREADS];
    const uint32_t col = blockIdx.y;
    const uint32_t* hv = heavy + (size_t)col * heavy_stride;
    const uint32_t nheavy = min(hv[0], heavy_stride - 1);
    const uint32_t* coff = chunk_offs + (size_t)col * (nbuckets + 1);
    const G1Xyzz* cs = chunk_sums + (size_t)col * chunk_stride;
    for (uint32_t h = blockIdx.x; h < nheavy; h += gridDim.x) {
        const uint32_t b = hv[1 + h];
        const uint32_t c0 = coff[b], nch = coff[b + 1] - c0;
        G1Xyzz acc = g1_xyzz_identity();
#pragma unroll 1
        for (uint32_t j = threadIdx.x; j < nch; j += TREE_THREADS) acc = g1_add(acc, cs[c0 + j]);
        acc = block_sum(acc, sh);
        if (threadIdx.x == 0) bucket_sums[(size_t)col * nbuckets + b] = acc;
        __syncthreads();
    }
}

// 10: sum_b (b+1) * B_b.  Thread t owns buckets [t*M, (t+1)*M): running sums give sum_j (j+1) B and S = sum B;
//     the block offset (t*M) * S is a small scalar multiple; then a block tree.
template <int MIN_CTAS>
__global__ void __launch_bounds__(TREE_THREADS, MIN_CTAS) k_reduce(const G1Xyzz* __restrict__ bucket_sums, uint32_t nbuckets, G1Xyzz* __restrict__ partials, uint32_t nparts, uint32_t per_thread) {
    __shared__ G1Xyzz sh[TREE_THREADS];
    const uint32_t col = blockIdx.y;
    const G1Xyzz* bs = bucket_sums + (size_t)col * nbuckets;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t lo = t * per_thread;
    G1Xyzz run = g1_xyzz_identity(), acc = g1_xyzz_identity();
    if (lo < nbuckets) {
        const uint32_t hi = min(lo + per_thread, nbuckets);
#pragma unroll 1
        for (uint32_t b = hi; b-- > lo;) {
            run = g1_add(run, bs[b]);
            acc = g1_add(acc, run);
        }
        if (lo > 0) acc = g1_add(acc, g1_mul_small(run, lo));
    }
    acc = block_sum(acc, sh);
    if (threadIdx.x == 0) partials[(size_t)col * nparts + blockIdx.x] = acc;
}
// 11: one block per column
__global__ void __launch_bounds__(TREE_THREADS) k_final(const G1Xyzz* __restrict__ partials, uint32_t nparts, G1Xyzz* __restrict__ out) {
    __shared__ G1Xyzz sh[TREE_THREADS];
    const uint32_t col = blockIdx.x;
    G1Xyzz acc = g1_xyzz_identity();
#pragma unroll 1
    for (uint32_t j = threadIdx.x; j < nparts; j += blockDim.x) acc = g1_add(acc, partials[(size_t)col * nparts + j]);
    acc = block_sum(acc, sh);
    if (threadIdx.x == 0) out[col] = acc;
}

// ---- four-lane cooperative variant of 11 (ec_coop.cuh) for g1_sum_run: a quad of lanes is one logical thread, a CTA holds COOP_LT of them ----
static constexpr int COOP_LT = TREE_THREADS / 4;
DEV G1Xyzz block_sum_coop(G1Xyzz v, G1Xyzz* sh) {
    const unsigned lt = threadIdx.x >> 2, q = threadIdx.x & 3;
    if (q == 0) sh[lt] = v;
    __syncthreads();
#pragma unroll 1
    for (unsigned s = COOP_LT / 2; s > 0; s >>= 1) {
        if (lt < s) { v = g1_add_coop4(v, sh[lt + s]); if (q == 0) sh[lt] = v; }
        __syncthreads();
    }
    return v;
}
__global__ void __launch_bounds__(TREE_THREADS) k_final_coop(const G1Xyzz* __restrict__ partials, uint32_t nparts, G1Xyzz* __restrict__ out) {
    __shared__ G1Xyzz sh[COOP_LT];
    const uint32_t col = blockIdx.x;
    G1Xyzz acc = g1_xyzz_identity();
#pragma unroll 1
    for (uint32_t j = threadIdx.x >> 2; j < nparts; j += COOP_LT) acc = g1_add_coop4(acc, partials[(size_t)col * nparts + j]);
    acc = block_sum_coop(acc, sh);
    if (threadIdx.x == 0) out[col] = acc;
}

// 12 (s > 1 windows per table level): per column, Horner over the s bucket-set results R_r (weight 2^(c*r)):
//    acc = R_(s-1);  acc = 2^c * acc + R_r for r = s-2 .. 0.   (s-1)*c doublings and s-1 additions per column.
__global__ void __launch_bounds__(32) k_subwindow_fold(const G1Xyzz* __restrict__ set_sums /*[col][s]*/, int s, int c, uint32_t batch, G1Xyzz* __restrict__ out) {
    const uint32_t col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= batch) return;
    const G1Xyzz* rs = set_sums + (size_t)col * s;
    G1Xyzz acc = rs[s - 1];
#pragma unroll 1
    for (int r = s - 2; r >= 0; --r) {
#pragma unroll 1
        for (int k = 0; k < c; ++k) acc = g1_dbl(acc);
        acc = g1_add(acc, rs[r]);
    }
    out[col] = acc;
}

// synthetic distinct bases for benchmarks / tests: out[i] = [h(seed, i)] * G, affine (G = (1, 2))
__global__ void __launch_bounds__(128) k_g1_generate(uint64_t seed, size_t n, G1Affine* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8];
    uint64_t z = seed + 0x9e3779b97f4a7c15ull * (uint64_t)(i + 1);
#pragma unroll
    for (int w = 0; w < 4; ++w) {
        z += 0x9e3779b97f4a7c15ull;
        uint64_t x = z; x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull; x = (x ^ (x >> 27)) * 0x94d049bb133111ebull; x ^= x >> 31;
        s[2 * w] = (uint32_t)x; s[2 * w + 1] = (uint32_t)(x >> 32);
    }
    s[7] &= 0x0fffffffu;        // < 2^252 < r
    G1Affine g; g.x = fp_one<FqTag>(); g.y = fp_one<FqTag>() + fp_one<FqTag>();
    G1Xyzz acc = g1_xyzz_identity();
#pragma unroll 1
    for (int b = 251; b >= 0; --b) {
        acc = g1_dbl(acc);
        if ((s[b >> 5] >> (b & 31)) & 1) acc = g1_add_mixed(acc, g);
    }
    out[i] = g1_to_affine(acc);
}
int g1_generate_run(uint64_t seed, size_t n, G1Affine* d_out, cudaStream_t st) {
    if (n == 0) return 0;
    k_g1_generate<<<div_up(n, 128), 128, 0, st>>>(seed, n, d_out); count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}

// out[i] = [scalars[i]] * base (affine): the n fixed-base multiplications of ParamsKZG::new / gen_srs
__global__ void __launch_bounds__(128) k_g1_fixed_base_mul(const Fr* __restrict__ scalars, size_t n, G1Affine base, G1Affine* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fr s = fp_from_mont(fp_load(scalars + i));
    G1Xyzz acc = g1_xyzz_identity();
#pragma unroll 1
    for (int b = 253; b >= 0; --b) {
        acc = g1_dbl(acc);
        if ((s.l[b >> 5] >> (b & 31)) & 1) acc = g1_add_mixed(acc, base);
    }
    out[i] = g1_to_affine(acc);
}
int g1_fixed_base_mul_run(const Fr* d_scalars, size_t n, const G1Affine& base, G1Affine* d_out, cudaStream_t st) {
    if (n == 0) return 0;
    k_g1_fixed_base_mul<<<div_up(n, 128), 128, 0, st>>>(d_scalars, n, base, d_out); count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}

int g1_sum_run(const G1Xyzz* d_points, size_t groups, size_t count, G1Xyzz* d_out, cudaStream_t st) {
    if (groups == 0) return 0;
    B200_CHECK(groups <= 0x7fffffffu && count <= 0xffffffffu, -1, "g1_sum: sizes out of range");
    k_final_coop<<<(unsigned)groups, TREE_THREADS, 0, st>>>(d_points, (uint32_t)count, d_out); count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
size_t msm_workspace_per_column(const MsmTable& t, size_t n) {
    const size_t nb = (size_t)t.s << (t.c - 1), ents = n * t.W;      // s bucket sets per column
    const size_t chunk_stride = nb + ents / 16 + 1;
    const size_t tile_counts = nb <= MSM_TILE_MAX_BUCKETS ? (ents + nb) * 4 : 0;     // msm_pick_recode bounds tiles * nb by ents + nb
    return ents * 4 + chunk_stride * (12 + sizeof(G1Xyzz)) + nb * (sizeof(G1Xyzz) + 24) + 65536 * (size_t)t.s + tile_counts;
}

int msm_run(const MsmTable& t, const Fr* d_scalars, size_t n, size_t stride, int batch, G1Xyzz* d_out, MsmWorkspace& ws, cudaStream_t st, size_t base_off) {
    B200_CHECK(base_off + n <= t.n, -1, "msm: pairs [%zu, %zu) but only %zu bases registered", base_off, base_off + n, t.n);
    B200_CHECK(batch > 0 && batch <= 65535, -1, "msm: batch %d out of range", batch);
    if (n == 0) {
        B200_CUDA(cudaMemsetAsync(d_out, 0, sizeof(G1Xyzz) * batch, st));
        return 0;
    }
    const int c = t.c, W = t.W, s = t.s;
    B200_CHECK((size_t)batch * s <= 65535, -1, "msm: batch %d x %d bucket sets out of range", batch, s);
    // s bucket sets of 2^(c-1) per column, laid out [col][r][b]: the same memory as batch * s virtual columns of 2^(c-1) buckets,
    // which is how the reduction (10, 11) sees them
    const uint32_t half = 1u << (c - 1), nb = half * (uint32_t)s;
    const int vcols = batch * s;
    const size_t ent_stride = (size_t)n * W;
    B200_CHECK(ent_stride < ((size_t)1 << 32), -1, "msm: n*W too large");
    const unsigned sms = (unsigned)sm_count();
    const MsmPlan plan = msm_plan(n, batch, c, s, W, (int)sms, config().msm_reduce_m, config().msm_reduce_threads);
    const uint32_t cap = plan.cap, heavy_stride = plan.heavy_stride, reduce_m = plan.reduce_m, reduce_threads = plan.reduce_threads;
    const uint32_t nparts = plan.nparts, final_threads = plan.final_threads;
    const size_t chunk_stride = plan.chunk_stride;
    const MsmRecodePlan rp = plan.recode;
    // counts region: hist | cursor | len_hist | len_cursor | heavy, zeroed every call (hist first: k_scan_buckets reads it as uint4).
    // The shared-counter path writes every hist word (k_tile_prefix) and has no cursor, so it zeroes from len_hist on.
    const size_t n_hist = (size_t)batch * nb, n_len = (size_t)batch * (cap + 1);
    if (ws.counts.ensure(plan.counts_bytes)) return -2;
    uint32_t* hist = ws.counts.as<uint32_t>();
    uint32_t* cursor = hist + n_hist;
    uint32_t* len_hist = cursor + n_hist;
    uint32_t* len_cursor = len_hist + n_len;
    uint32_t* heavy = len_cursor + n_len;
    uint32_t* zero_from = rp.tile ? len_hist : hist;
    const size_t zero_words = plan.counts_bytes / 4 - (size_t)(zero_from - hist);
    uint32_t* tile_counts = nullptr;
    const size_t tile_smem = (size_t)nb * 4;
    auto* count_k = s == 1 ? k_digits_tile<false, false> : k_digits_tile<false, true>;
    auto* place_k = s == 1 ? k_digits_tile<true, false> : k_digits_tile<true, true>;
    if (rp.tile) {
        if (ws.tile_counts.ensure(plan.tile_counts_bytes)) return -2;
        tile_counts = ws.tile_counts.as<uint32_t>();
        // the attribute belongs to the function on this device, not to the call: always the same limit, so concurrent callers with
        // other bucket counts cannot lower it under each other's launches (each launch still reserves only nb * 4 bytes)
        const int smem_limit = (int)(MSM_TILE_MAX_BUCKETS * 4);
        B200_CUDA(cudaFuncSetAttribute(count_k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit));
        B200_CUDA(cudaFuncSetAttribute(place_k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit));
    }
    // offsets: offs | chunk_offs | len_offs
    const size_t n_off = (size_t)batch * (nb + 1);
    if (ws.offs.ensure(plan.offs_bytes)) return -2;
    uint32_t* offs = ws.offs.as<uint32_t>();
    uint32_t* chunk_offs = offs + n_off;
    uint32_t* len_offs = chunk_offs + n_off;
    uint32_t* skew = len_offs + n_len;
    if (ws.ents.ensure(plan.ents_bytes)) return -2;
    uint32_t* ents = ws.ents.as<uint32_t>();
    if (ws.subs.ensure(plan.subs_bytes)) return -2;
    uint32_t* chunk_start = ws.subs.as<uint32_t>();
    uint32_t* chunk_len = chunk_start + (size_t)batch * chunk_stride;
    uint32_t* order = chunk_len + (size_t)batch * chunk_stride;
    // sums: chunk_sums | bucket_sums | partials | set_sums (s > 1: one result per bucket set, folded by k_subwindow_fold)
    if (ws.sums.ensure(plan.sums_bytes)) return -2;
    G1Xyzz* chunk_sums = ws.sums.as<G1Xyzz>();
    G1Xyzz* bucket_sums = chunk_sums + (size_t)batch * chunk_stride;
    G1Xyzz* partials = bucket_sums + (size_t)batch * nb;
    G1Xyzz* reduced = s > 1 ? partials + (size_t)vcols * nparts : d_out;

    ProfScope ps_total(PROF_MSM_TOTAL, st);
    B200_CUDA(cudaMemsetAsync(zero_from, 0, zero_words * 4, st));
    if (prof_enabled()) prof_mark(PROF_MSM_RECODE, st, true);
    const unsigned dig_blocks = min(div_up(n, 256), sms * 8u);
    const dim3 gd(dig_blocks, batch), gt(rp.tiles, batch);
    if (rp.tile) {
        count_k<<<gt, MSM_TILE_THREADS, tile_smem, st>>>(d_scalars, stride, (uint32_t)n, (uint32_t)t.n, (uint32_t)base_off, c, W, nb, rp.tile, tile_counts, nullptr, nullptr, 0, s);
        count_launch();
        k_tile_prefix<<<dim3(div_up(nb, 256), batch), 256, 0, st>>>(tile_counts, rp.tiles, nb, hist); count_launch();
    } else {
        if (s == 1) k_digits<false, false><<<gd, 256, 0, st>>>(d_scalars, stride, (uint32_t)n, (uint32_t)t.n, (uint32_t)base_off, c, W, nb, hist, nullptr, nullptr, 0, nullptr, 1);
        else k_digits<false, true><<<gd, 256, 0, st>>>(d_scalars, stride, (uint32_t)n, (uint32_t)t.n, (uint32_t)base_off, c, W, nb, hist, nullptr, nullptr, 0, nullptr, s);
        count_launch();
    }
    {
        ProfScope ps(PROF_MSM_SCAN, st);
        k_scan_buckets<<<batch, 1024, 0, st>>>(hist, offs, chunk_offs, nb, cap, skew); count_launch();
    }
    if (rp.tile) {
        place_k<<<gt, MSM_TILE_THREADS, tile_smem, st>>>(d_scalars, stride, (uint32_t)n, (uint32_t)t.n, (uint32_t)base_off, c, W, nb, rp.tile, tile_counts, offs, ents, ent_stride, s);
    } else if (s == 1) {
        k_digits<true, false><<<gd, 256, 0, st>>>(d_scalars, stride, (uint32_t)n, (uint32_t)t.n, (uint32_t)base_off, c, W, nb, cursor, offs, ents, ent_stride, skew, 1);
    } else {
        k_digits<true, true><<<gd, 256, 0, st>>>(d_scalars, stride, (uint32_t)n, (uint32_t)t.n, (uint32_t)base_off, c, W, nb, cursor, offs, ents, ent_stride, skew, s);
    }
    count_launch();
    k_fill_chunks<<<dim3(div_up(nb, 256), batch), 256, (cap + 1) * 4, st>>>(offs, chunk_offs, nb, cap, chunk_start, chunk_len, chunk_stride, len_hist, heavy, heavy_stride); count_launch();
    k_len_offsets<<<batch, 32, 0, st>>>(len_hist, len_offs, cap); count_launch();
    const unsigned ch_blocks = min(div_up(chunk_stride, 256), sms * 8u);
    k_order_chunks<<<dim3(ch_blocks, batch), 256, 0, st>>>(chunk_len, chunk_stride, chunk_offs, nb, len_offs, len_cursor, cap, order); count_launch();
    if (prof_enabled()) prof_mark(PROF_MSM_RECODE, st, false);
    const unsigned acc_blocks = min(div_up(chunk_stride, 128), sms * 16u);
    {
        ProfScope ps(PROF_MSM_ACCUMULATE, st);
        k_accumulate<<<dim3(acc_blocks, batch), 128, 0, st>>>(t.d_table, ents, ent_stride, chunk_start, chunk_len, order, chunk_stride, chunk_offs, nb, chunk_sums); count_launch();
    }
    ProfScope ps_tail(PROF_MSM_TAIL, st);
    k_combine<<<dim3(div_up(nb, 128), batch), 128, 0, st>>>(chunk_offs, nb, chunk_sums, chunk_stride, bucket_sums); count_launch();
    k_combine_heavy<<<dim3(32, batch), TREE_THREADS, 0, st>>>(heavy, heavy_stride, chunk_offs, nb, chunk_sums, chunk_stride, bucket_sums); count_launch();
    {
        ProfScope ps(PROF_MSM_REDUCE, st);
        k_reduce<1><<<dim3(nparts, vcols), reduce_threads, 0, st>>>(bucket_sums, half, partials, nparts, reduce_m); count_launch();
        k_final<<<vcols, final_threads, 0, st>>>(partials, nparts, reduced); count_launch();
    }
    if (s > 1) {
        ProfScope ps(PROF_MSM_FOLD, st);
        k_subwindow_fold<<<div_up((size_t)batch, 32), 32, 0, st>>>(reduced, s, c, (uint32_t)batch, d_out); count_launch();
    }
    B200_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace b200
