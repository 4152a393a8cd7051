// msm.cuh — internal interface of the BN254 G1 multi-scalar-multiplication engine (msm.cu).
#pragma once
#include "common.cuh"
#include "ec.cuh"

namespace b200 {

// Device-resident, window-precomputed base table for one SRS vector (ParamsKZG.g or .g_lagrange).
// The W = ceil(255 / c) windows are grouped s to a level; level j holds 2^(c*s*j) * P_i in affine form, L = ceil(W / s) levels.
// Window w reads level w / s and adds into bucket set w % s (2^(c-1) buckets each); the s set results are folded at the end
// with (s-1)*c doublings.  s = 1 (the full table) is one shared bucket set and no fold; larger s trades table memory
// (L * n * 64 B) for an s-fold bucket reduction (msm_pick_levels).
struct MsmTable {
    G1Affine* d_table = nullptr;   // [L][n]
    size_t n = 0;
    int c = 0;
    int W = 0;
    int s = 1;                     // windows per level (= bucket sets per column)
    int L = 0;                     // stored levels
    int device = 0;
    size_t bytes() const { return sizeof(G1Affine) * n * (size_t)L; }
};

struct MsmWorkspace {
    DevBuf counts, offs, ents, subs, sums, misc, tile_counts;
};

int msm_default_window(size_t n);
// The level policy: the smallest s whose ceil(W / s) * n * 64 B fits max_table_bytes, else s = W (L = 1: the bases alone,
// whatever the budget).  Pure host function.
inline void msm_pick_levels(size_t n, int c, size_t max_table_bytes, int* s, int* L) {
    const int W = (255 + c - 1) / c;
    const size_t level_bytes = sizeof(G1Affine) * n;
    for (int k = 1; k <= W; ++k) {
        const int l = (W + k - 1) / k;
        if (k == W || (size_t)l * level_bytes <= max_table_bytes) { *s = k; *L = l; return; }
    }
}
// Recoding with the bucket counters in shared memory (k_digits_tile): CTA (x, col) recodes the `tile` scalars [x * tile, (x + 1) * tile)
// of column col, `tiles` = ceil(n / tile) CTAs per column, and holds one 32-bit counter per bucket of the column.  Both recoding
// passes take this plan, so they cut the columns into the same tiles.  tile = 0: the bucket set does not fit in shared memory and the
// global-atomic k_digits runs instead.
struct MsmRecodePlan {
    uint32_t tile = 0, tiles = 0;
};
static constexpr uint32_t MSM_TILE_MAX_BUCKETS = 1u << 15;      // 128 KiB of counters, one CTA per SM
static constexpr uint32_t MSM_TILE_THREADS = 1024;
static constexpr size_t MSM_TILE_L2_BYTES = (size_t)16 << 20;   // entry-list bytes the placement pass may scatter into at once (of a 50 MB L2)
// Pure host function of the call shape and the SM count.  The tile is chosen so that
//   - the columns in flight (one CTA per SM) scatter into at most MSM_TILE_L2_BYTES of entry list, so the random 4-byte writes
//     merge in L2: tiles >= sms * n * W * 4 / MSM_TILE_L2_BYTES;
//   - a small batch still has one CTA per SM: tiles >= sms / batch;
//   - a tile makes at least as many entries (tile * W) as it has counters to clear and publish: tile >= nb / W.  This also keeps the
//     [col][tile][bucket] count matrix (tiles * nb words) no larger than n * W + nb words per column (msm_workspace_per_column);
// with the tile a multiple of the CTA size.
inline MsmRecodePlan msm_pick_recode(size_t n, int batch, uint32_t nb, int W, int sms) {
    MsmRecodePlan p;
    if (n == 0 || batch < 1 || W < 1 || sms < 1 || nb == 0 || nb > MSM_TILE_MAX_BUCKETS) return p;
    const size_t ents = n * (size_t)W;
    size_t tiles = ((size_t)sms * ents * 4 + MSM_TILE_L2_BYTES - 1) / MSM_TILE_L2_BYTES;
    const size_t fill = ((size_t)sms + batch - 1) / batch;
    if (tiles < fill) tiles = fill;
    size_t tile = (n + tiles - 1) / tiles;
    const size_t min_tile = (nb + W - 1) / W;
    if (tile < min_tile) tile = min_tile;
    tile = (tile + MSM_TILE_THREADS - 1) / MSM_TILE_THREADS * MSM_TILE_THREADS;
    p.tile = (uint32_t)tile;
    p.tiles = (uint32_t)((n + tile - 1) / tile);
    return p;
}
static constexpr int HEAVY_CHUNKS = 32;     // buckets with more chunks than this are summed by a whole block (k_combine_heavy)
static constexpr int REDUCE_M_MAX = 32;     // buckets per thread in k_reduce for large (work-bound) batches; small batches take fewer (latency)
static constexpr int TREE_THREADS = 256;

// Chunk length cap: aim for >= ~4 chunks per resident thread slot (SMs x 512 threads), a power of two in [16, 512].
inline uint32_t msm_pick_cap(size_t total_entries, int sms) {
    const size_t target = total_entries / ((size_t)sms * 512 * 4);
    uint32_t cap = 16;
    while (cap < 512 && cap < target) cap <<= 1;
    return cap;
}

// Launch geometry and workspace of one msm_run call: `batch` columns of n scalars against a table of window c, W windows and s
// bucket sets per column, on a device of `sms` SMs.  reduce_m / reduce_threads are the B200_MSM_REDUCE_M / _THREADS overrides
// (0 or out of range: the automatic choice).  Pure host function; msm_run launches exactly this.
struct MsmPlan {
    uint32_t cap = 0;               // entries per chunk at most (k_scan_buckets, k_fill_chunks)
    size_t chunk_stride = 0;        // chunk slots per column: >= the chunks any histogram of n * W entries can make
    uint32_t heavy_stride = 0;      // heavy-list words per column: a count, then room for every bucket of > HEAVY_CHUNKS chunks
    uint32_t reduce_m = 0, reduce_threads = 0;     // k_reduce: buckets per thread, threads per CTA
    uint32_t nparts = 0;            // k_reduce CTAs per bucket set, i.e. partials per bucket set that k_final adds
    uint32_t final_threads = 0;     // k_final threads per CTA
    MsmRecodePlan recode;
    // bytes each MsmWorkspace buffer is asked for
    size_t counts_bytes = 0, tile_counts_bytes = 0, offs_bytes = 0, ents_bytes = 0, subs_bytes = 0, sums_bytes = 0;
};
inline MsmPlan msm_plan(size_t n, int batch, int c, int s, int W, int sms, int reduce_m, int reduce_threads) {
    MsmPlan p;
    const uint32_t half = 1u << (c - 1), nb = half * (uint32_t)s;
    const size_t vcols = (size_t)batch * s, ent_stride = n * (size_t)W;
    p.cap = msm_pick_cap(ent_stride * batch, sms);
    p.chunk_stride = (size_t)nb + ent_stride / p.cap + 1;
    p.heavy_stride = (uint32_t)(ent_stride / ((size_t)p.cap * HEAVY_CHUNKS)) + 2;
    // Bucket reduction geometry.  A thread owns reduce_m consecutive buckets (2 * reduce_m dependent additions, then a small-multiple
    // fix-up and a block tree).  Large batches are work bound: 32 buckets per thread, 256-thread CTAs.  Small batches are bound by the
    // LATENCY of that dependent chain (a lone warp needs ~7.5 us per group addition, about 1000 cycles per field multiplication, twice its
    // throughput cost), so fewer buckets per thread and more, smaller CTAs win until the extra threads' fix-ups and tree levels cost more
    // than the shorter chain saves.  The table is the optimum per total bucket count of the sweep in tools/bench_msm_tail_sweep.py.
    const size_t all_buckets = (size_t)batch * nb;
    p.reduce_m = REDUCE_M_MAX; p.reduce_threads = TREE_THREADS;
    if (all_buckets <= ((size_t)1 << 15)) { p.reduce_m = 4; p.reduce_threads = 128; }
    else if (all_buckets <= ((size_t)1 << 18)) { p.reduce_m = 8; p.reduce_threads = 128; }
    else if (all_buckets <= ((size_t)5 << 17)) { p.reduce_m = 16; p.reduce_threads = 256; }
    else if (all_buckets < ((size_t)37 << 15)) { p.reduce_m = 32; p.reduce_threads = 128; }
    while (p.reduce_m > 1 && p.reduce_m > half) p.reduce_m >>= 1;
    if (reduce_m >= 1 && reduce_m <= 4096) p.reduce_m = (uint32_t)reduce_m;    // tuning override
    if (reduce_threads == 32 || reduce_threads == 64 || reduce_threads == 128 || reduce_threads == 256) p.reduce_threads = (uint32_t)reduce_threads;
    p.nparts = (((half + p.reduce_m - 1) / p.reduce_m) + p.reduce_threads - 1) / p.reduce_threads;
    p.final_threads = 32;
    while (p.final_threads < (uint32_t)TREE_THREADS && p.final_threads < p.nparts) p.final_threads <<= 1;
    p.recode = msm_pick_recode(n, batch, nb, W, sms);
    // counts: hist | cursor | len_hist | len_cursor | heavy;  offs: offs | chunk_offs | len_offs | skew;  subs: chunk start | length | order;
    // sums: chunk_sums | bucket_sums | partials | set_sums (s > 1)
    const size_t n_hist = (size_t)batch * nb, n_len = (size_t)batch * (p.cap + 1), n_off = (size_t)batch * (nb + 1);
    p.counts_bytes = (2 * n_hist + 2 * n_len + (size_t)batch * p.heavy_stride) * 4;
    p.tile_counts_bytes = p.recode.tile ? (size_t)batch * p.recode.tiles * nb * 4 : 0;
    p.offs_bytes = (2 * n_off + n_len + (size_t)batch) * 4;
    p.ents_bytes = (size_t)batch * ent_stride * 4;
    p.subs_bytes = (size_t)batch * p.chunk_stride * 4 * 3;
    p.sums_bytes = sizeof(G1Xyzz) * ((size_t)batch * p.chunk_stride + n_hist + vcols * p.nparts + (s > 1 ? vcols : 0));
    return p;
}
// Picks the window (c <= 0: msm_default_window) and the level count, and allocates the table.  Level 0 (the first n points)
// is left for the caller to fill, e.g. by uploading the bases straight into it.
int msm_table_alloc(MsmTable* t, size_t n, int c, size_t max_table_bytes);
// Fills levels 1 .. L-1 from level 0 on `st`.  d_bases != nullptr is first copied into level 0 (caller keeps ownership).
int msm_table_build(MsmTable* t, const G1Affine* d_bases, cudaStream_t st);
void msm_table_free(MsmTable* t);
// out[b] = sum_i scalars[b*stride + i] * P_(base_off + i)   (base_off + n <= table.n), XYZZ form, one point per column, on device.
// base_off > 0 is the base-split MSM: each device takes a contiguous range of the (scalar, base) pairs against its table replica.
// batch * t.s must not exceed 65535 (grid.y of the bucket reduction).
int msm_run(const MsmTable& t, const Fr* d_scalars, size_t n, size_t stride, int batch, G1Xyzz* d_out,
            MsmWorkspace& ws, cudaStream_t st, size_t base_off = 0);
int g1_fixed_base_mul_run(const Fr* d_scalars, size_t n, const G1Affine& base, G1Affine* d_out, cudaStream_t st);
// out[j] = scale * sum_i omega^(i j) * P_i over G1 (halo2 g_to_lagrange / ParamsKZG::downsize); affine in, affine out
int g1_fft_run(const G1Affine* d_in, uint32_t log_n, const Fr& omega, const Fr* scale, G1Affine* d_out, DevBuf& scratch, cudaStream_t st);
// SRS point check (k_g1_validate): a point is valid when x and y are canonical and it is (0, 0) or on y^2 = x^3 + 3.  For every
// invalid point i, *d_first = min(*d_first, i << 2 | reason); the caller sets *d_first to ~0 first.
enum G1Invalid : unsigned { G1_X_NOT_CANONICAL = 0, G1_Y_NOT_CANONICAL = 1, G1_NOT_ON_CURVE = 2, G1_VALID = 3 };
int g1_validate_run(const G1Affine* d_pts, size_t n, unsigned long long* d_first, cudaStream_t st);
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

// Where the windows of one scalar go in a table of `wpl` windows per level, low window first: window w reads level w / wpl and
// counts into bucket set r = w % wpl, whose first bucket is set_off = r * 2^(c-1); a digit d != 0 goes to bucket set_off + |d| - 1.
struct MsmWindowSlot {
    uint32_t level = 0, set_off = 0;
    int r = 0;
    HD void next(int c, int wpl) {
        set_off += 1u << (c - 1);
        if (++r == wpl) { r = 0; set_off = 0; ++level; }
    }
};

}  // namespace b200
