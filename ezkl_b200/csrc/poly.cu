// poly.cu — batched column-polynomial kernels over BN254 Fr for sm_90a.
//
// Replaces the CPU `parallelize` loops of halo2_proofs (UPSTREAM arithmetic.rs / poly.rs / poly/domain.rs):
//   Polynomial +,-,* and scalar ops, distribute_powers_zeta, divide_by_vanishing_poly, eval_polynomial,
//   kate_division, ff::BatchInvert and the running products / sums behind the permutation z(X) and mv-lookup phi(X)
//   columns (create_proof stages 2-9, SURVEY.md §3.1; entered from /root/reference/src/pfsys/mod.rs:456).
// The element-wise kernels are HBM-bound (96 / 64 B per element); scans and evaluation are chunked so that each
// thread does a serial run of CHUNK elements and only O(n / CHUNK) values go through the block/grid combine steps.
#include <cstring>
#include <vector>
#include "poly.cuh"

namespace b200 {

static constexpr int CHUNK = 16;
static constexpr int TB = 256;
static constexpr int TILE = CHUNK * TB;   // elements per block in the chunked kernels

__global__ void __launch_bounds__(256) k_poly_binary(int op, const Fr* __restrict__ a, const Fr* __restrict__ b, Fr s, Fr* __restrict__ out, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        Fr x = fp_load(a + i), r;
        if (op == POLY_ADD) r = x + fp_load(b + i);
        else if (op == POLY_SUB) r = x - fp_load(b + i);
        else if (op == POLY_MUL) r = x * fp_load(b + i);
        else if (op == POLY_SCALE) r = x * s;
        else r = x + s * fp_load(b + i);
        fp_store(out + i, r);
    }
}
__global__ void __launch_bounds__(256) k_poly_scale_cycle(const Fr* __restrict__ a, const Fr* __restrict__ consts, uint32_t period, Fr* __restrict__ out, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        fp_store(out + i, fp_load(a + i) * fp_load(consts + (i % period)));
}

// out[i] = sum_j scalars[j] * polys[j][i]   (one pass: each polynomial is read once, the sum lives in registers)
__global__ void __launch_bounds__(256) k_poly_lincomb(const Fr* const* __restrict__ polys, const Fr* __restrict__ scalars, uint32_t count, Fr* __restrict__ out, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        Fr acc = fp_zero<FrTag>();
#pragma unroll 1
        for (uint32_t j = 0; j < count; ++j) acc = acc + fp_load(scalars + j) * fp_load(polys[j] + i);
        fp_store(out + i, acc);
    }
}

static unsigned ew_grid(size_t n) { const unsigned gmax = (unsigned)sm_count() * 16u; unsigned g = div_up(n, 256); return g > gmax ? gmax : (g ? g : 1); }

int poly_binary(int op, const Fr* a, const Fr* b, const Fr* h_s, Fr* out, size_t n, cudaStream_t st) {
    if (n == 0) return 0;
    Fr s = h_s ? *h_s : fp_zero<FrTag>();
    k_poly_binary<<<ew_grid(n), 256, 0, st>>>(op, a, b, s, out, n); count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}
int poly_lincomb(const Fr* const* h_polys /*device addresses*/, const Fr* h_scalars, size_t count, Fr* out, size_t n, StagingRing& ring, cudaStream_t st) {
    if (n == 0) return 0;
    B200_CHECK(count < (1u << 24), -1, "poly_lincomb: too many terms");
    const size_t o_s = (sizeof(void*) * count + 31) & ~(size_t)31, total = o_s + sizeof(Fr) * count + 32;
    std::vector<uint8_t> blob(total, 0);
    if (count) { memcpy(blob.data(), h_polys, sizeof(void*) * count); memcpy(blob.data() + o_s, h_scalars, sizeof(Fr) * count); }
    const void* staged;
    if (int rc = ring.push(blob.data(), total, st, &staged)) return rc;
    const uint8_t* d = reinterpret_cast<const uint8_t*>(staged);
    k_poly_lincomb<<<ew_grid(n), 256, 0, st>>>(reinterpret_cast<const Fr* const*>(d), reinterpret_cast<const Fr*>(d + o_s), (uint32_t)count, out, n); count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}
int poly_scale_cycle(const Fr* a, const Fr* h_consts, uint32_t period, Fr* out, size_t n, StagingRing& ring, cudaStream_t st) {
    if (n == 0) return 0;
    B200_CHECK(period > 0, -1, "poly_scale_cycle: period 0");
    const void* d_consts;
    if (int rc = ring.push(h_consts, sizeof(Fr) * period, st, &d_consts)) return rc;
    k_poly_scale_cycle<<<ew_grid(n), 256, 0, st>>>(a, reinterpret_cast<const Fr*>(d_consts), period, out, n); count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}

// column y0 + blockIdx.y, cols[.] = (a, len): out[s] = sum_{t = s + q n < len} a[t] * cyc[t mod 3] * w^(mul * t mod 2^log_w), s < n.
// tab = [cyc[3] | lo | hi] with w^e = lo[e mod 2^lo_bits] * hi[e >> lo_bits].
__global__ void __launch_bounds__(256) k_poly_coset_fold(const FoldCol* __restrict__ cols, uint32_t y0, const Fr* __restrict__ tab, uint32_t lo_bits,
                                                         uint64_t mul, uint64_t emask, Fr* __restrict__ out_all, size_t out_stride, size_t n) {
    const size_t y = (size_t)y0 + blockIdx.y;
    const Fr* a = cols[y].a;
    const size_t len = cols[y].len;
    Fr* out = out_all + y * out_stride;
    const Fr* lo = tab + 3;
    const Fr* hi = lo + ((size_t)1 << lo_bits);
    const uint64_t lo_mask = ((uint64_t)1 << lo_bits) - 1;
    for (size_t s = (size_t)blockIdx.x * blockDim.x + threadIdx.x; s < n; s += (size_t)gridDim.x * blockDim.x) {
        Fr acc = fp_zero<FrTag>();
#pragma unroll 1
        for (size_t t = s; t < len; t += n) {
            const uint64_t e = (mul * t) & emask;
            acc = acc + fp_load(a + t) * (fp_load(tab + t % 3) * (fp_load(lo + (e & lo_mask)) * fp_load(hi + (e >> lo_bits))));
        }
        fp_store(out + s, acc);
    }
}
int poly_coset_fold(const FoldCol* d_cols, size_t n_cols, const Fr* d_tab, uint32_t lo_bits, uint32_t log_w, uint64_t mul, Fr* out, size_t out_stride, size_t n,
                    cudaStream_t st) {
    B200_CHECK(n > 0 && n_cols < (1ull << 32) && lo_bits <= log_w && log_w <= 28, -1, "poly_coset_fold: bad argument");
    for (size_t y0 = 0; y0 < n_cols; y0 += 65535) {          // one launch up to the grid's y limit
        const unsigned ny = (unsigned)(n_cols - y0 < 65535 ? n_cols - y0 : 65535);
        k_poly_coset_fold<<<dim3(ew_grid(n), ny), 256, 0, st>>>(d_cols, (uint32_t)y0, d_tab, lo_bits, mul, ((uint64_t)1 << log_w) - 1, out, out_stride, n);
        count_launch();
        B200_CUDA(cudaGetLastError());
    }
    return 0;
}

// ---- permutation keygen: sigma columns from the copy-constraint mapping -----------------------------------------------
// cell e = j * n + i of the mapping holds (column c, row r) of the cell its cycle maps (j, i) to; out[j * out_stride + i] =
// delta^c * omega^r.  tab = [delta^c, c < n_delta | lo | hi] with omega^r = lo[r mod 2^lo_bits] * hi[r >> lo_bits].  Per cell: 8 B read,
// 32 B written and two multiplications, so the kernel is HBM-bound; the tables stay in L1 / L2.
__global__ void __launch_bounds__(256) k_perm_sigmas(const uint2* __restrict__ map, size_t cells, uint32_t k, const Fr* __restrict__ tab, uint32_t n_delta,
                                                     uint32_t lo_bits, Fr* __restrict__ out, size_t out_stride, unsigned long long* __restrict__ invalid) {
    const uint32_t n_mask = (uint32_t)(((uint64_t)1 << k) - 1), lo_mask = (1u << lo_bits) - 1;
    const Fr* lo = tab + n_delta;
    const Fr* hi = lo + ((size_t)1 << lo_bits);
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < cells; e += (size_t)gridDim.x * blockDim.x) {
        const uint2 m = map[e];
        Fr v = fp_zero<FrTag>();
        if (m.x < n_delta && m.y <= n_mask) v = fp_load(tab + m.x) * (fp_load(lo + (m.y & lo_mask)) * fp_load(hi + (m.y >> lo_bits)));
        else if (invalid) atomicAdd(invalid, 1ull);
        fp_store(out + (e >> k) * out_stride + (e & n_mask), v);
    }
}
int perm_sigmas_run(const uint32_t* d_map, size_t n_columns, uint32_t k, const Fr* h_tab, size_t n_delta, uint32_t lo_bits, Fr* d_out, size_t out_stride,
                    unsigned long long* d_invalid, StagingRing& ring, cudaStream_t st) {
    B200_CHECK(k <= 28 && lo_bits <= k && n_delta < (1ull << 32) && out_stride >= ((size_t)1 << k), -1, "perm_sigmas: bad argument");
    if (n_columns == 0) return 0;
    const size_t tab_elems = n_delta + ((size_t)1 << lo_bits) + ((size_t)1 << (k - lo_bits)), cells = n_columns << k;
    const void* d_tab;
    if (int rc = ring.push(h_tab, sizeof(Fr) * tab_elems, st, &d_tab)) return rc;
    ProfScope ps(PROF_POLY, st);
    k_perm_sigmas<<<ew_grid(cells), 256, 0, st>>>(reinterpret_cast<const uint2*>(d_map), cells, k, reinterpret_cast<const Fr*>(d_tab), (uint32_t)n_delta, lo_bits,
                                                  d_out, out_stride, d_invalid);
    count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}

// ---- proving-key load (b200_pk_load, include/ezkl_b200.h) --------------------------------------------------------------------
// The check of one key column as halo2curves' Fr::from_raw_bytes makes it: one thread per element, 32 B read and one limb comparison,
// so HBM-bound.  Rows of a warp are consecutive, so its lowest failing lane is its lowest failing row: one atomicMin per warp at most,
// on (column << 32 | row), which keeps the lowest (column, row) of the call.
__global__ void __launch_bounds__(256) k_fr_validate(const Fr* __restrict__ col, size_t n, unsigned long long column, unsigned long long* __restrict__ first) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool bad = i < n && !fp_is_canonical(fp_load(col + i));
    const unsigned lanes = __ballot_sync(0xffffffffu, bad);
    if (lanes && (threadIdx.x & 31) == (unsigned)(__ffs(lanes) - 1)) atomicMin(first, (column << 32) | i);
}
int fr_validate_run(const Fr* d_col, size_t n, size_t column, unsigned long long* d_first, cudaStream_t st) {
    B200_CHECK(n <= ((size_t)1 << 32) && column < ((size_t)1 << 32), -1, "fr_validate: bad argument");
    if (n == 0) return 0;
    k_fr_validate<<<div_up(n, 256), 256, 0, st>>>(d_col, n, column, d_first); count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}
// out[j * n + i] = 1 (Montgomery) for lo[j] <= i < hi[j], else 0, for the three columns j < 3
struct FrRanges { uint64_t lo[3], hi[3]; };
__global__ void __launch_bounds__(256) k_fr_indicator(Fr* __restrict__ out, size_t n, FrRanges r) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned j = blockIdx.y;
    const uint64_t lo = j == 0 ? r.lo[0] : (j == 1 ? r.lo[1] : r.lo[2]), hi = j == 0 ? r.hi[0] : (j == 1 ? r.hi[1] : r.hi[2]);   // no local copy of r
    if (i < n) fp_store(out + j * n + i, i >= lo && i < hi ? fp_one<FrTag>() : fp_zero<FrTag>());
}
int fr_indicator_run(Fr* d_out, size_t n, const uint64_t lo[3], const uint64_t hi[3], cudaStream_t st) {
    if (n == 0) return 0;
    FrRanges r;
    for (int j = 0; j < 3; ++j) { r.lo[j] = lo[j]; r.hi[j] = hi[j]; }
    k_fr_indicator<<<dim3(div_up(n, 256), 3), 256, 0, st>>>(d_out, n, r); count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}

// ---- shared-memory helpers for one Fr per thread -------------------------------------------------------------
DEV Fr shf_get(const Fr* sh, uint32_t i) { return fp_load(sh + i); }
DEV void shf_put(Fr* sh, uint32_t i, const Fr& v) { fp_store(sh + i, v); }

// Weighted suffix-inclusive scan across the block: v[t] <- sum_{u >= t} v[u] * B^(u - t).  nthreads = blockDim.x.
// On return sh[u] holds thread u's result for every u (callers read their neighbour's value from it).
DEV Fr block_weighted_suffix(Fr v, Fr B, Fr* sh) {
    const uint32_t t = threadIdx.x, nt = blockDim.x;
    shf_put(sh, t, v);
    __syncthreads();
    for (uint32_t d = 1; d < nt; d <<= 1) {
        Fr add = fp_zero<FrTag>();
        const bool has = t + d < nt;
        if (has) add = B * shf_get(sh, t + d);
        __syncthreads();
        if (has) { v = v + add; shf_put(sh, t, v); }
        __syncthreads();
        B = B * B;
    }
    return v;
}
// Unweighted prefix-inclusive scan with a commutative op (product or sum).
template <bool PRODUCT>
DEV Fr block_prefix_inclusive(Fr v, Fr* sh) {
    const uint32_t t = threadIdx.x, nt = blockDim.x;
    shf_put(sh, t, v);
    __syncthreads();
    for (uint32_t d = 1; d < nt; d <<= 1) {
        Fr o = v;
        const bool has = t >= d;
        if (has) o = shf_get(sh, t - d);
        __syncthreads();
        if (has) { v = PRODUCT ? v * o : v + o; shf_put(sh, t, v); }
        __syncthreads();
    }
    return v;
}

// ---- evaluation / kate division (weighted suffix scans with multiplier x) --------------------------------------
struct WArgs { Fr x, xc, xt; };   // x, x^CHUNK, x^TILE

// chunk value V_t = sum_{j in chunk} a[j] x^(j - lo); block value = sum_t V_t (x^CHUNK)^t -> blk_val[blockIdx]
__global__ void __launch_bounds__(TB) k_wscan_block_values(const Fr* __restrict__ a, size_t stride, size_t m, const WArgs* __restrict__ wargs, Fr* __restrict__ blk_val, uint32_t nblk) {
    __shared__ Fr sh[TB];
    const WArgs w = wargs[blockIdx.y];
    const Fr* src = a + (size_t)blockIdx.y * stride;
    const size_t lo = (size_t)blockIdx.x * TILE + (size_t)threadIdx.x * CHUNK;
    Fr v = fp_zero<FrTag>();
    if (lo < m) {
        const size_t hi = lo + CHUNK < m ? lo + CHUNK : m;
        for (size_t j = hi; j-- > lo;) v = v * w.x + fp_load(src + j);
    }
    v = block_weighted_suffix(v, w.xc, sh);
    if (threadIdx.x == 0) fp_store(blk_val + (size_t)blockIdx.y * nblk + blockIdx.x, v);
}
// one block per polynomial: carry[blk] = sum_{u > blk} val[u] * XT^(u - blk - 1); total[p] = sum_u val[u] XT^u
__global__ void __launch_bounds__(1024) k_wscan_carries(const Fr* __restrict__ blk_val, uint32_t nblk, const WArgs* __restrict__ wargs, Fr* __restrict__ carry, Fr* __restrict__ total) {
    __shared__ Fr sh[1024];
    const WArgs w = wargs[blockIdx.x];
    const Fr* val = blk_val + (size_t)blockIdx.x * nblk;
    const uint32_t ipt = (nblk + blockDim.x - 1) / blockDim.x;
    const uint32_t lo = threadIdx.x * ipt, hi = min(lo + ipt, nblk);
    Fr v = fp_zero<FrTag>();
    for (uint32_t u = hi; u-- > lo && hi > lo;) v = v * w.xt + fp_load(val + u);
    Fr step = w.xt;                                       // xt^ipt (ipt is 1 unless there are more than 1024 block values)
    for (uint32_t e = 1; e < ipt; ++e) step = step * w.xt;
    Fr incl = block_weighted_suffix(v, step, sh);      // value of blocks >= lo, relative to block lo
    if (threadIdx.x == 0 && total) fp_store(total + blockIdx.x, incl);
    if (carry && lo < nblk) {
        // value of everything after this thread's last block, relative to block `hi`
        Fr c = (threadIdx.x + 1 < blockDim.x && hi < nblk) ? shf_get(sh, threadIdx.x + 1) : fp_zero<FrTag>();
        // note: thread t+1 starts at block lo + ipt = hi when hi == lo + ipt; if hi was clipped there is nothing after
        for (uint32_t u = hi; u-- > lo;) {
            fp_store(carry + (size_t)blockIdx.x * nblk + u, c);
            c = c * w.xt + fp_load(val + u);
        }
    }
}
// q[e] = sum_{f >= e} a[f] x^(f - e) for e < m  (a already offset by one coefficient for kate division)
__global__ void __launch_bounds__(TB) k_wscan_apply(const Fr* __restrict__ a, size_t m, const WArgs* __restrict__ wargs, const Fr* __restrict__ carry, Fr* __restrict__ q) {
    __shared__ Fr sh[TB];
    const WArgs w = wargs[0];
    const size_t lo = (size_t)blockIdx.x * TILE + (size_t)threadIdx.x * CHUNK;
    const size_t hi = lo + CHUNK < m ? lo + CHUNK : m;
    Fr v = fp_zero<FrTag>();
    if (lo < m) for (size_t j = hi; j-- > lo;) v = v * w.x + fp_load(a + j);
    const Fr blk_carry = fp_load(carry + blockIdx.x);
    if (threadIdx.x == TB - 1) v = v + w.xc * blk_carry;     // everything after this block, relative to the block end
    Fr incl = block_weighted_suffix(v, w.xc, sh);
    if (lo < m) {
        Fr c = threadIdx.x + 1 < TB ? shf_get(sh, threadIdx.x + 1) : blk_carry;
        // chunks clipped by m: the carry of a partially filled chunk must be relative to its nominal end (lo + CHUNK);
        // elements past m are zero, so stepping x over the gap is a multiplication by x^(gap)
        for (size_t g = hi; g < lo + CHUNK; ++g) c = c * w.x;
        for (size_t j = hi; j-- > lo;) { c = c * w.x + fp_load(a + j); fp_store(q + j, c); }
    }
}

static unsigned carry_threads(uint32_t nblk) { unsigned t = 32; while (t < nblk && t < 1024) t <<= 1; return t; }

static int upload_wargs(const Fr* h_x, int batch, StagingRing& ring, const WArgs** d_w, cudaStream_t st) {
    std::vector<WArgs> hw(batch);
    for (int p = 0; p < batch; ++p) { hw[p].x = h_x[p]; hw[p].xc = fp_pow_u64(h_x[p], CHUNK); hw[p].xt = fp_pow_u64(h_x[p], TILE); }
    const void* staged;
    if (int rc = ring.push(hw.data(), sizeof(WArgs) * batch, st, &staged)) return rc;
    *d_w = reinterpret_cast<const WArgs*>(staged);
    return 0;
}

int poly_eval(const Fr* coeffs, size_t stride, size_t n, const Fr* h_x, Fr* d_out, int batch, PolyWorkspace& ws, StagingRing& ring, cudaStream_t st) {
    B200_CHECK(batch > 0 && batch <= 65535, -1, "poly_eval: batch %d out of range", batch);
    if (n == 0) { B200_CUDA(cudaMemsetAsync(d_out, 0, sizeof(Fr) * batch, st)); return 0; }
    const uint32_t nblk = div_up(n, TILE);
    if (ws.scratch.ensure(sizeof(Fr) * (size_t)nblk * batch)) return -2;
    const WArgs* d_w;
    if (int rc = upload_wargs(h_x, batch, ring, &d_w, st)) return rc;
    Fr* blk_val = ws.scratch.as<Fr>();
    k_wscan_block_values<<<dim3(nblk, batch), TB, 0, st>>>(coeffs, stride, n, d_w, blk_val, nblk); count_launch();
    k_wscan_carries<<<batch, carry_threads(nblk), 0, st>>>(blk_val, nblk, d_w, nullptr, d_out); count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}

int poly_kate_division(const Fr* a, size_t n, const Fr* h_b, Fr* q, PolyWorkspace& ws, StagingRing& ring, cudaStream_t st) {
    B200_CHECK(n >= 1, -1, "kate_division: empty polynomial");
    if (n == 1) return 0;
    const size_t m = n - 1;
    const uint32_t nblk = div_up(m, TILE);
    if (ws.scratch.ensure(sizeof(Fr) * (size_t)nblk * 2)) return -2;
    const WArgs* d_w;
    if (int rc = upload_wargs(h_b, 1, ring, &d_w, st)) return rc;
    Fr* blk_val = ws.scratch.as<Fr>();
    Fr* carry = blk_val + nblk;
    k_wscan_block_values<<<dim3(nblk, 1), TB, 0, st>>>(a + 1, 0, m, d_w, blk_val, nblk); count_launch();
    k_wscan_carries<<<1, carry_threads(nblk), 0, st>>>(blk_val, nblk, d_w, carry, nullptr); count_launch();
    k_wscan_apply<<<nblk, TB, 0, st>>>(a + 1, m, d_w, carry, q); count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}

// ---- running product / sum (exclusive) --------------------------------------------------------------------------
template <bool PRODUCT> DEV Fr op_identity() { return PRODUCT ? fp_one<FrTag>() : fp_zero<FrTag>(); }
template <bool PRODUCT> DEV Fr op_apply(const Fr& a, const Fr& b) { return PRODUCT ? a * b : a + b; }

template <bool PRODUCT>
__global__ void __launch_bounds__(TB) k_scan_block_totals(const Fr* __restrict__ a_all, size_t a_stride, size_t n, Fr* __restrict__ blk_tot_all, uint32_t nblk) {
    __shared__ Fr sh[TB];
    const Fr* a = a_all + (size_t)blockIdx.y * a_stride;
    Fr* blk_tot = blk_tot_all + (size_t)blockIdx.y * nblk;
    const size_t lo = (size_t)blockIdx.x * TILE + (size_t)threadIdx.x * CHUNK;
    Fr v = op_identity<PRODUCT>();
    if (lo < n) { const size_t hi = lo + CHUNK < n ? lo + CHUNK : n; for (size_t j = lo; j < hi; ++j) v = op_apply<PRODUCT>(v, fp_load(a + j)); }
    v = block_prefix_inclusive<PRODUCT>(v, sh);
    if (threadIdx.x == TB - 1) fp_store(blk_tot + blockIdx.x, v);
}
template <bool PRODUCT>
__global__ void __launch_bounds__(1024) k_scan_block_prefixes(const Fr* __restrict__ blk_tot_all, uint32_t nblk, const Fr* __restrict__ inits, Fr* __restrict__ blk_pre_all) {
    __shared__ Fr sh[1024];
    const Fr* blk_tot = blk_tot_all + (size_t)blockIdx.x * nblk;
    Fr* blk_pre = blk_pre_all + (size_t)blockIdx.x * nblk;
    const Fr init = fp_load(inits + blockIdx.x);
    const uint32_t ipt = (nblk + blockDim.x - 1) / blockDim.x;
    const uint32_t lo = threadIdx.x * ipt, hi = min(lo + ipt, nblk);
    Fr v = op_identity<PRODUCT>();
    for (uint32_t u = lo; u < hi; ++u) v = op_apply<PRODUCT>(v, fp_load(blk_tot + u));
    Fr incl = block_prefix_inclusive<PRODUCT>(v, sh);
    Fr run = threadIdx.x ? op_apply<PRODUCT>(init, shf_get(sh, threadIdx.x - 1)) : init;
    for (uint32_t u = lo; u < hi; ++u) { fp_store(blk_pre + u, run); run = op_apply<PRODUCT>(run, fp_load(blk_tot + u)); }
}
template <bool PRODUCT>
__global__ void __launch_bounds__(TB) k_scan_apply(const Fr* __restrict__ a_all, size_t a_stride, size_t n, const Fr* __restrict__ blk_pre_all, uint32_t nblk, Fr* __restrict__ out_all, size_t out_stride) {
    __shared__ Fr sh[TB];
    const Fr* a = a_all + (size_t)blockIdx.y * a_stride;
    const Fr* blk_pre = blk_pre_all + (size_t)blockIdx.y * nblk;
    Fr* out = out_all + (size_t)blockIdx.y * out_stride;
    const size_t lo = (size_t)blockIdx.x * TILE + (size_t)threadIdx.x * CHUNK;
    const size_t hi = lo + CHUNK < n ? lo + CHUNK : n;
    Fr v = op_identity<PRODUCT>();
    if (lo < n) for (size_t j = lo; j < hi; ++j) v = op_apply<PRODUCT>(v, fp_load(a + j));
    Fr incl = block_prefix_inclusive<PRODUCT>(v, sh);
    if (lo < n) {
        Fr run = fp_load(blk_pre + blockIdx.x);
        if (threadIdx.x) run = op_apply<PRODUCT>(run, shf_get(sh, threadIdx.x - 1));
        for (size_t j = lo; j < hi; ++j) { Fr x = fp_load(a + j); fp_store(out + j, run); run = op_apply<PRODUCT>(run, x); }
    }
}

// `batch` independent columns a[p * a_stride ..] -> out[p * out_stride ..], one initial value each (h_inits: host array)
int poly_prefix_scan(bool product, const Fr* a, size_t a_stride, size_t n, const Fr* h_inits, Fr* out, size_t out_stride, int batch, PolyWorkspace& ws, StagingRing& ring,
                     cudaStream_t st) {
    if (n == 0 || batch == 0) return 0;
    B200_CHECK(batch > 0 && batch <= 65535, -1, "prefix_scan: batch %d out of range", batch);
    const uint32_t nblk = div_up(n, TILE);
    if (ws.scratch.ensure(sizeof(Fr) * (size_t)nblk * 2 * batch)) return -2;
    Fr* blk_tot = ws.scratch.as<Fr>();
    Fr* blk_pre = blk_tot + (size_t)nblk * batch;
    const void* staged;
    if (int rc = ring.push(h_inits, sizeof(Fr) * batch, st, &staged)) return rc;
    const Fr* d_inits = reinterpret_cast<const Fr*>(staged);
    const dim3 grid(nblk, batch);
    if (product) {
        k_scan_block_totals<true><<<grid, TB, 0, st>>>(a, a_stride, n, blk_tot, nblk); count_launch();
        k_scan_block_prefixes<true><<<batch, 1024, 0, st>>>(blk_tot, nblk, d_inits, blk_pre); count_launch();
        k_scan_apply<true><<<grid, TB, 0, st>>>(a, a_stride, n, blk_pre, nblk, out, out_stride); count_launch();
    } else {
        k_scan_block_totals<false><<<grid, TB, 0, st>>>(a, a_stride, n, blk_tot, nblk); count_launch();
        k_scan_block_prefixes<false><<<batch, 1024, 0, st>>>(blk_tot, nblk, d_inits, blk_pre); count_launch();
        k_scan_apply<false><<<grid, TB, 0, st>>>(a, a_stride, n, blk_pre, nblk, out, out_stride); count_launch();
    }
    B200_CUDA(cudaGetLastError());
    return 0;
}

// ---- batch inversion (Montgomery's trick per thread chunk, prefix products in scratch) -------------------------------
static constexpr int INV_CHUNK = 64;
__global__ void __launch_bounds__(128) k_batch_invert(Fr* __restrict__ a, Fr* __restrict__ pref, size_t n) {
    const size_t lo = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * INV_CHUNK;
    if (lo >= n) return;
    const size_t hi = lo + INV_CHUNK < n ? lo + INV_CHUNK : n;
    Fr run = fp_one<FrTag>();
    for (size_t j = lo; j < hi; ++j) {
        Fr x = fp_load(a + j);
        fp_store(pref + j, run);
        if (!fp_is_zero(x)) run = run * x;
    }
    Fr inv = fp_inv(run);
    for (size_t j = hi; j-- > lo;) {
        Fr x = fp_load(a + j);
        if (fp_is_zero(x)) continue;       // zeros stay zero (ff::BatchInvert)
        fp_store(a + j, inv * fp_load(pref + j));
        inv = inv * x;
    }
}

int poly_batch_invert(Fr* a, size_t n, PolyWorkspace& ws, cudaStream_t st) {
    if (n == 0) return 0;
    if (ws.scratch.ensure(sizeof(Fr) * n)) return -2;
    const size_t nthreads = (n + INV_CHUNK - 1) / INV_CHUNK;
    k_batch_invert<<<div_up(nthreads, 128), 128, 0, st>>>(a, ws.scratch.as<Fr>(), n); count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace b200
