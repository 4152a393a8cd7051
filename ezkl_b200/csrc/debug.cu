// debug.cu — small self-test entry points (b200_debug_*) used only by tests/ to localise a failure to one layer
// (field arithmetic, group law, digit recoding) before the composite kernels are blamed.  Not part of the drop-in ABI.
#include "debug.h"
#include "ec_coop.cuh"
#include "msm.cuh"
#include "ntt.cuh"

namespace b200 {
// ---- op tables: one HD dispatch function per family, called by the device kernel and by its host twin alike ---------------
// field ops on Montgomery words: 0 a + b, 1 a - b, 2 a * b, 3 inv(a), 4 from_mont(a), 5 sqr(a), 6 -a, 7 2a, 8 to_mont(a)
template <class Tag>
HD Fp<Tag> dbg_field(int op, const Fp<Tag>& x, const Fp<Tag>& y) {
    switch (op) {
        case 0: return x + y;
        case 1: return x - y;
        case 2: return x * y;
        case 3: return fp_inv(x);
        case 4: return fp_from_mont(x);
        case 5: return fp_sqr(x);
        case 6: return fp_neg(x);
        case 7: return fp_dbl(x);
        default: return fp_to_mont(x);
    }
}
// two-product ops: 0 a b + c d (fp_muladd2), 1 a b - c d (fp_mulsub2)
template <class Tag>
HD Fp<Tag> dbg_field4(int op, const Fp<Tag>& a, const Fp<Tag>& b, const Fp<Tag>& c, const Fp<Tag>& d) {
    return op == 0 ? fp_muladd2(a, b, c, d) : fp_mulsub2(a, b, c, d);
}
// affine in, affine out.  op 0: a + b; 1: 2a; 2: k a (k = b.x.l[0] as small integer); 3: a + 2b via g1_add (doubling branch when
// a == 2b); 4: a + (-a)
HD G1Affine dbg_g1(int op, const G1Affine& p, const G1Affine& q) {
    G1Xyzz r;
    if (op == 0) r = g1_add_mixed(g1_to_xyzz(p), q);
    else if (op == 1) r = g1_dbl(g1_to_xyzz(p));
    else if (op == 2) r = g1_mul_small(g1_to_xyzz(p), q.x.l[0]);
    else if (op == 3) r = g1_add(g1_to_xyzz(p), g1_dbl_affine(q));
    else r = g1_add_mixed(g1_to_xyzz(p), g1_neg(p));
    return g1_to_affine(r);
}
// XYZZ in, raw XYZZ words out (no normalisation).  op 0: g1_add(a, b); 1: g1_dbl(a); 2: g1_add_mixed(a, (b.x, b.y)); 3: g1_mul_small(a, k);
// 4: g1_to_affine(a) as (x, y, 0, 0); 5: g1_add_coop4(a, b) and 6: g1_dbl_coop4(a), device only (DBG_XYZZ_COOP and above).
enum { DBG_XYZZ_COOP = 5 };
HD G1Xyzz dbg_xyzz(int op, const G1Xyzz& a, const G1Xyzz& b, uint32_t k) {
    switch (op) {
        case 0: return g1_add(a, b);
        case 1: return g1_dbl(a);
        case 2: { G1Affine q; q.x = b.x; q.y = b.y; return g1_add_mixed(a, q); }
        case 3: return g1_mul_small(a, k);
        default: {
            const G1Affine q = g1_to_affine(a);
            G1Xyzz r = g1_xyzz_identity(); r.x = q.x; r.y = q.y;
            return r;
        }
    }
}

template <class Tag>
__global__ void k_dbg_field(int op, const Fp<Tag>* a, const Fp<Tag>* b, Fp<Tag>* o, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) fp_store(o + i, dbg_field(op, fp_load(a + i), fp_load(b + i)));
}
template <class Tag>
__global__ void k_dbg_field4(int op, const Fp<Tag>* a, const Fp<Tag>* b, const Fp<Tag>* c, const Fp<Tag>* d, Fp<Tag>* o, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) fp_store(o + i, dbg_field4(op, fp_load(a + i), fp_load(b + i), fp_load(c + i), fp_load(d + i)));
}
__global__ void k_dbg_g1(int op, const G1Affine* a, const G1Affine* b, G1Affine* o, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) o[i] = dbg_g1(op, a[i], b[i]);
}
// one element per thread; the cooperative ops take one element per quad (all four lanes load it, lane 0 writes), so consecutive
// elements are neighbouring quads of one warp and may take different branches
__global__ void k_dbg_xyzz(int op, const G1Xyzz* a, const G1Xyzz* b, const uint32_t* k, G1Xyzz* o, size_t n) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (op >= DBG_XYZZ_COOP) {
        const size_t i = t >> 2;
        if (i >= n) return;                 // a whole quad leaves together
        const G1Xyzz r = op == DBG_XYZZ_COOP ? g1_add_coop4(a[i], b[i]) : g1_dbl_coop4(a[i]);
        if ((t & 3) == 0) o[i] = r;
        return;
    }
    if (t < n) o[t] = dbg_xyzz(op, a[t], b[t], k[t]);
}
__global__ void k_dbg_xyzz_to_affine(const G1Xyzz* p, G1Affine* o, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) o[i] = g1_to_affine(p[i]);
}
// host twins' loops over the field op tables
template <class Tag> static void host_field_op(int op, const b200_fr* a, const b200_fr* b, b200_fr* out, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        Fp<Tag> x, y; memcpy(&x, &a[i], 32); memcpy(&y, &b[i], 32);
        const Fp<Tag> r = dbg_field(op, x, y); memcpy(&out[i], &r, 32);
    }
}
template <class Tag> static void host_field_op4(int op, const b200_fr* a, const b200_fr* b, const b200_fr* c, const b200_fr* d, b200_fr* out, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        Fp<Tag> w, x, y, z; memcpy(&w, &a[i], 32); memcpy(&x, &b[i], 32); memcpy(&y, &c[i], 32); memcpy(&z, &d[i], 32);
        const Fp<Tag> r = dbg_field4(op, w, x, y, z); memcpy(&out[i], &r, 32);
    }
}
// device copies of the HOST arrays of one debug call, freed when the call returns on any path
struct DbgStage {
    DevBuf bufs[6];
    int used = 0;
    template <class T> int in(const void* src, size_t bytes, T** d) {
        DevBuf& b = bufs[used++];
        if (b.ensure(bytes ? bytes : 1)) return -2;
        B200_CUDA(cudaMemcpy(b.p, src, bytes, cudaMemcpyHostToDevice));
        *d = b.as<T>();
        return 0;
    }
    template <class T> int out(size_t bytes, T** d) {
        DevBuf& b = bufs[used++];
        if (b.ensure(bytes ? bytes : 1)) return -2;
        *d = b.as<T>();
        return 0;
    }
    ~DbgStage() { for (DevBuf& b : bufs) b.release(); }
};
// What msm.cu (linked into this library for b200_debug_msm_base_off) needs from the product's capi.cu: default tuning, the SM count,
// and no event profiling.
static Config g_dbg_cfg;
const Config& config() { return g_dbg_cfg; }
int sm_count() {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) return 132;
    return v;
}
bool prof_enabled() { return false; }
void prof_mark(int, cudaStream_t, bool) {}
__global__ void k_dbg_digits(const Fr* s, int c, int W, int32_t* out, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr v = fp_from_mont(fp_load(s + i));
    uint32_t carry = 0;
    for (int w = 0; w < W; ++w) out[i * W + w] = msm_next_digit(v.l, c, &carry);
}
// ---- throughput microbenchmarks (register-resident loops; results written so nothing is optimised away) ---------
// variant 0: one dependent chain of Fq mulmods (PTX path); 1: two independent chains; 2: portable C++ mul;
// 3: chain of XYZZ mixed additions against a register-resident affine point; 4: Fq add/sub chain
template <int VARIANT>
__global__ void __launch_bounds__(256) k_bench_mul(Fq* out, int iters) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    Fq x = fp_one<FqTag>(), y = fp_one<FqTag>();
    x.l[0] ^= t; y.l[1] ^= (t * 2654435761u);
    if (VARIANT == 0) {
#pragma unroll 1
        for (int i = 0; i < iters; ++i) x = x * y;
    } else if (VARIANT == 1) {
        Fq z = y + y;
#pragma unroll 1
        for (int i = 0; i < iters; i += 2) { x = x * y; z = z * y; }
        x = x + z;
    } else if (VARIANT == 2) {
#pragma unroll 1
        for (int i = 0; i < iters; ++i) { Fq r; fp_mul_portable<FqTag>(r.l, x.l, y.l); x = r; }
    } else if (VARIANT == 3) {
        G1Affine g; g.x = x; g.y = y;
        G1Xyzz acc = g1_dbl_affine(g);
#pragma unroll 1
        for (int i = 0; i < iters; ++i) { acc = g1_add_mixed(acc, g); g.x.l[0] += 1; }
        x = acc.x + acc.y + acc.zz + acc.zzz;
    } else {
#pragma unroll 1
        for (int i = 0; i < iters; ++i) { x = x + y; y = y - x; }
    }
    fp_store(out + t, x);
}
// ---- raw integer-multiply pipe probes: v=0 mad.wide.u32 (no carry), 1 mad.lo.cc/madc.hi.cc pair chains, 2 mad.lo.u32, 3 DFMA
template <int V>
__global__ void __launch_bounds__(256) k_bench_pipe(uint64_t* out, int iters) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t a = t * 2654435761u + 12345u, b = t ^ 0x9e3779b9u;
    if (V == 0) {
        uint64_t c0 = t, c1 = t + 1, c2 = t + 2, c3 = t + 3, c4 = t + 4, c5 = t + 5, c6 = t + 6, c7 = t + 7;
#pragma unroll 1
        for (int i = 0; i < iters; ++i) {
            asm volatile("mad.wide.u32 %0, %8, %9, %0;\n\tmad.wide.u32 %1, %8, %9, %1;\n\tmad.wide.u32 %2, %8, %9, %2;\n\tmad.wide.u32 %3, %8, %9, %3;\n\t"
                         "mad.wide.u32 %4, %8, %9, %4;\n\tmad.wide.u32 %5, %8, %9, %5;\n\tmad.wide.u32 %6, %8, %9, %6;\n\tmad.wide.u32 %7, %8, %9, %7;"
                         : "+l"(c0), "+l"(c1), "+l"(c2), "+l"(c3), "+l"(c4), "+l"(c5), "+l"(c6), "+l"(c7) : "r"(a), "r"(b));
        }
        out[t] = c0 ^ c1 ^ c2 ^ c3 ^ c4 ^ c5 ^ c6 ^ c7;
    } else if (V == 1) {
        uint32_t e0 = t, e1 = 1, e2 = 2, e3 = 3, e4 = 4, e5 = 5, e6 = 6, e7 = 7, o0 = 8, o1 = 9, o2 = 10, o3 = 11, o4 = 12, o5 = 13, o6 = 14, o7 = 15;
#pragma unroll 1
        for (int i = 0; i < iters; ++i) {
            asm volatile("mad.lo.cc.u32 %0, %16, %17, %0;\n\tmadc.hi.cc.u32 %1, %16, %17, %1;\n\tmadc.lo.cc.u32 %2, %16, %17, %2;\n\tmadc.hi.cc.u32 %3, %16, %17, %3;\n\t"
                         "madc.lo.cc.u32 %4, %16, %17, %4;\n\tmadc.hi.cc.u32 %5, %16, %17, %5;\n\tmadc.lo.cc.u32 %6, %16, %17, %6;\n\tmadc.hi.u32 %7, %16, %17, %7;\n\t"
                         "mad.lo.cc.u32 %8, %16, %17, %8;\n\tmadc.hi.cc.u32 %9, %16, %17, %9;\n\tmadc.lo.cc.u32 %10, %16, %17, %10;\n\tmadc.hi.cc.u32 %11, %16, %17, %11;\n\t"
                         "madc.lo.cc.u32 %12, %16, %17, %12;\n\tmadc.hi.cc.u32 %13, %16, %17, %13;\n\tmadc.lo.cc.u32 %14, %16, %17, %14;\n\tmadc.hi.u32 %15, %16, %17, %15;"
                         : "+r"(e0), "+r"(e1), "+r"(e2), "+r"(e3), "+r"(e4), "+r"(e5), "+r"(e6), "+r"(e7), "+r"(o0), "+r"(o1), "+r"(o2), "+r"(o3), "+r"(o4), "+r"(o5), "+r"(o6), "+r"(o7)
                         : "r"(a), "r"(b));
        }
        out[t] = (uint64_t)(e0 ^ e1 ^ e2 ^ e3 ^ e4 ^ e5 ^ e6 ^ e7) << 32 | (o0 ^ o1 ^ o2 ^ o3 ^ o4 ^ o5 ^ o6 ^ o7);
    } else if (V == 2) {
        uint32_t c0 = t, c1 = 1, c2 = 2, c3 = 3, c4 = 4, c5 = 5, c6 = 6, c7 = 7;
#pragma unroll 1
        for (int i = 0; i < iters; ++i) {
            asm volatile("mad.lo.u32 %0, %8, %9, %0;\n\tmad.lo.u32 %1, %8, %9, %1;\n\tmad.lo.u32 %2, %8, %9, %2;\n\tmad.lo.u32 %3, %8, %9, %3;\n\t"
                         "mad.lo.u32 %4, %8, %9, %4;\n\tmad.lo.u32 %5, %8, %9, %5;\n\tmad.lo.u32 %6, %8, %9, %6;\n\tmad.lo.u32 %7, %8, %9, %7;"
                         : "+r"(c0), "+r"(c1), "+r"(c2), "+r"(c3), "+r"(c4), "+r"(c5), "+r"(c6), "+r"(c7) : "r"(a), "r"(b));
        }
        out[t] = c0 ^ c1 ^ c2 ^ c3 ^ c4 ^ c5 ^ c6 ^ c7;
    } else {
        double x = (double)a, y = 1.0 + 1e-9 * (double)(b & 1023), c0 = t, c1 = 1, c2 = 2, c3 = 3, c4 = 4, c5 = 5, c6 = 6, c7 = 7;
#pragma unroll 1
        for (int i = 0; i < iters; ++i) {
            c0 = fma(x, y, c0); c1 = fma(x, y, c1); c2 = fma(x, y, c2); c3 = fma(x, y, c3); c4 = fma(x, y, c4); c5 = fma(x, y, c5); c6 = fma(x, y, c6); c7 = fma(x, y, c7);
        }
        out[t] = (uint64_t)(c0 + c1 + c2 + c3 + c4 + c5 + c6 + c7);
    }
}
}  // namespace b200
using namespace b200;

#pragma GCC visibility push(default)
extern "C" {
// all pointers are HOST pointers; the call stages, runs one kernel and copies back
int b200_debug_field_op(int field, int op, const b200_fr* a, const b200_fr* b, b200_fr* out, size_t n) {
    if (n == 0) return 0;
    DbgStage st;
    Fr *da, *db, *dout;
    if (int rc = st.in(a, 32 * n, &da)) return rc;
    if (int rc = st.in(b, 32 * n, &db)) return rc;
    if (int rc = st.out(32 * n, &dout)) return rc;
    if (field == 0) k_dbg_field<FrTag><<<div_up(n, 128), 128>>>(op, da, db, dout, n);
    else k_dbg_field<FqTag><<<div_up(n, 128), 128>>>(op, (const Fq*)da, (const Fq*)db, (Fq*)dout, n);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemcpy(out, dout, 32 * n, cudaMemcpyDeviceToHost));
    return 0;
}
int b200_debug_field_op4(int field, int op, const b200_fr* a, const b200_fr* b, const b200_fr* c, const b200_fr* d, b200_fr* out, size_t n) {
    if (n == 0) return 0;
    DbgStage st;
    Fr *da, *db, *dc, *dd, *dout;
    if (int rc = st.in(a, 32 * n, &da)) return rc;
    if (int rc = st.in(b, 32 * n, &db)) return rc;
    if (int rc = st.in(c, 32 * n, &dc)) return rc;
    if (int rc = st.in(d, 32 * n, &dd)) return rc;
    if (int rc = st.out(32 * n, &dout)) return rc;
    if (field == 0) k_dbg_field4<FrTag><<<div_up(n, 128), 128>>>(op, da, db, dc, dd, dout, n);
    else k_dbg_field4<FqTag><<<div_up(n, 128), 128>>>(op, (const Fq*)da, (const Fq*)db, (const Fq*)dc, (const Fq*)dd, (Fq*)dout, n);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemcpy(out, dout, 32 * n, cudaMemcpyDeviceToHost));
    return 0;
}
int b200_debug_g1_op(int op, const b200_g1_affine* a, const b200_g1_affine* b, b200_g1_affine* out, size_t n) {
    if (n == 0) return 0;
    DbgStage st;
    G1Affine *da, *db, *dout;
    if (int rc = st.in(a, 64 * n, &da)) return rc;
    if (int rc = st.in(b, 64 * n, &db)) return rc;
    if (int rc = st.out(64 * n, &dout)) return rc;
    k_dbg_g1<<<div_up(n, 64), 64>>>(op, da, db, dout, n);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemcpy(out, dout, 64 * n, cudaMemcpyDeviceToHost));
    return 0;
}
int b200_debug_g1_xyzz_op(int op, const b200_g1_xyzz* a, const b200_g1_xyzz* b, const uint32_t* k, b200_g1_xyzz* out, size_t n) {
    if (op < 0 || op > DBG_XYZZ_COOP + 1) return -1;
    if (n == 0) return 0;
    DbgStage st;
    G1Xyzz *da, *db, *dout;
    uint32_t* dk;
    if (int rc = st.in(a, 128 * n, &da)) return rc;
    if (int rc = st.in(b, 128 * n, &db)) return rc;
    if (int rc = st.in(k, 4 * n, &dk)) return rc;
    if (int rc = st.out(128 * n, &dout)) return rc;
    const size_t threads = op >= DBG_XYZZ_COOP ? 4 * n : n;
    k_dbg_xyzz<<<div_up(threads, 64), 64>>>(op, da, db, dk, dout, n);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemcpy(out, dout, 128 * n, cudaMemcpyDeviceToHost));
    return 0;
}
int b200_debug_digits(const b200_fr* s, size_t n, int c, int32_t* out /* n * ceil(255/c) */) {
    const int W = (255 + c - 1) / c;
    void *ds, *dout;
    B200_CUDA(cudaMalloc(&ds, 32 * n)); B200_CUDA(cudaMalloc(&dout, 4 * n * W));
    B200_CUDA(cudaMemcpy(ds, s, 32 * n, cudaMemcpyHostToDevice));
    k_dbg_digits<<<div_up(n, 128), 128>>>((const Fr*)ds, c, W, (int32_t*)dout, n);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemcpy(out, dout, 4 * n * W, cudaMemcpyDeviceToHost));
    cudaFree(ds); cudaFree(dout);
    return 0;
}
// returns elapsed ms for `iters` operations per thread on blocks x threads threads
int b200_debug_bench(int variant, int iters, int blocks, int threads, float* ms) {
    Fq* d; B200_CUDA(cudaMalloc(&d, sizeof(Fq) * (size_t)blocks * threads));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int rep = 0; rep < 2; ++rep) {
        cudaEventRecord(e0);
        switch (variant) {
            case 0: k_bench_mul<0><<<blocks, threads>>>(d, iters); break;
            case 1: k_bench_mul<1><<<blocks, threads>>>(d, iters); break;
            case 2: k_bench_mul<2><<<blocks, threads>>>(d, iters); break;
            case 3: k_bench_mul<3><<<blocks, threads>>>(d, iters); break;
            default: k_bench_mul<4><<<blocks, threads>>>(d, iters); break;
        }
        cudaEventRecord(e1);
        B200_CUDA(cudaEventSynchronize(e1));
    }
    B200_CUDA(cudaEventElapsedTime(ms, e0, e1));
    cudaFree(d); cudaEventDestroy(e0); cudaEventDestroy(e1);
    return 0;
}
// returns elapsed ms; ops per thread per iteration: 8 (v0, v2, v3) or 16 (v1)
int b200_debug_bench_pipe(int variant, int iters, int blocks, int threads, float* ms) {
    uint64_t* d; B200_CUDA(cudaMalloc(&d, 8 * (size_t)blocks * threads));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int rep = 0; rep < 2; ++rep) {
        cudaEventRecord(e0);
        switch (variant) {
            case 0: k_bench_pipe<0><<<blocks, threads>>>(d, iters); break;
            case 1: k_bench_pipe<1><<<blocks, threads>>>(d, iters); break;
            case 2: k_bench_pipe<2><<<blocks, threads>>>(d, iters); break;
            default: k_bench_pipe<3><<<blocks, threads>>>(d, iters); break;
        }
        cudaEventRecord(e1);
        B200_CUDA(cudaEventSynchronize(e1));
    }
    B200_CUDA(cudaEventElapsedTime(ms, e0, e1));
    cudaFree(d); cudaEventDestroy(e0); cudaEventDestroy(e1);
    return 0;
}
// host-only: the same recoding routine compiled for the CPU (lets the not-gpu tests check it without a device)
int b200_debug_digits_host(const b200_fr* s_canonical, size_t n, int c, int32_t* out) {
    const int W = (255 + c - 1) / c;
    for (size_t i = 0; i < n; ++i) {
        uint32_t v[8]; memcpy(v, &s_canonical[i], 32);
        uint32_t carry = 0;
        for (int w = 0; w < W; ++w) out[i * W + w] = msm_next_digit(v, c, &carry);
    }
    return 0;
}
// host-only: where each digit of the recoding above goes in a table of `wpl` windows per level (the slot walk k_digits runs):
// out[(i * W + w) * 4 + {0, 1, 2, 3}] = level, bucket set, bucket (-1 for a zero digit), sign (-1, 0, 1)
int b200_debug_digit_slots_host(const b200_fr* s_canonical, size_t n, int c, int wpl, int32_t* out) {
    const int W = (255 + c - 1) / c;
    for (size_t i = 0; i < n; ++i) {
        uint32_t v[8]; memcpy(v, &s_canonical[i], 32);
        uint32_t carry = 0;
        MsmWindowSlot slot;
        for (int w = 0; w < W; ++w) {
            const int32_t d = msm_next_digit(v, c, &carry);
            int32_t* o = out + ((size_t)i * W + w) * 4;
            o[0] = (int32_t)slot.level; o[1] = slot.r;
            o[2] = d ? (int32_t)(slot.set_off + (uint32_t)(d < 0 ? -d : d) - 1u) : -1;
            o[3] = d < 0 ? -1 : (d > 0 ? 1 : 0);
            slot.next(c, wpl);
        }
    }
    return 0;
}
// host-only: the base-table level policy (msm.cuh)
int b200_debug_msm_pick_levels(size_t n, int c, size_t max_table_bytes, int* s, int* L) {
    msm_pick_levels(n, c, max_table_bytes, s, L);
    return 0;
}
// host-only: the recoding tile policy (msm.cuh): out = {tile, tiles}; tile = 0 when the global-atomic recoding runs
int b200_debug_msm_recode_plan(size_t n, int batch, uint32_t nbuckets, int W, int sm_count, uint32_t* out /* 2 */) {
    const MsmRecodePlan p = msm_pick_recode(n, batch, nbuckets, W, sm_count);
    out[0] = p.tile; out[1] = p.tiles;
    return 0;
}
// host-only: the launch geometry and workspace of msm_run (msm_plan, msm.cuh) for `batch` columns of n scalars against a table of window
// c with s windows per level, on a device of sm_count SMs, with the reduction overrides reduce_m / reduce_threads (0: automatic).
// out = {cap, chunk_stride, heavy_stride, reduce_m, reduce_threads, nparts, final_threads, recode tile, recode tiles, bytes of counts,
// tile_counts, offs, ents, subs and sums, msm_workspace_per_column}.  -1 for a shape msm_run rejects.
int b200_debug_msm_plan(size_t n, int batch, int c, int s, int sm_count, int reduce_m, int reduce_threads, uint64_t* out /* 16 */) {
    if (c < 4 || c > 24) return -1;
    const int W = (255 + c - 1) / c;
    if (n == 0 || batch < 1 || s < 1 || s > W || (size_t)batch * s > 65535 || n * W >= ((size_t)1 << 32) || sm_count < 1) return -1;
    const MsmPlan p = msm_plan(n, batch, c, s, W, sm_count, reduce_m, reduce_threads);
    MsmTable t;
    t.n = n; t.c = c; t.W = W; t.s = s; t.L = (W + s - 1) / s;
    const uint64_t v[16] = {p.cap, p.chunk_stride, p.heavy_stride, p.reduce_m, p.reduce_threads, p.nparts, p.final_threads, p.recode.tile, p.recode.tiles,
                            p.counts_bytes, p.tile_counts_bytes, p.offs_bytes, p.ents_bytes, p.subs_bytes, p.sums_bytes, msm_workspace_per_column(t, n)};
    memcpy(out, v, sizeof v);
    return 0;
}
// msm_run with base_off > 0 (the base-split MSM that only a multi-device call makes in the product) on the current device.
// scalars [batch][n] and bases [table_n] are HOST arrays; out[b] = sum_i scalars[b][i] * bases[base_off + i] in affine form.
// The table is built with window c under max_table_bytes (0: every level).  The MSM code is msm.cu, linked into this library.
int b200_debug_msm_base_off(const b200_fr* scalars, size_t n, int batch, const b200_g1_affine* bases, size_t table_n, int c,
                            size_t max_table_bytes, size_t base_off, b200_g1_affine* out) {
    if (n == 0 || batch < 1 || batch > 4096 || base_off + n > table_n || c < 4 || c > 22) return -1;
    MsmTable t;
    MsmWorkspace ws;
    void *d_sc = nullptr, *d_xyzz = nullptr, *d_aff = nullptr;
    auto run = [&]() -> int {
        if (int rc = msm_table_alloc(&t, table_n, c, max_table_bytes ? max_table_bytes : ~(size_t)0)) return rc;
        B200_CUDA(cudaMemcpy(t.d_table, bases, sizeof(G1Affine) * table_n, cudaMemcpyHostToDevice));
        if (int rc = msm_table_build(&t, nullptr, 0)) return rc;
        B200_CUDA(cudaMalloc(&d_sc, sizeof(Fr) * n * batch));
        B200_CUDA(cudaMalloc(&d_xyzz, sizeof(G1Xyzz) * batch));
        B200_CUDA(cudaMalloc(&d_aff, sizeof(G1Affine) * batch));
        B200_CUDA(cudaMemcpy(d_sc, scalars, sizeof(Fr) * n * batch, cudaMemcpyHostToDevice));
        if (int rc = msm_run(t, (const Fr*)d_sc, n, n, batch, (G1Xyzz*)d_xyzz, ws, 0, base_off)) return rc;
        k_dbg_xyzz_to_affine<<<div_up(batch, 32), 32>>>((const G1Xyzz*)d_xyzz, (G1Affine*)d_aff, (size_t)batch);
        B200_CUDA(cudaGetLastError());
        B200_CUDA(cudaMemcpy(out, d_aff, sizeof(G1Affine) * batch, cudaMemcpyDeviceToHost));
        return 0;
    };
    const int rc = run();
    DevBuf* bufs[] = {&ws.counts, &ws.offs, &ws.ents, &ws.subs, &ws.sums, &ws.misc, &ws.tile_counts};
    for (DevBuf* b : bufs) b->release();
    msm_table_free(&t);
    if (d_sc) cudaFree(d_sc);
    if (d_xyzz) cudaFree(d_xyzz);
    if (d_aff) cudaFree(d_aff);
    return rc;
}
// host-only: the NTT pass geometry (ntt.cuh) of a 2^log_n transform of `batch` polynomials on a device of `sm_count` SMs.
// out[pass * 7 + {0..6}] = kernel (1: k_ntt_pass, 2: k_ntt_pass2), logm, log_g, threads, dynamic shared memory bytes, grid.x,
// inter-pass twiddle (0: none, the last pass; 1: full omega^e table; 2: two-level t_lo / t_hi tables).  Returns the pass count.
int b200_debug_ntt_plan_host(uint32_t log_n, int batch, int sm_count, int64_t* out /* 3 * 7 */) {
    if (log_n < 1 || log_n > 28 || batch < 1 || batch > 65535 || sm_count < 1) return -1;
    int npass, logm[3];
    ntt_choose_passes(log_n, &npass, logm);
    for (int i = 0; i < npass; ++i) {
        const NttPassShape sh = ntt_pass_shape(npass, logm, i);
        const NttPassGeom g = ntt_pass_geometry((uint32_t)logm[i], sh.inner_cnt, sh.lines, batch, sm_count);
        int64_t* o = out + 7 * i;
        o[0] = g.kernel; o[1] = logm[i]; o[2] = g.log_g; o[3] = g.threads; o[4] = (int64_t)g.smem; o[5] = (int64_t)g.grid_x;
        o[6] = i == npass - 1 ? 0 : (g.kernel == 2 && ntt_full_table(log_n, npass) ? 1 : 2);     // k_ntt_pass reads t_lo / t_hi only
    }
    return npass;
}
// host-only twins of the calls above: the same op tables compiled for the CPU, through the portable path (not-gpu tests and
// the host tail, normalize_host, run this code)
int b200_debug_host_g1_op(int op, const b200_g1_affine* a, const b200_g1_affine* b, b200_g1_affine* out, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        G1Affine p, q; memcpy(&p, &a[i], 64); memcpy(&q, &b[i], 64);
        const G1Affine o = dbg_g1(op, p, q); memcpy(&out[i], &o, 64);
    }
    return 0;
}
int b200_debug_host_g1_xyzz_op(int op, const b200_g1_xyzz* a, const b200_g1_xyzz* b, const uint32_t* k, b200_g1_xyzz* out, size_t n) {
    if (op < 0 || op >= DBG_XYZZ_COOP) return -1;           // the cooperative ops exist on the device only
    for (size_t i = 0; i < n; ++i) {
        G1Xyzz p, q; memcpy(&p, &a[i], 128); memcpy(&q, &b[i], 128);
        const G1Xyzz o = dbg_xyzz(op, p, q, k[i]); memcpy(&out[i], &o, 128);
    }
    return 0;
}
int b200_debug_host_field_op(int field, int op, const b200_fr* a, const b200_fr* b, b200_fr* out, size_t n) {
    if (field == 0) host_field_op<FrTag>(op, a, b, out, n); else host_field_op<FqTag>(op, a, b, out, n);
    return 0;
}
int b200_debug_host_field_op4(int field, int op, const b200_fr* a, const b200_fr* b, const b200_fr* c, const b200_fr* d, b200_fr* out, size_t n) {
    if (field == 0) host_field_op4<FrTag>(op, a, b, c, d, out, n); else host_field_op4<FqTag>(op, a, b, c, d, out, n);
    return 0;
}
}
#pragma GCC visibility pop
