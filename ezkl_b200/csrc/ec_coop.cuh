// ec_coop.cuh — four-lane cooperative XYZZ addition / doubling for latency-bound final sums (k_final_coop in msm.cu, behind
// g1_sum_run: b200_g1_sum_dev and the cross-device combine of b200_msm_sharded_dev).
//
// A final sum is a chain of DEPENDENT group operations per column with little parallelism (a lone warp pays the
// latency of its 14 multiplications back to back on every addition, about twice their throughput cost).  Here the four lanes of a quad hold identical copies of the operands and each computes ONE of the independent products
// of a formula level, the products are exchanged with quad-wide shuffles, and the cheap additions are done redundantly by all four:
// an addition is 4 multiplication levels deep instead of 14 (doubling: 3 instead of 9), at 14 of 16 (10 of 12) lane-multiplications
// of useful work.  Results are bit-identical to g1_add / g1_dbl (same formulas, exact arithmetic); every lane of the quad returns the
// same point.  All four lanes of a quad must call together; different quads of a warp may diverge (the shuffles use the quad's mask).
#pragma once
#include "ec.cuh"

namespace b200 {

#if defined(__CUDACC__)
DEV unsigned quad_mask() { return 0xFu << (threadIdx.x & 28u); }
DEV Fq quad_bcast(const Fq& v, int src, unsigned mask) {
    Fq r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = __shfl_sync(mask, v.l[i], src, 4);
    return r;
}
DEV Fq sel4(int q, const Fq& v0, const Fq& v1, const Fq& v2, const Fq& v3) {
    Fq r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = q == 0 ? v0.l[i] : (q == 1 ? v1.l[i] : (q == 2 ? v2.l[i] : v3.l[i]));
    return r;
}
// 2 * p  (dbl-2008-s-1): levels {U^2, X^2} {U V, X V, M^2, V ZZ} {M (S - X3), W Y, W ZZZ}
DEV G1Xyzz g1_dbl_coop4(const G1Xyzz& p) {
    if (g1_is_identity(p)) return p;
    const int q = threadIdx.x & 3;
    const unsigned mask = quad_mask();
    const Fq u = fp_dbl(p.y);
    Fq m = sel4(q, u, p.x, u, p.x);
    m = m * m;
    const Fq v = quad_bcast(m, 0, mask), xx = quad_bcast(m, 1, mask);
    const Fq mm = fp_dbl(xx) + xx;
    m = sel4(q, u, p.x, mm, v) * sel4(q, v, v, mm, p.zz);
    const Fq w = quad_bcast(m, 0, mask), s = quad_bcast(m, 1, mask), m2 = quad_bcast(m, 2, mask), zz3 = quad_bcast(m, 3, mask);
    G1Xyzz r;
    r.x = m2 - fp_dbl(s);
    m = sel4(q, mm, w, w, w) * sel4(q, s - r.x, p.y, p.zzz, p.zzz);
    const Fq t1 = quad_bcast(m, 0, mask), t2 = quad_bcast(m, 1, mask);
    r.y = t1 - t2;
    r.zz = zz3;
    r.zzz = quad_bcast(m, 2, mask);
    return r;
}
// a + b  (add-2008-s), complete: levels {X1 ZZ2, X2 ZZ1, Y1 ZZZ2, Y2 ZZZ1} {P^2, R^2, ZZ1 ZZ2, ZZZ1 ZZZ2} {P PP, U1 PP, ZZ12 PP} {R (Q - X3), S1 PPP, ZZZ12 PPP}
DEV G1Xyzz g1_add_coop4(const G1Xyzz& a, const G1Xyzz& b) {
    if (g1_is_identity(a)) return b;
    if (g1_is_identity(b)) return a;
    const int q = threadIdx.x & 3;
    const unsigned mask = quad_mask();
    Fq m = sel4(q, a.x, b.x, a.y, b.y) * sel4(q, b.zz, a.zz, b.zzz, a.zzz);
    const Fq u1 = quad_bcast(m, 0, mask), u2 = quad_bcast(m, 1, mask), s1 = quad_bcast(m, 2, mask), s2 = quad_bcast(m, 3, mask);
    const Fq p = u2 - u1, r = s2 - s1;
    if (fp_is_zero(p)) {
        if (fp_is_zero(r)) return g1_dbl_coop4(a);
        return g1_xyzz_identity();
    }
    m = sel4(q, p, r, a.zz, a.zzz) * sel4(q, p, r, b.zz, b.zzz);
    const Fq pp = quad_bcast(m, 0, mask), rr = quad_bcast(m, 1, mask), zz12 = quad_bcast(m, 2, mask), zzz12 = quad_bcast(m, 3, mask);
    m = sel4(q, p, u1, zz12, zz12) * pp;
    const Fq ppp = quad_bcast(m, 0, mask), qq = quad_bcast(m, 1, mask);
    G1Xyzz o;
    o.zz = quad_bcast(m, 2, mask);
    o.x = rr - ppp - fp_dbl(qq);
    m = sel4(q, r, s1, zzz12, zzz12) * sel4(q, qq - o.x, ppp, ppp, ppp);
    const Fq t1 = quad_bcast(m, 0, mask), t2 = quad_bcast(m, 1, mask);
    o.y = t1 - t2;
    o.zzz = quad_bcast(m, 2, mask);
    return o;
}
#endif

}  // namespace b200
