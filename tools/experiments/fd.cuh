// fd.cuh — BN254 Fr / Fq Montgomery arithmetic on 5 x 52-bit limbs with the limb products formed on the FP64 pipe.
//
// Why a second multiplier: every hot kernel of this library is bound by ONE pipe, the one IMAD / IMAD.WIDE issue on, while the
// FP64 pipe has nothing to do (not measured on the H100).  The H100 SXM keeps a full-rate FP64 pipe (64 DFMA/clk/SM nominal), so a
// multiplier whose product array runs on DFMA can execute NEXT TO the integer one (different warps of the same kernel) and raise
// the SM's multiply throughput above what either pipe gives alone.
//
// Representation: Fd = 5 limbs of 52 bits held in uint64 (the integer 0 <= v < 2^260), Montgomery radix R' = 2^260.
// A limb product a_j * b_i < 2^104 is split exactly with two fused multiply-adds in round-toward-zero mode
//     hi = fma_rz(a, b, 2^104)                = 2^104 + floor(ab / 2^52) * 2^52        (ulp of [2^104, 2^105) is 2^52)
//     lo = fma_rz(a, b, (2^104 + 2^52) - hi)  = 2^52 + (ab mod 2^52)                   (exact)
// Both results have a pinned exponent, so their raw bit patterns minus the exponent constants are the two 52-bit halves and
// the column sums are plain 64-bit integer additions on the ALU pipe (two terms per IADD3 / IADD3.X pair).  The exponent
// constants have a zero low word and fold into the immediate of the first IADD3.X of each column.
// (Technique: Emmart, Zheng, Weems, "Faster modular exponentiation using double precision floating point arithmetic on the
// GPU", ARITH 2018; restated from the paper's description for a 254-bit modulus and a CIOS schedule.)
//
// fd_mul(a, b) = a * b * 2^-260 mod N, result < 2N with normalised limbs, for ANY normalised inputs < 2^260.  Multiplying a
// value held in the wire format's radix (x * 2^256, include/ezkl_b200.h) by a CONSTANT stored as c * 2^260 returns
// (x c) * 2^256: data keeps its wire radix when only the constants (twiddles, table entries) are kept in R' form.
#pragma once
#include <math.h>
#include "../../ezkl_b200/csrc/field.cuh"

namespace b200 {

struct FdFqTag {
    using Wire = FqTag;
    HD static uint64_t mod(int i) {
        constexpr uint64_t M[5] = {0x8c16d87cfd47ull, 0x916871ca8d3c2ull, 0x181585d97816aull, 0xa029b85045b68ull, 0x30644e72e131ull};
        return M[i];
    }
    static constexpr uint64_t NINV = 0x20782e4866389ull;      // -N^-1 mod 2^52
};
struct FdFrTag {
    using Wire = FrTag;
    HD static uint64_t mod(int i) {
        constexpr uint64_t M[5] = {0x1f593f0000001ull, 0x4879b9709143eull, 0x181585d2833e8ull, 0xa029b85045b68ull, 0x30644e72e131ull};
        return M[i];
    }
    static constexpr uint64_t NINV = 0x1f593efffffffull;
};

template <class T> struct Fd { uint64_t l[5]; };

static constexpr uint64_t FD_MASK = (1ull << 52) - 1;
static constexpr uint64_t FD_EL = 0x4330000000000000ull;      // bit pattern of 2^52
static constexpr uint64_t FD_EH = 0x4670000000000000ull;      // bit pattern of 2^104

#if defined(__CUDA_ARCH__)
DEV double fd_fma_rz(double a, double b, double c) { return __fma_rz(a, b, c); }
DEV uint64_t fd_bits(double x) { return (uint64_t)__double_as_longlong(x); }
DEV double fd_from_bits(uint64_t x) { return __longlong_as_double((long long)x); }
#else
// host build: the caller (tests) sets fesetround(FE_TOWARDZERO); every other FP operation in this file is exact
inline double fd_fma_rz(double a, double b, double c) { return fma(a, b, c); }
inline uint64_t fd_bits(double x) { uint64_t r; memcpy(&r, &x, 8); return r; }
inline double fd_from_bits(uint64_t x) { double r; memcpy(&r, &x, 8); return r; }
#endif

// integer limb (< 2^52) -> double holding the same integer
HD double fd_limb_to_double(uint64_t v) { return fd_from_bits(v | FD_EL) - 0x1p52; }

template <class T>
HD Fd<T> fd_mul(const Fd<T>& a, const Fd<T>& b) {
    const double C104 = 0x1p104, C2 = 0x1p104 + 0x1p52;
    double ad[5], bd[5], nd[5];
#pragma unroll
    for (int j = 0; j < 5; ++j) { ad[j] = fd_limb_to_double(a.l[j]); bd[j] = fd_limb_to_double(b.l[j]); nd[j] = (double)T::mod(j); }
    const double ninv = (double)T::NINV;
    uint64_t t[10];
#pragma unroll
    for (int j = 0; j < 10; ++j) t[j] = 0;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
#pragma unroll
        for (int j = 0; j < 5; ++j) {
            const double hi = fd_fma_rz(ad[j], bd[i], C104);
            const double lo = fd_fma_rz(ad[j], bd[i], C2 - hi);
            t[i + j] += fd_bits(lo) - FD_EL;
            t[i + j + 1] += fd_bits(hi) - FD_EH;
        }
        // q = t[i] * (-N^-1) mod 2^52, then t += q * N: column i becomes a multiple of 2^52
        const double md = fd_limb_to_double(t[i] & FD_MASK);
        const double qh = fd_fma_rz(md, ninv, C104);
        const double q = fd_fma_rz(md, ninv, C2 - qh) - 0x1p52;
#pragma unroll
        for (int j = 0; j < 5; ++j) {
            const double hi = fd_fma_rz(q, nd[j], C104);
            const double lo = fd_fma_rz(q, nd[j], C2 - hi);
            t[i + j] += fd_bits(lo) - FD_EL;
            t[i + j + 1] += fd_bits(hi) - FD_EH;
        }
        t[i + 1] += t[i] >> 52;
    }
    Fd<T> r;
    uint64_t c = 0;
#pragma unroll
    for (int k = 0; k < 5; ++k) { const uint64_t v = t[5 + k] + c; r.l[k] = k < 4 ? (v & FD_MASK) : v; c = v >> 52; }
    return r;
}

// ---- wire (8 x u32 = 256-bit integer) <-> 52-bit limbs: pure bit re-slicing, no change of Montgomery radix -----------------
template <class T>
HD Fd<T> fd_from_wire(const Fp<typename T::Wire>& x) {
    const uint64_t v0 = x.l[0] | ((uint64_t)x.l[1] << 32), v1 = x.l[2] | ((uint64_t)x.l[3] << 32), v2 = x.l[4] | ((uint64_t)x.l[5] << 32),
                   v3 = x.l[6] | ((uint64_t)x.l[7] << 32);
    Fd<T> r;
    r.l[0] = v0 & FD_MASK;
    r.l[1] = ((v0 >> 52) | (v1 << 12)) & FD_MASK;
    r.l[2] = ((v1 >> 40) | (v2 << 24)) & FD_MASK;
    r.l[3] = ((v2 >> 28) | (v3 << 36)) & FD_MASK;
    r.l[4] = v3 >> 16;
    return r;
}
// requires normalised limbs and a value < 2^256
template <class T>
HD Fp<typename T::Wire> fd_to_wire(const Fd<T>& a) {
    const uint64_t v0 = a.l[0] | (a.l[1] << 52), v1 = (a.l[1] >> 12) | (a.l[2] << 40), v2 = (a.l[2] >> 24) | (a.l[3] << 28), v3 = (a.l[3] >> 36) | (a.l[4] << 16);
    Fp<typename T::Wire> r;
    r.l[0] = (uint32_t)v0; r.l[1] = (uint32_t)(v0 >> 32); r.l[2] = (uint32_t)v1; r.l[3] = (uint32_t)(v1 >> 32);
    r.l[4] = (uint32_t)v2; r.l[5] = (uint32_t)(v2 >> 32); r.l[6] = (uint32_t)v3; r.l[7] = (uint32_t)(v3 >> 32);
    return r;
}

}  // namespace b200
