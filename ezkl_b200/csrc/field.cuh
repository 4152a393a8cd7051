// field.cuh — BN254 Fr / Fq Montgomery arithmetic on 8 x 32-bit limbs, host + device.
//
// Wire format = halo2curves' raw SerdeObject form (SURVEY.md Appendix B): 4 x u64 little-endian limbs in Montgomery
// form, R = 2^256; on a little-endian machine that is bit-identical to the 8 x u32 limb array used here, so host
// buffers coming from Rust `&[Fr]` are consumed zero-copy.  Replaces halo2curves 0.7.0 src/bn256/{fr,fq}.rs
// (un-vendored dependency; call sites /root/reference/src/pfsys/mod.rs:20-22).
//
// Device path: generated single-asm-block PTX carry chains (fp_ptx.cuh, validated by fp_gen.py's interpreter).
// Host path: portable C++ CIOS, used by the library's own host-side tail
// (final point normalisation) and by the host unit tests of the EC formulas.
#pragma once
#include <stdint.h>
#include "fp_ptx.cuh"

#if defined(__CUDACC__)
#define HD __host__ __device__ __forceinline__
#define DEV __device__ __forceinline__
#else
#define HD inline
#define DEV inline
#endif

namespace b200 {

struct FrTag {
    static constexpr uint32_t INV = 0xefffffffu;
    HD static uint32_t mod(int i) {
        constexpr uint32_t M[8] = {0xf0000001u, 0x43e1f593u, 0x79b97091u, 0x2833e848u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
        return M[i];
    }
    HD static uint32_t one(int i) {   // R mod r
        constexpr uint32_t V[8] = {0x4ffffffbu, 0xac96341cu, 0x9f60cd29u, 0x36fc7695u, 0x7879462eu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u};
        return V[i];
    }
    HD static uint32_t r2(int i) {    // R^2 mod r
        constexpr uint32_t V[8] = {0xae216da7u, 0x1bb8e645u, 0xe35c59e3u, 0x53fe3ab1u, 0x53bb8085u, 0x8c49833du, 0x7f4e44a5u, 0x0216d0b1u};
        return V[i];
    }
};
struct FqTag {
    static constexpr uint32_t INV = 0xe4866389u;
    HD static uint32_t mod(int i) {
        constexpr uint32_t M[8] = {0xd87cfd47u, 0x3c208c16u, 0x6871ca8du, 0x97816a91u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
        return M[i];
    }
    HD static uint32_t one(int i) {   // R mod p
        constexpr uint32_t V[8] = {0xc58f0d9du, 0xd35d438du, 0xf5c70b3du, 0x0a78eb28u, 0x7879462cu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u};
        return V[i];
    }
    HD static uint32_t r2(int i) {    // R^2 mod p
        constexpr uint32_t V[8] = {0x538afa89u, 0xf32cfc5bu, 0xd44501fbu, 0xb5e71911u, 0x0a417ff6u, 0x47ab1effu, 0xcab8351fu, 0x06d89f71u};
        return V[i];
    }
};

// ------------------------------------------------------------------------------------------------------
// The element type.  alignas(16): global loads/stores are two 128-bit transactions per element.
template <class Tag>
struct alignas(16) Fp {
    uint32_t l[8];
};
using Fr = Fp<FrTag>;
using Fq = Fp<FqTag>;

// ---- portable implementations (host; fp_mul_portable also runs on the device in debug.cu's k_bench_mul<2>) ----------
template <class Tag>
HD void fp_mul_portable(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    uint32_t t[10];
#pragma unroll
    for (int i = 0; i < 10; ++i) t[i] = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        uint64_t c = 0, s;
#pragma unroll
        for (int j = 0; j < 8; ++j) { s = (uint64_t)a[j] * b[i] + t[j] + c; t[j] = (uint32_t)s; c = s >> 32; }
        s = (uint64_t)t[8] + c; t[8] = (uint32_t)s; t[9] = (uint32_t)(s >> 32);
        uint32_t m = t[0] * Tag::INV;
        c = ((uint64_t)m * Tag::mod(0) + t[0]) >> 32;
#pragma unroll
        for (int j = 1; j < 8; ++j) { s = (uint64_t)m * Tag::mod(j) + t[j] + c; t[j - 1] = (uint32_t)s; c = s >> 32; }
        s = (uint64_t)t[8] + c; t[7] = (uint32_t)s; t[8] = t[9] + (uint32_t)(s >> 32);
    }
    // t < 2M: conditional subtract
    uint32_t d[8]; uint64_t br = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { uint64_t s = (uint64_t)t[j] - Tag::mod(j) - br; d[j] = (uint32_t)s; br = (s >> 32) & 1; }
    bool ge = (t[8] != 0) || (br == 0);
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = ge ? d[j] : t[j];
}
template <class Tag>
HD void fp_add_portable(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    uint32_t t[8], d[8]; uint64_t c = 0, br = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { uint64_t s = (uint64_t)a[j] + b[j] + c; t[j] = (uint32_t)s; c = s >> 32; }
#pragma unroll
    for (int j = 0; j < 8; ++j) { uint64_t s = (uint64_t)t[j] - Tag::mod(j) - br; d[j] = (uint32_t)s; br = (s >> 32) & 1; }
    bool ge = (br == 0);
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = ge ? d[j] : t[j];
}
template <class Tag>
HD void fp_sub_portable(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    uint32_t t[8]; uint64_t br = 0, c = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { uint64_t s = (uint64_t)a[j] - b[j] - br; t[j] = (uint32_t)s; br = (s >> 32) & 1; }
    uint32_t mask = br ? 0xffffffffu : 0u;
#pragma unroll
    for (int j = 0; j < 8; ++j) { uint64_t s = (uint64_t)t[j] + (Tag::mod(j) & mask) + c; r[j] = (uint32_t)s; c = s >> 32; }
}

// ---- dispatch ----------------------------------------------------------------------------------------------
template <class Tag> struct PtxOps;
#if defined(__CUDA_ARCH__)
template <> struct PtxOps<FrTag> {
    DEV static void mul(uint32_t* r, const uint32_t* a, const uint32_t* b) { fr_mul_ptx(r, a, b); }
    DEV static void add(uint32_t* r, const uint32_t* a, const uint32_t* b) { fr_add_ptx(r, a, b); }
    DEV static void sub(uint32_t* r, const uint32_t* a, const uint32_t* b) { fr_sub_ptx(r, a, b); }
    DEV static void mul2(uint32_t* r, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d) { fr_mul2_ptx(r, a, b, c, d); }
    DEV static void sqr(uint32_t* r, const uint32_t* a) { fr_sqr_ptx(r, a); }
};
template <> struct PtxOps<FqTag> {
    DEV static void mul(uint32_t* r, const uint32_t* a, const uint32_t* b) { fq_mul_ptx(r, a, b); }
    DEV static void add(uint32_t* r, const uint32_t* a, const uint32_t* b) { fq_add_ptx(r, a, b); }
    DEV static void sub(uint32_t* r, const uint32_t* a, const uint32_t* b) { fq_sub_ptx(r, a, b); }
    DEV static void mul2(uint32_t* r, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d) { fq_mul2_ptx(r, a, b, c, d); }
    DEV static void sqr(uint32_t* r, const uint32_t* a) { fq_sqr_ptx(r, a); }
};
#endif

template <class Tag> HD Fp<Tag> operator*(const Fp<Tag>& a, const Fp<Tag>& b) {
    Fp<Tag> r;
#if defined(__CUDA_ARCH__)
    PtxOps<Tag>::mul(r.l, a.l, b.l);
#else
    fp_mul_portable<Tag>(r.l, a.l, b.l);
#endif
    return r;
}
template <class Tag> HD Fp<Tag> operator+(const Fp<Tag>& a, const Fp<Tag>& b) {
    Fp<Tag> r;
#if defined(__CUDA_ARCH__)
    PtxOps<Tag>::add(r.l, a.l, b.l);
#else
    fp_add_portable<Tag>(r.l, a.l, b.l);
#endif
    return r;
}
template <class Tag> HD Fp<Tag> operator-(const Fp<Tag>& a, const Fp<Tag>& b) {
    Fp<Tag> r;
#if defined(__CUDA_ARCH__)
    PtxOps<Tag>::sub(r.l, a.l, b.l);
#else
    fp_sub_portable<Tag>(r.l, a.l, b.l);
#endif
    return r;
}
// dedicated squaring on the device (fp_gen.py: gen_sqr, 36 limb products instead of 64); the host build computes a * a
template <class Tag> HD Fp<Tag> fp_sqr(const Fp<Tag>& a) {
#if defined(__CUDA_ARCH__)
    Fp<Tag> r;
    PtxOps<Tag>::sqr(r.l, a.l);
    return r;
#else
    return a * a;
#endif
}
template <class Tag> HD Fp<Tag> fp_dbl(const Fp<Tag>& a) { return a + a; }
template <class Tag> HD Fp<Tag> fp_zero() {
    Fp<Tag> r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = 0;
    return r;
}
template <class Tag> HD Fp<Tag> fp_one() {
    Fp<Tag> r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = Tag::one(i);
    return r;
}
template <class Tag> HD bool fp_is_zero(const Fp<Tag>& a) {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) o |= a.l[i];
    return o == 0;
}
template <class Tag> HD bool fp_eq(const Fp<Tag>& a, const Fp<Tag>& b) {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) o |= a.l[i] ^ b.l[i];
    return o == 0;
}
template <class Tag> HD Fp<Tag> fp_neg(const Fp<Tag>& a) { return fp_zero<Tag>() - a; }
// the 8 limbs, read as one 256-bit integer, are below the modulus: the encoding check of halo2curves' from_raw_bytes, for Fr and Fq alike
template <class Tag> HD bool fp_is_canonical(const Fp<Tag>& a) {
#pragma unroll
    for (int i = 7; i >= 0; --i) if (a.l[i] != Tag::mod(i)) return a.l[i] < Tag::mod(i);
    return false;
}
// a*b + c*d and a*b - c*d with ONE Montgomery reduction on the device (fp_gen.py: gen_mul2, 466 instructions against
// 312 + 312 + 25); the host build composes them from the single-product operators.
template <class Tag> HD Fp<Tag> fp_muladd2(const Fp<Tag>& a, const Fp<Tag>& b, const Fp<Tag>& c, const Fp<Tag>& d) {
#if defined(__CUDA_ARCH__)
    Fp<Tag> r;
    PtxOps<Tag>::mul2(r.l, a.l, b.l, c.l, d.l);
    return r;
#else
    return a * b + c * d;
#endif
}
template <class Tag> HD Fp<Tag> fp_mulsub2(const Fp<Tag>& a, const Fp<Tag>& b, const Fp<Tag>& c, const Fp<Tag>& d) {
#if defined(__CUDA_ARCH__)
    return fp_muladd2(a, b, fp_neg(c), d);
#else
    return a * b - c * d;
#endif
}
// Montgomery <-> canonical
template <class Tag> HD Fp<Tag> fp_from_mont(const Fp<Tag>& a) {
    Fp<Tag> one_c = fp_zero<Tag>(); one_c.l[0] = 1;
    return a * one_c;
}
template <class Tag> HD Fp<Tag> fp_to_mont(const Fp<Tag>& a) {
    Fp<Tag> r2;
#pragma unroll
    for (int i = 0; i < 8; ++i) r2.l[i] = Tag::r2(i);
    return a * r2;
}
// a^(M-2) (Fermat); 0 -> 0.  Not unrolled: ~380 multiplications, used off the hot loops only.
template <class Tag> HD Fp<Tag> fp_inv(const Fp<Tag>& a) {
    uint32_t e[8];
    {
        uint64_t br = 2;   // e = M - 2
        for (int i = 0; i < 8; ++i) { uint64_t s = (uint64_t)Tag::mod(i) - br; e[i] = (uint32_t)s; br = (s >> 32) & 1; }
    }
    Fp<Tag> acc = fp_one<Tag>();
#pragma unroll 1
    for (int i = 253; i >= 0; --i) {
        acc = acc * acc;
        if ((e[i >> 5] >> (i & 31)) & 1) acc = acc * a;
    }
    return acc;
}
// small power, exponent as u64 (square-and-multiply)
template <class Tag> HD Fp<Tag> fp_pow_u64(const Fp<Tag>& a, uint64_t e) {
    Fp<Tag> acc = fp_one<Tag>();
#pragma unroll 1
    for (int i = 63; i >= 0; --i) {
        acc = acc * acc;
        if ((e >> i) & 1) acc = acc * a;
    }
    return acc;
}

#if defined(__CUDACC__)
// 2 x 128-bit global accesses per element
template <class Tag> DEV Fp<Tag> fp_load(const Fp<Tag>* p) {
    Fp<Tag> r;
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 lo = q[0], hi = q[1];
    r.l[0] = lo.x; r.l[1] = lo.y; r.l[2] = lo.z; r.l[3] = lo.w;
    r.l[4] = hi.x; r.l[5] = hi.y; r.l[6] = hi.z; r.l[7] = hi.w;
    return r;
}
template <class Tag> DEV void fp_store(Fp<Tag>* p, const Fp<Tag>& v) {
    uint4* q = reinterpret_cast<uint4*>(p);
    q[0] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
    q[1] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}
#endif

}  // namespace b200
