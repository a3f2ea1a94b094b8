// field.cuh — 255-bit Pasta field arithmetic for sm_90a: 8 x u32 limbs, Montgomery form (R = 2^256).
//
// Replaces, on the device, what the reference gets from ark-ff's Fp256<MontBackend<_,4>> (crate not in the
// reference tree; constants from curves/src/pasta/fields/fp.rs:8-80 and fq.rs:8-79).  The in-memory format is
// identical to the reference's: 4 x u64 little-endian Montgomery limbs == 8 x u32 little-endian limbs.
//
// Multiplication is a word-serial Montgomery product on two carry-save accumulators P ("aligned with limb 0")
// and S ("aligned with limb 1"): products of the even limbs of a with b_i tile P in contiguous 64-bit slots, the
// odd limbs tile S, so every row is one mad.lo.cc/madc.hi.cc carry chain, which ptxas fuses pairwise into
// IMAD.WIDE.U32(.X) — 4 per chain.  Both Pasta moduli have the shape
//      m = 1 + m1*2^32 + m2*2^64 + m3*2^96 + 2^254        (limbs 4..6 zero, limb 7 = 2^30, m == 1 mod 2^32)
// so -m^{-1} mod 2^32 = 2^32-1 (the quotient digit is just -t0, no multiply) and a reduction row needs only
// four wide multiplies (m1, m2, m3, 2^30) instead of eight.
//
// Every primitive below is also compiled for the HOST (carry flag emulated in a thread-local) so that the exact
// instruction sequences can be unit-tested on a machine without a GPU (tests/test_device_math_host.py).
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define ZK_HD __host__ __device__ __forceinline__
#define ZK_HDC __host__ __device__ constexpr
#define ZK_D __device__ __forceinline__
#else
#define ZK_HD inline
#define ZK_HDC constexpr
#define ZK_D inline
#endif

namespace zkb {

// ------------------------------------------------------------------------------------------------ carry chains
#if defined(__CUDA_ARCH__)
#define ZK_ASM asm volatile
ZK_D uint32_t add_cc(uint32_t a, uint32_t b) { uint32_t r; ZK_ASM("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
ZK_D uint32_t addc_cc(uint32_t a, uint32_t b) { uint32_t r; ZK_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
ZK_D uint32_t addc(uint32_t a, uint32_t b) { uint32_t r; ZK_ASM("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
ZK_D uint32_t sub_cc(uint32_t a, uint32_t b) { uint32_t r; ZK_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
ZK_D uint32_t subc_cc(uint32_t a, uint32_t b) { uint32_t r; ZK_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
ZK_D uint32_t subc(uint32_t a, uint32_t b) { uint32_t r; ZK_ASM("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
ZK_D uint32_t mul_lo(uint32_t a, uint32_t b) { uint32_t r; ZK_ASM("mul.lo.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
ZK_D uint32_t mul_hi(uint32_t a, uint32_t b) { uint32_t r; ZK_ASM("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
// plain 64-bit product unpacked into halves: ptxas keeps it a stand-alone IMAD.WIDE.U32 (a mul.lo/mul.hi pair followed by
// carry adds is re-fused into the carry-chained IMAD.WIDE.U32.X)
ZK_D void mul_wide_split(uint32_t a, uint32_t b, uint32_t& lo, uint32_t& hi) {
    uint64_t t;
    ZK_ASM("mul.wide.u32 %0, %1, %2;" : "=l"(t) : "r"(a), "r"(b));
    ZK_ASM("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(t));
}
ZK_D uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; ZK_ASM("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
ZK_D uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; ZK_ASM("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
ZK_D uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; ZK_ASM("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
ZK_D uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; ZK_ASM("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
#else
// Host emulation of the PTX condition-code carry flag (CC.CF): same semantics, one flag per thread.
inline uint32_t& zk_cf() { static thread_local uint32_t cf = 0; return cf; }
inline uint32_t add_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b; zk_cf() = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t addc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b + zk_cf(); zk_cf() = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t addc(uint32_t a, uint32_t b) { return (uint32_t)((uint64_t)a + b + zk_cf()); }
// PTX: sub.cc writes CF = borrow; subc consumes it as borrow-in
inline uint32_t sub_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b; zk_cf() = (uint32_t)((t >> 32) & 1); return (uint32_t)t; }
inline uint32_t subc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b - zk_cf(); zk_cf() = (uint32_t)((t >> 32) & 1); return (uint32_t)t; }
inline uint32_t subc(uint32_t a, uint32_t b) { return (uint32_t)((uint64_t)a - b - zk_cf()); }
inline uint32_t mul_lo(uint32_t a, uint32_t b) { return (uint32_t)((uint64_t)a * b); }
inline uint32_t mul_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline void mul_wide_split(uint32_t a, uint32_t b, uint32_t& lo, uint32_t& hi) { uint64_t t = (uint64_t)a * b; lo = (uint32_t)t; hi = (uint32_t)(t >> 32); }
inline uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (uint64_t)mul_lo(a, b) + c; zk_cf() = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (uint64_t)mul_lo(a, b) + c + zk_cf(); zk_cf() = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (uint64_t)mul_hi(a, b) + c + zk_cf(); zk_cf() = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { return (uint32_t)((uint64_t)mul_hi(a, b) + c + zk_cf()); }
#endif

// ------------------------------------------------------------------------------------------------ field parameters
// Limbs are 32-bit little-endian views of the 4 x u64 constants in the reference.
struct FpParams {  // curves/src/pasta/fields/fp.rs:31-50
    static constexpr uint32_t M1 = 0x992d30edu, M2 = 0x094cf91bu, M3 = 0x224698fcu;
    static ZK_HDC uint32_t R(int i) {
        constexpr uint32_t t[8] = {0xfffffffdu, 0x34786d38u, 0xe41914adu, 0x992c350bu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x3fffffffu};
        return t[i];
    }
    static ZK_HDC uint32_t R2(int i) {
        constexpr uint32_t t[8] = {0x0000000fu, 0x8c78ecb3u, 0x8b0de0e7u, 0xd7d30dbdu, 0xc3c95d18u, 0x7797a99bu, 0x7b9cb714u, 0x096d41afu};
        return t[i];
    }
    // 2^32-th root of unity 5^T, Montgomery form (fp.rs:24-27)
    static ZK_HDC uint32_t ROOT(int i) {
        constexpr uint32_t t[8] = {0xbad6dbf0u, 0xa28db849u, 0xd3b539dfu, 0x9083cd03u, 0x9dc8448eu, 0xfba6b9cau, 0x7b89c6dau, 0x3ec92874u};
        return t[i];
    }
};
struct FqParams {  // curves/src/pasta/fields/fq.rs:29-48
    static constexpr uint32_t M1 = 0x8c46eb21u, M2 = 0x0994a8ddu, M3 = 0x224698fcu;
    static ZK_HDC uint32_t R(int i) {
        constexpr uint32_t t[8] = {0xfffffffdu, 0x5b2b3e9cu, 0xe3420567u, 0x992c350bu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x3fffffffu};
        return t[i];
    }
    static ZK_HDC uint32_t R2(int i) {
        constexpr uint32_t t[8] = {0x0000000fu, 0xfc9678ffu, 0x891a16e3u, 0x67bb433du, 0x04ccf590u, 0x7fae2310u, 0x7ccfdaa9u, 0x096d41afu};
        return t[i];
    }
    static ZK_HDC uint32_t ROOT(int i) {
        constexpr uint32_t t[8] = {0x8c9942deu, 0x21807742u, 0x21b60494u, 0xcc495789u, 0xb2efbee2u, 0xac2e5d27u, 0x7f2db056u, 0x0b79fa89u};
        return t[i];
    }
};
constexpr uint32_t M7 = 0x40000000u;  // both fields: bit 254

struct alignas(16) fe {
    uint32_t v[8];
};

template <class F> ZK_HD fe fe_one() {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = F::R(i);
    return r;
}
template <class F> ZK_HD fe fe_r2() {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = F::R2(i);
    return r;
}
ZK_HD fe fe_zero() {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = 0;
    return r;
}
ZK_HD bool fe_is_zero(const fe& a) {
    return (a.v[0] | a.v[1] | a.v[2] | a.v[3] | a.v[4] | a.v[5] | a.v[6] | a.v[7]) == 0;
}
ZK_HD bool fe_eq(const fe& a, const fe& b) {
    uint32_t d = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) d |= a.v[i] ^ b.v[i];
    return d == 0;
}

// r = (t >= m) ? t - m : t     (t < 2m)
template <class F> ZK_HD void fe_cond_sub(fe& t) {
    uint32_t d[8];
    d[0] = sub_cc(t.v[0], 1u);
    d[1] = subc_cc(t.v[1], F::M1);
    d[2] = subc_cc(t.v[2], F::M2);
    d[3] = subc_cc(t.v[3], F::M3);
    d[4] = subc_cc(t.v[4], 0u);
    d[5] = subc_cc(t.v[5], 0u);
    d[6] = subc_cc(t.v[6], 0u);
    d[7] = subc_cc(t.v[7], M7);
    uint32_t borrow = subc(0u, 0u);  // 0xffffffff if t < m
#pragma unroll
    for (int i = 0; i < 8; i++) t.v[i] = borrow ? t.v[i] : d[i];
}

// a < m ?  (is the 256-bit integer a canonical field element)
template <class F> ZK_HD bool fe_lt_modulus(const fe& a) {
    const uint32_t m[8] = {1u, F::M1, F::M2, F::M3, 0u, 0u, 0u, M7};
    for (int i = 7; i >= 0; i--) {
        if (a.v[i] != m[i]) return a.v[i] < m[i];
    }
    return false;
}

template <class F> ZK_HD fe fe_add(const fe& a, const fe& b) {
    fe r;
    r.v[0] = add_cc(a.v[0], b.v[0]);
#pragma unroll
    for (int i = 1; i < 7; i++) r.v[i] = addc_cc(a.v[i], b.v[i]);
    r.v[7] = addc(a.v[7], b.v[7]);  // a + b < 2^256
    fe_cond_sub<F>(r);
    return r;
}

template <class F> ZK_HD fe fe_sub(const fe& a, const fe& b) {
    fe r;
    r.v[0] = sub_cc(a.v[0], b.v[0]);
#pragma unroll
    for (int i = 1; i < 8; i++) r.v[i] = subc_cc(a.v[i], b.v[i]);
    uint32_t mask = subc(0u, 0u);  // all ones if a < b
    r.v[0] = add_cc(r.v[0], 1u & mask);
    r.v[1] = addc_cc(r.v[1], F::M1 & mask);
    r.v[2] = addc_cc(r.v[2], F::M2 & mask);
    r.v[3] = addc_cc(r.v[3], F::M3 & mask);
    r.v[4] = addc_cc(r.v[4], 0u);
    r.v[5] = addc_cc(r.v[5], 0u);
    r.v[6] = addc_cc(r.v[6], 0u);
    r.v[7] = addc(r.v[7], M7 & mask);
    return r;
}

template <class F> ZK_HD fe fe_neg(const fe& a) {
    if (fe_is_zero(a)) return a;
    fe r;
    r.v[0] = sub_cc(1u, a.v[0]);
    r.v[1] = subc_cc(F::M1, a.v[1]);
    r.v[2] = subc_cc(F::M2, a.v[2]);
    r.v[3] = subc_cc(F::M3, a.v[3]);
    r.v[4] = subc_cc(0u, a.v[4]);
    r.v[5] = subc_cc(0u, a.v[5]);
    r.v[6] = subc_cc(0u, a.v[6]);
    r.v[7] = subc(M7, a.v[7]);
    return r;
}

template <class F> ZK_HD fe fe_dbl(const fe& a) { return fe_add<F>(a, a); }

// One Montgomery reduction row on the carry-save pair (P, S):  t += q*m with q = -t0, making P[0] == 0.
//   chain alpha: P0 + q (carry is worth S0), q*m1 -> S0:S1, q*m3 -> S2:S3, q*2^30 -> S6:S7 (shifts)
//   chain beta : q*m2 -> P2:P3, carry rippled to P8
template <class F> ZK_HD void mont_reduce_row(uint32_t (&P)[9], uint32_t (&S)[9]) {
    // q = -P0 through sub.cc (flag unused): a plain negation gets folded by ptxas into the low half of the next
    // multiply (p0 * -m1), which splits every IMAD.WIDE of the row into IMAD + IMAD.HI (checked in SASS).
    uint32_t q = sub_cc(0u, P[0]);
    (void)add_cc(P[0], q);
    S[0] = madc_lo_cc(q, F::M1, S[0]);
    S[1] = madc_hi_cc(q, F::M1, S[1]);
    S[2] = madc_lo_cc(q, F::M3, S[2]);
    S[3] = madc_hi_cc(q, F::M3, S[3]);
    S[4] = addc_cc(S[4], 0u);
    S[5] = addc_cc(S[5], 0u);
    S[6] = addc_cc(S[6], q << 30);   // q * 2^30 with two shifts: keeps the (quarter-rate) IMAD.WIDE pipe for real products
    S[7] = addc_cc(S[7], q >> 2);
    S[8] = addc(S[8], 0u);
    P[2] = mad_lo_cc(q, F::M2, P[2]);
    P[3] = madc_hi_cc(q, F::M2, P[3]);
    P[4] = addc_cc(P[4], 0u);
    P[5] = addc_cc(P[5], 0u);
    P[6] = addc_cc(P[6], 0u);
    P[7] = addc_cc(P[7], 0u);
    P[8] = addc(P[8], 0u);
}

// ZK_MUL_PLAIN_PER_ROW — pipe-balancing experiment prepared for the next GPU round (DESIGN.md "next levers"); 0 = the shipped,
// measured form (the macro below then expands to exactly the original instruction sequence).  K = 1..6: the K highest products
// a_j * b_i of every row (j = 7, 6, 5, ...) become PLAIN wide multiplies — cheaper on the FMA pipe than the carry-chained form
// (tools/ubench/pipes.cu measures both), and off the carry chains — added in with two carry adds each on the ALU pipe.  Bit-exact in
// every setting (tests/test_device_math_host.py builds them all).
#ifndef ZK_MUL_PLAIN_PER_ROW
#define ZK_MUL_PLAIN_PER_ROW 0
#endif

// Montgomery product a*b/R mod m, fully reduced.  Inputs < m.
template <class F> ZK_HD fe fe_mul(const fe& a, const fe& b) {
    uint32_t P[9], S[9];
    // row 0: P = a_even * b0, S = a_odd * b0
    {
        const uint32_t bi = b.v[0];
        P[0] = mul_lo(a.v[0], bi); P[1] = mul_hi(a.v[0], bi);
        P[2] = mul_lo(a.v[2], bi); P[3] = mul_hi(a.v[2], bi);
        P[4] = mul_lo(a.v[4], bi); P[5] = mul_hi(a.v[4], bi);
        P[6] = mul_lo(a.v[6], bi); P[7] = mul_hi(a.v[6], bi);
        P[8] = 0;
        S[0] = mul_lo(a.v[1], bi); S[1] = mul_hi(a.v[1], bi);
        S[2] = mul_lo(a.v[3], bi); S[3] = mul_hi(a.v[3], bi);
        S[4] = mul_lo(a.v[5], bi); S[5] = mul_hi(a.v[5], bi);
        S[6] = mul_lo(a.v[7], bi); S[7] = mul_hi(a.v[7], bi);
        S[8] = 0;
    }
    mont_reduce_row<F>(P, S);
#pragma unroll
    for (int i = 1; i < 8; i++) {
        // shift right one limb: t' = S + P1 + (P[2..8] << 32); then t' += a * b_i
        const uint32_t bi = b.v[i];
        uint32_t nP[9], nS[9];
#if ZK_MUL_PLAIN_PER_ROW > 0
        // products a_j * b_i, j >= 8 - ZK_MUL_PLAIN_PER_ROW, as stand-alone wide multiplies (off the carry chains)
        uint32_t tl[8], th[8];
#pragma unroll
        for (int j = 8 - ZK_MUL_PLAIN_PER_ROW; j < 8; j++) mul_wide_split(a.v[j], bi, tl[j], th[j]);
#define ZK_ROW_PAIR(dst, k, j, add_lo, add_hi)                                                   \
        if (j >= 8 - ZK_MUL_PLAIN_PER_ROW) { dst[k] = addc_cc(tl[j], add_lo); dst[k + 1] = addc_cc(th[j], add_hi); } \
        else { dst[k] = madc_lo_cc(a.v[j], bi, add_lo); dst[k + 1] = madc_hi_cc(a.v[j], bi, add_hi); }
#else
#define ZK_ROW_PAIR(dst, k, j, add_lo, add_hi) { dst[k] = madc_lo_cc(a.v[j], bi, add_lo); dst[k + 1] = madc_hi_cc(a.v[j], bi, add_hi); }
#endif
        nP[0] = add_cc(S[0], P[1]);                  // carry is worth nS[0]
        ZK_ROW_PAIR(nS, 0, 1, P[2], P[3])
        ZK_ROW_PAIR(nS, 2, 3, P[4], P[5])
        ZK_ROW_PAIR(nS, 4, 5, P[6], P[7])
        ZK_ROW_PAIR(nS, 6, 7, P[8], 0u)
        nS[8] = addc(0u, 0u);
        nP[0] = mad_lo_cc(a.v[0], bi, nP[0]);
        nP[1] = madc_hi_cc(a.v[0], bi, S[1]);
        ZK_ROW_PAIR(nP, 2, 2, S[2], S[3])
        ZK_ROW_PAIR(nP, 4, 4, S[4], S[5])
        ZK_ROW_PAIR(nP, 6, 6, S[6], S[7])
        nP[8] = addc(S[8], 0u);
#undef ZK_ROW_PAIR
        mont_reduce_row<F>(nP, nS);
#pragma unroll
        for (int k = 0; k < 9; k++) { P[k] = nP[k]; S[k] = nS[k]; }
    }
    // final shift: r = S + P1 + (P[2..8] << 32)  (< 2m < 2^256)
    fe r;
    r.v[0] = add_cc(S[0], P[1]);
    r.v[1] = addc_cc(S[1], P[2]);
    r.v[2] = addc_cc(S[2], P[3]);
    r.v[3] = addc_cc(S[3], P[4]);
    r.v[4] = addc_cc(S[4], P[5]);
    r.v[5] = addc_cc(S[5], P[6]);
    r.v[6] = addc_cc(S[6], P[7]);
    r.v[7] = addc(S[7], P[8]);
    fe_cond_sub<F>(r);
    return r;
}

template <class F> ZK_HD fe fe_sqr(const fe& a) { return fe_mul<F>(a, a); }

// Out-of-line product for the LATENCY-bound kernels (the reduction tails of the MSM run a handful of point additions per
// thread): a point addition with 14 inlined products is ~56 KB of straight-line code that every launch streams through a cold
// instruction cache; with the product behind a call it is ~3 KB plus one 4 KB body.  The throughput kernels keep the inlined form.
#if defined(__CUDACC__)
template <class F> __device__ __noinline__ fe fe_mul_call(fe a, fe b) { return fe_mul<F>(a, b); }
#else
template <class F> inline fe fe_mul_call(fe a, fe b) { return fe_mul<F>(a, b); }
#endif
// product selected by the code-size policy of the caller
template <class F, bool COMPACT> ZK_HD fe fe_mulx(const fe& a, const fe& b) {
#if defined(__CUDA_ARCH__)
    if (COMPACT) return fe_mul_call<F>(a, b);
#endif
    return fe_mul<F>(a, b);
}

// canonical integer (8 x u32) -> Montgomery and back (ark: from_bigint / into_bigint)
template <class F> ZK_HD fe fe_to_mont(const fe& a) { return fe_mul<F>(a, fe_r2<F>()); }
template <class F> ZK_HD fe fe_from_mont(const fe& a) {
    fe one = fe_zero();
    one.v[0] = 1;
    return fe_mul<F>(a, one);
}

// a^e for a small public exponent (square-and-multiply, MSB first)
template <class F> ZK_HD fe fe_pow_u64(const fe& a, uint64_t e) {
    fe acc = fe_one<F>();
    bool started = false;
    for (int i = 63; i >= 0; i--) {
        if (started) acc = fe_sqr<F>(acc);
        if ((e >> i) & 1) { acc = started ? fe_mul<F>(acc, a) : a; started = true; }
    }
    return acc;
}

// a^(m-2): Fermat inverse, 0 -> 0.  m - 2 = 2^254 + (m_low - 2).
template <class F> ZK_HD fe fe_inv(const fe& a) {
    // exponent limbs (32-bit LE) of m - 2
    const uint32_t e[8] = {0xffffffffu, F::M1 - 1u, F::M2, F::M3, 0u, 0u, 0u, M7};
    // (m0 = 1, so m - 2 borrows: limb0 = 0xffffffff, limb1 = M1 - 1)
    fe acc = fe_one<F>();
    bool started = false;
    for (int i = 255; i >= 0; i--) {
        if (started) acc = fe_sqr<F>(acc);
        if ((e[i >> 5] >> (i & 31)) & 1) { acc = started ? fe_mul<F>(acc, a) : a; started = true; }
    }
    return acc;
}

}  // namespace zkb
