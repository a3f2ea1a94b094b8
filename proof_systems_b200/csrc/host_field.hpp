// host_field.hpp — host-side (CPU) Pasta field and XYZZ group arithmetic for the O(c) FINISHING steps of the MSM
// (the bit-sliced bucket sums come back from the GPU as c points; the host does the c doublings / additions that are
// strictly serial) and for into_affine() of results.  This is product code, independent of oracle/; it never sees more
// than a few hundred points per call and is not a fallback for any kernel.
//
// 4 x u64 Montgomery limbs, CIOS with unsigned __int128 (constants: curves/src/pasta/fields/fp.rs:31-50,80, fq.rs:29-48,79).
#pragma once
#include <cstdint>
#include <cstring>

namespace zkb {
namespace host {

struct HFp {
    static constexpr uint64_t M[4] = {0x992d30ed00000001ULL, 0x224698fc094cf91bULL, 0x0ULL, 0x4000000000000000ULL};
    static constexpr uint64_t R[4] = {0x34786d38fffffffdULL, 0x992c350be41914adULL, 0xffffffffffffffffULL, 0x3fffffffffffffffULL};
    static constexpr uint64_t R2[4] = {0x8c78ecb30000000fULL, 0xd7d30dbd8b0de0e7ULL, 0x7797a99bc3c95d18ULL, 0x096d41af7b9cb714ULL};
    static constexpr uint64_t INV = 11037532056220336127ULL;
    // 2^32-th root of unity 5^T, Montgomery form (fp.rs:24-27; field.cuh's FpParams::ROOT)
    static constexpr uint64_t ROOT[4] = {0xa28db849bad6dbf0ULL, 0x9083cd03d3b539dfULL, 0xfba6b9ca9dc8448eULL, 0x3ec928747b89c6daULL};
};
struct HFq {
    static constexpr uint64_t M[4] = {0x8c46eb2100000001ULL, 0x224698fc0994a8ddULL, 0x0ULL, 0x4000000000000000ULL};
    static constexpr uint64_t R[4] = {0x5b2b3e9cfffffffdULL, 0x992c350be3420567ULL, 0xffffffffffffffffULL, 0x3fffffffffffffffULL};
    static constexpr uint64_t R2[4] = {0xfc9678ff0000000fULL, 0x67bb433d891a16e3ULL, 0x7fae231004ccf590ULL, 0x096d41af7ccfdaa9ULL};
    static constexpr uint64_t INV = 10108024940646105087ULL;
    static constexpr uint64_t ROOT[4] = {0x218077428c9942deULL, 0xcc49578921b60494ULL, 0xac2e5d27b2efbee2ULL, 0x0b79fa897f2db056ULL};
};

struct hfe {
    uint64_t l[4];
};
typedef unsigned __int128 u128;

inline bool is_zero(const hfe& a) { return (a.l[0] | a.l[1] | a.l[2] | a.l[3]) == 0; }
template <class P> inline hfe one() { hfe r; memcpy(r.l, P::R, 32); return r; }
inline hfe zero() { hfe r; memset(r.l, 0, 32); return r; }

template <class P> inline bool geq_mod(const uint64_t* a) {
    for (int i = 3; i >= 0; i--) {
        if (a[i] > P::M[i]) return true;
        if (a[i] < P::M[i]) return false;
    }
    return true;
}
template <class P> inline void sub_mod(uint64_t* a) {
    uint64_t br = 0;
    for (int i = 0; i < 4; i++) {
        u128 d = (u128)a[i] - P::M[i] - br;
        a[i] = (uint64_t)d;
        br = (uint64_t)(d >> 64) & 1;
    }
}
template <class P> inline hfe add(const hfe& a, const hfe& b) {
    hfe r;
    u128 c = 0;
    for (int i = 0; i < 4; i++) { c += (u128)a.l[i] + b.l[i]; r.l[i] = (uint64_t)c; c >>= 64; }
    if (geq_mod<P>(r.l)) sub_mod<P>(r.l);
    return r;
}
template <class P> inline hfe sub(const hfe& a, const hfe& b) {
    hfe r;
    uint64_t br = 0;
    for (int i = 0; i < 4; i++) { u128 d = (u128)a.l[i] - b.l[i] - br; r.l[i] = (uint64_t)d; br = (uint64_t)(d >> 64) & 1; }
    if (br) {
        u128 c = 0;
        for (int i = 0; i < 4; i++) { c += (u128)r.l[i] + P::M[i]; r.l[i] = (uint64_t)c; c >>= 64; }
    }
    return r;
}
template <class P> inline hfe dbl(const hfe& a) { return add<P>(a, a); }
template <class P> inline hfe mul(const hfe& a, const hfe& b) {
    uint64_t t[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; i++) {
        u128 c = 0;
        for (int j = 0; j < 4; j++) { c += (u128)a.l[j] * b.l[i] + t[j]; t[j] = (uint64_t)c; c >>= 64; }
        c += t[4];
        t[4] = (uint64_t)c;
        t[5] = (uint64_t)(c >> 64);
        uint64_t q = t[0] * P::INV;
        c = ((u128)q * P::M[0] + t[0]) >> 64;
        for (int j = 1; j < 4; j++) { c += (u128)q * P::M[j] + t[j]; t[j - 1] = (uint64_t)c; c >>= 64; }
        c += t[4];
        t[3] = (uint64_t)c;
        t[4] = t[5] + (uint64_t)(c >> 64);
    }
    if (t[4] || geq_mod<P>(t)) sub_mod<P>(t);
    hfe r;
    memcpy(r.l, t, 32);
    return r;
}
template <class P> inline hfe sqr(const hfe& a) { return mul<P>(a, a); }
template <class P> inline hfe inv(const hfe& a) {
    uint64_t e[4];
    memcpy(e, P::M, 32);
    e[0] -= 2;
    hfe acc = one<P>();
    bool started = false;
    for (int i = 255; i >= 0; i--) {
        if (started) acc = sqr<P>(acc);
        if ((e[i / 64] >> (i % 64)) & 1) { acc = started ? mul<P>(acc, a) : a; started = true; }
    }
    return acc;
}
// a^e (square and multiply from the top bit; a^0 = 1)
template <class P> inline hfe pow_u64(const hfe& a, uint64_t e) {
    hfe acc = one<P>();
    for (int i = 63; i >= 0; i--) {
        acc = sqr<P>(acc);
        if ((e >> i) & 1) acc = mul<P>(acc, a);
    }
    return acc;
}
// the generator of the 2^log_n subgroup, (5^T)^(2^(32 - log_n)) (log_n <= 32): ark's Radix2EvaluationDomain group_gen, the same
// element the NTT tables are built from (ntt.cu)
template <class P> inline hfe root_of_unity(unsigned log_n) {
    hfe w;
    memcpy(w.l, P::ROOT, 32);
    for (unsigned i = log_n; i < 32; i++) w = sqr<P>(w);
    return w;
}

struct hxyzz { hfe X, Y, ZZ, ZZZ; };
struct haffine { hfe x, y; };
struct hjac { hfe X, Y, Z; };

inline hxyzz identity() { hxyzz r; r.X = r.Y = r.ZZ = r.ZZZ = zero(); return r; }
inline bool is_inf(const hxyzz& p) { return is_zero(p.ZZ); }

template <class P> inline hxyzz pdbl(const hxyzz& p) {
    if (is_inf(p)) return p;
    hfe U = dbl<P>(p.Y), V = sqr<P>(U), W = mul<P>(U, V), S = mul<P>(p.X, V);
    hfe xx = sqr<P>(p.X), M = add<P>(dbl<P>(xx), xx);
    hxyzz r;
    r.X = sub<P>(sqr<P>(M), dbl<P>(S));
    r.Y = sub<P>(mul<P>(M, sub<P>(S, r.X)), mul<P>(W, p.Y));
    r.ZZ = mul<P>(V, p.ZZ);
    r.ZZZ = mul<P>(W, p.ZZZ);
    return r;
}
template <class P> inline hxyzz padd(const hxyzz& p, const hxyzz& q) {
    if (is_inf(q)) return p;
    if (is_inf(p)) return q;
    hfe U1 = mul<P>(p.X, q.ZZ), U2 = mul<P>(q.X, p.ZZ), S1 = mul<P>(p.Y, q.ZZZ), S2 = mul<P>(q.Y, p.ZZZ);
    hfe Pd = sub<P>(U2, U1), Rd = sub<P>(S2, S1);
    if (is_zero(Pd)) {
        if (is_zero(Rd)) return pdbl<P>(p);
        return identity();
    }
    hfe PP = sqr<P>(Pd), PPP = mul<P>(Pd, PP), Q = mul<P>(U1, PP);
    hxyzz r;
    r.X = sub<P>(sub<P>(sqr<P>(Rd), PPP), dbl<P>(Q));
    r.Y = sub<P>(mul<P>(Rd, sub<P>(Q, r.X)), mul<P>(S1, PPP));
    r.ZZ = mul<P>(mul<P>(p.ZZ, q.ZZ), PP);
    r.ZZZ = mul<P>(mul<P>(p.ZZZ, q.ZZZ), PPP);
    return r;
}
template <class P> inline hxyzz from_affine(const haffine& a) {
    hxyzz r;
    if (is_zero(a.x) && is_zero(a.y)) return identity();
    r.X = a.x; r.Y = a.y; r.ZZ = one<P>(); r.ZZZ = one<P>();
    return r;
}
// into_affine(): x = X/ZZ, y = Y/ZZZ; identity -> (0, 0)
template <class P> inline haffine to_affine(const hxyzz& p) {
    haffine r;
    if (is_inf(p)) { r.x = zero(); r.y = zero(); return r; }
    hfe t = inv<P>(mul<P>(p.ZZ, p.ZZZ));
    r.x = mul<P>(p.X, mul<P>(t, p.ZZZ));
    r.y = mul<P>(p.Y, mul<P>(t, p.ZZ));
    return r;
}
// XYZZ -> Jacobian (X:Y:Z), x = X/Z^2, y = Y/Z^3, without inversion: Z = ZZZ, X' = X*ZZ^2 (ZZZ^2 = ZZ^3), Y' = Y*ZZZ^2.
// Identity -> (1, 1, 0), arkworks' Projective::zero().
template <class P> inline hjac to_jacobian(const hxyzz& p) {
    hjac r;
    if (is_inf(p)) { r.X = one<P>(); r.Y = one<P>(); r.Z = zero(); return r; }
    r.X = mul<P>(p.X, sqr<P>(p.ZZ));
    r.Y = mul<P>(p.Y, sqr<P>(p.ZZZ));
    r.Z = p.ZZZ;
    return r;
}
template <class P> inline hxyzz from_jacobian(const hjac& j) {
    hxyzz r;
    if (is_zero(j.Z)) return identity();
    r.X = j.X; r.Y = j.Y; r.ZZ = sqr<P>(j.Z); r.ZZZ = mul<P>(r.ZZ, j.Z);
    return r;
}
// [k]P, k canonical 4 x u64 (used for h * blinder in mask_custom: one scalar per commitment chunk)
template <class P> inline hxyzz scalar_mul(const hxyzz& p, const uint64_t k[4]) {
    hxyzz acc = identity();
    for (int i = 255; i >= 0; i--) {
        acc = pdbl<P>(acc);
        if ((k[i / 64] >> (i % 64)) & 1) acc = padd<P>(acc, p);
    }
    return acc;
}

}  // namespace host
}  // namespace zkb
