// hash_to_curve.cuh — the generators of `SRS::create` (poly-commitment/src/ipa.rs:234-265, 561-590, 751-778): a point of
// y^2 = x^3 + 5 from a Blake2b-512 digest.  Three steps, each restated from its source:
//   blake2b_512        RFC 7693, unkeyed, 64-byte digest, a message of at most one 128-byte block
//   digest_to_field    point_of_random_bytes (ipa.rs:234-265): digest bytes 0..30 as bits[8i + j] = (d[i] >> j) & 1, read with
//                      BigInt::from_bits_be (bits[0] is the most significant bit), an element of the curve's base field
//   bw_to_group        BWParameters::to_group / get_xy (groupmap/src/lib.rs): the first of three candidate x whose x^3 + 5 has a
//                      square root, y the root Tonelli-Shanks returns (field_sqrt.cuh).  The Pasta cofactor is 1.
// Compiled for the host as well (tests/host_math/h2c_host.cpp), like field.cuh.
#pragma once
#include "field_sqrt.cuh"

namespace zkb {

// ------------------------------------------------------------------------------------------------ Blake2b-512
ZK_HDC uint64_t blake2b_iv(int i) {
    constexpr uint64_t t[8] = {0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                               0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull};
    return t[i];
}
// message word schedule of round r (rounds 10 and 11 repeat 0 and 1)
ZK_HDC int blake2b_sigma(int r, int k) {
    constexpr unsigned char t[10][16] = {
        {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
        {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
        {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
        {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
        {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0}};
    return t[r % 10][k];
}
ZK_HD uint64_t rotr64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }
ZK_HD void blake2b_g(uint64_t (&v)[16], int a, int b, int c, int d, uint64_t x, uint64_t y) {
    v[a] = v[a] + v[b] + x; v[d] = rotr64(v[d] ^ v[a], 32);
    v[c] = v[c] + v[d];     v[b] = rotr64(v[b] ^ v[c], 24);
    v[a] = v[a] + v[b] + y; v[d] = rotr64(v[d] ^ v[a], 16);
    v[c] = v[c] + v[d];     v[b] = rotr64(v[b] ^ v[c], 63);
}
// Blake2b-512 of a message of len <= 128 bytes, given as 16 little-endian words zero-padded past len; digest byte i is
// (h[i / 8] >> (8 * (i % 8))) & 0xff.  One compression, the final one.
ZK_HD void blake2b_512(const uint64_t (&m)[16], unsigned len, uint64_t (&h)[8]) {
    uint64_t v[16];
#pragma unroll
    for (int i = 0; i < 8; i++) { h[i] = blake2b_iv(i); v[i + 8] = blake2b_iv(i); }
    h[0] ^= 0x01010040ull;            // parameter block: digest length 64, key length 0, fanout 1, depth 1
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = h[i];
    v[12] ^= len;                     // byte counter t (< 2^64)
    v[14] = ~v[14];                   // final block
#pragma unroll
    for (int r = 0; r < 12; r++) {
        blake2b_g(v, 0, 4, 8, 12, m[blake2b_sigma(r, 0)], m[blake2b_sigma(r, 1)]);
        blake2b_g(v, 1, 5, 9, 13, m[blake2b_sigma(r, 2)], m[blake2b_sigma(r, 3)]);
        blake2b_g(v, 2, 6, 10, 14, m[blake2b_sigma(r, 4)], m[blake2b_sigma(r, 5)]);
        blake2b_g(v, 3, 7, 11, 15, m[blake2b_sigma(r, 6)], m[blake2b_sigma(r, 7)]);
        blake2b_g(v, 0, 5, 10, 15, m[blake2b_sigma(r, 8)], m[blake2b_sigma(r, 9)]);
        blake2b_g(v, 1, 6, 11, 12, m[blake2b_sigma(r, 10)], m[blake2b_sigma(r, 11)]);
        blake2b_g(v, 2, 7, 8, 13, m[blake2b_sigma(r, 12)], m[blake2b_sigma(r, 13)]);
        blake2b_g(v, 3, 4, 9, 14, m[blake2b_sigma(r, 14)], m[blake2b_sigma(r, 15)]);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] ^= v[i] ^ v[i + 8];
}

// ------------------------------------------------------------------------------------------------ digest -> base field
ZK_HD uint32_t brev32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __brev(x);
#else
    x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);
    x = ((x >> 2) & 0x33333333u) | ((x & 0x33333333u) << 2);
    x = ((x >> 4) & 0x0f0f0f0fu) | ((x & 0x0f0f0f0fu) << 4);
    x = ((x >> 8) & 0x00ff00ffu) | ((x & 0x00ff00ffu) << 8);
    return (x >> 16) | (x << 16);
#endif
}
// t = sum_{i < 31} rev8(d[i]) * 256^(30 - i), canonical (8 x u32 little-endian).  Bit 8i + j of the digest (little-endian bit
// order) is bit 247 - (8i + j) of t: t is the 248-bit reversal of the digest's low 31 bytes, i.e. the 256-bit reversal of
// those bytes shifted down by 8.  t < 2^248 < modulus, so from_bigint cannot fail.
ZK_HD fe digest_to_field(const uint64_t (&h)[8]) {
    uint32_t d[8];
#pragma unroll
    for (int k = 0; k < 4; k++) { d[2 * k] = (uint32_t)h[k]; d[2 * k + 1] = (uint32_t)(h[k] >> 32); }
    d[7] &= 0x00ffffffu;              // digest byte 31 is not used
    uint32_t r[8];
#pragma unroll
    for (int k = 0; k < 8; k++) r[k] = brev32(d[7 - k]);
    fe t;
#pragma unroll
    for (int k = 0; k < 7; k++) t.v[k] = (r[k] >> 8) | (r[k + 1] << 24);
    t.v[7] = r[7] >> 8;
    return t;
}

// ------------------------------------------------------------------------------------------------ BW group map
// BWParameters::setup for y^2 = x^3 + 5 (groupmap/src/lib.rs): u = 1 (the first u with u^3 + 5 != 0), fu = u^3 + 5 = 6, and
// inv_three_u_squared = 1 / (3 u^2), sqrt_neg_three_u_squared = sqrt(-3 u^2) (ark's root), sqrt_neg_three_u_squared_minus_u_over_2
// = (sqrt(-3 u^2) - u) / 2; Montgomery form, 32-bit little-endian limbs.  tests/test_h2c_host.py pins them to the derivation.
enum { BW_FU, BW_INV_THREE_U2, BW_SQRT_NEG_THREE_U2, BW_SQRT_NEG_THREE_U2_MINUS_U_OVER_2 };
struct BwFp {
    static ZK_HDC uint32_t C(int c, int i) {
        constexpr uint32_t t[4][8] = {
            {0xffffffe9u, 0x3cf09ab4u, 0x2a159e85u, 0xeba8415bu, 0xfffffffcu, 0xffffffffu, 0xffffffffu, 0x3fffffffu},
            {0x55555555u, 0x22464506u, 0xa791024cu, 0xf4932256u, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x3fffffffu},
            {0xc3342a76u, 0x9f4f7638u, 0x6dcd8aadu, 0xb3fde93eu, 0x90f48cccu, 0x54cedab9u, 0x4f42f0ecu, 0x2bb0093bu},
            {0x619a153du, 0x02021cf6u, 0x4980b78eu, 0x9e8c2697u, 0xc87a4666u, 0x2a676d5cu, 0xa7a17876u, 0x15d8049du}};
        return t[c][i];
    }
};
struct BwFq {
    static ZK_HDC uint32_t C(int c, int i) {
        constexpr uint32_t t[4][8] = {
            {0xffffffe9u, 0x65a0e008u, 0x23a4d418u, 0xeba8415bu, 0xfffffffcu, 0xffffffffu, 0xffffffffu, 0x3fffffffu},
            {0x55555555u, 0x7be85c4au, 0xa7791d0bu, 0xf4932256u, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x3fffffffu},
            {0x00222240u, 0xc78c8885u, 0x8787b03eu, 0xf7abb348u, 0x26b65651u, 0x0584ebf6u, 0x1048b620u, 0x243a53f1u},
            {0x80111122u, 0x7c541a84u, 0x56ed29dau, 0x40630b9cu, 0x135b2b29u, 0x02c275fbu, 0x88245b10u, 0x121d29f8u}};
        return t[c][i];
    }
};
template <class F> struct BwOf;
template <> struct BwOf<FpParams> { using type = BwFp; };
template <> struct BwOf<FqParams> { using type = BwFq; };

template <class F> ZK_HD fe bw_const(int c) {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = BwOf<F>::type::C(c, i);
    return r;
}

// to_group(t) (t Montgomery): (x, y) Montgomery.  alpha = 1 / (t^2 (t^2 + fu)), 0 when that product is 0 (fe_inv maps 0 to 0,
// as the reference's unwrap_or_else(zero)).  Returns false only if no candidate is on the curve, which the map rules out.
template <class F> ZK_HDT bool bw_to_group(const fe& t, fe& x_out, fe& y_out) {
    const fe u = fe_one<F>();
    const fe fu = bw_const<F>(BW_FU);
    const fe t2 = fe_sqr<F>(t);
    const fe t2_fu = fe_add<F>(t2, fu);
    const fe alpha = fe_inv<F>(fe_mul<F>(t2, t2_fu));
    // x1 = sqrt_neg_three_u_squared_minus_u_over_2 - t2^2 alpha sqrt_neg_three_u_squared
    const fe x1 = fe_sub<F>(bw_const<F>(BW_SQRT_NEG_THREE_U2_MINUS_U_OVER_2), fe_mul<F>(fe_mul<F>(fe_sqr<F>(t2), alpha), bw_const<F>(BW_SQRT_NEG_THREE_U2)));
    fe five = fe_zero();
    five.v[0] = 5;
    const fe b = fe_to_mont<F>(five);
    // one square root per attempt, the candidates in the reference's order: x1, x2 = -u - x1, x3 = u - (t2 + fu)^2 (alpha (t2 + fu)) / (3 u^2)
    fe x = x1;
    for (int k = 0; k < 3; k++) {
        if (k == 1) x = fe_sub<F>(fe_neg<F>(u), x1);
        if (k == 2)
            x = fe_sub<F>(u, fe_mul<F>(fe_mul<F>(fe_sqr<F>(t2_fu), fe_mul<F>(alpha, t2_fu)), bw_const<F>(BW_INV_THREE_U2)));
        if (fe_sqrt<F>(fe_add<F>(fe_mul<F>(fe_sqr<F>(x), x), b), y_out)) { x_out = x; return true; }
    }
    return false;
}

// point_of_random_bytes of a message of at most 128 bytes (16 little-endian words, zero-padded)
template <class F> ZK_HDT bool point_of_message(const uint64_t (&m)[16], unsigned len, fe& x, fe& y) {
    uint64_t h[8];
    blake2b_512(m, len, h);
    return bw_to_group<F>(fe_to_mont<F>(digest_to_field(h)), x, y);
}

}  // namespace zkb
