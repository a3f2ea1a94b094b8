// field_sqrt.cuh — the square root of ark-ff's Tonelli-Shanks (two-adicity 32, fp.rs:21 / fq.rs:19: the 2^32-th root of unity is
// the ROOT constant of field.cuh), step for step, so that it returns the same one of the two roots as the reference.  Shared by
// point decompression (decompress.cu) and SRS generation (srs_gen.cu); compiled for the host as well, like field.cuh.
#pragma once
#include "field.cuh"

#if defined(__CUDACC__)
#define ZK_HDT __host__ __device__
#else
#define ZK_HDT
#endif

namespace zkb {

// a^e for a 255-bit public exponent given as 8 x u32 (MSB first square-and-multiply)
template <class F> ZK_HDT fe fe_pow_256(const fe& a, const uint32_t (&e)[8]) {
    fe acc = fe_one<F>();
    bool started = false;
    for (int i = 255; i >= 0; i--) {
        if (started) acc = fe_sqr<F>(acc);
        if ((e[i >> 5] >> (i & 31)) & 1u) { acc = started ? fe_mul<F>(acc, a) : a; started = true; }
    }
    return acc;
}

// Square root in a field with m - 1 = 2^32 * T, T odd.  Returns false when a is a non-residue.
template <class F> ZK_HDT bool fe_sqrt(const fe& a, fe& out) {
    if (fe_is_zero(a)) { out = a; return true; }
    // (T - 1) / 2 where T = (m - 1) >> 32: from the modulus limbs {1, M1, M2, M3, 0, 0, 0, 2^30}
    const uint32_t T[8] = {F::M1, F::M2, F::M3, 0u, 0u, 0u, M7, 0u};
    uint32_t e[8];
#pragma unroll
    for (int i = 0; i < 8; i++) e[i] = (T[i] >> 1) | (i < 7 ? (T[i + 1] << 31) : 0u);   // T is odd: (T - 1) / 2 == T >> 1
    fe w = fe_pow_256<F>(a, e);       // a^((T-1)/2)
    fe x = fe_mul<F>(a, w);           // a^((T+1)/2)
    fe b = fe_mul<F>(x, w);           // a^T
    fe z;
#pragma unroll
    for (int i = 0; i < 8; i++) z.v[i] = F::ROOT(i);   // generator of the 2^32 subgroup
    const fe one = fe_one<F>();
    unsigned v = 32;
    while (!fe_eq(b, one)) {
        unsigned k = 0;
        fe b2 = b;
        while (!fe_eq(b2, one)) {
            b2 = fe_sqr<F>(b2);
            if (++k >= v) return false;   // b has order 2^v: a is not a square
        }
        fe ww = z;
        for (unsigned j = 0; j + k + 1 < v; j++) ww = fe_sqr<F>(ww);
        z = fe_sqr<F>(ww);
        b = fe_mul<F>(b, z);
        x = fe_mul<F>(x, ww);
        v = k;
    }
    out = x;
    return true;
}

}  // namespace zkb
