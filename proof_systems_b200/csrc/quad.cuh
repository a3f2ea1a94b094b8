// quad.cuh — latency-optimised XYZZ point addition: FOUR lanes cooperate on ONE addition.
//
// The reduction tails of the MSM (per-bucket sums of task partials, bit-sliced bucket sums) are chains of DEPENDENT
// point additions executed by very few warps; a serial add-2008-s is 14 field multiplications back to back (several
// microseconds at one warp per scheduler).  Its data-flow is only four multiplications deep, so a quad computes
//     stage 1   U1 = X1*ZZ2     U2 = X2*ZZ1     S1 = Y1*ZZZ2      S2 = Y2*ZZZ1
//     stage 2   PP = P^2        RR = R^2        ZZ12 = ZZ1*ZZ2    ZZZ12 = ZZZ1*ZZZ2        (P = U2-U1, R = S2-S1)
//     stage 3   PPP = P*PP      Q = U1*PP       ZZ3 = ZZ12*PP     W = ZZZ12*P
//     stage 4   (idle)          Ya = R*(Q-X3)   Yb = S1*PPP       ZZZ3 = W*PP              (X3 = RR-PPP-2Q, Y3 = Ya-Yb)
// one multiplication per lane per stage, operands exchanged with warp shuffles: ~3x lower latency for ~15% more work.
//
// Contract: the four lanes 4k..4k+3 of a quad hold IDENTICAL p and q and all receive the identical sum; EVERY lane of the
// warp must call the function (full-mask shuffles) — idle quads pass identities.  Identity operands and the exceptional
// cases P == Q / P == -Q are resolved after the shuffles (the latter by the serial formula; they are rare).
#pragma once
#include "common.cuh"

namespace zkb {

__device__ __forceinline__ fe sel_fe(bool c, const fe& a, const fe& b) {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = c ? a.v[i] : b.v[i];
    return r;
}

// COMPACT: the four stage products and the serial fall-back go through the out-of-line product (field.cuh).  Measured neutral
// to slightly worse for the quad kernels (unlike the serial per-bucket pass, msm.cu), so the default is the inlined form.
template <class F, bool COMPACT = false> __device__ __forceinline__ xyzz_t xyzz_add_quad(const xyzz_t& p, const xyzz_t& q) {
    const unsigned lane = threadIdx.x & 31, r = lane & 3, base = lane & ~3u;
    const bool r0 = r == 0, r1 = r == 1, r2 = r == 2, odd = (r & 1) != 0, lo = r < 2;
    // stage 1
    fe m1 = fe_mulx<F, COMPACT>(sel_fe(r0, p.X, sel_fe(r1, q.X, sel_fe(r2, p.Y, q.Y))),
                      sel_fe(r0, q.ZZ, sel_fe(r1, p.ZZ, sel_fe(r2, q.ZZZ, p.ZZZ))));  // U1 | U2 | S1 | S2
    fe o1 = shfl_xor_fe(m1, 1);
    fe d = odd ? fe_sub<F>(m1, o1) : fe_sub<F>(o1, m1);   // lanes 0,1: P = U2-U1      lanes 2,3: R = S2-S1
    fe d2 = shfl_xor_fe(d, 2);
    fe Pd = sel_fe(lo, d, d2), Rd = sel_fe(lo, d2, d);
    fe first = sel_fe(odd, o1, m1);                       // lanes 0,1: U1            lanes 2,3: S1
    // stage 2
    fe m2 = fe_mulx<F, COMPACT>(sel_fe(r0, Pd, sel_fe(r1, Rd, sel_fe(r2, p.ZZ, p.ZZZ))),
                      sel_fe(r0, Pd, sel_fe(r1, Rd, sel_fe(r2, q.ZZ, q.ZZZ))));      // PP | RR | ZZ12 | ZZZ12
    fe PP = shfl_fe(m2, base);
    // stage 3
    fe m3 = fe_mulx<F, COMPACT>(sel_fe(r0, Pd, sel_fe(r1, first, m2)), sel_fe(r == 3, Pd, PP));  // PPP | Q | ZZ3 | W
    fe PPP = shfl_fe(m3, base);
    fe X3 = fe_sub<F>(fe_sub<F>(m2, PPP), fe_dbl<F>(m3));  // meaningful in lane 1 (RR - PPP - 2Q)
    // stage 4
    fe m4 = fe_mulx<F, COMPACT>(sel_fe(lo, Rd, sel_fe(r2, first, m3)), sel_fe(lo, fe_sub<F>(m3, X3), sel_fe(r2, PPP, PP)));  // - | Ya | Yb | ZZZ3
    fe Yb = shfl_fe(m4, base + 2);
    fe Y3 = fe_sub<F>(m4, Yb);                             // meaningful in lane 1
    xyzz_t res;
    res.X = shfl_fe(X3, base + 1);
    res.Y = shfl_fe(Y3, base + 1);
    res.ZZ = shfl_fe(m3, base + 2);
    res.ZZZ = shfl_fe(m4, base + 3);
    // exceptional cases, uniform within the quad, no shuffles below this line
    const bool pinf = xyzz_is_inf(p), qinf = xyzz_is_inf(q);
    if (qinf) return p;
    if (pinf) return q;
    if (fe_is_zero(Pd)) return xyzz_add<F, COMPACT>(p, q);  // same x: doubling or identity
    return res;
}

// Block-wide sum of one partial per QUAD (replicated in its four lanes) through shared memory with re-compaction.
// blockDim.x a power of two in [32, 4 * capacity of sm]; sm holds blockDim.x / 4 points.  Result valid in quad 0.
template <class F> __device__ __forceinline__ xyzz_t block_tree_sum_quad(xyzz_t acc, xyzz_t* sm) {
    const unsigned tid = threadIdx.x, qd = tid >> 2, nq = blockDim.x >> 2;
    if ((tid & 3) == 0) store_xyzz(sm + qd, acc);
    __syncthreads();
#pragma unroll 1
    for (unsigned stride = nq >> 1; stride >= 1; stride >>= 1) {
        // a warp takes part while its first quad is live; its dead quads add identities so the shuffles stay uniform
        if (((tid & ~31u) >> 2) < stride) {
            xyzz_t o = qd < stride ? load_xyzz(sm + qd + stride) : xyzz_identity();
            acc = xyzz_add_quad<F>(acc, o);
            if ((tid & 3) == 0 && qd < stride) store_xyzz(sm + qd, acc);
        }
        __syncthreads();
    }
    return acc;  // valid in quad 0
}

}  // namespace zkb
