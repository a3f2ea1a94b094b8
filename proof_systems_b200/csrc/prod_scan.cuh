// prod_scan.cuh — the multiplicative prefix scan shared by the aggregation polynomials (perm.cu's z, lookup.cu's lookup
// aggregation): a block-level exclusive product and the one-CTA scan over the block totals.  A three-level scan is then three
// launches (per-block products, k_block_product_scan, apply), so no kernel waits on a flag another CTA writes.
#pragma once
#include "common.cuh"
#include "field.cuh"

namespace zkb {

// exclusive prefix product of v over the block's THREADS threads (thread 0 gets one); *total: the product over all of them.  Every
// thread of the block calls it.
template <class FS, unsigned THREADS> __device__ __forceinline__ fe block_exclusive_product(const fe& v, fe& total) {
    __shared__ fe warp_tot[THREADS / 32];
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    fe incl = v;
#pragma unroll
    for (unsigned d = 1; d < 32; d <<= 1) {
        const fe up = shfl_up_fe(incl, d);
        if (lane >= d) incl = fe_mul<FS>(incl, up);
    }
    fe excl = shfl_up_fe(incl, 1);
    if (lane == 0) excl = fe_one<FS>();
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    total = warp_tot[0];
#pragma unroll
    for (unsigned k = 1; k < THREADS / 32; k++) {
        if (k == warp) excl = fe_mul<FS>(excl, total);      // total is the product of the warps before this one here
        total = fe_mul<FS>(total, warp_tot[k]);
    }
    return excl;
}

// one block of THREADS: tot[b] <- product of tot[0 .. b - 1] (exclusive), each thread over a contiguous segment of the nb totals
template <class FS, unsigned THREADS> __global__ void __launch_bounds__(THREADS) k_block_product_scan(fe* tot, size_t nb) {
    const size_t per = (nb + THREADS - 1) / THREADS;
    const size_t b0 = threadIdx.x * per, b1 = b0 + per < nb ? b0 + per : nb;
    fe p = fe_one<FS>();
    for (size_t b = b0; b < b1; b++) p = fe_mul<FS>(p, load_fe(tot + b));
    fe all;
    fe run = block_exclusive_product<FS, THREADS>(p, all);
    for (size_t b = b0; b < b1; b++) {
        const fe v = load_fe(tot + b);
        store_fe(tot + b, run);
        run = fe_mul<FS>(run, v);
    }
}

}  // namespace zkb
