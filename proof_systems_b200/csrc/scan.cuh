// scan.cuh — the block-level prefix scan behind the library's multi-launch scans, over any associative operation: the field
// product (MulOp, the aggregation polynomials of aggreg.cuh) and the u32 sum (AddU32, lookup.cu's sorted-column offsets).  A
// three-level scan is three launches (per-block scans writing one total per block, k_scan_block_totals, an apply), so no kernel
// waits on a flag another CTA writes.
#pragma once
#include "common.cuh"
#include "field.cuh"

namespace zkb {

// an associative operation with its identity: T, identity(), apply(a, b)
template <class FS> struct MulOp {
    using T = fe;
    static __device__ __forceinline__ fe identity() { return fe_one<FS>(); }
    static __device__ __forceinline__ fe apply(const fe& a, const fe& b) { return fe_mul<FS>(a, b); }
};
struct AddU32 {
    using T = uint32_t;
    static __device__ __forceinline__ uint32_t identity() { return 0; }
    static __device__ __forceinline__ uint32_t apply(uint32_t a, uint32_t b) { return a + b; }
};

__device__ __forceinline__ fe shfl_up(const fe& a, unsigned d) { return shfl_up_fe(a, d); }
__device__ __forceinline__ uint32_t shfl_up(uint32_t a, unsigned d) { return __shfl_up_sync(0xffffffffu, a, d); }

// exclusive prefix of v over the block's THREADS threads (thread 0 gets the identity); total: all of them combined.  Every thread
// of the block calls it.
template <class Op, unsigned THREADS> __device__ __forceinline__ typename Op::T block_exclusive_scan(const typename Op::T& v, typename Op::T& total) {
    using T = typename Op::T;
    __shared__ T warp_tot[THREADS / 32];
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T incl = v;
#pragma unroll
    for (unsigned d = 1; d < 32; d <<= 1) {
        const T up = shfl_up(incl, d);
        if (lane >= d) incl = Op::apply(incl, up);
    }
    T excl = shfl_up(incl, 1);
    if (lane == 0) excl = Op::identity();
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    total = warp_tot[0];
#pragma unroll
    for (unsigned k = 1; k < THREADS / 32; k++) {
        if (k == warp) excl = Op::apply(excl, total);       // total combines the warps before this one here
        total = Op::apply(total, warp_tot[k]);
    }
    return excl;
}

// one block of THREADS: tot[b] <- tot[0] op .. op tot[b - 1] (exclusive), each thread over a contiguous segment of the nb totals
template <class Op, unsigned THREADS> __global__ void __launch_bounds__(THREADS) k_scan_block_totals(typename Op::T* tot, size_t nb) {
    using T = typename Op::T;
    const size_t per = (nb + THREADS - 1) / THREADS;
    const size_t b0 = threadIdx.x * per, b1 = b0 + per < nb ? b0 + per : nb;
    T p = Op::identity();
    for (size_t b = b0; b < b1; b++) p = Op::apply(p, tot[b]);
    T all;
    T run = block_exclusive_scan<Op, THREADS>(p, all);
    for (size_t b = b0; b < b1; b++) {
        const T v = tot[b];
        tot[b] = run;
        run = Op::apply(run, v);
    }
}

}  // namespace zkb
