// aggreg.cuh — the aggregation polynomials' common pipeline (perm.cu's z, lookup.cu's lookup aggregation): given per-row factors
// num[j] and den[j] for rows j < end,
//   r[j] = num[j] / den[j], with 1 / 0 := 0 (ark_ff::batch_inversion skips zero entries and leaves them zero)
//   z[0] = 1, z[j + 1] = z[j] r[j] for j < last, and the flag z[last] == 1
// as three launches: k_agg_ratios (16 rows per thread, one inversion each by Montgomery's trick, the block scan and the
// block-local prefixes), k_scan_block_totals (scan.cuh) and k_agg_apply (the block prefixes, the flag, and the caller's Tail in
// the first warp of the last block, which writes the rows after `last`).  Field arithmetic is exact, so this association order
// gives the reference's bits.
//
// Rows: the caller's kernel argument, with a type Cursor and two device methods, called in row order by each thread:
//   Cursor start(size_t j0) const                                     the thread's state at its first row
//   void row(Cursor& c, size_t j, fe& num, fe& den) const             the factors of row j
// Tail: void operator()(fe* z, size_t last, unsigned lane) const       run by the 32 lanes of one warp
#pragma once
#include "ctx.hpp"
#include "scan.cuh"

namespace zkb {

constexpr unsigned AGG_THREADS = 128;                         // every kernel below: 4 warps
constexpr unsigned AGG_ROWS = 16;                             // consecutive rows per thread of k_agg_ratios (one inversion each)
constexpr unsigned AGG_BLOCK_ROWS = AGG_THREADS * AGG_ROWS;   // rows per block, one block total each

inline size_t agg_blocks(size_t end) { return (end + AGG_BLOCK_ROWS - 1) / AGG_BLOCK_ROWS; }

// rows [AGG_ROWS t, AGG_ROWS (t + 1)) of thread t below `end`: z[j] = num[j] * (product of the thread's earlier nonzero den),
// r[j] = den[j]; one inversion; backward, r[j] = num[j] / den[j].  Then the block's exclusive scan of the per-thread products of
// r below `last`, and z[j] = (product of r[i], i < j, within the block) for j <= last.  Block totals go to block_tot.
template <class FS, class Rows>
__global__ void __launch_bounds__(AGG_THREADS) k_agg_ratios(const __grid_constant__ Rows rows, fe* z, fe* r, fe* block_tot, size_t end, size_t last) {
    const size_t j0 = ((size_t)blockIdx.x * AGG_THREADS + threadIdx.x) * AGG_ROWS;
    const size_t j1 = j0 + AGG_ROWS < end ? j0 + AGG_ROWS : end;
    fe tot = fe_one<FS>();
    if (j0 < j1) {
        typename Rows::Cursor c = rows.start(j0);
        fe acc = fe_one<FS>();
        for (size_t j = j0; j < j1; j++) {
            fe num, den;
            rows.row(c, j, num, den);
            store_fe(z + j, fe_mul<FS>(num, acc));
            store_fe(r + j, den);
            if (!fe_is_zero(den)) acc = fe_mul<FS>(acc, den);
        }
        // inv = 1 / (product of the nonzero den[i], j0 <= i <= j), so r[j] = inv * z[j]; a zero den gives r[j] = 0
        fe inv = fe_inv<FS>(acc);
        for (size_t j = j1; j-- > j0;) {
            const fe den = load_fe(r + j);
            fe rj = fe_zero();
            if (!fe_is_zero(den)) {
                rj = fe_mul<FS>(inv, load_fe(z + j));
                inv = fe_mul<FS>(inv, den);
            }
            store_fe(r + j, rj);
            if (j < last) tot = fe_mul<FS>(tot, rj);
        }
    }
    fe block_total;
    fe run = block_exclusive_scan<MulOp<FS>, AGG_THREADS>(tot, block_total);
    if (threadIdx.x == 0) store_fe(block_tot + blockIdx.x, block_total);
    for (size_t j = j0; j < j1 && j <= last; j++) {
        store_fe(z + j, run);
        if (j < last) run = fe_mul<FS>(run, load_fe(r + j));
    }
}

// blocks 0 .. gridDim.x - 2: z[j] *= tot[j / AGG_BLOCK_ROWS] for j <= last, and the flag z[last] == 1; the last block's first
// warp: the tail
template <class FS, class Tail>
__global__ void __launch_bounds__(AGG_THREADS) k_agg_apply(fe* z, const fe* __restrict__ tot, size_t last, unsigned* final_is_one,
                                                           const __grid_constant__ Tail tail) {
    if (blockIdx.x + 1 < gridDim.x) {
        const size_t j = (size_t)blockIdx.x * AGG_THREADS + threadIdx.x;
        if (j > last) return;
        fe v = load_fe(z + j);
        const size_t b = j / AGG_BLOCK_ROWS;
        if (b) {
            v = fe_mul<FS>(v, load_fe_nc(tot + b));
            store_fe(z + j, v);
        }
        if (j == last) *final_is_one = fe_eq(v, fe_one<FS>()) ? 1u : 0u;
        return;
    }
    if (threadIdx.x < 32) tail(z, last, threadIdx.x);
}

// the three launches on ctx->stream (the caller holds the context lock).  Scratch: r of `end` elements, block_tot of
// agg_blocks(end), and the flag.
template <class FS, class Rows, class Tail>
int agg_launch(zk_ctx* ctx, const Rows& rows, const Tail& tail, fe* z, fe* r, fe* block_tot, size_t end, size_t last, unsigned* d_flag) {
    const size_t blocks = agg_blocks(end);
    cudaStream_t st = ctx->stream;
    k_agg_ratios<FS><<<(unsigned)blocks, AGG_THREADS, 0, st>>>(rows, z, r, block_tot, end, last);
    ZK_CUDA(cudaGetLastError());
    k_scan_block_totals<MulOp<FS>, AGG_THREADS><<<1, AGG_THREADS, 0, st>>>(block_tot, blocks);
    ZK_CUDA(cudaGetLastError());
    k_agg_apply<FS><<<(unsigned)((last + AGG_THREADS) / AGG_THREADS + 1), AGG_THREADS, 0, st>>>(z, block_tot, last, d_flag, tail);
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 3;
    return ZK_OK;
}

}  // namespace zkb
