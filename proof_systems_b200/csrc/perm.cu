// perm.cu — the permutation aggregation polynomial z (kimchi/src/circuits/polynomials/permutation.rs:447-574, `perm_aggreg`) on
// the device, from the resident witness and permutation_coefficients8, so z never has to be built on the host and uploaded.
// With n = |d1|, last = n - zk_rows and sid[j] = omega^j:
//   num[j] = prod_{k<7} (w_k[j] + beta shift_k omega^j + gamma)      den[j] = prod_{k<7} (w_k[j] + beta sigma_k[s j] + gamma)
//   r[j]   = num[j] / den[j], with 1 / 0 := 0 (ark_ff::batch_inversion skips zero entries and leaves them zero)
//   z[0] = 1, z[j + 1] = z[j] r[j] for j < last           a multiplicative prefix scan over rows 0 .. last - 1:
//                                                           k_perm_ratios (ratios, per-thread and per-block prefixes),
//                                                           k_block_product_scan (the block totals, prod_scan.cuh),
//                                                           k_perm_apply
//   z[last + 1] = rand0, z[last + 2] = rand1                the reference's two F::rand(rng) draws, in its order
//   z[j + 1] = z[j] r[j] for j = last + 2 .. n - 2          zk_rows - 3 rows, one warp of k_perm_apply
//   final value: z[last] == 1; z = interpolate(z) over d1   the library's inverse NTT, in place
// No kernel waits on another CTA: the scan's three levels are three launches.  Field arithmetic is exact, so this association
// order gives the reference's bits.
#include <cstring>
#include <mutex>

#include "../../include/zkb200.h"
#include "ctx.hpp"
#include "prod_scan.cuh"

using namespace zkb;

namespace zkb {

constexpr unsigned PA_THREADS = 128;                       // every kernel below: 4 warps
constexpr unsigned PA_ROWS = 16;                           // consecutive rows per thread of k_perm_ratios (one inversion each)
constexpr unsigned PA_BLOCK_ROWS = PA_THREADS * PA_ROWS;   // rows per block, one block total each

struct PermAggArgs {
    const fe* w[7];     // witness columns over d1
    const fe* sigma[7]; // permutation_coefficients8 (or any s n evaluations), read at s j
    const fe* ulo;      // omega^j from the forward transform's tables (ntt.cuh): ulo[j & 1023] * mid[(j >> 10) & 1023] * hi2[j >> 20]
    const fe* mid;
    const fe* hi2;
    fe* z;              // the caller's buffer: num * (product of the thread's earlier nonzero den), then the block-local prefixes
    fe* r;              // scratch, n: den, then r = num / den for every row (the tail reads its rows from here)
    fe* block_tot;      // scratch: each block's product of r over its rows below `last`
    size_t n;
    size_t last;        // n - zk_rows
    size_t sigma_stride;
    fe beta, gamma;
    fe bshift[7];       // beta * shift_k
};

// rows [PA_ROWS t, PA_ROWS (t + 1)) of thread t: num and den, Montgomery's trick over the thread's nonzero den (one inversion),
// r into a.r; the block's exclusive scan of the per-thread products below `last`; then z[j] = (product of r[i], i < j, within the
// block) for j <= last.  Block totals go to a.block_tot.
template <class FS> __global__ void __launch_bounds__(PA_THREADS) k_perm_ratios(const __grid_constant__ PermAggArgs a) {
    const size_t j0 = ((size_t)blockIdx.x * PA_THREADS + threadIdx.x) * PA_ROWS;
    const size_t j1 = j0 + PA_ROWS < a.n ? j0 + PA_ROWS : a.n;
    fe tot = fe_one<FS>();
    if (j0 < a.n) {
        // forward: z[j] = num[j] * (product of the nonzero den[i], j0 <= i < j), r[j] = den[j]
        fe x = load_fe_nc(a.ulo + (j0 & 1023));
        if ((j0 >> 10) & 1023) x = fe_mul<FS>(x, load_fe_nc(a.mid + ((j0 >> 10) & 1023)));
        if (j0 >> 20) x = fe_mul<FS>(x, load_fe_nc(a.hi2 + (j0 >> 20)));
        const fe omega = load_fe_nc(a.ulo + 1);
        fe acc = fe_one<FS>();
        for (size_t j = j0; j < j1; j++) {
            fe wg = fe_add<FS>(load_fe_nc(a.w[0] + j), a.gamma);
            fe num = fe_add<FS>(wg, fe_mul<FS>(x, a.bshift[0]));
            fe den = fe_add<FS>(wg, fe_mul<FS>(a.beta, load_fe_nc(a.sigma[0] + a.sigma_stride * j)));
#pragma unroll 1
            for (unsigned k = 1; k < 7; k++) {
                wg = fe_add<FS>(load_fe_nc(a.w[k] + j), a.gamma);
                num = fe_mul<FS>(num, fe_add<FS>(wg, fe_mul<FS>(x, a.bshift[k])));
                den = fe_mul<FS>(den, fe_add<FS>(wg, fe_mul<FS>(a.beta, load_fe_nc(a.sigma[k] + a.sigma_stride * j))));
            }
            store_fe(a.z + j, fe_mul<FS>(num, acc));
            store_fe(a.r + j, den);
            if (!fe_is_zero(den)) acc = fe_mul<FS>(acc, den);
            x = fe_mul<FS>(x, omega);
        }
        // backward: inv = 1 / (product of the nonzero den[i], j0 <= i <= j), so r[j] = inv * z[j]; a zero den gives r[j] = 0
        fe inv = fe_inv<FS>(acc);
        for (size_t j = j1; j-- > j0;) {
            const fe den = load_fe(a.r + j);
            fe r = fe_zero();
            if (!fe_is_zero(den)) {
                r = fe_mul<FS>(inv, load_fe(a.z + j));
                inv = fe_mul<FS>(inv, den);
            }
            store_fe(a.r + j, r);
            if (j < a.last) tot = fe_mul<FS>(tot, r);
        }
    }
    fe block_total;
    fe run = block_exclusive_product<FS, PA_THREADS>(tot, block_total);
    if (threadIdx.x == 0) store_fe(a.block_tot + blockIdx.x, block_total);
    for (size_t j = j0; j < j1 && j <= a.last; j++) {
        store_fe(a.z + j, run);
        if (j < a.last) run = fe_mul<FS>(run, load_fe(a.r + j));
    }
}

// blocks 0 .. gridDim.x - 2: z[j] *= tot[j / PA_BLOCK_ROWS] for j <= last, and the final-value flag z[last] == 1;
// the last block's first warp: z[last + 1] = rand0, z[last + 2] = rand1, then z[j + 1] = z[j] r[j] for j = last + 2 .. n - 2 as a
// warp scan, 32 rows per step
template <class FS> __global__ void __launch_bounds__(PA_THREADS) k_perm_apply(fe* z, const fe* __restrict__ tot, const fe* __restrict__ r,
                                                                             size_t n, size_t last, const fe rand0, const fe rand1,
                                                                             unsigned* final_is_one) {
    if (blockIdx.x + 1 < gridDim.x) {
        const size_t j = (size_t)blockIdx.x * PA_THREADS + threadIdx.x;
        if (j > last) return;
        fe v = load_fe(z + j);
        const size_t b = j / PA_BLOCK_ROWS;
        if (b) {
            v = fe_mul<FS>(v, load_fe_nc(tot + b));
            store_fe(z + j, v);
        }
        if (j == last) *final_is_one = fe_eq(v, fe_one<FS>()) ? 1u : 0u;
        return;
    }
    if (threadIdx.x >= 32) return;
    const unsigned lane = threadIdx.x;
    if (lane == 0) {
        store_fe(z + last + 1, rand0);
        store_fe(z + last + 2, rand1);
    }
    fe carry = rand1;
    for (size_t base = last + 2; base < n - 1; base += 32) {
        const size_t j = base + lane;
        fe v = j < n - 1 ? load_fe_nc(r + j) : fe_one<FS>();
#pragma unroll
        for (unsigned d = 1; d < 32; d <<= 1) {
            const fe up = shfl_up_fe(v, d);
            if (lane >= d) v = fe_mul<FS>(v, up);
        }
        v = fe_mul<FS>(carry, v);
        if (j < n - 1) store_fe(z + j + 1, v);
        carry = shfl_fe(v, 31);
    }
}

template <class T>
static int perm_aggreg_impl(zk_ctx* ctx, unsigned log_n, size_t zk_rows, const void* const d_w[7], const void* const d_sigma[7],
                            size_t sigma_stride, const uint64_t beta[4], const uint64_t gamma[4], const uint64_t shifts[28],
                            const uint64_t rand[8], fe* d_z, int* final_is_one) {
    using namespace host;
    using FS = typename T::Dev; using HP = typename T::Host;
    const size_t n = (size_t)1 << log_n, last = n - zk_rows;
    PermAggArgs a{};
    for (int k = 0; k < 7; k++) { a.w[k] = (const fe*)d_w[k]; a.sigma[k] = (const fe*)d_sigma[k]; }
    a.z = d_z; a.n = n; a.last = last; a.sigma_stride = sigma_stride;
    hfe hb;
    memcpy(hb.l, beta, 32);
    memcpy(&a.beta, beta, 32);
    memcpy(&a.gamma, gamma, 32);
    for (int k = 0; k < 7; k++) {
        hfe s;
        memcpy(s.l, shifts + 4 * k, 32);
        const hfe bs = mul<HP>(hb, s);
        memcpy(&a.bshift[k], bs.l, 32);
    }
    fe r0, r1;
    memcpy(&r0, rand, 32);
    memcpy(&r1, rand + 4, 32);

    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    PinnedSlots* pin = ctx_pinned(ctx);
    if (!pin) return ZK_ERR_CUDA;
    int rc = ctx_ntt_table_ptrs(ctx, T::id, log_n, false, &a.ulo, &a.mid, &a.hi2);
    if (rc) return rc;
    // context scratch: r over d1 | block totals | the final-value flag
    const size_t blocks = (n + PA_BLOCK_ROWS - 1) / PA_BLOCK_ROWS;
    Layout lay;
    const size_t o_r = lay.add(n * sizeof(fe)), o_tot = lay.add(blocks * sizeof(fe)), o_flag = lay.add(sizeof(unsigned));
    rc = ctx->d_perm.ensure(lay.total);
    if (rc) return rc;
    a.r = ctx->d_perm.at<fe>(o_r);
    a.block_tot = ctx->d_perm.at<fe>(o_tot);
    unsigned* d_flag = ctx->d_perm.at<unsigned>(o_flag);
    k_perm_ratios<FS><<<(unsigned)blocks, PA_THREADS, 0, st>>>(a);
    ZK_CUDA(cudaGetLastError());
    k_block_product_scan<FS, PA_THREADS><<<1, PA_THREADS, 0, st>>>(a.block_tot, blocks);
    ZK_CUDA(cudaGetLastError());
    k_perm_apply<FS><<<(unsigned)((last + PA_THREADS) / PA_THREADS + 1), PA_THREADS, 0, st>>>(d_z, a.block_tot, a.r, n, last, r0, r1, d_flag);
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 3;
    rc = ctx_ntt_device(ctx, T::id, d_z, log_n, 1, 0, /* inverse = */ 1, /* coset = */ 0);     // Evaluations::interpolate
    if (rc) return rc;
    ZK_CUDA(cudaMemcpyAsync(&pin->perm_final, d_flag, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    ZK_CUDA(cudaStreamSynchronize(st));
    *final_is_one = pin->perm_final ? 1 : 0;
    return ZK_OK;
}

// [p, p + bytes) and [q, q + qbytes) share a byte
static bool overlaps(const void* p, size_t bytes, const void* q, size_t qbytes) {
    const uintptr_t a = (uintptr_t)p, b = (uintptr_t)q;
    return a < b + qbytes && b < a + bytes;
}

}  // namespace zkb

extern "C" int zk_perm_aggreg_dev(zk_ctx* ctx, int field_id, unsigned log_n, size_t zk_rows, const void* const d_w[7],
                                  const void* const d_sigma[7], uint64_t sigma_len, const uint64_t beta[4], const uint64_t gamma[4],
                                  const uint64_t shifts[28], const uint64_t rand[8], void* d_z, int* final_is_one) {
    if (!ctx || !d_w || !d_sigma || !beta || !gamma || !shifts || !rand || !d_z || !final_is_one) { zk_set_error("perm_aggreg: null argument"); return ZK_ERR_INVALID; }
    for (int k = 0; k < 7; k++)
        if (!d_w[k] || !d_sigma[k]) { zk_set_error("perm_aggreg: column %d is null", k); return ZK_ERR_INVALID; }
    if (int rc = check_field("perm_aggreg", field_id)) return rc;
    if (int rc = check_log_n("perm_aggreg", log_n)) return rc;
    const size_t n = (size_t)1 << log_n;
    // kimchi: 3 <= zk_rows < n (constraints.rs), so both random rows lie inside the domain and z[n - zk_rows] exists
    if (zk_rows < 3 || zk_rows >= n) { zk_set_error("perm_aggreg: zk_rows %zu is not in [3, %zu)", zk_rows, n); return ZK_ERR_INVALID; }
    if (sigma_len == 0 || sigma_len % n || sigma_len / n > 8) {
        zk_set_error("perm_aggreg: sigma has %llu evaluations, not 1 .. 8 times %zu", (unsigned long long)sigma_len, n);
        return ZK_ERR_INVALID;
    }
    if (!canonical(field_id, beta) || !canonical(field_id, gamma)) { zk_set_error("perm_aggreg: beta or gamma is not a canonical field element"); return ZK_ERR_INVALID; }
    for (int k = 0; k < 7; k++)
        if (!canonical(field_id, shifts + 4 * k)) { zk_set_error("perm_aggreg: shift %d is not a canonical field element", k); return ZK_ERR_INVALID; }
    for (int k = 0; k < 2; k++)
        if (!canonical(field_id, rand + 4 * k)) { zk_set_error("perm_aggreg: random value %d is not a canonical field element", k); return ZK_ERR_INVALID; }
    for (int k = 0; k < 7; k++)
        if (overlaps(d_z, n * sizeof(fe), d_w[k], n * sizeof(fe)) || overlaps(d_z, n * sizeof(fe), d_sigma[k], sigma_len * sizeof(fe))) {
            zk_set_error("perm_aggreg: d_z overlaps column %d", k);
            return ZK_ERR_INVALID;
        }
    return with_field(field_id, [&](auto f) {
        return perm_aggreg_impl<decltype(f)>(ctx, log_n, zk_rows, d_w, d_sigma, (size_t)(sigma_len / n), beta, gamma, shifts, rand, (fe*)d_z, final_is_one);
    });
}
