// evals.cu — the prover's evaluations at zeta and zeta*omega on the device (kimchi/src/prover.rs:1009-1058), over the columns the
// d8 pipeline left resident (zk_ntt_dev / zk_ntt_dev_oop, zk_index_cache_section), so nothing but the few hundred results crosses PCIe.
//
// kimchi/src/lagrange_basis_evaluations.rs and utils/src/{dense_polynomial,chunked_polynomial}.rs, restated:
//   LagrangeBasisEvaluations::new(m, D(n), x) (:242-258)                                   -> zk_lagrange_evals_dev
//     n <= m (new_with_segment_size_1, :126-198): l_i = (x^n - 1) / (w^-i t_0 (x - w^i)), t_0 = prod_{j>=1} (1 - w^j) = n, through
//            batch_inversion_and_mul, which skips zero denominators: for x in the domain the numerator is 0 and every l_i is 0.
//            Here l_i = c / (x w^-i - 1) with c = (x^n - 1) / n computed once on the host — the same field elements; the
//            denominators are inverted with Montgomery's trick over the strided set of LB_SEG elements each thread owns (one
//            Fermat inversion per thread, zero denominators skipped and left zero), w^-i taken from the inverse NTT's tables.
//     n > m  (new_with_chunked_segments, :203-240): c = n / m vectors, vector k = iFFT(n) of (x^0 .. x^{m-1} at k m .. (k+1) m - 1,
//            0 elsewhere): one fill kernel for the c power vectors, then ONE batched inverse NTT through the library's own path.
//   evaluate(p) (:72-109) / evaluate_boolean(p) (:116-131)                                  -> zk_lagrange_evaluate_dev
//     chunk k of point t: sum_i p[stride i] * l_{t,k}[i]   (boolean: sum of l_{t,k}[i] over p[stride i] != 0), stride = |p| / n.
//     Stage 1: block (slice, column, pair group) reads p[stride i] ONCE for up to EV_PAIRS (point, chunk) pairs — in the prover's
//     case (2 points, <= 4 chunks) every pair — and writes one partial sum per pair; stage 2 (k_sum_partials) adds the partials.
//   to_chunked_polynomial(c, s).evaluate_chunks(x) (dense_polynomial.rs:50-69, chunked_polynomial.rs:21-28) -> zk_poly_evaluate_chunks_dev
//     chunk k = Horner of coefficients k s .. (k+1) s - 1 (zero past the end of the polynomial); more than c chunks is the
//     reference's assert_eq! and ZK_ERR_LENGTH here.  A thread runs Horner over HS_SEG coefficients of one chunk for up to HS_PTS
//     points at once (the coefficients are read once for all of them), scales by x^{segment start}, and the block's sum is one partial.
// Field arithmetic is exact: the two-stage sums give the bits of the reference's serial sums.
#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/zkb200.h"
#include "ctx.hpp"
#include "poly.cuh"

using namespace zkb;

namespace zkb {

constexpr unsigned EV_THREADS = 128;     // every kernel below: 4 warps
constexpr unsigned LB_SEG = 16;          // unchunked basis: elements per thread (one inversion each)
constexpr unsigned LB_RUN = 16;          // chunked basis: consecutive powers per thread (one exponentiation each)
constexpr unsigned EV_PAIRS = 8;         // column evaluation: (point, chunk) accumulators per thread
constexpr unsigned HS_PTS = 4;           // coefficient evaluation: points per thread
constexpr unsigned HS_SEG = 32;          // coefficient evaluation: coefficients per thread

// sum of acc[k] (k < cnt, uniform over the block) over the block's 128 threads; thread k < cnt writes the sum of accumulator k to
// out[k * out_stride]
template <class FS, unsigned K> __device__ __forceinline__ void block_sum_store(const fe (&acc)[K], unsigned cnt, fe* out, size_t out_stride) {
    __shared__ fe part[EV_THREADS / 32][K];
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (unsigned k = 0; k < K; k++) {
        if (k < cnt) {
            fe v = acc[k];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) v = fe_add<FS>(v, shfl_down_fe(v, off));
            if (lane == 0) part[warp][k] = v;
        }
    }
    __syncthreads();
    if (threadIdx.x < cnt) {
        fe s = part[0][threadIdx.x];
#pragma unroll
        for (unsigned w = 1; w < EV_THREADS / 32; w++) s = fe_add<FS>(s, part[w][threadIdx.x]);
        store_fe(out + threadIdx.x * out_stride, s);
    }
}

// out[o] = sum_{s < nparts} part[o * nparts + s]: one block per output
template <class FS> __global__ void __launch_bounds__(EV_THREADS) k_sum_partials(const fe* __restrict__ part, size_t nparts, fe* out) {
    const fe* p = part + (size_t)blockIdx.x * nparts;
    fe acc[1] = {fe_zero()};
    for (size_t s = threadIdx.x; s < nparts; s += EV_THREADS) acc[0] = fe_add<FS>(acc[0], load_fe(p + s));
    block_sum_store<FS, 1>(acc, 1, out + blockIdx.x, 1);
}

// ------------------------------------------------------------------------------------------------ basis, n <= max_poly_size
struct LagBasisArgs {
    const fe* ulo;      // w^-i from the inverse transform's unscaled tables (domain_point, ntt.cuh)
    const fe* mid;
    const fe* hi2;
    fe* out;
    size_t n;
    size_t threads;     // thread t owns i = t, t + threads, ...
    fe x;
    fe c;               // (x^n - 1) / n
};

template <class FS> __device__ __forceinline__ fe lag_denominator(const LagBasisArgs& a, size_t i) {
    const fe w = domain_point<FS>(a.ulo, a.mid, a.hi2, i);
    return fe_sub<FS>(fe_mul<FS>(a.x, w), fe_one<FS>());       // x w^-i - 1 = w^-i (x - w^i)
}

template <class FS> __global__ void __launch_bounds__(EV_THREADS) k_lagrange_basis(const __grid_constant__ LagBasisArgs a) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.n || t >= a.threads) return;
    // forward: out[i] = product of this thread's nonzero denominators before i
    fe acc = fe_one<FS>();
    for (size_t i = t; i < a.n; i += a.threads) {
        const fe d = lag_denominator<FS>(a, i);
        store_fe(a.out + i, acc);
        if (!fe_is_zero(d)) acc = fe_mul<FS>(acc, d);
    }
    // inv = c / (product of all of them); backward: out[i] = inv * prefix_i = c / d_i, then inv *= d_i
    fe inv = fe_mul<FS>(fe_inv<FS>(acc), a.c);
    for (size_t i = t + ((a.n - 1 - t) / a.threads) * a.threads;; i -= a.threads) {
        const fe d = lag_denominator<FS>(a, i);
        if (fe_is_zero(d)) {
            store_fe(a.out + i, fe_zero());
        } else {
            store_fe(a.out + i, fe_mul<FS>(inv, load_fe(a.out + i)));
            inv = fe_mul<FS>(inv, d);
        }
        if (i < a.threads) break;
    }
}

// ------------------------------------------------------------------------------------------------ basis, n > max_poly_size
// element e of the chunks x n output: vector k = e >> log_n holds x^(j - k m) at j = e & (n - 1) in [k m, (k + 1) m), 0 elsewhere.
// A thread writes LB_RUN consecutive elements: one exponentiation, then one product per element (consecutive in-range elements
// always have consecutive exponents: the element after a vector's range is out of range or the first of the next vector).
template <class FS> __global__ void __launch_bounds__(EV_THREADS) k_chunked_powers(fe* out, unsigned log_n, size_t m, size_t total, const fe x) {
    const size_t e0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * LB_RUN;
    if (e0 >= total) return;
    const size_t n_mask = ((size_t)1 << log_n) - 1;
    fe v = fe_zero();
    bool have = false;
    for (size_t e = e0; e < e0 + LB_RUN && e < total; e++) {
        const size_t lo = (e >> log_n) * m, j = e & n_mask;
        if (j >= lo && j < lo + m) {
            v = have ? fe_mul<FS>(v, x) : fe_pow_u64<FS>(x, j - lo);
            have = true;
            store_fe(out + e, v);
        } else {
            have = false;
            store_fe(out + e, fe_zero());
        }
    }
}

// ------------------------------------------------------------------------------------------------ evaluate / evaluate_boolean
struct EvalCol {
    const fe* p;
    uint64_t stride;    // |p| / n
    uint32_t boolean;
    uint32_t reserved;
};

struct LagEvalArgs {
    const EvalCol* cols;       // device
    const fe* const* bases;    // device: n_points pointers, each chunks x n
    fe* partial;               // [(col * n_pairs + pair) * blocks_x + block]
    size_t n;
    unsigned chunks, n_pairs, blocks_x;
};

// grid (blocks_x, n_cols, pair groups): pair = point * chunks + chunk
template <class FS> __global__ void __launch_bounds__(EV_THREADS) k_lagrange_evaluate(const __grid_constant__ LagEvalArgs a) {
    const unsigned pair0 = blockIdx.z * EV_PAIRS, cnt = min(EV_PAIRS, a.n_pairs - pair0);
    const EvalCol c = a.cols[blockIdx.y];
    const fe* b[EV_PAIRS];
    fe acc[EV_PAIRS];
#pragma unroll
    for (unsigned k = 0; k < EV_PAIRS; k++) {
        acc[k] = fe_zero();
        const unsigned pair = pair0 + (k < cnt ? k : 0);
        b[k] = a.bases[pair / a.chunks] + (size_t)(pair % a.chunks) * a.n;
    }
    for (size_t i = (size_t)blockIdx.x * EV_THREADS + threadIdx.x; i < a.n; i += (size_t)a.blocks_x * EV_THREADS) {
        const fe p = load_fe_nc(c.p + c.stride * i);           // once for every pair of the group
        const bool nz = !fe_is_zero(p);
#pragma unroll
        for (unsigned k = 0; k < EV_PAIRS; k++) {
            if (k < cnt) {
                if (c.boolean) {
                    if (nz) acc[k] = fe_add<FS>(acc[k], load_fe_nc(b[k] + i));   // evaluate_boolean: a nonzero value counts as one
                } else {
                    acc[k] = fe_add<FS>(acc[k], fe_mul<FS>(p, load_fe_nc(b[k] + i)));
                }
            }
        }
    }
    block_sum_store<FS, EV_PAIRS>(acc, cnt, a.partial + ((size_t)blockIdx.y * a.n_pairs + pair0) * a.blocks_x + blockIdx.x, a.blocks_x);
}

// ------------------------------------------------------------------------------------------------ evaluate_chunks
struct DevPoly {
    const fe* c;
    uint64_t len;
};

struct ChunkEvalArgs {
    const DevPoly* polys;      // device
    const fe* points;          // device, n_points
    fe* partial;               // [((poly * n_points + point) * covered + chunk) * bpc + block of the chunk]
    uint64_t chunk_size;
    unsigned n_points, covered, spc, bpc;   // chunks holding coefficients, segments per chunk, blocks per chunk
};

// grid (covered * bpc, n_polys, point groups)
template <class FS> __global__ void __launch_bounds__(EV_THREADS) k_evaluate_chunks(const __grid_constant__ ChunkEvalArgs a) {
    const unsigned pt0 = blockIdx.z * HS_PTS, cnt = min(HS_PTS, a.n_points - pt0);
    const unsigned ch = blockIdx.x / a.bpc, blk = blockIdx.x % a.bpc, s = blk * EV_THREADS + threadIdx.x;
    const DevPoly poly = a.polys[blockIdx.y];
    fe x[HS_PTS], acc[HS_PTS];
#pragma unroll
    for (unsigned k = 0; k < HS_PTS; k++) {
        acc[k] = fe_zero();
        x[k] = load_fe_nc(a.points + pt0 + (k < cnt ? k : 0));
    }
    const uint64_t off = (uint64_t)s * HS_SEG, start = (uint64_t)ch * a.chunk_size + off;
    uint64_t end = start + HS_SEG;
    if (end > (uint64_t)(ch + 1) * a.chunk_size) end = (uint64_t)(ch + 1) * a.chunk_size;
    if (end > poly.len) end = poly.len;
    if (s < a.spc && start < end) {
#pragma unroll 1
        for (uint64_t j = end; j-- > start;) {
            const fe cj = load_fe_nc(poly.c + j);
#pragma unroll
            for (unsigned k = 0; k < HS_PTS; k++)
                if (k < cnt) acc[k] = fe_add<FS>(fe_mul<FS>(acc[k], x[k]), cj);
        }
        if (off) {
#pragma unroll
            for (unsigned k = 0; k < HS_PTS; k++)
                if (k < cnt) acc[k] = fe_mul<FS>(acc[k], fe_pow_u64<FS>(x[k], off));
        }
    }
    const size_t stride = (size_t)a.covered * a.bpc;
    block_sum_store<FS, HS_PTS>(acc, cnt, a.partial + ((size_t)blockIdx.y * a.n_points + pt0) * stride + (size_t)ch * a.bpc + blk, stride);
}

template <class FS> int launch_sum(const fe* part, size_t nparts, fe* out, size_t n_out, cudaStream_t st) {
    for (size_t o = 0; o < n_out; o += 65535) {
        const unsigned blocks = (unsigned)std::min<size_t>(n_out - o, 65535);
        k_sum_partials<FS><<<blocks, EV_THREADS, 0, st>>>(part + o * nparts, nparts, out + o);
    }
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

template <class FS> static fe host_basis_scale(const fe& x, unsigned log_n) {
    // (x^n - 1) / n: the numerator of batch_inversion_and_mul over t_0 = prod_{j>=1} (1 - w^j) = n
    fe n = fe_zero();
    n.v[0] = 1u << log_n;
    return fe_mul<FS>(fe_sub<FS>(fe_pow_u64<FS>(x, (uint64_t)1 << log_n), fe_one<FS>()), fe_inv<FS>(fe_to_mont<FS>(n)));
}

// the chunks holding coefficients, segments per chunk and blocks per chunk of evaluate_chunks over polynomials of up to max_len
static void chunk_plan(uint64_t max_len, size_t chunk_size, uint64_t* covered, uint64_t* spc, uint64_t* bpc) {
    *covered = (max_len + chunk_size - 1) / chunk_size;
    *spc = (std::min<uint64_t>(chunk_size, max_len) + HS_SEG - 1) / HS_SEG;
    *bpc = (*spc + EV_THREADS - 1) / EV_THREADS;
}

int ctx_evaluate_chunks(zk_ctx* ctx, int field_id, const zk_dev_poly* polys, size_t n_polys, size_t chunk_size, const uint64_t* points_mont,
                        size_t n_points, std::vector<uint8_t>& stage, const fe** d_res, uint64_t* covered_out) {
    uint64_t max_len = 0;
    for (size_t k = 0; k < n_polys; k++) max_len = std::max(max_len, polys[k].len);
    uint64_t covered, spc, bpc;
    chunk_plan(max_len, chunk_size, &covered, &spc, &bpc);
    *covered_out = covered;
    const size_t n_cov = n_polys * n_points * covered;
    if (n_cov == 0) return ZK_OK;
    cudaStream_t st = ctx->stream;
    // context scratch: polynomial table | points | partial sums | results
    Layout lay;
    const size_t o_pol = lay.add(n_polys * sizeof(DevPoly)), o_pts = lay.add(n_points * sizeof(fe));
    const size_t o_part = lay.add(n_cov * bpc * sizeof(fe)), o_res = lay.add(n_cov * sizeof(fe));
    int rc = ctx->d_evals.ensure(lay.total);
    if (rc) return rc;
    stage.assign(o_part, 0);
    for (size_t k = 0; k < n_polys; k++) {
        const DevPoly d{(const fe*)polys[k].d_coeffs, polys[k].len};
        memcpy(stage.data() + o_pol + k * sizeof(DevPoly), &d, sizeof(DevPoly));
    }
    memcpy(stage.data() + o_pts, points_mont, n_points * sizeof(fe));
    ZK_CUDA(cudaMemcpyAsync(ctx->d_evals.p, stage.data(), stage.size(), cudaMemcpyHostToDevice, st));
    ChunkEvalArgs a{};
    a.polys = ctx->d_evals.at<const DevPoly>(o_pol); a.points = ctx->d_evals.at<const fe>(o_pts); a.partial = ctx->d_evals.at<fe>(o_part);
    a.chunk_size = chunk_size; a.n_points = (unsigned)n_points; a.covered = (unsigned)covered; a.spc = (unsigned)spc; a.bpc = (unsigned)bpc;
    const dim3 grid((unsigned)(covered * bpc), (unsigned)n_polys, (unsigned)((n_points + HS_PTS - 1) / HS_PTS));
    fe* res = ctx->d_evals.at<fe>(o_res);
    rc = with_field(field_id, [&](auto f) {
        using FS = typename decltype(f)::Dev;
        k_evaluate_chunks<FS><<<grid, EV_THREADS, 0, st>>>(a); return launch_sum<FS>(a.partial, bpc, res, n_cov, st);
    });
    if (rc) return rc;
    ctx->launches += 1 + (n_cov + 65534) / 65535;
    *d_res = res;
    return ZK_OK;
}

}  // namespace zkb

extern "C" {

size_t zk_lagrange_evals_chunks(size_t domain_size, size_t max_poly_size) {
    if (domain_size == 0 || max_poly_size == 0) return 0;
    if (domain_size <= max_poly_size) return 1;
    return domain_size % max_poly_size ? 0 : domain_size / max_poly_size;
}

int zk_lagrange_evals_dev(zk_ctx* ctx, int field_id, unsigned log_n, size_t max_poly_size, const uint64_t x_mont[4], void* d_out) {
    if (!ctx || !x_mont || !d_out) { zk_set_error("lagrange_evals: null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_field("lagrange_evals", field_id)) return rc;
    if (int rc = check_log_n("lagrange_evals", log_n)) return rc;
    if (max_poly_size == 0) { zk_set_error("lagrange_evals: max_poly_size is 0"); return ZK_ERR_INVALID; }
    const size_t n = (size_t)1 << log_n, chunks = zk_lagrange_evals_chunks(n, max_poly_size);
    if (chunks == 0) { zk_set_error("lagrange_evals: domain size %zu is not a multiple of max_poly_size %zu", n, max_poly_size); return ZK_ERR_INVALID; }
    if (!canonical(field_id, x_mont)) { zk_set_error("lagrange_evals: x is not a canonical field element"); return ZK_ERR_INVALID; }
    fe x;
    memcpy(&x, x_mont, 32);
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    if (chunks == 1) {
        LagBasisArgs a{};
        int rc = ctx_ntt_table_ptrs(ctx, field_id, log_n, true, &a.ulo, &a.mid, &a.hi2);
        if (rc) return rc;
        a.out = (fe*)d_out; a.n = n; a.x = x;
        a.threads = (n + LB_SEG - 1) / LB_SEG;
        const unsigned blocks = (unsigned)((a.threads + EV_THREADS - 1) / EV_THREADS);
        with_field(field_id, [&](auto f) {
            using FS = typename decltype(f)::Dev;
            a.c = host_basis_scale<FS>(x, log_n); k_lagrange_basis<FS><<<blocks, EV_THREADS, 0, st>>>(a);
        });
        ZK_CUDA(cudaGetLastError());
        ctx->launches += 1;
        return ZK_OK;
    }
    const size_t total = chunks * n, threads = (total + LB_RUN - 1) / LB_RUN;
    const unsigned blocks = (unsigned)((threads + EV_THREADS - 1) / EV_THREADS);
    with_field(field_id, [&](auto f) { k_chunked_powers<typename decltype(f)::Dev><<<blocks, EV_THREADS, 0, st>>>((fe*)d_out, log_n, max_poly_size, total, x); });
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 1;
    return ctx_ntt_device(ctx, field_id, (fe*)d_out, log_n, chunks, 0, /* inverse = */ 1, /* coset = */ 0);
}

int zk_lagrange_evaluate_dev(zk_ctx* ctx, int field_id, const void* const* d_bases, size_t n_points, unsigned log_n, size_t chunks,
                             const zk_eval_column* cols, size_t n_cols, uint64_t* out) {
    if (!ctx || (!d_bases && n_points) || (!cols && n_cols) || (!out && n_points && n_cols)) { zk_set_error("lagrange_evaluate: null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_field("lagrange_evaluate", field_id)) return rc;
    if (int rc = check_log_n("lagrange_evaluate", log_n)) return rc;
    const size_t n = (size_t)1 << log_n;
    // a basis of D(n) has 1 vector, or n / max_poly_size for a divisor max_poly_size < n: chunks divides n either way
    if (chunks == 0 || chunks > n || n % chunks) { zk_set_error("lagrange_evaluate: %zu chunks cannot belong to a basis of a domain of %zu", chunks, n); return ZK_ERR_INVALID; }
    if (n_cols > 65535) { zk_set_error("lagrange_evaluate: %zu columns, at most 65535", n_cols); return ZK_ERR_INVALID; }
    for (size_t p = 0; p < n_points; p++)
        if (!d_bases[p]) { zk_set_error("lagrange_evaluate: basis %zu is null", p); return ZK_ERR_INVALID; }
    std::vector<EvalCol> hc(n_cols);
    for (size_t k = 0; k < n_cols; k++) {
        const zk_eval_column& c = cols[k];
        if (!c.d_evals) { zk_set_error("lagrange_evaluate: column %zu is null", k); return ZK_ERR_INVALID; }
        if (c.len == 0 || c.len % n) { zk_set_error("lagrange_evaluate: column %zu has %llu evaluations, not a positive multiple of %zu", k, (unsigned long long)c.len, n); return ZK_ERR_INVALID; }
        hc[k] = EvalCol{(const fe*)c.d_evals, c.len / n, c.boolean ? 1u : 0u, 0u};
    }
    const size_t n_pairs = n_points * chunks;
    if (n_pairs == 0 || n_cols == 0) return ZK_OK;
    if (n_pairs > (size_t)65535 * EV_PAIRS) { zk_set_error("lagrange_evaluate: %zu (point, chunk) pairs, at most %u", n_pairs, 65535 * EV_PAIRS); return ZK_ERR_INVALID; }

    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    int sms = 0;
    ZK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ctx->device));
    const size_t groups = (n_pairs + EV_PAIRS - 1) / EV_PAIRS;
    // slices of at least 16 elements per thread, and about 8 blocks per SM over the whole grid
    const size_t by_len = std::max<size_t>(1, n / (EV_THREADS * 16)), by_fill = std::max<size_t>(1, (size_t)sms * 8 / (n_cols * groups));
    const unsigned blocks_x = (unsigned)std::min<size_t>(std::min(by_len, by_fill), 65535);
    const size_t n_out = n_cols * n_pairs;
    // context scratch: column table | basis pointers | partial sums | results
    Layout lay;
    const size_t o_col = lay.add(n_cols * sizeof(EvalCol)), o_bas = lay.add(n_points * sizeof(fe*));
    const size_t o_part = lay.add(n_out * blocks_x * sizeof(fe)), o_res = lay.add(n_out * sizeof(fe));
    int rc = ctx->d_evals.ensure(lay.total);
    if (rc) return rc;
    std::vector<uint8_t> stage(o_part, 0);
    memcpy(stage.data() + o_col, hc.data(), n_cols * sizeof(EvalCol));
    memcpy(stage.data() + o_bas, d_bases, n_points * sizeof(fe*));
    ZK_CUDA(cudaMemcpyAsync(ctx->d_evals.p, stage.data(), stage.size(), cudaMemcpyHostToDevice, st));
    LagEvalArgs a{};
    a.cols = ctx->d_evals.at<const EvalCol>(o_col); a.bases = ctx->d_evals.at<const fe* const>(o_bas); a.partial = ctx->d_evals.at<fe>(o_part);
    a.n = n; a.chunks = (unsigned)chunks; a.n_pairs = (unsigned)n_pairs; a.blocks_x = blocks_x;
    const dim3 grid(blocks_x, (unsigned)n_cols, (unsigned)groups);
    fe* res = ctx->d_evals.at<fe>(o_res);
    rc = with_field(field_id, [&](auto f) {
        using FS = typename decltype(f)::Dev;
        k_lagrange_evaluate<FS><<<grid, EV_THREADS, 0, st>>>(a); return launch_sum<FS>(a.partial, blocks_x, res, n_out, st);
    });
    if (rc) return rc;
    ctx->launches += 1 + (n_out + 65534) / 65535;
    ZK_CUDA(cudaMemcpyAsync(out, res, n_out * sizeof(fe), cudaMemcpyDeviceToHost, st));
    ZK_CUDA(cudaStreamSynchronize(st));      // `stage` is a local, `out` is the caller's
    return ZK_OK;
}

int zk_poly_evaluate_chunks_dev(zk_ctx* ctx, int field_id, const zk_dev_poly* polys, size_t n_polys, size_t num_chunks, size_t chunk_size,
                                const uint64_t* points_mont, size_t n_points, uint64_t* out) {
    if (!ctx || (!polys && n_polys) || (!points_mont && n_points) || (!out && n_polys && n_points && num_chunks)) { zk_set_error("evaluate_chunks: null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_field("evaluate_chunks", field_id)) return rc;
    if (chunk_size == 0) { zk_set_error("evaluate_chunks: chunk_size is 0"); return ZK_ERR_INVALID; }
    if (n_polys > 65535) { zk_set_error("evaluate_chunks: %zu polynomials, at most 65535", n_polys); return ZK_ERR_INVALID; }
    if (n_points > (size_t)65535 * HS_PTS) { zk_set_error("evaluate_chunks: %zu points, at most %u", n_points, 65535 * HS_PTS); return ZK_ERR_INVALID; }
    for (size_t t = 0; t < n_points; t++)
        if (!canonical(field_id, points_mont + 4 * t)) { zk_set_error("evaluate_chunks: point %zu is not a canonical field element", t); return ZK_ERR_INVALID; }
    uint64_t max_len = 0;
    for (size_t k = 0; k < n_polys; k++) {
        if (!polys[k].d_coeffs && polys[k].len) { zk_set_error("evaluate_chunks: polynomial %zu is null", k); return ZK_ERR_INVALID; }
        max_len = std::max(max_len, polys[k].len);
    }
    for (size_t k = 0; k < n_polys; k++)
        if ((polys[k].len + chunk_size - 1) / chunk_size > num_chunks) {     // to_chunked_polynomial's assert_eq!(chunk_polys.len(), num_chunks)
            zk_set_error("evaluate_chunks: polynomial %zu has %llu coefficients, more than %zu chunks of %zu", k, (unsigned long long)polys[k].len, num_chunks, chunk_size);
            return ZK_ERR_LENGTH;
        }
    const size_t n_out = n_polys * n_points * num_chunks;
    if (n_out == 0) return ZK_OK;
    memset(out, 0, n_out * sizeof(fe));                 // chunks past the end of every polynomial: the zero polynomial
    uint64_t covered, spc, bpc;
    chunk_plan(max_len, chunk_size, &covered, &spc, &bpc);
    if (covered == 0) return ZK_OK;
    if (covered * bpc > 0x7fffffffu) { zk_set_error("evaluate_chunks: %llu coefficients per polynomial are too many", (unsigned long long)max_len); return ZK_ERR_INVALID; }
    const size_t n_cov = n_polys * n_points * covered;

    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    std::vector<uint8_t> stage;
    const fe* res = nullptr;
    int rc = ctx_evaluate_chunks(ctx, field_id, polys, n_polys, chunk_size, points_mont, n_points, stage, &res, &covered);
    if (rc) return rc;
    std::vector<fe> h(n_cov);
    ZK_CUDA(cudaMemcpyAsync(h.data(), res, n_cov * sizeof(fe), cudaMemcpyDeviceToHost, st));
    ZK_CUDA(cudaStreamSynchronize(st));
    // (poly, point, chunk < covered) -> out[(poly * n_points + point) * num_chunks + chunk]
    for (size_t q = 0; q < n_polys * n_points; q++) memcpy(out + 4 * q * num_chunks, h.data() + q * covered, covered * sizeof(fe));
    return ZK_OK;
}

}  // extern "C"
