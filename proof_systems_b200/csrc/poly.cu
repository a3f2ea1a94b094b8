// poly.cu — the polynomial tail of the quotient on the device (SURVEY.md §8f row 3): what the prover does between the iFFTs of
// t4 / t8 and the commitment to t (kimchi/src/prover.rs:905-918):
//     let mut f = t4.interpolate() + t8.interpolate();  f += &public_poly;          -> zk_poly_add_dev (coefficient-wise, in HBM)
//     let (quotient, res) = f.divide_by_vanishing_poly(index.cs.domain.d1);           -> zk_poly_divide_by_vanishing_dev
//     if !res.is_zero() { Err("rest of division by vanishing polynomial") }           -> the call's remainder flag
//     quotient += &bnd;                                                               -> zk_poly_add_dev
// Dividing by Z_H = x^n - 1 in coefficient form is a suffix sum over every residue class of the exponents mod n:
//     f = q (x^n - 1) + r   <=>   q_i = sum_{k >= 1} f_{i + k n},   r_i = sum_{k >= 0} f_{i + k n}  (i < n)
// (ark-poly's DensePolynomial::divide_by_vanishing_poly computes the same sums chunk by chunk).  One thread per residue class:
// 32 B read and 32 B written per coefficient — a pure HBM stream.  The quotient then feeds zk_msm_dev chunk by chunk without
// leaving the device (commit_non_hiding's MSMs take Montgomery scalars as they lie).
#include <cstring>
#include <mutex>

#include "../../include/zkb200.h"
#include "ctx.hpp"

using namespace zkb;

namespace zkb {

template <class FS> __global__ void k_vec_add(fe* dst, const fe* __restrict__ src, size_t len) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= len) return;
    store_fe(dst + i, fe_add<FS>(load_fe(dst + i), load_fe_nc(src + i)));
}

// thread i < n walks its residue class from the top coefficient down: before f[j] is added, acc = sum of the class above j = q[j]
template <class FS> __global__ void k_divide_by_vanishing(const fe* __restrict__ f, size_t len, size_t n, fe* quot, unsigned* nonzero_remainder) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || i >= len) return;
    fe acc = fe_zero();
    for (size_t j = i + ((len - 1 - i) / n) * n;; j -= n) {       // the class's largest index below len, then down to i
        if (len > n && j < len - n) store_fe(quot + j, acc);      // the quotient has len - n coefficients
        acc = fe_add<FS>(acc, load_fe_nc(f + j));
        if (j < n) break;
    }
    if (!fe_is_zero(acc)) atomicOr(nonzero_remainder, 1u);        // r_i = the sum of the whole class
}

}  // namespace zkb

extern "C" {

int zk_poly_add_dev(zk_ctx* ctx, int field_id, void* d_dst, const void* d_src, size_t len) {
    if (!ctx || ((!d_dst || !d_src) && len)) { zk_set_error("poly_add: null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_field("poly_add", field_id)) return rc;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    if (len == 0) return ZK_OK;
    const unsigned blocks = (unsigned)((len + 255) / 256);
    with_field(field_id, [&](auto f) { k_vec_add<typename decltype(f)::Dev><<<blocks, 256, 0, ctx->stream>>>((fe*)d_dst, (const fe*)d_src, len); });
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 1;
    return ZK_OK;
}

int zk_poly_divide_by_vanishing_dev(zk_ctx* ctx, int field_id, const void* d_f, size_t len, unsigned log_n, void* d_quot, int* remainder_is_zero) {
    if (!ctx || !d_f || !remainder_is_zero) { zk_set_error("divide_by_vanishing: null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_field("divide_by_vanishing", field_id)) return rc;
    if (int rc = check_log_n("divide_by_vanishing", log_n)) return rc;
    const size_t n = (size_t)1 << log_n;
    if (len > n && !d_quot) { zk_set_error("divide_by_vanishing: null quotient buffer"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    PinnedSlots* pin = ctx_pinned(ctx);
    if (!pin) return ZK_ERR_CUDA;
    if (int rc = ctx->d_flag.ensure(sizeof(unsigned))) return rc;
    unsigned* d_flag = ctx->d_flag.at<unsigned>();
    ZK_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(unsigned), ctx->stream));
    const unsigned blocks = (unsigned)((n + 127) / 128);
    with_field(field_id, [&](auto f) { k_divide_by_vanishing<typename decltype(f)::Dev><<<blocks, 128, 0, ctx->stream>>>((const fe*)d_f, len, n, (fe*)d_quot, d_flag); });
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 1;
    ZK_CUDA(cudaMemcpyAsync(&pin->remainder, d_flag, sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    *remainder_is_zero = pin->remainder == 0;
    return ZK_OK;
}

}  // extern "C"
