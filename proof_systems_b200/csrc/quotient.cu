// quotient.cu — first pointwise evaluator of the d8 pipeline (SURVEY.md §8f row 3): the permutation part of kimchi's quotient
// polynomial, computed over the d8 evaluations where they already live — the device — between the FFT(8n) that produced them
// (zk_ntt_dev_oop, kimchi/src/circuits/constraints.rs:488-507) and the iFFT(8n) that follows the quotient (prover.rs:907).
//
// kimchi/src/circuits/polynomials/permutation.rs:223-357, `perm` (the `bnd` part is two polynomial divisions on z, O(n) host work):
//     perm(x) = alpha0 * zkpm(x) * ( z(x)       * prod_{k < 7} (w_k(x) + gamma + beta * shift_k * x)
//                                  - z(x omega) * prod_{k < 7} (w_k(x) + gamma + beta * sigma_k(x)) )
// in evaluation form over d8: x_i = omega_8n^i, z(x omega) = z[(i + 8) mod 8n] (lagrange.d8.next.z, constraints.rs:497-505),
// zkpm = precomputations().permutation_vanishing_polynomial_l, sigma_k = column_evaluations.permutation_coefficients8[k].
// One thread per point of d8: 16 resident arrays read once (512 B), one written; ~35 field multiplications.
#include <cstring>
#include <mutex>

#include "../../include/zkb200.h"
#include "ctx.hpp"

using namespace zkb;

namespace zkb {

struct PermQuotArgs {
    const fe* w[7];     // the 7 permuted witness columns over d8
    const fe* sigma[7]; // permutation_coefficients8
    const fe* z;
    const fe* zkpm;
    const fe* ulo;      // x_i = omega_m^i from the forward transform's tables (domain_point, ntt.cuh)
    const fe* mid;
    const fe* hi2;
    fe* out;
    size_t m;
    unsigned next_shift;
    fe beta, gamma, alpha0;
    fe shift[7];
};

template <class FS> __global__ void __launch_bounds__(128) k_perm_quotient(const __grid_constant__ PermQuotArgs a) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.m) return;
    const fe bx = fe_mul<FS>(a.beta, domain_point<FS>(a.ulo, a.mid, a.hi2, i));
    size_t inext = i + a.next_shift;
    if (inext >= a.m) inext -= a.m;
    fe shifts = load_fe_nc(a.z + i), sigmas = load_fe_nc(a.z + inext);
#pragma unroll 1
    for (unsigned k = 0; k < 7; k++) {
        const fe wg = fe_add<FS>(load_fe_nc(a.w[k] + i), a.gamma);
        shifts = fe_mul<FS>(shifts, fe_add<FS>(wg, fe_mul<FS>(bx, a.shift[k])));
        sigmas = fe_mul<FS>(sigmas, fe_add<FS>(wg, fe_mul<FS>(a.beta, load_fe_nc(a.sigma[k] + i))));
    }
    const fe r = fe_mul<FS>(fe_mul<FS>(fe_sub<FS>(shifts, sigmas), a.alpha0), load_fe_nc(a.zkpm + i));
    store_fe(a.out + i, r);
}

}  // namespace zkb

extern "C" int zk_perm_quotient_dev(zk_ctx* ctx, int field_id, unsigned log_m, const void* const d_w[7], const void* d_z, const void* const d_sigma[7],
                                    const void* d_zkpm, const uint64_t beta[4], const uint64_t gamma[4], const uint64_t alpha0[4],
                                    const uint64_t shifts[28], unsigned next_shift, void* d_out) {
    if (!ctx || !d_w || !d_z || !d_sigma || !d_zkpm || !beta || !gamma || !alpha0 || !shifts || !d_out) { zk_set_error("perm_quotient: null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_field("perm_quotient", field_id)) return rc;
    if (int rc = check_log_n("perm_quotient", log_m, "log_m")) return rc;
    const size_t m = (size_t)1 << log_m;
    if (next_shift >= m) { zk_set_error("perm_quotient: shift %u does not fit a domain of %zu", next_shift, m); return ZK_ERR_INVALID; }
    for (int k = 0; k < 7; k++)
        if (!d_w[k] || !d_sigma[k]) { zk_set_error("perm_quotient: column %d is null", k); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    PermQuotArgs a{};
    int rc = ctx_ntt_table_ptrs(ctx, field_id, log_m, false, &a.ulo, &a.mid, &a.hi2);
    if (rc) return rc;
    for (int k = 0; k < 7; k++) { a.w[k] = (const fe*)d_w[k]; a.sigma[k] = (const fe*)d_sigma[k]; }
    a.z = (const fe*)d_z; a.zkpm = (const fe*)d_zkpm; a.out = (fe*)d_out;
    a.m = m; a.next_shift = next_shift;
    memcpy(&a.beta, beta, 32); memcpy(&a.gamma, gamma, 32); memcpy(&a.alpha0, alpha0, 32);
    memcpy(a.shift, shifts, 7 * 32);
    const unsigned blocks = (unsigned)((m + 127) / 128);
    with_field(field_id, [&](auto f) { k_perm_quotient<typename decltype(f)::Dev><<<blocks, 128, 0, ctx->stream>>>(a); });
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 1;
    return ZK_OK;
}
