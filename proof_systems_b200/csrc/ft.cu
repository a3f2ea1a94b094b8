// ft.cu — the ft polynomial of Maller's optimisation (kimchi/src/prover.rs:1147-1206) on the device, from the resident quotient t
// and the linearisation's evaluation-form terms (kimchi: sigma_6 over d8 scaled by perm_scalar), so only ft's length and ft(zeta
// omega) cross PCIe.  With n = |d1|, m = max_poly_size and num_chunks = 1 if n < m else n / m (prover.rs:208-212):
//   f_eval[i] = sum_k coeff_k * term_k[(len_k / n) i]                                  k_combine (poly.cuh)
//   f = interpolate(f_eval) over d1                                                    the library's inverse NTT
//   ft = f.to_chunked_polynomial(num_chunks, m).linearize(zeta^m)                       k_linearize_add, scale0 = 1
//      - t.to_chunked_polynomial(7 num_chunks, m).linearize(zeta^m).scale(zeta^n - 1)   k_linearize_add, scale0 = -(zeta^n - 1)
//   ft_len: one past the last nonzero coefficient (linearize trims trailing zeros, and so does ark-poly's subtraction)
//                                                                                      k_last_nonzero
//   ft_eval1 = ft.evaluate(zeta omega)                                                 evaluate_chunks (evals.cu): one chunk of m
// Both linearisations accumulate into the caller's ft buffer, zeroed first, so all m coefficients are written and the tail past
// ft_len is zero (evaluating all m of them gives ft(zeta omega): trailing zeros do not change a Horner sum).  Field arithmetic is
// exact, so this order of the sums gives the reference's bits.
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/zkb200.h"
#include "poly.cuh"

using namespace zkb;

namespace zkb {

constexpr unsigned FT_THREADS = 128;

// *out = max(*out, 1 + the largest i < len with a[i] != 0): one atomic per warp that holds a nonzero coefficient
__global__ void __launch_bounds__(FT_THREADS) k_last_nonzero(const fe* __restrict__ a, size_t len, unsigned long long* out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long v = i < len && !fe_is_zero(load_fe_nc(a + i)) ? (unsigned long long)i + 1 : 0;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v = max(v, __shfl_down_sync(0xffffffffu, v, off));
    if ((threadIdx.x & 31) == 0 && v) atomicMax(out, v);
}

template <class T>
static int ft_impl(zk_ctx* ctx, unsigned log_n, size_t m, std::vector<CombineDesc>& terms, const fe* d_t, size_t t_len, const uint64_t zeta_mont[4],
                   fe* d_ft, size_t* ft_len, uint64_t ft_eval1[4]) {
    using namespace host;
    using FS = typename T::Dev; using HP = typename T::Host;
    const size_t n = (size_t)1 << log_n;
    // host scalars: zeta^m, -(zeta^n - 1) = 1 - zeta^n, zeta omega (omega: the generator of d1)
    hfe zeta;
    memcpy(zeta.l, zeta_mont, 32);
    const hfe zeta_m = pow_u64<HP>(zeta, m), neg_zh = sub<HP>(one<HP>(), pow_u64<HP>(zeta, n)), zeta_omega = mul<HP>(zeta, root_of_unity<HP>(log_n));
    fe fzm, fneg, fone = fe_one<FS>();
    memcpy(&fzm, &zeta_m, 32);
    memcpy(&fneg, &neg_zh, 32);

    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    PinnedSlots* pin = ctx_pinned(ctx);
    if (!pin) return ZK_ERR_CUDA;
    // context scratch: f (n elements, only with terms) | term descriptors | the length counter
    Layout lay;
    const size_t o_f = lay.add((terms.empty() ? 0 : n) * sizeof(fe)), o_desc = lay.add(terms.size() * sizeof(CombineDesc));
    const size_t o_len = lay.add(sizeof(unsigned long long));
    int rc = ctx->d_ft.ensure(lay.total);
    if (rc) return rc;
    fe* d_f = ctx->d_ft.at<fe>(o_f);
    CombineDesc* d_desc = ctx->d_ft.at<CombineDesc>(o_desc);
    unsigned long long* d_len = ctx->d_ft.at<unsigned long long>(o_len);
    ZK_CUDA(cudaMemsetAsync(d_len, 0, sizeof(unsigned long long), st));
    ZK_CUDA(cudaMemsetAsync(d_ft, 0, m * sizeof(fe), st));
    const unsigned lin_blocks = (unsigned)((m + FT_THREADS - 1) / FT_THREADS);
    if (!terms.empty()) {                         // f = 0 without terms: it adds nothing
        ZK_CUDA(cudaMemcpyAsync(d_desc, terms.data(), terms.size() * sizeof(CombineDesc), cudaMemcpyHostToDevice, st));
        k_combine<FS><<<(unsigned)((n + FT_THREADS - 1) / FT_THREADS), FT_THREADS, 0, st>>>(d_desc, (unsigned)terms.size(), d_f, n);
        ZK_CUDA(cudaGetLastError());
        ctx->launches += 1;
        rc = ctx_ntt_device(ctx, T::id, d_f, log_n, 1, 0, /* inverse = */ 1, /* coset = */ 0);     // Evaluations::interpolate
        if (rc) return rc;
        k_linearize_add<FS><<<lin_blocks, FT_THREADS, 0, st>>>(d_ft, d_f, n, m, (unsigned)((n + m - 1) / m), fzm, fone);
        ZK_CUDA(cudaGetLastError());
        ctx->launches += 1;
    }
    if (t_len) {
        k_linearize_add<FS><<<lin_blocks, FT_THREADS, 0, st>>>(d_ft, d_t, t_len, m, (unsigned)((t_len + m - 1) / m), fzm, fneg);
        ZK_CUDA(cudaGetLastError());
        ctx->launches += 1;
    }
    k_last_nonzero<<<lin_blocks, FT_THREADS, 0, st>>>(d_ft, m, d_len);
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 1;
    const zk_dev_poly ft{d_ft, m};
    std::vector<uint8_t> stage;
    const fe* d_eval = nullptr;
    uint64_t covered = 0;
    rc = ctx_evaluate_chunks(ctx, T::id, &ft, 1, m, zeta_omega.l, 1, stage, &d_eval, &covered);
    if (rc) return rc;
    ZK_CUDA(cudaMemcpyAsync(&pin->ft_len, d_len, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    ZK_CUDA(cudaMemcpyAsync(&pin->ft_eval1, d_eval, sizeof(fe), cudaMemcpyDeviceToHost, st));
    ZK_CUDA(cudaStreamSynchronize(st));
    *ft_len = (size_t)pin->ft_len;
    memcpy(ft_eval1, &pin->ft_eval1, 32);
    return ZK_OK;
}

}  // namespace zkb

extern "C" int zk_prover_ft_dev(zk_ctx* ctx, int field_id, unsigned log_n, size_t max_poly_size, const zk_lin_term* terms, size_t n_terms,
                                const void* d_t, size_t t_len, const uint64_t zeta_mont[4], void* d_ft, size_t* ft_len, uint64_t ft_eval1[4]) {
    if (!ctx || (!terms && n_terms) || (!d_t && t_len) || !zeta_mont || !d_ft || !ft_len || !ft_eval1) { zk_set_error("prover_ft: null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_field("prover_ft", field_id)) return rc;
    if (int rc = check_log_n("prover_ft", log_n)) return rc;
    if (max_poly_size == 0) { zk_set_error("prover_ft: max_poly_size is 0"); return ZK_ERR_INVALID; }
    const size_t n = (size_t)1 << log_n, m = max_poly_size;
    if (n >= m && n % m) { zk_set_error("prover_ft: domain size %zu is not a multiple of max_poly_size %zu", n, m); return ZK_ERR_INVALID; }
    if (!canonical(field_id, zeta_mont)) { zk_set_error("prover_ft: zeta is not a canonical field element"); return ZK_ERR_INVALID; }
    if (n_terms > 0xffffffffu) { zk_set_error("prover_ft: %zu terms are too many", n_terms); return ZK_ERR_INVALID; }
    std::vector<CombineDesc> descs(n_terms);
    for (size_t k = 0; k < n_terms; k++) {
        const zk_lin_term& t = terms[k];
        if (!t.d_evals) { zk_set_error("prover_ft: term %zu is null", k); return ZK_ERR_INVALID; }
        // CombineDesc's 32-bit stride: kimchi's domains d1 .. d8 (len = n, 2n, 4n or 8n; 3n ... 7n are accepted too)
        if (t.len == 0 || t.len % n || t.len / n > 8) { zk_set_error("prover_ft: term %zu has %llu evaluations, not 1 .. 8 times %zu", k, (unsigned long long)t.len, n); return ZK_ERR_INVALID; }
        if (!canonical(field_id, t.coeff)) { zk_set_error("prover_ft: coefficient of term %zu is not a canonical field element", k); return ZK_ERR_INVALID; }
        descs[k].p = (const fe*)t.d_evals;
        descs[k].len = (uint32_t)n;
        descs[k].stride = (uint32_t)(t.len / n);
        memcpy(&descs[k].scale, t.coeff, 32);
    }
    const size_t num_chunks = n < m ? 1 : n / m;
    if ((t_len + m - 1) / m > 7 * num_chunks) {     // t.to_chunked_polynomial(7 * num_chunks, m)'s assert_eq!
        zk_set_error("prover_ft: t has %zu coefficients, more than %zu chunks of %zu", t_len, 7 * num_chunks, m);
        return ZK_ERR_LENGTH;
    }
    return with_field(field_id, [&](auto f) { return ft_impl<decltype(f)>(ctx, log_n, m, descs, (const fe*)d_t, t_len, zeta_mont, (fe*)d_ft, ft_len, ft_eval1); });
}
