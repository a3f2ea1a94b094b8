// accumulator.cu — the recursion accumulators of a batch of proofs (poly-commitment/src/utils.rs:204-312, the same code as
// kimchi-stubs/src/urs_utils.rs:10-101) behind two C-ABI calls, zk_srs_accumulator_check and zk_srs_accumulator_generate
// (include/zkb200.h).  An accumulator is sg_i = <b_poly_coefficients(chal_i), g>; the reference's cost is one dense MSM over g per
// accumulator (generate) or one MSM over g || comms with the challenge polynomials of the whole batch summed into its scalars (check).
//
// Both build the challenge polynomials from the product tables of bpoly.cuh (the convention of zk_srs_verify):
//   * check: S[j] = sum_i (-r^i) s_i[j] (k_bpoly_tables + k_bpoly_sum, two launches for the batch), S through the fused MSM over
//     the resident generator table, and the k commitments with scalars r^i as a transient plain base set; the host adds the two.
//   * generate: per group of at most ctx->msm.batch accumulators (and at most ACC_EXPAND_BUDGET bytes of expanded scalars), one
//     table launch, one expansion launch (k_bpoly_expand, one vector per accumulator) and one fused ctx_msm_many.
#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/zkb200.h"
#include "bpoly.cuh"
#include "ctx.hpp"

using namespace zkb;

namespace zkb {
namespace {

constexpr size_t ACC_EXPAND_BUDGET = (size_t)256 << 20;   // generate: expanded scalars of one group (8 vectors at |g| = 2^20)

unsigned ceil_log2(size_t n) {
    unsigned K = 0;
    while (((size_t)1 << K) < n) K++;
    return K;
}

// rounds = n_chals / k as the reference derives it, refused where it panics: k = 0 with challenges (assert_eq!(chals.len(), 0)),
// fewer challenges than accumulators (% 0) and a remainder (assert_eq!(chals.len() % rounds, 0)); k = 0 without challenges: 0
int derive_rounds(const char* what, size_t k, size_t n_chals, size_t* rounds) {
    *rounds = 0;
    if (k == 0) {
        if (n_chals) { zk_set_error("%s: %zu challenges for no accumulators", what, n_chals); return ZK_ERR_INVALID; }
        return ZK_OK;
    }
    if (n_chals < k) { zk_set_error("%s: %zu challenges for %zu accumulators leave 0 rounds", what, n_chals, k); return ZK_ERR_INVALID; }
    *rounds = n_chals / k;
    if (n_chals % *rounds) { zk_set_error("%s: %zu challenges are not a multiple of %zu rounds", what, n_chals, *rounds); return ZK_ERR_INVALID; }
    return ZK_OK;
}

// the table input of vectors [first, first + cnt): rev[i][t] = chal_i[R - 1 - t] for t < min(R, K), zero above (bpoly.cuh)
void reversed_challenges(const uint64_t* chals, size_t first, size_t cnt, size_t R, unsigned K, std::vector<host::hfe>& rev) {
    rev.assign(std::max<size_t>(1, cnt * K), host::zero());
    const size_t used = std::min<size_t>(R, K);
    for (size_t i = 0; i < cnt; i++)
        for (size_t t = 0; t < used; t++) memcpy(&rev[i * K + t], chals + 4 * ((first + i) * R + R - 1 - t), 32);
}

template <class C>
int check_impl(zk_srs* srs, const uint64_t* comms_xy, size_t k, const uint64_t* chals, size_t R, const uint64_t* r_mont, int* out_ok,
               uint64_t* out_sum_xyz) {
    using namespace host;
    using FS = typename C::FS; using HP = typename C::HP; using HS = typename C::HS;
    zk_ctx* ctx = srs->ctx;
    cudaStream_t st = ctx->stream;
    const size_t len = srs->n;
    const unsigned K = (unsigned)R, L = (K + 1) / 2, H = K - L;
    // rs[i] = r^i (the commitments' scalars), w[i] = -r^i (folded into the high tables: S = -sum_i r^i s_i)
    hfe r, ri = one<HS>();
    memcpy(&r, r_mont, 32);
    std::vector<hfe> rev, rs(k), w(k);
    reversed_challenges(chals, 0, k, R, K, rev);
    for (size_t i = 0; i < k; i++) {
        rs[i] = ri;
        w[i] = sub<HS>(zero(), ri);
        ri = mul<HS>(ri, r);
    }
    // scratch: S, lo tables, hi tables, rev, weights, commitment scalars | commitments (affine)
    const size_t n_lo = k << L, n_hi = k << H;
    Layout lay;
    const size_t o_fe = lay.add((len + n_lo + n_hi + rev.size() + 2 * k) * sizeof(fe)), o_pts = lay.add(k * sizeof(affine_t));
    int rc = ctx->d_verify.ensure(lay.total);
    if (rc) return rc;
    fe* d_S = ctx->d_verify.at<fe>(o_fe);
    fe* d_lo = d_S + len;
    fe* d_hi = d_lo + n_lo;
    fe* d_rev = d_hi + n_hi;
    fe* d_w = d_rev + rev.size();
    fe* d_rs = d_w + k;
    affine_t* d_pts = ctx->d_verify.at<affine_t>(o_pts);
    ZK_CUDA(cudaMemcpyAsync(d_rev, rev.data(), rev.size() * sizeof(fe), cudaMemcpyHostToDevice, st));
    ZK_CUDA(cudaMemcpyAsync(d_w, w.data(), k * sizeof(fe), cudaMemcpyHostToDevice, st));
    ZK_CUDA(cudaMemcpyAsync(d_rs, rs.data(), k * sizeof(fe), cudaMemcpyHostToDevice, st));
    ZK_CUDA(cudaMemcpyAsync(d_pts, comms_xy, k * sizeof(affine_t), cudaMemcpyHostToDevice, st));
    const size_t n_tab = n_lo + n_hi;
    k_bpoly_tables<FS><<<(unsigned)((n_tab + 127) / 128), 128, 0, st>>>(d_rev, d_w, (unsigned)k, K, L, d_lo, d_hi);
    ZK_CUDA(cudaGetLastError());
    k_bpoly_sum<FS><<<(unsigned)((len + 127) / 128), 128, 0, st>>>(d_lo, d_hi, (unsigned)k, L, H, d_S, len);
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 2;

    // <S, g> over the resident table, then <rs, comms> as a transient plain base set
    uint64_t out_g[12], out_c[12];
    const fe* s_ptr = d_S;
    rc = ctx_msm_many(ctx, srs->g, 0, len, &s_ptr, 1, /*mont=*/1, 0, out_g);
    if (rc) return rc;
    zk_bases cb;
    cb.ctx = ctx;
    cb.b.curve = srs->curve;
    cb.b.n = k;
    cb.b.c = 0;
    cb.b.nwin = 0;
    cb.b.d_points = d_pts;
    const fe* c_ptr = d_rs;
    rc = ctx_msm_many(ctx, &cb, 0, k, &c_ptr, 1, /*mont=*/1, 0, out_c);
    if (rc) return rc;

    hjac jg, jc;
    memcpy(&jg, out_g, 96);
    memcpy(&jc, out_c, 96);
    const hxyzz sum = padd<HP>(from_jacobian<HP>(jg), from_jacobian<HP>(jc));
    *out_ok = is_inf(sum) ? 1 : 0;
    if (out_sum_xyz) {
        const hjac js = to_jacobian<HP>(sum);
        memcpy(out_sum_xyz, &js, 96);
    }
    return ZK_OK;
}

template <class C>
int generate_impl(zk_srs* srs, size_t m, const uint64_t* chals, size_t R, uint64_t* out_xy) {
    using namespace host;
    using FS = typename C::FS; using HP = typename C::HP; using HS = typename C::HS;
    zk_ctx* ctx = srs->ctx;
    cudaStream_t st = ctx->stream;
    const size_t len = srs->n;
    const unsigned K = ceil_log2(len), L = (K + 1) / 2, H = K - L;
    const size_t group = std::max<size_t>(1, std::min<size_t>(std::min<size_t>((size_t)std::max(ctx->msm.batch, 1), MSM_MAX_BATCH),
                                                                          ACC_EXPAND_BUDGET / (len * sizeof(fe))));
    // scratch: expanded scalars, lo tables, hi tables, rev, weights (all one) of one group
    const size_t n_lo = group << L, n_hi = group << H, n_rev = std::max<size_t>(1, group * K);
    Layout lay;
    const size_t o_fe = lay.add((group * len + n_lo + n_hi + n_rev + group) * sizeof(fe));
    int rc = ctx->d_verify.ensure(lay.total);
    if (rc) return rc;
    fe* d_s = ctx->d_verify.at<fe>(o_fe);
    fe* d_lo = d_s + group * len;
    fe* d_hi = d_lo + n_lo;
    fe* d_rev = d_hi + n_hi;
    fe* d_w = d_rev + n_rev;
    const std::vector<hfe> ones(group, one<HS>());
    ZK_CUDA(cudaMemcpyAsync(d_w, ones.data(), group * sizeof(fe), cudaMemcpyHostToDevice, st));
    std::vector<hfe> rev;
    std::vector<uint64_t> jac(12 * group);
    const fe* ptrs[MSM_MAX_BATCH];
    for (size_t first = 0; first < m; first += group) {
        const size_t cnt = std::min(group, m - first);
        reversed_challenges(chals, first, cnt, R, K, rev);     // pageable: the copy has consumed rev when it returns
        ZK_CUDA(cudaMemcpyAsync(d_rev, rev.data(), rev.size() * sizeof(fe), cudaMemcpyHostToDevice, st));
        const size_t n_tab = (cnt << L) + (cnt << H);
        k_bpoly_tables<FS><<<(unsigned)((n_tab + 127) / 128), 128, 0, st>>>(d_rev, d_w, (unsigned)cnt, K, L, d_lo, d_hi);
        ZK_CUDA(cudaGetLastError());
        k_bpoly_expand<FS><<<dim3((unsigned)((len + 127) / 128), (unsigned)cnt), 128, 0, st>>>(d_lo, d_hi, L, H, d_s, len);
        ZK_CUDA(cudaGetLastError());
        ctx->launches += 2;
        for (size_t j = 0; j < cnt; j++) ptrs[j] = d_s + j * len;
        rc = ctx_msm_many(ctx, srs->g, 0, len, ptrs, cnt, /*mont=*/1, 0, jac.data());
        if (rc) return rc;
        for (size_t j = 0; j < cnt; j++) {
            hjac p;
            memcpy(&p, jac.data() + 12 * j, 96);
            const haffine a = to_affine<HP>(from_jacobian<HP>(p));   // into_affine(): the identity is (0, 0)
            memcpy(out_xy + 8 * (first + j), &a, 64);
        }
    }
    return ZK_OK;
}

}  // namespace
}  // namespace zkb

extern "C" int zk_srs_accumulator_check(zk_srs* srs, const uint64_t* comms_xy, size_t n_comms, const uint64_t* chals_mont, size_t n_chals,
                                        const uint64_t r_mont[4], int* out_ok, uint64_t out_sum_xyz[12]) {
    static const char* what = "accumulator_check";
    if (!srs || (!comms_xy && n_comms) || (!chals_mont && n_chals) || !r_mont || !out_ok) { zk_set_error("%s: null argument", what); return ZK_ERR_INVALID; }
    size_t R;
    int rc = derive_rounds(what, n_comms, n_chals, &R);
    if (rc) return rc;
    if (n_comms == 0) {           // the reference returns true without an MSM
        *out_ok = 1;
        if (out_sum_xyz) {
            const host::hjac id = with_curve(srs->curve, [](auto c) { return host::to_jacobian<typename decltype(c)::HP>(host::identity()); });
            memcpy(out_sum_xyz, &id, 96);
        }
        return ZK_OK;
    }
    if (R >= 8 * sizeof(size_t) - 1 || ((size_t)1 << R) != srs->n) {      // assert_eq!(terms.len(), n)
        zk_set_error("%s: %zu rounds give 2^%zu coefficients per accumulator, the SRS has %zu points", what, R, R, srs->n);
        return ZK_ERR_LENGTH;
    }
    zk_ctx* ctx = srs->ctx;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    return with_curve(srs->curve, [&](auto c) { return check_impl<decltype(c)>(srs, comms_xy, n_comms, chals_mont, R, r_mont, out_ok, out_sum_xyz); });
}

extern "C" int zk_srs_accumulator_generate(zk_srs* srs, size_t num_comms, const uint64_t* chals_mont, size_t n_chals, uint64_t* out_xy,
                                           size_t capacity_points, size_t* out_points) {
    static const char* what = "accumulator_generate";
    if (!srs || (!chals_mont && n_chals) || !out_points) { zk_set_error("%s: null argument", what); return ZK_ERR_INVALID; }
    size_t R;
    int rc = derive_rounds(what, num_comms, n_chals, &R);
    if (rc) return rc;
    const size_t m = R ? n_chals / R : 0;      // one accumulator per chunk of `rounds` challenges, trailing chunks included
    *out_points = m;
    if (m == 0) return ZK_OK;
    if (capacity_points < m) { zk_set_error("%s: %zu points do not fit the capacity %zu", what, m, capacity_points); return ZK_ERR_INVALID; }
    if (!out_xy) { zk_set_error("%s: null argument", what); return ZK_ERR_INVALID; }
    zk_ctx* ctx = srs->ctx;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    return with_curve(srs->curve, [&](auto c) { return generate_impl<decltype(c)>(srs, m, chals_mont, R, out_xy); });
}
