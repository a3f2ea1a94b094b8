// srs.cu — host-side mirror of poly_commitment::ipa::SRS<G> (poly-commitment/src/ipa.rs:56-75 and the `impl SRS<G>`
// at :596-800) for the commitment entry points that sit on the MSM hot path.  The chunking / padding / sub-sampling
// POLICY is restated here; every group operation of size n runs on the device through the resident-bases MSM.
//
//   commit_non_hiding                 ipa.rs:638-683
//   commit_evaluations_non_hiding     ipa.rs:706-728  + PolyComm::multi_scalar_mul, commitment.rs:350-394
//   mask_custom                       ipa.rs:605-622
//   get_lagrange_basis (cache entry)  ipa.rs:780-795  (the basis itself is provided by the caller: the reference
//                                     computes it with a group iFFT, ipa.rs:1065-1172 — SURVEY.md §8f row 2, "next")
#include <cstring>
#include <map>
#include <vector>

#include "../../include/zkb200.h"
#include "ctx.hpp"
#include "msm.cuh"

using namespace zkb;

// SRS::mask_custom (ipa.rs:605-622): chunk_i + blinder_i * h; one scalar multiplication per chunk, host side.
template <class HP, class HS> static void mask_one(const uint64_t* chunk, const uint64_t* blinder_mont, const uint64_t* h, uint64_t* out) {
    using namespace host;
    haffine c, hh;
    memcpy(&c, chunk, 64);
    memcpy(&hh, h, 64);
    hfe b;
    memcpy(&b, blinder_mont, 32);
    hfe one_raw = zero();
    one_raw.l[0] = 1;
    hfe canon = mul<HS>(b, one_raw);  // into_bigint
    hxyzz m = scalar_mul<HP>(from_affine<HP>(hh), canon.l);
    haffine r = to_affine<HP>(padd<HP>(m, from_affine<HP>(c)));
    memcpy(out, &r, 64);
}

extern "C" {

int zk_srs_create(zk_ctx* ctx, int curve_id, const uint64_t* g_xy, size_t n, const uint64_t h_xy[8], int window_bits, zk_srs** out) {
    if (!ctx || !out || !g_xy || !h_xy || n == 0) { zk_set_error("srs_create: null/empty argument"); return ZK_ERR_INVALID; }
    zk_bases* g = nullptr;
    int rc = zk_bases_upload(ctx, curve_id, g_xy, n, window_bits, 0, &g);
    if (rc) return rc;
    zk_srs* s = new zk_srs();
    s->ctx = ctx; s->curve = curve_id; s->n = n; s->g = g;
    memcpy(s->h, h_xy, 64);
    *out = s;
    return ZK_OK;
}

void zk_srs_destroy(zk_srs* srs) {
    if (!srs) return;
    for (auto& kv : srs->lagrange) zk_bases_free(kv.second);
    zk_bases_free(srs->g);
    delete srs;
}

size_t zk_srs_max_poly_size(const zk_srs* srs) { return srs ? srs->n : 0; }

static size_t basis_chunks(const zk_srs* srs, size_t domain_size) { return (domain_size + srs->n - 1) / srs->n; }   // n.div_ceil(srs_size), ipa.rs:1145

int zk_srs_add_lagrange_basis(zk_srs* srs, size_t domain_size, const uint64_t* basis_xy, int window_bits) {
    if (!srs || !basis_xy || domain_size == 0) { zk_set_error("add_lagrange_basis: null/empty argument"); return ZK_ERR_INVALID; }
    // a domain larger than the SRS has ceil(domain / |g|) chunks per element (ipa.rs:1145-1171): basis_xy is chunk-major,
    // chunk c's domain_size points at basis_xy + 8 * c * domain_size
    const size_t chunks = basis_chunks(srs, domain_size);
    zk_bases* b = nullptr;
    int rc = zk_bases_upload(srs->ctx, srs->curve, basis_xy, domain_size * chunks, window_bits, 0, &b);
    if (rc) return rc;
    auto it = srs->lagrange.find(domain_size);
    if (it != srs->lagrange.end()) { zk_bases_free(it->second); it->second = b; }
    else srs->lagrange.emplace(domain_size, b);
    return ZK_OK;
}

size_t zk_srs_lagrange_basis_chunks(const zk_srs* srs, size_t domain_size) {
    return srs && domain_size ? basis_chunks(srs, domain_size) : 0;
}

// SRS::get_lagrange_basis_from_domain_size (ipa.rs:780-788) -> SRS::lagrange_basis (ipa.rs:1065-1172), on the device:
// group iFFT of g[0..domain_size) + normalisation; the basis is registered (with its window table) for
// commit_evaluations_non_hiding.  Already registered sizes return at once, like the reference's cache.
int zk_srs_lagrange_basis(zk_srs* srs, size_t domain_size, int window_bits) {
    if (!srs || domain_size == 0 || (domain_size & (domain_size - 1))) { zk_set_error("lagrange_basis: domain size must be a power of two"); return ZK_ERR_INVALID; }
    if (srs->lagrange.count(domain_size)) return ZK_OK;
    if (domain_size > ((size_t)1 << 30)) { zk_set_error("lagrange_basis: domain %zu too large", domain_size); return ZK_ERR_INVALID; }
    unsigned log_n = 0;
    while (((size_t)1 << log_n) < domain_size) log_n++;
    const size_t chunks = basis_chunks(srs, domain_size);
    zk_ctx* ctx = srs->ctx;
    DevScratch d_out;                    // transient: freed on every return
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        ZK_CUDA(cudaSetDevice(ctx->device));
        if (int rc = d_out.ensure(chunks * domain_size * sizeof(affine_t))) return rc;
        unsigned nl = 0;
        int rc = ZK_OK;
        for (size_t c = 0; c < chunks && rc == ZK_OK; c++)
            rc = with_curve(srs->curve, [&](auto cv) {
                using C = decltype(cv);
                return lagrange_basis_build<typename C::F, typename C::FS>(srs->g->b, log_n, (unsigned)c, d_out.at<affine_t>() + c * domain_size, ctx->stream, &nl);
            });
        ctx->launches += nl;
        if (rc) return rc;
    }
    zk_bases* b = nullptr;
    int rc = zk_bases_upload(ctx, srs->curve, d_out.at<const uint64_t>(), chunks * domain_size, window_bits, /*points_on_device=*/1, &b);
    if (rc == ZK_OK) srs->lagrange.emplace(domain_size, b);
    return rc;
}

// Copy a registered basis back to the host (affine, n x 8 u64): what get_lagrange_basis(domain) derefs to.
int zk_srs_get_lagrange_basis(zk_srs* srs, size_t domain_size, uint64_t* out_xy, size_t capacity_points) {
    if (!srs || !out_xy) { zk_set_error("get_lagrange_basis: null argument"); return ZK_ERR_INVALID; }
    auto it = srs->lagrange.find(domain_size);
    if (it == srs->lagrange.end()) { zk_set_error("get_lagrange_basis: no basis for domain size %zu", domain_size); return ZK_ERR_INVALID; }
    const size_t total = domain_size * basis_chunks(srs, domain_size);     // chunk-major
    if (capacity_points < total) { zk_set_error("get_lagrange_basis: capacity %zu < %zu", capacity_points, total); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(srs->ctx->mu);
    ZK_CUDA(cudaSetDevice(srs->ctx->device));
    ZK_CUDA(cudaMemcpyAsync(out_xy, it->second->b.d_points, total * sizeof(affine_t), cudaMemcpyDeviceToHost, srs->ctx->stream));
    ZK_CUDA(cudaStreamSynchronize(srs->ctx->stream));
    return ZK_OK;
}

// SRS::commit_non_hiding (ipa.rs:638-683)
int zk_srs_commit_non_hiding(zk_srs* srs, const uint64_t* coeffs_mont, size_t len, size_t num_chunks, uint64_t* out_xy, size_t out_capacity, size_t* out_chunks) {
    if (!srs || !out_xy || !out_chunks || (!coeffs_mont && len)) { zk_set_error("commit_non_hiding: null argument"); return ZK_ERR_INVALID; }
    // plnm.is_zero() (ark-poly: no coefficients, or all of them zero) -> vec![G::zero()]; otherwise the chunk count comes from
    // plnm.len() AS GIVEN (ipa.rs:646-676 never trims: an untrimmed coefficient vector with a zero tail still yields
    // ceil(len / |g|) chunks, the last ones the identity)
    bool all_zero = true;
    for (size_t i = 0; i < 4 * len && all_zero; i++) all_zero = coeffs_mont[i] == 0;
    if (all_zero) len = 0;
    const size_t n = srs->n;
    size_t produced = len == 0 ? 1 : (len + n - 1) / n;       // is_zero -> vec![G::zero()]
    size_t total = produced > num_chunks ? produced : num_chunks;  // pad with G::zero() up to num_chunks (ipa.rs:678-680)
    *out_chunks = total;
    if (total > out_capacity) { zk_set_error("commit_non_hiding: %zu chunks do not fit the output capacity %zu", total, out_capacity); return ZK_ERR_INVALID; }
    memset(out_xy, 0, total * 64);  // identity chunks
    if (len == 0) return ZK_OK;
    // `len < |g|`: one msm on g[..len]; `len == |g|`: the reference splits in two halves and adds (same group element);
    // `len > |g|`: one msm_bigint per chunk of |g| coefficients, the last one shorter (ipa.rs:663-676).
    size_t k = produced;
    std::vector<uint64_t> jac(12 * k);
    if (k == 1 || len % n == 0) {
        size_t per = k == 1 ? len : n;
        int rc = zk_msm_batch(srs->ctx, srs->g, 0, per, coeffs_mont, k, /*mont=*/1, 0, jac.data());
        if (rc) return rc;
    } else {
        int rc = zk_msm_batch(srs->ctx, srs->g, 0, n, coeffs_mont, k - 1, 1, 0, jac.data());
        if (rc) return rc;
        rc = zk_msm(srs->ctx, srs->g, 0, len - (k - 1) * n, coeffs_mont + 4 * (k - 1) * n, 1, 0, jac.data() + 12 * (k - 1));
        if (rc) return rc;
    }
    for (size_t j = 0; j < k; j++) {
        int rc = zk_jacobian_to_affine(srs->curve, jac.data() + 12 * j, out_xy + 8 * j);
        if (rc) return rc;
    }
    return ZK_OK;
}

// SRS::commit_evaluations_non_hiding (ipa.rs:706-728) -> PolyComm::multi_scalar_mul (commitment.rs:350-394)
int zk_srs_commit_evaluations_non_hiding(zk_srs* srs, size_t domain_size, const uint64_t* evals_mont, size_t evals_domain_size, uint64_t out_xy[8]) {
    if (!srs || !evals_mont || !out_xy) { zk_set_error("commit_evaluations: null argument"); return ZK_ERR_INVALID; }
    auto it = srs->lagrange.find(domain_size);
    if (it == srs->lagrange.end()) { zk_set_error("commit_evaluations: no Lagrange basis registered for domain size %zu", domain_size); return ZK_ERR_INVALID; }
    if (domain_size > evals_domain_size) {
        // the reference panics: "desired commitment domain size greater than evaluations' domain size" (ipa.rs:723-725)
        zk_set_error("desired commitment domain size (%zu) greater than evaluations' domain size (%zu)", domain_size, evals_domain_size);
        return ZK_ERR_INVALID;
    }
    if (evals_domain_size % domain_size) { zk_set_error("commit_evaluations: %zu is not a multiple of %zu", evals_domain_size, domain_size); return ZK_ERR_INVALID; }
    const uint64_t* sc = evals_mont;
    std::vector<uint64_t> sub;
    if (evals_domain_size != domain_size) {   // v[i] = evals[s * i]  (ipa.rs:717-722)
        size_t s = evals_domain_size / domain_size;
        sub.resize(4 * domain_size);
        for (size_t i = 0; i < domain_size; i++) memcpy(&sub[4 * i], evals_mont + 4 * s * i, 32);
        sc = sub.data();
    }
    // PolyComm::multi_scalar_mul (commitment.rs:350-394): one MSM per chunk of the basis elements, all with the same scalars
    const size_t chunks = basis_chunks(srs, domain_size);
    if (chunks == 1) {
        uint64_t jac[12];
        int rc = zk_msm(srs->ctx, it->second, 0, domain_size, sc, /*mont=*/1, 0, jac);
        if (rc) return rc;
        return zk_jacobian_to_affine(srs->curve, jac, out_xy);
    }
    for (size_t c = 0; c < chunks; c++) {
        uint64_t jac[12];
        int rc = zk_msm(srs->ctx, it->second, c * domain_size, domain_size, sc, /*mont=*/1, 0, jac);
        if (rc) return rc;
        rc = zk_jacobian_to_affine(srs->curve, jac, out_xy + 8 * c);
        if (rc) return rc;
    }
    return ZK_OK;
}

// k independent commit_evaluations_non_hiding calls on the same domain (the reference issues the 15 witness columns from
// rayon workers at once, kimchi/src/prover.rs:329-351): evals_mont = k x domain_size, out_xy = k x 8.
int zk_srs_commit_evaluations_batch(zk_srs* srs, size_t domain_size, const uint64_t* evals_mont, size_t k, uint64_t* out_xy) {
    if (!srs || (!evals_mont && k) || (!out_xy && k)) { zk_set_error("commit_evaluations_batch: null argument"); return ZK_ERR_INVALID; }
    auto it = srs->lagrange.find(domain_size);
    if (it == srs->lagrange.end()) { zk_set_error("commit_evaluations: no Lagrange basis registered for domain size %zu", domain_size); return ZK_ERR_INVALID; }
    if (basis_chunks(srs, domain_size) != 1) { zk_set_error("commit_evaluations_batch: chunked bases (domain %zu > srs %zu) go through zk_srs_commit_evaluations_non_hiding", domain_size, srs->n); return ZK_ERR_INVALID; }
    std::vector<uint64_t> jac(12 * k);
    int rc = zk_msm_batch(srs->ctx, it->second, 0, domain_size, evals_mont, k, /*mont=*/1, 0, jac.data());
    if (rc) return rc;
    for (size_t j = 0; j < k; j++) {
        rc = zk_jacobian_to_affine(srs->curve, jac.data() + 12 * j, out_xy + 8 * j);
        if (rc) return rc;
    }
    return ZK_OK;
}

int zk_srs_mask_custom(zk_srs* srs, const uint64_t* chunks_xy, size_t n_chunks, const uint64_t* blinders_mont, size_t n_blinders, uint64_t* out_xy) {
    if (!srs || !chunks_xy || !blinders_mont || !out_xy) { zk_set_error("mask_custom: null argument"); return ZK_ERR_INVALID; }
    if (n_chunks != n_blinders) {
        zk_set_error("BlindersDontMatch(%zu, %zu)", n_blinders, n_chunks);  // poly-commitment/src/error.rs:3-9
        return ZK_ERR_LENGTH;
    }
    for (size_t i = 0; i < n_chunks; i++)
        with_curve(srs->curve, [&](auto c) { mask_one<typename decltype(c)::HP, typename decltype(c)::HS>(chunks_xy + 8 * i, blinders_mont + 4 * i, srs->h, out_xy + 8 * i); });
    return ZK_OK;
}

}  // extern "C"
