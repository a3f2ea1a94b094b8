// open.cu — SRS::open (poly-commitment/src/ipa.rs:823-1061) behind one C-ABI call, zk_srs_open (include/zkb200.h).
//
// Device: combine_polys (poly-commitment/src/utils.rs:103-202: one kernel sums every coefficient-form chunk scaled by its
// power of polyscale, another the sub-sampled evaluation-form entries, then the NTT library interpolates and a third kernel
// linearises the chunks), b_init (ipa.rs:876-888: every thread raises the evaluation points to its own index), the combined
// inner product, the folding rounds of ipa.cu with h and U as extra bases, and the last MSM pair
//     sg = <s, g>            delta = <d s, g> + (d b0) U + r_delta h   ==  (g0 + b0 U) d + r_delta h      (ipa.rs:1030-1038)
// Host: the O(1)-per-round field arithmetic (u^-1, r_prime, z1, z2), the O(c) tails of the MSMs, the window rows of h and U
// (255 doublings + one batch inversion), and the caller's sponge / group map behind the callbacks.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/zkb200.h"
#include "ipa.hpp"
#include "msm.cuh"
#include "poly.cuh"

using namespace zkb;

namespace zkb {

// b[j] = sum_i scale_i * elm_i^j   (ipa.rs:876-888; pows(padded_length, e))
template <class FS> __global__ void k_b_init(const fe* __restrict__ elm, const fe* __restrict__ scales, unsigned n_elm, fe* b, size_t n) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    fe acc = fe_zero();
    for (unsigned i = 0; i < n_elm; i++) acc = fe_add<FS>(acc, fe_mul<FS>(fe_pow_u64<FS>(load_fe_nc(elm + i), (uint64_t)j), load_fe_nc(scales + i)));
    store_fe(b + j, acc);
}

// out1 = (s, 0, 0)   out2 = (d * s, r_delta, d * b0)      (b0 = b[0] on the device)
template <class FS> __global__ void k_final_scalars(const fe* __restrict__ s, size_t len, fe d, fe r_delta, const fe* __restrict__ b0, fe* out1, fe* out2) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < len) {
        const fe v = load_fe_nc(s + t);
        store_fe(out1 + t, v);
        store_fe(out2 + t, fe_mul<FS>(v, d));
    } else if (t == len) {
        store_fe(out1 + len, fe_zero()); store_fe(out1 + len + 1, fe_zero());
        store_fe(out2 + len, r_delta); store_fe(out2 + len + 1, fe_mul<FS>(load_fe(b0), d));
    }
}

// rows[w * n_pts + e] = 2^(c w) * P_e, affine (one batch inversion) — the table layout of msm.cuh for the extra points
template <class HP> static void host_window_rows(const uint64_t* pts_xy, size_t n_pts, unsigned c, unsigned rows, std::vector<host::haffine>& out) {
    using namespace host;
    std::vector<hxyzz> all(rows * n_pts);
    for (size_t e = 0; e < n_pts; e++) {
        haffine a;
        memcpy(&a, pts_xy + 8 * e, 64);
        hxyzz cur = from_affine<HP>(a);
        for (unsigned w = 0; w < rows; w++) {
            if (w) for (unsigned k = 0; k < c; k++) cur = pdbl<HP>(cur);
            all[w * n_pts + e] = cur;
        }
    }
    // x = X / ZZ, y = Y / ZZZ with ONE inversion of prod (ZZ * ZZZ)
    const size_t m = all.size();
    std::vector<hfe> z(m), pre(m + 1);
    pre[0] = one<HP>();
    for (size_t i = 0; i < m; i++) {
        z[i] = is_inf(all[i]) ? one<HP>() : mul<HP>(all[i].ZZ, all[i].ZZZ);
        pre[i + 1] = mul<HP>(pre[i], z[i]);
    }
    hfe acc = inv<HP>(pre[m]);
    out.resize(m);
    for (size_t i = m; i-- > 0;) {
        const hfe zi = mul<HP>(acc, pre[i]);   // 1 / z[i]
        acc = mul<HP>(acc, z[i]);
        if (is_inf(all[i])) { out[i].x = zero(); out[i].y = zero(); continue; }
        out[i].x = mul<HP>(all[i].X, mul<HP>(zi, all[i].ZZZ));
        out[i].y = mul<HP>(all[i].Y, mul<HP>(zi, all[i].ZZ));
    }
}

struct PtrKind {
    const fe* dev = nullptr;    // usable from kernels as is (device memory, or page-locked host memory mapped into the device)
    bool staged = false;
};

template <class C>
static int open_impl(zk_srs* srs, const zk_open_poly* polys, size_t n_polys, const uint64_t* elm_mont, size_t n_elm, const uint64_t polyscale[4],
                     const uint64_t evalscale[4], const uint64_t* rng, const zk_open_transcript* tr, uint64_t* out_lr_xy, unsigned rounds,
                     uint64_t out_delta_xy[8], uint64_t out_z1[4], uint64_t out_z2[4], uint64_t out_sg_xy[8]) {
    using namespace host;
    using FS = typename C::FS; using HP = typename C::HP; using HS = typename C::HS;
    zk_ctx* ctx = srs->ctx;
    cudaStream_t st = ctx->stream;
    // ZKB200_TRACE_OPEN=1: wall-clock split of one call on stderr (diagnostic; tools/open_time.py)
    static const bool trace = getenv("ZKB200_TRACE_OPEN") != nullptr;
    using clk = std::chrono::steady_clock;
    const auto t_begin = clk::now();
    auto ms_since = [](clk::time_point t0) { return std::chrono::duration<double, std::milli>(clk::now() - t0).count(); };
    double tr_lr = 0, tr_host = 0, tr_fold = 0;
    const size_t srs_len = srs->n, n0 = (size_t)1 << rounds;
    const MsmBases& gb = srs->g->b;
    const unsigned c = gb.c, rows = c ? gb.nwin : 1;

    // ---- combine_polys, host side: the scale of every term and the combined blinder (utils.rs:127-177)
    hfe ps, es;
    memcpy(&ps, polyscale, 32);
    memcpy(&es, evalscale, 32);
    hfe scale = one<HS>(), combined_comm = zero();
    std::vector<CombineDesc> coeff_terms, eval_terms;
    size_t degree = 0, stage_elems = 0;
    std::vector<PtrKind> kinds(n_polys);
    for (size_t k = 0; k < n_polys; k++) {
        const zk_open_poly& p = polys[k];
        if ((!p.data && p.len) || (!p.blinders && p.n_blinders)) { zk_set_error("open: polynomial %zu has a null pointer", k); return ZK_ERR_INVALID; }
        cudaPointerAttributes attr;
        const bool known = p.len && cudaPointerGetAttributes(&attr, p.data) == cudaSuccess;
        if (!known) cudaGetLastError();
        if (known && (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged)) kinds[k].dev = (const fe*)p.data;
        else if (known && attr.type == cudaMemoryTypeHost && attr.devicePointer) kinds[k].dev = (const fe*)attr.devicePointer;
        else { kinds[k].staged = true; stage_elems += p.len; }
        if (p.domain_size) {
            if (degree && degree != p.domain_size) { zk_set_error("open: evaluation-form polynomials on different domains (%zu, %zu)", degree, p.domain_size); return ZK_ERR_INVALID; }
            if (p.len % p.domain_size || (p.domain_size & (p.domain_size - 1))) { zk_set_error("open: %zu evaluations do not tile a domain of %zu", p.len, p.domain_size); return ZK_ERR_INVALID; }
            degree = p.domain_size;
        }
    }
    // ---- device scratch: staged polynomial data, evaluation part, elm, scales, blinders | extra bases | descriptors
    unsigned log_deg = 0;
    while (((size_t)1 << log_deg) < degree) log_deg++;
    if (degree && log_deg > 30) { zk_set_error("open: evaluation domain too large"); return ZK_ERR_INVALID; }
    const size_t small_fe = n_elm * 2 + 2 * (size_t)rounds + 8;
    const size_t max_terms = n_polys + [&] { size_t t = 0; for (size_t k = 0; k < n_polys; k++) t += polys[k].n_blinders; return t; }();
    Layout lay;
    const size_t o_fe = lay.add((stage_elems + degree + small_fe) * sizeof(fe)), o_extra = lay.add(rows * 2 * sizeof(affine_t));
    const size_t o_desc = lay.add(max_terms * sizeof(CombineDesc));
    int rc = ctx->d_open.ensure(lay.total);
    if (rc) return rc;
    fe* d_stage = ctx->d_open.at<fe>(o_fe);
    fe* d_evals = d_stage + stage_elems;
    fe* d_small = d_evals + degree;                       // elm | eval scales | rand_l, rand_r ...
    affine_t* d_extra = ctx->d_open.at<affine_t>(o_extra);
    CombineDesc* d_descs = ctx->d_open.at<CombineDesc>(o_desc);
    {
        size_t off = 0;
        for (size_t k = 0; k < n_polys; k++) {
            if (!kinds[k].staged) continue;
            ZK_CUDA(cudaMemcpyAsync(d_stage + off, polys[k].data, polys[k].len * sizeof(fe), cudaMemcpyHostToDevice, st));
            kinds[k].dev = d_stage + off;
            off += polys[k].len;
        }
    }
    for (size_t k = 0; k < n_polys; k++) {
        const zk_open_poly& p = polys[k];
        if (p.domain_size) {
            CombineDesc d{};
            d.p = kinds[k].dev; d.len = (uint32_t)p.domain_size; d.stride = (uint32_t)(p.len / p.domain_size);
            memcpy(&d.scale, &scale, 32);
            if (p.len) eval_terms.push_back(d);
            for (size_t j = 0; j < p.n_blinders; j++) {
                hfe bl; memcpy(&bl, p.blinders + 4 * j, 32);
                combined_comm = add<HS>(combined_comm, mul<HS>(bl, scale));
                scale = mul<HS>(scale, ps);
            }
        } else {
            size_t off = 0;
            for (size_t j = 0; j < p.n_blinders; j++) {
                const size_t lo = std::min(off, p.len), hi = std::min(off + srs_len, p.len);
                if (hi > lo) {
                    CombineDesc d{};
                    d.p = kinds[k].dev + lo; d.len = (uint32_t)(hi - lo); d.stride = 1;
                    memcpy(&d.scale, &scale, 32);
                    coeff_terms.push_back(d);
                }
                hfe bl; memcpy(&bl, p.blinders + 4 * j, 32);
                combined_comm = add<HS>(combined_comm, mul<HS>(bl, scale));
                scale = mul<HS>(scale, ps);
                off += srs_len;
            }
        }
    }
    // ---- the rounds' state: a and b are built in place
    zk_ipa* s = nullptr;
    rc = ctx->d_ipa.ensure(ipa_storage_bytes(n0));
    if (rc) return rc;
    rc = ipa_create(ctx, srs->g, n0, &s, ctx->d_ipa.p);
    if (rc) return rc;
    struct Guard { zk_ipa* s; ~Guard() { cudaStreamSynchronize(s->ctx->stream); delete s; } } guard{s};
    std::vector<CombineDesc> all_terms(coeff_terms);
    all_terms.insert(all_terms.end(), eval_terms.begin(), eval_terms.end());
    if (!all_terms.empty()) ZK_CUDA(cudaMemcpyAsync(d_descs, all_terms.data(), all_terms.size() * sizeof(CombineDesc), cudaMemcpyHostToDevice, st));
    k_combine<FS><<<(unsigned)((n0 + 127) / 128), 128, 0, st>>>(d_descs, (unsigned)coeff_terms.size(), s->d_a, n0);
    ctx->launches += 1;
    if (degree) {
        k_combine<FS><<<(unsigned)((degree + 127) / 128), 128, 0, st>>>(d_descs + coeff_terms.size(), (unsigned)eval_terms.size(), d_evals, degree);
        ZK_CUDA(cudaGetLastError());
        rc = ctx_ntt_device(ctx, C::scalar_field, d_evals, log_deg, 1, 0, /*inverse=*/1, 0);     // Evaluations::interpolate (utils.rs:195-197)
        if (rc) return rc;
        const unsigned num_chunks = (unsigned)((degree + srs_len - 1) / srs_len);
        fe zeta;
        memcpy(&zeta, polyscale, 32);
        k_linearize_add<FS><<<(unsigned)((srs_len + 127) / 128), 128, 0, st>>>(s->d_a, d_evals, degree, srs_len, num_chunks, zeta, fe_one<FS>());
        ctx->launches += 2;
    }
    // ---- b_init and the combined inner product (ipa.rs:876-896)
    std::vector<hfe> small(small_fe);
    {
        hfe sc = one<HS>();
        for (size_t i = 0; i < n_elm; i++) {
            memcpy(&small[i], elm_mont + 4 * i, 32);
            small[n_elm + i] = sc;
            sc = mul<HS>(sc, es);
        }
        memcpy(&small[2 * n_elm], rng, 2 * (size_t)rounds * 32);
    }
    ZK_CUDA(cudaMemcpyAsync(d_small, small.data(), small_fe * sizeof(fe), cudaMemcpyHostToDevice, st));
    k_b_init<FS><<<(unsigned)((n0 + 127) / 128), 128, 0, st>>>(d_small, d_small + n_elm, (unsigned)n_elm, s->d_b, n0);
    ctx->launches += 1;
    ZK_CUDA(cudaGetLastError());
    rc = ipa_inner_product<FS>(s, s->d_a, s->d_b, n0, s->d_part + IP_BLOCKS);
    if (rc) return rc;
    ZK_CUDA(cudaMemcpyAsync(s->h_ip, s->d_part + IP_BLOCKS, sizeof(fe), cudaMemcpyDeviceToHost, st));
    ZK_CUDA(cudaStreamSynchronize(st));
    uint64_t cip[4], u_xy[8];
    memcpy(cip, s->h_ip, 32);
    if (tr->u_base(tr->user, cip, u_xy) != 0) { zk_set_error("open: the u_base callback failed"); return ZK_ERR_INVALID; }
    // ---- h and U as extra bases: their window rows, laid out like the table
    {
        uint64_t pts[16];
        memcpy(pts, srs->h, 64);
        memcpy(pts + 8, u_xy, 64);
        std::vector<haffine> rws;
        host_window_rows<HP>(pts, 2, c, rows, rws);
        ZK_CUDA(cudaMemcpyAsync(d_extra, rws.data(), rws.size() * sizeof(haffine), cudaMemcpyHostToDevice, st));
        ZK_CUDA(cudaStreamSynchronize(st));     // rws is a local
    }
    s->d_extra = d_extra;
    s->d_rand = d_small + 2 * n_elm;
    const double tr_setup = ms_since(t_begin);
    // ---- the folding rounds (ipa.rs:929-1007)
    std::vector<hfe> chals(rounds), chal_invs(rounds);
    for (unsigned r = 0; r < rounds; r++) {
        uint64_t l_jac[12], r_jac[12];
        const auto t_r0 = clk::now();
        rc = ipa_round_lr(s, l_jac, r_jac, nullptr, nullptr);
        if (rc) return rc;
        const auto t_r1 = clk::now();
        uint64_t* lr = out_lr_xy + 16 * (size_t)r;
        zk_jacobian_to_affine(srs->curve, l_jac, lr);
        zk_jacobian_to_affine(srs->curve, r_jac, lr + 8);
        uint64_t u[4];
        if (tr->round(tr->user, r, lr, lr + 8, u) != 0) { zk_set_error("open: the round callback failed"); return ZK_ERR_INVALID; }
        memcpy(&chals[r], u, 32);
        if (is_zero(chals[r])) { zk_set_error("open: zero challenge"); return ZK_ERR_INVALID; }
        chal_invs[r] = inv<HS>(chals[r]);
        const auto t_r2 = clk::now();
        rc = ipa_round_fold(s, chals[r].l, chal_invs[r].l);
        if (rc) return rc;
        if (trace) {
            tr_lr += std::chrono::duration<double, std::milli>(t_r1 - t_r0).count();
            tr_host += std::chrono::duration<double, std::milli>(t_r2 - t_r1).count();
            tr_fold += ms_since(t_r2);
        }
    }
    const auto t_final = clk::now();
    // ---- a0, r_prime, then sg and delta as one MSM pair (ipa.rs:1009-1038)
    hfe a0;
    ZK_CUDA(cudaMemcpyAsync(s->h_ip, s->d_a, sizeof(fe), cudaMemcpyDeviceToHost, st));
    hfe r_prime = combined_comm;
    for (unsigned r = 0; r < rounds; r++) {
        hfe rl, rr;
        memcpy(&rl, rng + 8 * (size_t)r, 32);
        memcpy(&rr, rng + 8 * (size_t)r + 4, 32);
        r_prime = add<HS>(r_prime, add<HS>(mul<HS>(rl, chal_invs[r]), mul<HS>(rr, chals[r])));
    }
    hfe d, r_delta;
    memcpy(&d, rng + 8 * (size_t)rounds, 32);
    memcpy(&r_delta, rng + 8 * (size_t)rounds + 4, 32);
    const size_t len = std::min(n0, gb.n), stride = n0 + 2;
    fe fd, frd;
    memcpy(&fd, &d, 32);
    memcpy(&frd, &r_delta, 32);
    k_final_scalars<FS><<<(unsigned)((len + 1 + 127) / 128), 128, 0, st>>>(s->d_s[s->cur], len, fd, frd, s->d_b, s->d_sc, s->d_sc + stride);
    ctx->launches += 1;
    ZK_CUDA(cudaGetLastError());
    const fe* scs[2] = {s->d_sc, s->d_sc + stride};
    uint64_t fin[24];
    rc = ctx_msm_many(ctx, srs->g, 0, len, scs, 2, /*mont=*/1, 0, fin, d_extra, 2);     // synchronises: a0 has landed too
    if (rc) return rc;
    memcpy(&a0, s->h_ip, 32);
    zk_jacobian_to_affine(srs->curve, fin, out_sg_xy);
    zk_jacobian_to_affine(srs->curve, fin + 12, out_delta_xy);
    uint64_t cch[4];
    if (tr->final_challenge(tr->user, out_delta_xy, cch) != 0) { zk_set_error("open: the final_challenge callback failed"); return ZK_ERR_INVALID; }
    hfe cc;
    memcpy(&cc, cch, 32);
    const hfe z1 = add<HS>(mul<HS>(a0, cc), d), z2 = add<HS>(mul<HS>(r_prime, cc), r_delta);
    memcpy(out_z1, &z1, 32);
    memcpy(out_z2, &z2, 32);
    if (trace)
        fprintf(stderr, "[zk_srs_open] setup (combine, b, <a,b>, U rows) %.3f ms | %u rounds: L/R MSM pairs %.3f, host (affine, transcript, 1/u) %.3f, fold launches %.3f | "
                        "final (sg, delta, z) %.3f | total %.3f ms\n", tr_setup, rounds, tr_lr, tr_host, tr_fold, ms_since(t_final), ms_since(t_begin));
    return ZK_OK;
}

}  // namespace zkb

extern "C" int zk_srs_open(zk_srs* srs, const zk_open_poly* polys, size_t n_polys, const uint64_t* elm_mont, size_t n_elm,
                           const uint64_t polyscale[4], const uint64_t evalscale[4], const uint64_t* rng_scalars, size_t n_rng_scalars,
                           const zk_open_transcript* transcript, uint64_t* out_lr_xy, size_t lr_capacity_rounds, size_t* out_rounds,
                           uint64_t out_delta_xy[8], uint64_t out_z1[4], uint64_t out_z2[4], uint64_t out_sg_xy[8]) {
    if (!srs || (!polys && n_polys) || (!elm_mont && n_elm) || !polyscale || !evalscale || !rng_scalars || !transcript || !out_rounds ||
        !out_delta_xy || !out_z1 || !out_z2 || !out_sg_xy) { zk_set_error("open: null argument"); return ZK_ERR_INVALID; }
    if (!transcript->u_base || !transcript->round || !transcript->final_challenge) { zk_set_error("open: transcript callback missing"); return ZK_ERR_INVALID; }
    unsigned rounds = 0;                          // math::ceil_log2(self.g.len())
    while (((size_t)1 << rounds) < srs->n) rounds++;
    *out_rounds = rounds;
    if (n_rng_scalars != 2 * (size_t)rounds + 2) { zk_set_error("open: %zu random scalars given, 2 * %u + 2 needed", n_rng_scalars, rounds); return ZK_ERR_LENGTH; }
    if (rounds > lr_capacity_rounds || (rounds && !out_lr_xy)) { zk_set_error("open: room for %zu (l, r) pairs, %u needed", lr_capacity_rounds, rounds); return ZK_ERR_LENGTH; }
    zk_ctx* ctx = srs->ctx;
    std::lock_guard<std::mutex> lk(ctx->mu);   // held across the callbacks: they must not call into this context
    ZK_CUDA(cudaSetDevice(ctx->device));
    return with_curve(srs->curve, [&](auto c) {
        return open_impl<decltype(c)>(srs, polys, n_polys, elm_mont, n_elm, polyscale, evalscale, rng_scalars, transcript, out_lr_xy, rounds, out_delta_xy, out_z1, out_z2, out_sg_xy);
    });
}
