// verify.cu — SRS::verify (poly-commitment/src/ipa.rs:301-502) behind one C-ABI call, zk_srs_verify (include/zkb200.h).
//
// The reference builds one MSM over  h || g || padding || (per proof: sg, U, L_j, R_j ..., commitment chunks, U, delta)  and compares
// it with zero.  Here it is split in two:
//   * the g part: S[j] = sum_i sg_rand_base^i s_i[j], s_i = b_poly_coefficients(chal_i) (commitment.rs:464-476: bit t of j selects
//     chal_i[k_i - 1 - t]).  Per proof, a table of the products over the low L bits of j and one over the high K - L bits (the
//     weight folded into the high table) are built by k_verify_tables; k_verify_s then costs one product and one addition per
//     (proof, j).  Two launches for the whole batch, whatever its size.  S runs through the fused MSM pipeline over the resident
//     generator table (ctx_msm_many, Montgomery scalars).
//   * the proof points: h, then per proof sg, U (its two scalars merged), L_j, R_j, the commitment chunks, delta — about
//     2k + 4 + #chunks points per proof — as a transient plain base set (no window table) of the same pipeline.
// Host: the callbacks (the caller's sponge and group map), the O(k + #chunks) scalar arithmetic per proof (one batch inversion of
// all challenges, b0 = sum_i evalscale^i b_poly(chal, elm_i) in O(k) per point, commitment.rs:426-436), and the sum of the two
// Jacobian results.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/zkb200.h"
#include "ctx.hpp"
#include "msm.cuh"

using namespace zkb;

namespace zkb {

// Per proof i (blockIdx-linear index over B x (2^L + 2^H) entries):
//   lo[i][e] = prod_{t < L, bit t of e} rev[i][t]           hi[i][e] = w[i] * prod_{t < H, bit t of e} rev[i][L + t]
// rev[i][t] = chal_i[k_i - 1 - t] for t < k_i and 0 above, so the entries of j >= 2^k_i vanish (the proof's s covers 2^k_i entries)
template <class FS>
__global__ void k_verify_tables(const fe* __restrict__ rev, const fe* __restrict__ w, unsigned B, unsigned K, unsigned L, fe* lo, fe* hi) {
    const unsigned H = K - L;
    const size_t per = ((size_t)1 << L) + ((size_t)1 << H);
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= per * B) return;
    const unsigned i = (unsigned)(idx / per);
    size_t e = idx % per;
    const fe* r = rev + (size_t)i * K;
    if (e < ((size_t)1 << L)) {
        fe v = fe_one<FS>();
        for (unsigned t = 0; t < L; t++)
            if ((e >> t) & 1) v = fe_mul<FS>(v, load_fe_nc(r + t));
        store_fe(lo + ((size_t)i << L) + e, v);
    } else {
        e -= (size_t)1 << L;
        fe v = load_fe_nc(w + i);
        for (unsigned t = 0; t < H; t++)
            if ((e >> t) & 1) v = fe_mul<FS>(v, load_fe_nc(r + L + t));
        store_fe(hi + ((size_t)i << H) + e, v);
    }
}

// S[j] = sum_i lo[i][j mod 2^L] * hi[i][j >> L],  j < len
template <class FS>
__global__ void k_verify_s(const fe* __restrict__ lo, const fe* __restrict__ hi, unsigned B, unsigned L, unsigned H, fe* S, size_t len) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= len) return;
    const size_t jl = j & (((size_t)1 << L) - 1), jh = j >> L;
    fe acc = fe_zero();
    for (unsigned i = 0; i < B; i++)
        acc = fe_add<FS>(acc, fe_mul<FS>(load_fe_nc(lo + ((size_t)i << L) + jl), load_fe_nc(hi + ((size_t)i << H) + jh)));
    store_fe(S + j, acc);
}

template <class C>
static int verify_impl(zk_srs* srs, const zk_verify_proof* batch, size_t B, const uint64_t* rng, int* out_ok, uint64_t* out_sum_xyz) {
    using namespace host;
    using FS = typename C::FS; using HP = typename C::HP; using HS = typename C::HS;
    zk_ctx* ctx = srs->ctx;
    cudaStream_t st = ctx->stream;
    // ZKB200_TRACE_VERIFY=1: wall-clock split of one call on stderr (diagnostic; tools/verify_time.py)
    static const bool trace = getenv("ZKB200_TRACE_VERIFY") != nullptr;
    using clk = std::chrono::steady_clock;
    auto ms = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    const auto t0 = clk::now();
    unsigned K = 0;                                  // max_rounds = math::ceil_log2(self.g.len())
    while (((size_t)1 << K) < srs->n) K++;
    const size_t len = srs->n;
    hfe rand_base, sg_rand_base;
    memcpy(&rand_base, rng, 32);
    memcpy(&sg_rand_base, rng + 4, 32);

    // ---- the transcripts, proof by proof in batch order (ipa.rs:372-383)
    std::vector<hfe> chals, us(B), cs(B);
    std::vector<haffine> ubase(B);
    std::vector<size_t> chal_off(B + 1, 0);
    for (size_t i = 0; i < B; i++) chal_off[i + 1] = chal_off[i] + batch[i].n_rounds;
    chals.resize(chal_off[B]);
    for (size_t i = 0; i < B; i++) {
        const zk_verify_proof& p = batch[i];
        const zk_open_transcript* tr = p.transcript;
        if (tr->u_base(tr->user, p.combined_inner_product, (uint64_t*)&ubase[i]) != 0) { zk_set_error("verify: proof %zu: the u_base callback failed", i); return ZK_ERR_INVALID; }
        for (size_t j = 0; j < p.n_rounds; j++) {
            uint64_t u[4];
            if (tr->round(tr->user, (unsigned)j, p.lr_xy + 16 * j, p.lr_xy + 16 * j + 8, u) != 0) { zk_set_error("verify: proof %zu: the round callback failed", i); return ZK_ERR_INVALID; }
            memcpy(&chals[chal_off[i] + j], u, 32);
        }
        uint64_t c[4];
        if (tr->final_challenge(tr->user, p.delta_xy, c) != 0) { zk_set_error("verify: proof %zu: the final_challenge callback failed", i); return ZK_ERR_INVALID; }
        memcpy(&cs[i], c, 32);
    }
    const auto t_tr = clk::now();

    // ---- chal_inv: ark_ff::batch_inversion over every challenge of the batch (zeros are skipped and stay zero)
    const size_t nc = chals.size();
    std::vector<hfe> chal_inv(nc, zero()), pre(nc + 1);
    pre[0] = one<HS>();
    for (size_t t = 0; t < nc; t++) pre[t + 1] = is_zero(chals[t]) ? pre[t] : mul<HS>(pre[t], chals[t]);
    {
        hfe acc = inv<HS>(pre[nc]);
        for (size_t t = nc; t-- > 0;) {
            if (is_zero(chals[t])) continue;
            chal_inv[t] = mul<HS>(acc, pre[t]);
            acc = mul<HS>(acc, chals[t]);
        }
    }

    // ---- the proof points and their scalars (ipa.rs:404-499): h first, then per proof sg, U, (L_j, R_j)..., chunks, delta
    size_t n_pts = 1;
    for (size_t i = 0; i < B; i++) {
        n_pts += 3 + 2 * batch[i].n_rounds;
        for (size_t q = 0; q < batch[i].n_comms; q++) n_pts += batch[i].comm_chunks[q];
    }
    std::vector<haffine> pts(n_pts);
    std::vector<hfe> sc(n_pts);
    const unsigned L = (K + 1) / 2, H = K - L;
    std::vector<hfe> rev((size_t)B * (K ? K : 1), zero()), wts(B);
    memcpy(&pts[0], srs->h, 64);
    hfe h_scalar = zero(), r_i = one<HS>(), w_i = one<HS>();
    size_t at = 1;
    auto put = [&](const uint64_t* xy, const hfe& s) { memcpy(&pts[at], xy, 64); sc[at] = s; at++; };
    for (size_t i = 0; i < B; i++) {
        const zk_verify_proof& p = batch[i];
        const hfe* ch = chals.data() + chal_off[i];
        const hfe* ci = chal_inv.data() + chal_off[i];
        const size_t k = p.n_rounds;
        hfe z1, z2, cip, es, ps;
        memcpy(&z1, p.z1, 32); memcpy(&z2, p.z2, 32); memcpy(&cip, p.combined_inner_product, 32);
        memcpy(&es, p.evalscale, 32); memcpy(&ps, p.polyscale, 32);
        // b0 = sum_e evalscale^e b_poly(chal, elm_e),  b_poly(chal, x) = prod_t (1 + chal[t] x^(2^(k-1-t)))   (commitment.rs:426-436)
        hfe b0 = zero(), esc = one<HS>();
        std::vector<hfe> pow2(k ? k : 1);
        for (size_t e = 0; e < p.n_elm; e++) {
            hfe x;
            memcpy(&x, p.elm + 4 * e, 32);
            if (k) pow2[0] = x;
            for (size_t t = 1; t < k; t++) pow2[t] = sqr<HS>(pow2[t - 1]);
            hfe term = one<HS>();
            for (size_t t = 0; t < k; t++) term = mul<HS>(term, add<HS>(one<HS>(), mul<HS>(ch[t], pow2[k - 1 - t])));
            b0 = add<HS>(b0, mul<HS>(esc, term));
            esc = mul<HS>(esc, es);
        }
        const hfe rz1 = mul<HS>(r_i, z1), rc = mul<HS>(cs[i], r_i);
        h_scalar = sub<HS>(h_scalar, mul<HS>(r_i, z2));                              // - rand_base_i z2 H
        put(p.sg_xy, sub<HS>(sub<HS>(zero(), rz1), w_i));                             // (- rand_base_i z1 - sg_rand_base_i) sg
        put((const uint64_t*)&ubase[i], sub<HS>(mul<HS>(rc, cip), mul<HS>(rz1, b0))); // (rand_base_i c cip - rand_base_i z1 b0) U
        for (size_t j = 0; j < k; j++) {
            put(p.lr_xy + 16 * j, mul<HS>(rc, ci[j]));                               // rand_base_i c u_j^-1 L_j
            put(p.lr_xy + 16 * j + 8, mul<HS>(rc, ch[j]));                           // rand_base_i c u_j R_j
        }
        hfe psi = one<HS>();                                                          // combine_commitments (commitment.rs:724-744)
        size_t off = 0;
        for (size_t q = 0; q < p.n_comms; q++)
            for (size_t t = 0; t < p.comm_chunks[q]; t++, off++) {
                put(p.comm_xy + 8 * off, mul<HS>(rc, psi));
                psi = mul<HS>(psi, ps);
            }
        put(p.delta_xy, r_i);                                                         // rand_base_i delta
        for (size_t t = 0; t < k; t++) rev[i * K + t] = ch[k - 1 - t];
        wts[i] = w_i;
        r_i = mul<HS>(r_i, rand_base);
        w_i = mul<HS>(w_i, sg_rand_base);
    }
    sc[0] = h_scalar;
    const auto t_host = clk::now();

    // ---- device scratch: S, lo tables, hi tables, rev, weights, proof scalars | proof points (affine)
    const size_t n_lo = (size_t)B << L, n_hi = (size_t)B << H;
    Layout lay;
    const size_t o_fe = lay.add((len + n_lo + n_hi + rev.size() + B + n_pts) * sizeof(fe)), o_pts = lay.add(n_pts * sizeof(affine_t));
    int rc = ctx->d_verify.ensure(lay.total);
    if (rc) return rc;
    fe* d_S = ctx->d_verify.at<fe>(o_fe);
    fe* d_lo = d_S + len;
    fe* d_hi = d_lo + n_lo;
    fe* d_rev = d_hi + n_hi;
    fe* d_w = d_rev + rev.size();
    fe* d_sc = d_w + B;
    affine_t* d_pts = ctx->d_verify.at<affine_t>(o_pts);
    ZK_CUDA(cudaMemcpyAsync(d_rev, rev.data(), rev.size() * sizeof(fe), cudaMemcpyHostToDevice, st));
    ZK_CUDA(cudaMemcpyAsync(d_w, wts.data(), B * sizeof(fe), cudaMemcpyHostToDevice, st));
    ZK_CUDA(cudaMemcpyAsync(d_sc, sc.data(), n_pts * sizeof(fe), cudaMemcpyHostToDevice, st));
    ZK_CUDA(cudaMemcpyAsync(d_pts, pts.data(), n_pts * sizeof(affine_t), cudaMemcpyHostToDevice, st));
    const size_t n_tab = n_lo + n_hi;
    k_verify_tables<FS><<<(unsigned)((n_tab + 127) / 128), 128, 0, st>>>(d_rev, d_w, (unsigned)B, K, L, d_lo, d_hi);
    ZK_CUDA(cudaGetLastError());
    k_verify_s<FS><<<(unsigned)((len + 127) / 128), 128, 0, st>>>(d_lo, d_hi, (unsigned)B, L, H, d_S, len);
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 2;
    if (trace) ZK_CUDA(cudaStreamSynchronize(st));
    const auto t_s = clk::now();

    // ---- <S, g> over the resident table, then the proof points as a transient plain base set
    uint64_t out_g[12], out_p[12];
    const fe* s_ptr = d_S;
    rc = ctx_msm_many(ctx, srs->g, 0, len, &s_ptr, 1, /*mont=*/1, 0, out_g);
    if (rc) return rc;
    const auto t_g = clk::now();
    zk_bases pb;
    pb.ctx = ctx;
    pb.b.curve = srs->curve;
    pb.b.n = n_pts;
    pb.b.c = 0;
    pb.b.nwin = 0;
    pb.b.d_points = d_pts;
    const fe* p_ptr = d_sc;
    rc = ctx_msm_many(ctx, &pb, 0, n_pts, &p_ptr, 1, /*mont=*/1, 0, out_p);
    if (rc) return rc;
    const auto t_p = clk::now();

    hjac jg, jp;
    memcpy(&jg, out_g, 96);
    memcpy(&jp, out_p, 96);
    const hxyzz sum = padd<HP>(from_jacobian<HP>(jg), from_jacobian<HP>(jp));
    *out_ok = is_inf(sum) ? 1 : 0;
    if (out_sum_xyz) {
        const hjac js = to_jacobian<HP>(sum);
        memcpy(out_sum_xyz, &js, 96);
    }
    if (trace)
        fprintf(stderr, "[zk_srs_verify] %zu proofs, %zu proof points | transcript callbacks %.3f ms | host scalars %.3f | s-vector kernels %.3f | "
                        "g MSM %.3f | proof-point MSM %.3f | total %.3f ms\n",
                B, n_pts, ms(t0, t_tr), ms(t_tr, t_host), ms(t_host, t_s), ms(t_s, t_g), ms(t_g, t_p), ms(t0, clk::now()));
    return ZK_OK;
}

}  // namespace zkb

extern "C" int zk_srs_verify(zk_srs* srs, const zk_verify_proof* batch, size_t n, const uint64_t rng_scalars[8], int* out_ok,
                             uint64_t out_sum_xyz[12]) {
    if (!srs || (!batch && n) || !rng_scalars || !out_ok) { zk_set_error("verify: null argument"); return ZK_ERR_INVALID; }
    unsigned K = 0;
    while (((size_t)1 << K) < srs->n) K++;
    for (size_t i = 0; i < n; i++) {
        const zk_verify_proof& p = batch[i];
        const zk_open_transcript* tr = p.transcript;
        size_t chunks = 0;
        for (size_t q = 0; p.comm_chunks && q < p.n_comms; q++) chunks += p.comm_chunks[q];
        if ((!p.lr_xy && p.n_rounds) || !p.delta_xy || !p.z1 || !p.z2 || !p.sg_xy || (!p.elm && p.n_elm) || !p.polyscale || !p.evalscale ||
            (!p.comm_chunks && p.n_comms) || (!p.comm_xy && chunks) || !p.combined_inner_product || !tr || !tr->u_base || !tr->round ||
            !tr->final_challenge) { zk_set_error("verify: proof %zu has a null pointer", i); return ZK_ERR_INVALID; }
        if (p.n_rounds > K) { zk_set_error("verify: proof %zu has %zu rounds, the SRS of %zu points allows %u", i, p.n_rounds, srs->n, K); return ZK_ERR_LENGTH; }
    }
    if (n == 0) {                 // the reference's MSM of all-zero scalars is the identity
        *out_ok = 1;
        if (out_sum_xyz) {
            const host::hjac id = with_curve(srs->curve, [](auto c) { return host::to_jacobian<typename decltype(c)::HP>(host::identity()); });
            memcpy(out_sum_xyz, &id, 96);
        }
        return ZK_OK;
    }
    zk_ctx* ctx = srs->ctx;
    std::lock_guard<std::mutex> lk(ctx->mu);   // held across the callbacks: they must not call into this context
    ZK_CUDA(cudaSetDevice(ctx->device));
    return with_curve(srs->curve, [&](auto c) { return verify_impl<decltype(c)>(srs, batch, n, rng_scalars, out_ok, out_sum_xyz); });
}
