// ipa.cu — device-resident state for the folding rounds of the IPA opening proof, SRS::open
// (poly-commitment/src/ipa.rs:929-1007).  The coefficient vector a and the evaluation vector b are folded in HBM; the bases are
// NEVER folded: after j rounds with challenges u_1..u_j the reference's folded bases are
//     g_j[i] = sum_t s_j[t] * g[t * m_j + i],      m_j = n / 2^j,   s_j = b_poly_coefficients(u_1..u_j)  (commitment.rs:565-581)
// so the round's two commitments are MSMs over the ORIGINAL, resident, table-precomputed SRS points with expanded scalars
//     L_j = <a_hi, g_j,lo> = sum_{t, i < h} (a[h + i] s_j[t]) g[t m_j + i]          (h = m_j / 2; ipa.rs:943-961)
//     R_j = <a_lo, g_j,hi> = sum_{t, i < h} (a[i] s_j[t])     g[t m_j + h + i]
// and the final base g0 (the proof's `sg`) is <s_k, g>.  That replaces log2(n) rounds of per-point scalar multiplications
// (G::combine_one_endo, commitment.rs:539 / combine.rs:292-342 — latency-bound chains of ~380 group operations per point) by
// the throughput-bound MSM pipeline of msm.cu; the group elements produced are the same.  L and R of a round are ONE fused
// pipeline (two bucket groups).  Two ways to drive the rounds:
//   zk_ipa_*      the bare rounds: the host owns the Fiat-Shamir sponge, rand_l / rand_r, h and u_base; it finishes L and R
//                 (two scalar multiplications each), squeezes u, and asks for the fold
//   zk_srs_open   (open.cu) the whole SRS::open: h and U are two extra points of the same MSMs, their scalars (the blinders and
//                 the inner products) are appended on the device, so a round returns the finished L and R
//     a <- a_lo + u^-1 a_hi,   b <- b_lo + u b_hi,   s <- (s[t], u s[t])_t          (ipa.rs:980-1006)
// SURVEY.md §8f row 1.
#include <mutex>

#include "../../include/zkb200.h"
#include "ipa.hpp"
#include "msm.cuh"

using namespace zkb;

namespace zkb {

// partial[blockIdx] = sum over the block's strided share of x[i] * y[i]  (Montgomery in, Montgomery out)
template <class FS> __global__ void __launch_bounds__(IP_THREADS) k_inner_product(const fe* __restrict__ x, const fe* __restrict__ y, size_t m, fe* partial) {
    __shared__ fe sm[IP_THREADS];
    fe acc = fe_zero();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (size_t)gridDim.x * blockDim.x)
        acc = fe_add<FS>(acc, fe_mul<FS>(load_fe_nc(x + i), load_fe_nc(y + i)));
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (unsigned s = blockDim.x >> 1; s >= 1; s >>= 1) {
        if (threadIdx.x < s) sm[threadIdx.x] = fe_add<FS>(sm[threadIdx.x], sm[threadIdx.x + s]);
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = sm[0];
}
template <class FS> __global__ void __launch_bounds__(IP_BLOCKS) k_inner_product_final(const fe* __restrict__ partial, fe* out) {
    __shared__ fe sm[IP_BLOCKS];
    sm[threadIdx.x] = partial[threadIdx.x];
    __syncthreads();
    for (unsigned s = IP_BLOCKS >> 1; s >= 1; s >>= 1) {
        if (threadIdx.x < s) sm[threadIdx.x] = fe_add<FS>(sm[threadIdx.x], sm[threadIdx.x + s]);
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = sm[0];
}

// v[i] <- v[i] + c * v[i + half]
template <class FS> __global__ void k_fold_field(fe* v, size_t half, fe c) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= half) return;
    store_fe(v + i, fe_add<FS>(load_fe(v + i), fe_mul<FS>(load_fe(v + i + half), c)));
}

// s_new[2t] = s[t], s_new[2t + 1] = u * s[t]
template <class FS> __global__ void k_expand_challenges(const fe* __restrict__ s_old, fe* s_new, size_t count, fe u) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    fe v = load_fe_nc(s_old + t);
    store_fe(s_new + 2 * t, v);
    store_fe(s_new + 2 * t + 1, fe_mul<FS>(v, u));
}

// sc[t * m + i] = (right ? (i >= h ? a[i - h] : 0) : (i < h ? a[h + i] : 0)) * s[t],  m = 2h
template <class FS> __global__ void k_expand_scalars(fe* sc, const fe* __restrict__ a, const fe* __restrict__ s, size_t n0, size_t h, int right) {
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n0) return;
    const size_t m = 2 * h, t = idx / m, i = idx % m;
    fe v = fe_zero();
    if (right ? (i >= h) : (i < h)) v = fe_mul<FS>(load_fe_nc(a + (right ? i - h : i + h)), load_fe_nc(s + t));
    store_fe(sc + idx, v);
}

// the scalars of the two extra points (h, U) behind the `len` base scalars of L and of R:  (rand_l, <a_hi, b_lo>), (rand_r, <a_lo, b_hi>)
__global__ void k_tail_scalars(fe* sc_l, fe* sc_r, size_t len, const fe* __restrict__ rand_lr, const fe* __restrict__ ips) {
    if (threadIdx.x == 0) { store_fe(sc_l + len, load_fe(rand_lr)); store_fe(sc_l + len + 1, load_fe(ips)); }
    if (threadIdx.x == 1) { store_fe(sc_r + len, load_fe(rand_lr + 1)); store_fe(sc_r + len + 1, load_fe(ips + 1)); }
}

template <class FS> int ipa_inner_product(zk_ipa* s, const fe* x, const fe* y, size_t m, fe* d_out) {
    k_inner_product<FS><<<IP_BLOCKS, IP_THREADS, 0, s->ctx->stream>>>(x, y, m, s->d_part);
    k_inner_product_final<FS><<<1, IP_BLOCKS, 0, s->ctx->stream>>>(s->d_part, d_out);
    ZK_CUDA(cudaGetLastError());
    s->ctx->launches += 2;
    return ZK_OK;
}
template int ipa_inner_product<FpParams>(zk_ipa*, const fe*, const fe*, size_t, fe*);
template int ipa_inner_product<FqParams>(zk_ipa*, const fe*, const fe*, size_t, fe*);

// L and R of one round: both scalar vectors are expanded on the main stream, the two MSMs run as ONE fused pipeline
template <class FS> static int ipa_expand_and_msm(zk_ipa* s, size_t h, uint64_t out_l_xyz[12], uint64_t out_r_xyz[12]) {
    zk_ctx* ctx = s->ctx;
    const unsigned blocks = (unsigned)((s->n0 + 255) / 256);
    const size_t stride = s->n0 + 2;                                    // room for the two extra scalars
    fe *sc_l = s->d_sc, *sc_r = s->d_sc + stride;
    k_expand_scalars<FS><<<blocks, 256, 0, ctx->stream>>>(sc_l, s->d_a, s->d_s[s->cur], s->n0, h, 0);
    k_expand_scalars<FS><<<blocks, 256, 0, ctx->stream>>>(sc_r, s->d_a, s->d_s[s->cur], s->n0, h, 1);
    ctx->launches += 2;
    const size_t len = s->n0 < s->bases->b.n ? s->n0 : s->bases->b.n;   // positions past the SRS are identity padding
    const bool extras = s->d_extra != nullptr;
    if (extras) {
        k_tail_scalars<<<1, 32, 0, ctx->stream>>>(sc_l, sc_r, len, s->d_rand + 2 * s->round, s->d_part + IP_BLOCKS);
        ctx->launches += 1;
    }
    ZK_CUDA(cudaGetLastError());
    const fe* scs[2] = {sc_l, sc_r};
    uint64_t out[24];
    int rc = ctx_msm_many(ctx, s->bases, 0, len, scs, 2, /*mont=*/1, 0, out, s->d_extra, extras ? 2 : 0);
    if (rc) return rc;
    memcpy(out_l_xyz, out, 96);
    memcpy(out_r_xyz, out + 12, 96);
    return ZK_OK;
}

// one device allocation: a | b | s0 | s1 | sc_L (+2) | sc_R (+2) | partials (+ two inner products)
size_t ipa_storage_bytes(size_t n) { return (6 * n + 4 + IP_BLOCKS + 2) * sizeof(fe); }

int ipa_create(zk_ctx* ctx, const zk_bases* bases, size_t n, zk_ipa** out, void* storage) {
    if (n < 1 || (n & (n - 1))) { zk_set_error("ipa: n must be a power of two (the reference pads to a power of two, ipa.rs:848-850)"); return ZK_ERR_INVALID; }
    if (bases->b.n > n || (n > 1 && 2 * bases->b.n <= n)) { zk_set_error("ipa: n = %zu is not the SRS size %zu rounded up to a power of two", n, bases->b.n); return ZK_ERR_INVALID; }
    PinnedSlots* pin = ctx_pinned(ctx);
    if (!pin) return ZK_ERR_CUDA;
    auto s = std::make_unique<zk_ipa>();
    s->ctx = ctx; s->curve = bases->b.curve; s->n = s->n0 = n; s->bases = bases;
    if (!storage) {
        if (int rc = s->storage.ensure(ipa_storage_bytes(n))) return rc;
        storage = s->storage.p;
    }
    s->d_a = (fe*)storage;
    s->d_b = s->d_a + n; s->d_s[0] = s->d_a + 2 * n; s->d_s[1] = s->d_a + 3 * n; s->d_sc = s->d_a + 4 * n; s->d_part = s->d_a + 6 * n + 4;
    s->h_ip = pin->ip;
    // s_0 = (1), staged through the curve's slot (PinnedSlots::s0)
    const fe* one = with_curve(s->curve, [&](auto c) { using C = decltype(c); return &(pin->s0[C::scalar_field] = fe_one<typename C::FS>()); });
    if (cudaError_t e = cudaMemcpyAsync(s->d_s[0], one, sizeof(fe), cudaMemcpyHostToDevice, ctx->stream)) {
        zk_set_error("ipa: %s", cudaGetErrorString(e));
        return ZK_ERR_CUDA;
    }
    *out = s.release();
    return ZK_OK;
}

int ipa_round_lr(zk_ipa* s, uint64_t out_l_xyz[12], uint64_t out_r_xyz[12], uint64_t out_ip_l[4], uint64_t out_ip_r[4]) {
    if (s->n < 2) { zk_set_error("ipa_round_lr: folding is complete"); return ZK_ERR_INVALID; }
    zk_ctx* ctx = s->ctx;
    const size_t h = s->n / 2;
    int rc = with_curve(s->curve, [&](auto c) {
        using FS = typename decltype(c)::FS;
        // inner products <a_hi, b_lo>, <a_lo, b_hi>
        if (int e = ipa_inner_product<FS>(s, s->d_a + h, s->d_b, h, s->d_part + IP_BLOCKS)) return e;
        if (int e = ipa_inner_product<FS>(s, s->d_a, s->d_b + h, h, s->d_part + IP_BLOCKS + 1)) return e;
        if (out_ip_l) ZK_CUDA(cudaMemcpyAsync(s->h_ip, s->d_part + IP_BLOCKS, 2 * sizeof(fe), cudaMemcpyDeviceToHost, ctx->stream));
        return ipa_expand_and_msm<FS>(s, h, out_l_xyz, out_r_xyz);
    });
    if (rc) return rc;
    if (out_ip_l) {
        ZK_CUDA(cudaStreamSynchronize(ctx->stream));
        memcpy(out_ip_l, &s->h_ip[0], 32);
        memcpy(out_ip_r, &s->h_ip[1], 32);
    }
    return ZK_OK;
}

int ipa_round_fold(zk_ipa* s, const uint64_t u_mont[4], const uint64_t u_inv_mont[4]) {
    if (s->n < 2) { zk_set_error("ipa_round_fold: folding is complete"); return ZK_ERR_INVALID; }
    zk_ctx* ctx = s->ctx;
    const size_t h = s->n / 2, count = s->n0 / s->n;   // count = 2^j challenges products so far
    fe u, ui;
    memcpy(u.v, u_mont, 32);
    memcpy(ui.v, u_inv_mont, 32);
    const unsigned blocks = (unsigned)((h + 127) / 128), sblocks = (unsigned)((count + 127) / 128);
    with_curve(s->curve, [&](auto c) {
        using FS = typename decltype(c)::FS;
        k_fold_field<FS><<<blocks, 128, 0, ctx->stream>>>(s->d_a, h, ui);
        k_fold_field<FS><<<blocks, 128, 0, ctx->stream>>>(s->d_b, h, u);
        k_expand_challenges<FS><<<sblocks, 128, 0, ctx->stream>>>(s->d_s[s->cur], s->d_s[s->cur ^ 1], count, u);
    });
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 3;
    s->cur ^= 1;
    s->n = h;
    s->round += 1;
    return ZK_OK;
}


// g'[i] = g[i] + [k] g[h + i], k canonical; see zk_points_fold_dev
template <class F> __global__ void __launch_bounds__(64) k_fold_bases(const affine_t* __restrict__ g, size_t h, fe k, affine_t* out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= h) return;
    const affine_t lo = g[i], hi = g[h + i];
    xyzz_t acc = affine_is_inf(hi) ? xyzz_identity() : xyzz_scalar_mul<F>(xyzz_from_affine<F>(hi), k);
    if (!affine_is_inf(lo)) acc = xyzz_madd<F>(acc, lo);
    out[i] = xyzz_to_affine<F>(acc);
}

}  // namespace zkb

extern "C" {

int zk_ipa_begin(zk_ctx* ctx, const zk_bases* bases, const uint64_t* a_mont, const uint64_t* b_mont, size_t n, zk_ipa** out) {
    if (!ctx || !bases || !a_mont || !b_mont || !out) { zk_set_error("ipa_begin: null argument"); return ZK_ERR_INVALID; }
    if (ctx_root(bases->ctx) != ctx_root(ctx)) { zk_set_error("ipa_begin: bases belong to another context"); return ZK_ERR_INVALID; }
    if (n < 2) { zk_set_error("ipa_begin: n must be a power of two >= 2 (the reference pads to a power of two, ipa.rs:848-850)"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    zk_ipa* s = nullptr;
    int rc = ipa_create(ctx, bases, n, &s);
    if (rc) return rc;
    std::unique_ptr<zk_ipa> owner(s);
    cudaError_t e = cudaMemcpyAsync(s->d_a, a_mont, n * sizeof(fe), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(s->d_b, b_mont, n * sizeof(fe), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        zk_set_error("ipa_begin: %s", cudaGetErrorString(e));
        return ZK_ERR_CUDA;
    }
    *out = owner.release();
    return ZK_OK;
}

void zk_ipa_free(zk_ipa* s) {
    if (!s) return;
    std::lock_guard<std::mutex> lk(s->ctx->mu);
    cudaSetDevice(s->ctx->device);
    delete s;
}

size_t zk_ipa_len(const zk_ipa* s) { return s ? s->n : 0; }

int zk_ipa_round_lr(zk_ipa* s, uint64_t out_l_xyz[12], uint64_t out_r_xyz[12], uint64_t out_ip_l[4], uint64_t out_ip_r[4]) {
    if (!s || !out_l_xyz || !out_r_xyz || !out_ip_l || !out_ip_r) { zk_set_error("ipa_round_lr: null argument"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(s->ctx->mu);
    ZK_CUDA(cudaSetDevice(s->ctx->device));
    return ipa_round_lr(s, out_l_xyz, out_r_xyz, out_ip_l, out_ip_r);
}

int zk_ipa_round_fold(zk_ipa* s, const uint64_t u_mont[4], const uint64_t u_inv_mont[4]) {
    if (!s || !u_mont || !u_inv_mont) { zk_set_error("ipa_round_fold: null argument"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(s->ctx->mu);
    ZK_CUDA(cudaSetDevice(s->ctx->device));
    return ipa_round_fold(s, u_mont, u_inv_mont);
}

// The reference's own per-round base fold, g'[i] = g[i] + [u] g[h + i]  (`G::combine_one_endo`, ipa.rs:1002-1006 /
// combine.rs:292-342), as a device building block: one thread per output point, a double-and-add chain over the bits of u
// (leading zeros skipped, so a 128-bit endo-form challenge costs half of a full one) and one inversion back to affine.
// The opening path does NOT use it (never-folded bases, header comment); it is here so that the two designs can be timed
// against each other on the same machine (tools/fold_vs_never_fold.py, DESIGN.md 4.4) and is parity-tested like everything else.
int zk_points_fold_dev(zk_ctx* ctx, int curve_id, const void* d_g, size_t h, const uint64_t u_mont[4], void* d_out) {
    if (!ctx || !u_mont || ((!d_g || !d_out) && h)) { zk_set_error("points_fold: null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_curve("points_fold", curve_id)) return rc;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    if (h == 0) return ZK_OK;
    host::hfe um, unit = host::zero();
    memcpy(&um, u_mont, 32);
    unit.l[0] = 1;
    const unsigned blocks = (unsigned)((h + 63) / 64);
    with_curve(curve_id, [&](auto c) {
        using C = decltype(c);
        const host::hfe uc = host::mul<typename C::HS>(um, unit);     // canonical u = u_mont / R: a Montgomery product with the integer 1
        fe k;
        memcpy(&k, &uc, 32);
        k_fold_bases<typename C::F><<<blocks, 64, 0, ctx->stream>>>((const affine_t*)d_g, h, k, (affine_t*)d_out);
    });
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 1;
    return ZK_OK;
}

// Current state: copies min(len, capacity) leading elements of a and b (Montgomery); out_g_xyz (optional) receives the first
// current folded base g_j[0] in Jacobian form — after the last fold that is g0 = <b_poly_coefficients(chals), g>, the
// proof's `sg` (one MSM over the resident table).
int zk_ipa_read(zk_ipa* s, uint64_t* out_a, uint64_t* out_b, size_t capacity, uint64_t out_g_xyz[12]) {
    if (!s) { zk_set_error("ipa_read: null argument"); return ZK_ERR_INVALID; }
    zk_ctx* ctx = s->ctx;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    const size_t m = s->n < capacity ? s->n : capacity;
    if (out_a && m) ZK_CUDA(cudaMemcpyAsync(out_a, s->d_a, m * sizeof(fe), cudaMemcpyDeviceToHost, ctx->stream));
    if (out_b && m) ZK_CUDA(cudaMemcpyAsync(out_b, s->d_b, m * sizeof(fe), cudaMemcpyDeviceToHost, ctx->stream));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    if (out_g_xyz) {
        if (s->n != 1) { zk_set_error("ipa_read: the folded base is available after the last round only"); return ZK_ERR_INVALID; }
        const size_t len = s->n0 < s->bases->b.n ? s->n0 : s->bases->b.n;
        return ctx_msm_device(ctx, s->bases, 0, len, s->d_s[s->cur], /*mont=*/1, 0, out_g_xyz);
    }
    return ZK_OK;
}

}  // extern "C"
