// perm.cu — the permutation aggregation polynomial z (kimchi/src/circuits/polynomials/permutation.rs:447-574, `perm_aggreg`) on
// the device, from the resident witness and permutation_coefficients8, so z never has to be built on the host and uploaded.
// With n = |d1|, last = n - zk_rows and sid[j] = omega^j:
//   num[j] = prod_{k<7} (w_k[j] + beta shift_k omega^j + gamma)      den[j] = prod_{k<7} (w_k[j] + beta sigma_k[s j] + gamma)
//   r[j]   = num[j] / den[j] for j < n, z[0] = 1, z[j + 1] = z[j] r[j] for j < last, the flag z[last] == 1:
//                                                           aggreg.cuh with end = n (PermRows)
//   z[last + 1] = rand0, z[last + 2] = rand1                the reference's two F::rand(rng) draws, in its order
//   z[j + 1] = z[j] r[j] for j = last + 2 .. n - 2          zk_rows - 3 rows, a warp scan (PermTail)
//   z = interpolate(z) over d1                              the library's inverse NTT, in place
#include <cstring>
#include <mutex>

#include "../../include/zkb200.h"
#include "aggreg.cuh"

using namespace zkb;

namespace zkb {

template <class FS> struct PermRows {
    const fe* w[7];     // witness columns over d1
    const fe* sigma[7]; // permutation_coefficients8 (or any s n evaluations), read at s j
    const fe* ulo;      // omega^j from the forward transform's tables (domain_point, ntt.cuh)
    const fe* mid;
    const fe* hi2;
    size_t sigma_stride;
    fe beta, gamma;
    fe bshift[7];       // beta * shift_k

    struct Cursor { fe x, omega; };     // x = omega^j
    __device__ Cursor start(size_t j0) const { return {domain_point<FS>(ulo, mid, hi2, j0), load_fe_nc(ulo + 1)}; }
    __device__ void row(Cursor& c, size_t j, fe& num, fe& den) const {
        fe wg = fe_add<FS>(load_fe_nc(w[0] + j), gamma);
        num = fe_add<FS>(wg, fe_mul<FS>(c.x, bshift[0]));
        den = fe_add<FS>(wg, fe_mul<FS>(beta, load_fe_nc(sigma[0] + sigma_stride * j)));
#pragma unroll 1
        for (unsigned k = 1; k < 7; k++) {
            wg = fe_add<FS>(load_fe_nc(w[k] + j), gamma);
            num = fe_mul<FS>(num, fe_add<FS>(wg, fe_mul<FS>(c.x, bshift[k])));
            den = fe_mul<FS>(den, fe_add<FS>(wg, fe_mul<FS>(beta, load_fe_nc(sigma[k] + sigma_stride * j))));
        }
        c.x = fe_mul<FS>(c.x, c.omega);
    }
};

// z[last + 1] = rand0, z[last + 2] = rand1, then z[j + 1] = z[j] r[j] for j = last + 2 .. n - 2 as a warp scan, 32 rows per step
template <class FS> struct PermTail {
    const fe* r;
    size_t n;
    fe rand0, rand1;

    __device__ void operator()(fe* z, size_t last, unsigned lane) const {
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
};

template <class T>
static int perm_aggreg_impl(zk_ctx* ctx, unsigned log_n, size_t zk_rows, const void* const d_w[7], const void* const d_sigma[7],
                            size_t sigma_stride, const uint64_t beta[4], const uint64_t gamma[4], const uint64_t shifts[28],
                            const uint64_t rand[8], fe* d_z, int* final_is_one) {
    using namespace host;
    using FS = typename T::Dev; using HP = typename T::Host;
    const size_t n = (size_t)1 << log_n, last = n - zk_rows;
    PermRows<FS> a{};
    for (int k = 0; k < 7; k++) { a.w[k] = (const fe*)d_w[k]; a.sigma[k] = (const fe*)d_sigma[k]; }
    a.sigma_stride = sigma_stride;
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
    PermTail<FS> tail{};
    tail.n = n;
    memcpy(&tail.rand0, rand, 32);
    memcpy(&tail.rand1, rand + 4, 32);

    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    PinnedSlots* pin = ctx_pinned(ctx);
    if (!pin) return ZK_ERR_CUDA;
    int rc = ctx_ntt_table_ptrs(ctx, T::id, log_n, false, &a.ulo, &a.mid, &a.hi2);
    if (rc) return rc;
    // context scratch: r over d1 | block totals | the final-value flag
    Layout lay;
    const size_t o_r = lay.add(n * sizeof(fe)), o_tot = lay.add(agg_blocks(n) * sizeof(fe)), o_flag = lay.add(sizeof(unsigned));
    rc = ctx->d_perm.ensure(lay.total);
    if (rc) return rc;
    fe* r = ctx->d_perm.at<fe>(o_r);
    unsigned* d_flag = ctx->d_perm.at<unsigned>(o_flag);
    tail.r = r;
    rc = agg_launch<FS>(ctx, a, tail, d_z, r, ctx->d_perm.at<fe>(o_tot), n, last, d_flag);
    if (rc) return rc;
    rc = ctx_ntt_device(ctx, T::id, d_z, log_n, 1, 0, /* inverse = */ 1, /* coset = */ 0);     // Evaluations::interpolate
    if (rc) return rc;
    ZK_CUDA(cudaMemcpyAsync(&pin->agg_final, d_flag, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    ZK_CUDA(cudaStreamSynchronize(st));
    *final_is_one = pin->agg_final ? 1 : 0;
    return ZK_OK;
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
