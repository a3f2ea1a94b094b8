// poly.cuh — coefficient / evaluation-form kernels shared by the opening proof's combine_polys (open.cu) and the ft polynomial of
// Maller's optimisation (ft.cu): a scaled, strided sum of evaluation-form columns, and the linearisation of a chunked polynomial.
#pragma once
#include "ctx.hpp"

namespace zkb {

struct alignas(16) CombineDesc {
    const fe* p;        // element i of the term is p[i * stride]
    uint32_t len;       // number of elements the term contributes (i < len): any d1 up to 2^30
    uint32_t stride;    // 1, 2, 4 or 8 for kimchi's domains d1 .. d8
    fe scale;           // Montgomery
};
static_assert(sizeof(CombineDesc) == 48, "layout");

// out[i] = sum_d scale_d * p_d[i * stride_d]  (i < len_d), i < n_out
template <class FS> __global__ void k_combine(const CombineDesc* __restrict__ descs, unsigned nd, fe* out, size_t n_out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out) return;
    fe acc = fe_zero();
    for (unsigned d = 0; d < nd; d++) {
        const uint32_t len = descs[d].len;
        if (i < len) acc = fe_add<FS>(acc, fe_mul<FS>(load_fe_nc(descs[d].p + i * (size_t)descs[d].stride), load_fe_nc(&descs[d].scale)));
    }
    store_fe(out + i, acc);
}

// a[i] += sum_k scale0 * zeta^k * e[k * chunk + i]   (scale0 * to_chunked_polynomial(num_chunks, chunk).linearize(zeta),
// utils/src/chunked_polynomial.rs:34-51; combine_polys passes scale0 = 1, utils.rs:190-199)
template <class FS> __global__ void k_linearize_add(fe* a, const fe* __restrict__ e, size_t e_len, size_t chunk, unsigned num_chunks, fe zeta, fe scale0) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= chunk) return;
    fe acc = load_fe(a + i), scale = scale0;
    for (unsigned k = 0; k < num_chunks; k++) {
        const size_t j = (size_t)k * chunk + i;
        if (j < e_len) acc = fe_add<FS>(acc, fe_mul<FS>(load_fe_nc(e + j), scale));
        scale = fe_mul<FS>(scale, zeta);
    }
    store_fe(a + i, acc);
}

// evaluate_chunks on the device with the context lock held (evals.cu): the values of the covered chunks of every polynomial at
// every point land in device scratch, *d_res[(poly * n_points + point) * covered + chunk], covered = ceil(max len / chunk_size).
// Nothing is synchronised; `stage` holds the tables' host copy and must outlive the launches.
int ctx_evaluate_chunks(zk_ctx* ctx, int field_id, const zk_dev_poly* polys, size_t n_polys, size_t chunk_size, const uint64_t* points_mont,
                        size_t n_points, std::vector<uint8_t>& stage, const fe** d_res, uint64_t* covered);

}  // namespace zkb
