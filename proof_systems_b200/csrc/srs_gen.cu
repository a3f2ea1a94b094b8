// srs_gen.cu — the points of `SRS::create(depth)` (poly-commitment/src/ipa.rs:751-778) generated on the device:
//   g[i] = point_of_random_bytes(Blake2b512(u32_be(i)))                i < depth
//   h    = point_of_random_bytes(Blake2b512(b"srs_misc" || u32_be(0)))
// One thread per point, grid-stride; item `depth` is h.  The hash, the packing and the group map are in hash_to_curve.cuh.
#include "common.cuh"
#include "hash_to_curve.cuh"

namespace zkb {

template <class F> __global__ void __launch_bounds__(128) k_srs_generate(affine_t* out, size_t depth) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i <= depth; i += stride) {
        uint64_t m[16] = {};
        unsigned len;
        if (i < depth) {
            const uint32_t k = (uint32_t)i;                 // the reference's `i as u32`; depth <= 2^32 (zk_srs_generate)
            m[0] = __byte_perm(k, 0, 0x0123);               // u32_be(i): the big-endian bytes as the low word's first four bytes
            len = 4;
        } else {
            m[0] = 0x6373696d5f737273ull;                   // "srs_misc" little-endian; u32_be(0) is the zero word m[1]
            len = 12;
        }
        affine_t r;
        if (!point_of_message<F>(m, len, r.x, r.y)) r.x = r.y = fe_zero();   // unreachable: the map always finds a point
        store_affine(out + i, r);
    }
}

template <class F> int srs_generate_points(affine_t* d_out, size_t depth, int sm_count, cudaStream_t st) {
    const size_t blocks = std::min<size_t>((depth + 1 + 127) / 128, (size_t)sm_count * 16);
    k_srs_generate<F><<<(unsigned)blocks, 128, 0, st>>>(d_out, depth);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}
template int srs_generate_points<FpParams>(affine_t*, size_t, int, cudaStream_t);
template int srs_generate_points<FqParams>(affine_t*, size_t, int, cudaStream_t);

}  // namespace zkb
