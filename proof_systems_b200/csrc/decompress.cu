// decompress.cu — device-side ingestion of the reference's compressed points (SURVEY.md §8f row 4).
//
// srs/pallas.srs and srs/vesta.srs store every generator in ark-serialize's compressed short-Weierstrass form, as used by
// the SerdeAs adapter (utils/src/serialization.rs:65-106; layout verified against the files, SURVEY.md Appendix B):
//     32 bytes little-endian canonical x  ||  1 flag byte:  bit 7 = "y is the larger of {y, p - y}",  bit 6 = infinity.
// One thread per point: y = sqrt(x^3 + 5) by Tonelli-Shanks (field_sqrt.cuh), sign chosen by the flag, output affine in
// Montgomery form.
#include "common.cuh"
#include "field_sqrt.cuh"

namespace zkb {

// canonical a > canonical b ?  (both Montgomery on input)
template <class F> __device__ bool fe_canonical_gt(const fe& a, const fe& b) {
    const fe ca = fe_from_mont<F>(a), cb = fe_from_mont<F>(b);
    for (int i = 7; i >= 0; i--) {
        if (ca.v[i] != cb.v[i]) return ca.v[i] > cb.v[i];
    }
    return false;
}

__device__ __forceinline__ fe load_le_bytes(const uint8_t* p) {
    fe r;
#pragma unroll
    for (int k = 0; k < 8; k++) r.v[k] = (uint32_t)p[4 * k] | ((uint32_t)p[4 * k + 1] << 8) | ((uint32_t)p[4 * k + 2] << 16) | ((uint32_t)p[4 * k + 3] << 24);
    return r;
}
__device__ __forceinline__ void store_le_bytes(uint8_t* p, const fe& a) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
        p[4 * k] = (uint8_t)a.v[k]; p[4 * k + 1] = (uint8_t)(a.v[k] >> 8); p[4 * k + 2] = (uint8_t)(a.v[k] >> 16); p[4 * k + 3] = (uint8_t)(a.v[k] >> 24);
    }
}

template <class F> __global__ void __launch_bounds__(128) k_decompress(const uint8_t* __restrict__ in, affine_t* out, size_t n, unsigned* bad) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* p = in + 33 * i;
    const uint8_t flags = p[32];
    affine_t r;
    r.x = fe_zero();
    r.y = fe_zero();
    // ark-serialize's SWFlags::from_u8 accepts exactly three flag values (0x00, 0x80, 0x40): stray low bits and the
    // infinity + sign combination are rejected, and the field deserialiser checks x < modulus (what the reference's
    // deserialize_with_mode(Compress::Yes, Validate::Yes) enforces through SerdeAs, utils/src/serialization.rs:65-106).
    const fe xc = load_le_bytes(p);
    if ((flags & 0x3f) != 0 || (flags & 0xc0) == 0xc0 || !fe_lt_modulus<F>(xc)) {
        atomicAdd(bad, 1u);
        store_affine(out + i, r);
        return;
    }
    if (!(flags & 0x40)) {
        const fe x = fe_to_mont<F>(xc);
        fe five = fe_zero();
        five.v[0] = 5;
        const fe rhs = fe_add<F>(fe_mul<F>(fe_sqr<F>(x), x), fe_to_mont<F>(five));   // x^3 + 5  (pallas.rs / vesta.rs: a = 0, b = 5)
        fe y;
        if (!fe_sqrt<F>(rhs, y)) { atomicAdd(bad, 1u); store_affine(out + i, r); return; }
        const fe ny = fe_neg<F>(y);
        const bool y_larger = fe_canonical_gt<F>(y, ny);
        const bool want_larger = (flags & 0x80) != 0;
        r.x = x;
        r.y = (want_larger == y_larger) ? y : ny;
    }
    store_affine(out + i, r);
}

// ark-serialize uncompressed, unchecked (SerdeAsUnchecked, utils/src/serialization.rs:108-146; the srs/test_*.srs layout):
// 32 B LE canonical x || 32 B LE canonical y || flag byte (bit 6 = infinity).  No curve check, as in the reference.
template <class F> __global__ void __launch_bounds__(128) k_from_uncompressed(const uint8_t* __restrict__ in, affine_t* out, size_t n, unsigned* bad) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* p = in + 65 * i;
    affine_t r;
    r.x = fe_zero();
    r.y = fe_zero();
    if (!(p[64] & 0x40)) {
        const fe xc = load_le_bytes(p), yc = load_le_bytes(p + 32);
        if (!fe_lt_modulus<F>(xc) || !fe_lt_modulus<F>(yc)) atomicAdd(bad, 1u);   // not a canonical field element
        r.x = fe_to_mont<F>(xc);
        r.y = fe_to_mont<F>(yc);
    }
    store_affine(out + i, r);
}

// affine Montgomery -> 33-byte compressed form (the inverse of k_decompress): what PolyComm / OpeningProof serialise to
// (utils/src/serialization.rs:65-84).  The identity is x = 0, flags = 0x40.
template <class F> __global__ void __launch_bounds__(128) k_compress(const affine_t* __restrict__ in, uint8_t* out, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const affine_t a = load_affine_nc(in + i);
    uint8_t* p = out + 33 * i;
    if (affine_is_inf(a)) {
        store_le_bytes(p, fe_zero());
        p[32] = 0x40;
        return;
    }
    store_le_bytes(p, fe_from_mont<F>(a.x));
    p[32] = fe_canonical_gt<F>(a.y, fe_neg<F>(a.y)) ? 0x80 : 0x00;
}

// Synthetic on-curve points for benchmarks and tests that need more bases than the reference ships (BASELINE config 4: 2^20
// points; srs/*.srs hold 2^16): point i = the first x in the sequence H(seed, i, 0), H(seed, i, 1), ... (splitmix64 words, below
// 2^254, read as a Montgomery residue) for which x^3 + 5 is a square, with the root Tonelli-Shanks returns.  Deterministic in
// (curve, seed, i); about two attempts per point.
template <class F> __global__ void __launch_bounds__(128) k_synthetic_points(affine_t* out, size_t n, uint64_t seed) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe five = fe_zero();
    five.v[0] = 5;
    const fe b = fe_to_mont<F>(five);
    for (uint64_t attempt = 0;; attempt++) {
        fe x;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            uint64_t z = seed + 0x9E3779B97F4A7C15ull * (4 * (uint64_t)i + k + 1) + 0xD1B54A32D192ED03ull * attempt;
            z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
            z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
            z ^= z >> 31;
            if (k == 3) z &= (1ull << 62) - 1;
            x.v[2 * k] = (uint32_t)z; x.v[2 * k + 1] = (uint32_t)(z >> 32);
        }
        fe y;
        if (fe_sqrt<F>(fe_add<F>(fe_mul<F>(fe_sqr<F>(x), x), b), y) && !fe_is_zero(y)) {
            affine_t r;
            r.x = x; r.y = y;
            store_affine(out + i, r);
            return;
        }
    }
}
template <class F> int points_synthetic(affine_t* d_out, size_t n, uint64_t seed, cudaStream_t st) {
    if (n) k_synthetic_points<F><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(d_out, n, seed);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}
template int points_synthetic<FpParams>(affine_t*, size_t, uint64_t, cudaStream_t);
template int points_synthetic<FqParams>(affine_t*, size_t, uint64_t, cudaStream_t);

template <class F> int points_from_uncompressed(const uint8_t* d_in, affine_t* d_out, size_t n, unsigned* d_bad, cudaStream_t st) {
    ZK_CUDA(cudaMemsetAsync(d_bad, 0, sizeof(unsigned), st));
    if (n) k_from_uncompressed<F><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(d_in, d_out, n, d_bad);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}
template int points_from_uncompressed<FpParams>(const uint8_t*, affine_t*, size_t, unsigned*, cudaStream_t);
template int points_from_uncompressed<FqParams>(const uint8_t*, affine_t*, size_t, unsigned*, cudaStream_t);

template <class F> int points_compress(const affine_t* d_in, uint8_t* d_out, size_t n, cudaStream_t st) {
    if (n) k_compress<F><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(d_in, d_out, n);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}
template int points_compress<FpParams>(const affine_t*, uint8_t*, size_t, cudaStream_t);
template int points_compress<FqParams>(const affine_t*, uint8_t*, size_t, cudaStream_t);

template <class F> int points_decompress(const uint8_t* d_in, affine_t* d_out, size_t n, unsigned* d_bad, cudaStream_t st) {
    ZK_CUDA(cudaMemsetAsync(d_bad, 0, sizeof(unsigned), st));
    if (n) k_decompress<F><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(d_in, d_out, n, d_bad);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}
template int points_decompress<FpParams>(const uint8_t*, affine_t*, size_t, unsigned*, cudaStream_t);
template int points_decompress<FqParams>(const uint8_t*, affine_t*, size_t, unsigned*, cudaStream_t);

}  // namespace zkb
