// group_ntt.cu — Lagrange-basis commitments on the device: the inverse radix-2 FFT over GROUP elements that
// SRS::lagrange_basis runs on the CPU (poly-commitment/src/ipa.rs:1065-1172, single-chunk case domain <= |g|):
//     L_i = sum_j (w^{-ij} / n) * g[j]          (ark-poly's ifft_in_place is generic over DomainCoeff, ipa.rs:1161)
// followed by batch normalisation (ipa.rs:1164).  The result is exactly the data stored in srs/test_{pallas,vesta}.srs,
// which is the parity target (tests/test_gpu_lagrange.py).
//
// Setup-time work (once per SRS and domain size), so the shape is simple: log n radix-2 DIF layers over an XYZZ array
// in global memory, one thread per butterfly  (u, v) -> (u + v, [w^{-j 2^s}] (u - v)),  the twiddle multiplication being a
// 255-bit double-and-add; then one pass that scales by n^-1, undoes the bit reversal and converts to affine.
// ~(n/2 log n + n) scalar multiplications: 0.6 M at n = 2^16.
#include <algorithm>

#include "msm.cuh"

namespace zkb {

// tw[i] = w^{-i} as a CANONICAL integer, i < count (w = n-th root of unity of the scalar field); ninv[0] = n^-1 canonical
template <class FS> __global__ void k_gntt_twiddles(fe* tw, fe* ninv, unsigned log_n, unsigned count) {
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    fe w;
#pragma unroll
    for (int k = 0; k < 8; k++) w.v[k] = FS::ROOT(k);
    for (unsigned k = log_n; k < 32; k++) w = fe_sqr<FS>(w);
    fe wi = fe_inv<FS>(w);
    store_fe(tw + i, fe_from_mont<FS>(fe_pow_u64<FS>(wi, i)));
    if (i == 0) {
        fe nn = fe_zero();
        nn.v[0] = 1u << log_n;
        store_fe(ninv, fe_from_mont<FS>(fe_inv<FS>(fe_to_mont<FS>(nn))));
    }
}

// a[start + j] = g[j] for j < terms, the identity elsewhere (one chunk of a chunked basis, ipa.rs:1145-1160; start = 0, terms = n
// for the plain case)
template <class F> __global__ void k_gntt_load(const affine_t* __restrict__ g, xyzz_t* a, unsigned n, unsigned start, unsigned terms) {
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool live = i >= start && i - start < terms;
    store_xyzz(a + i, live ? xyzz_from_affine<F>(load_affine_nc(g + (i - start))) : xyzz_identity());
}

// one DIF layer: half = n >> (s+1); butterfly k: (i0, i1 = i0 + half); twiddle exponent j << s
template <class F> __global__ void __launch_bounds__(128) k_gntt_layer(xyzz_t* a, const fe* __restrict__ tw, unsigned log_n, unsigned s) {
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned n = 1u << log_n, half = n >> (s + 1);
    if (k >= n / 2) return;
    const unsigned grp = k / half, j = k - grp * half;
    const unsigned i0 = grp * 2 * half + j, i1 = i0 + half;
    xyzz_t u = load_xyzz(a + i0), v = load_xyzz(a + i1);
    store_xyzz(a + i0, xyzz_add<F>(u, v));
    xyzz_t d = xyzz_add<F>(u, xyzz_neg<F>(v));
    if (j != 0) d = xyzz_scalar_mul<F>(d, load_fe_nc(tw + ((size_t)j << s)));
    store_xyzz(a + i1, d);
}

// out[bitrev(i)] = affine([n^-1] a[i])
template <class F> __global__ void __launch_bounds__(128) k_gntt_finish(const xyzz_t* __restrict__ a, const fe* __restrict__ ninv, affine_t* out, unsigned log_n) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (1u << log_n)) return;
    xyzz_t p = xyzz_scalar_mul<F>(load_xyzz(a + i), load_fe_nc(ninv));
    const unsigned r = log_n ? (__brev(i) >> (32 - log_n)) : 0;
    store_affine(out + r, xyzz_to_affine<F>(p));
}

// d_out: n affine points (device).  g: resident generators (row 0 of the table is the points themselves).
// Chunk `chunk` of the basis of a domain larger than the SRS (ipa.rs:1145-1171): the inverse FFT of the vector that holds
// g[0 .. terms) at positions chunk * |g| .. and the identity elsewhere; chunk 0 with n <= |g| is the ordinary basis.
template <class F, class FS> int lagrange_basis_build(const MsmBases& g, unsigned log_n, unsigned chunk, affine_t* d_out, cudaStream_t st, unsigned* launches) {
    const unsigned n = 1u << log_n;
    const size_t start = (size_t)chunk * g.n;
    if (start >= n && !(chunk == 0 && n <= g.n)) { zk_set_error("lagrange_basis: chunk %u outside a domain of %u over %zu generators", chunk, n, g.n); return ZK_ERR_INVALID; }
    const unsigned terms = (unsigned)std::min<size_t>(g.n, n - start);
    DevScratch a_mem, tw_mem;
    if (int rc = a_mem.ensure((size_t)n * sizeof(xyzz_t))) return rc;
    if (int rc = tw_mem.ensure(((size_t)n / 2 + 2) * sizeof(fe))) return rc;
    xyzz_t* a = a_mem.at<xyzz_t>();
    fe* tw = tw_mem.at<fe>();
    fe* ninv = tw + n / 2 + 1;
    const unsigned ntw = n / 2 ? n / 2 : 1;
    k_gntt_twiddles<FS><<<(ntw + 127) / 128, 128, 0, st>>>(tw, ninv, log_n, ntw);
    k_gntt_load<F><<<(n + 127) / 128, 128, 0, st>>>(g.d_points, a, n, (unsigned)start, terms);
    for (unsigned s = 0; s < log_n; s++) k_gntt_layer<F><<<(n / 2 + 127) / 128, 128, 0, st>>>(a, tw, log_n, s);
    k_gntt_finish<F><<<(n + 127) / 128, 128, 0, st>>>(a, ninv, d_out, log_n);
    cudaError_t e = cudaGetLastError();
    cudaError_t e2 = cudaStreamSynchronize(st);
    if (e != cudaSuccess || e2 != cudaSuccess) { zk_set_error("lagrange_basis: %s", cudaGetErrorString(e != cudaSuccess ? e : e2)); return ZK_ERR_CUDA; }
    if (launches) *launches += 3 + log_n;
    return ZK_OK;
}

template int lagrange_basis_build<FpParams, FqParams>(const MsmBases&, unsigned, unsigned, affine_t*, cudaStream_t, unsigned*);
template int lagrange_basis_build<FqParams, FpParams>(const MsmBases&, unsigned, unsigned, affine_t*, cudaStream_t, unsigned*);

}  // namespace zkb
