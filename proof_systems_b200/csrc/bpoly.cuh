// bpoly.cuh — the coefficients of challenge polynomials, s = b_poly_coefficients(chal) (poly-commitment/src/commitment.rs:464-476:
// s[j] = prod over the set bits t of j of chal[k - 1 - t]), built from two product tables per challenge vector.  Shared by
// zk_srs_verify (verify.cu: one weighted sum over the whole batch) and the recursion accumulators (accumulator.cu: the weighted sum
// for the check, one vector per accumulator for generate).
//
// Table convention: K = ceil_log2(|g|), L = ceil(K / 2), H = K - L; vector i's challenges enter reversed and zero-padded to K,
//   rev[i][t] = chal_i[R_i - 1 - t] for t < min(R_i, K), 0 above,
// so the entries j >= 2^R_i vanish (the vector covers 2^R_i entries; msm_bigint's truncation to g[..2^R_i]) and R_i > K uses only
// the last K challenges, the ones the first 2^K coefficients depend on.
#pragma once
#include "common.cuh"

namespace zkb {

// Per vector i (blockIdx-linear index over B x (2^L + 2^H) entries):
//   lo[i][e] = prod_{t < L, bit t of e} rev[i][t]           hi[i][e] = w[i] * prod_{t < H, bit t of e} rev[i][L + t]
template <class FS>
__global__ void k_bpoly_tables(const fe* __restrict__ rev, const fe* __restrict__ w, unsigned B, unsigned K, unsigned L, fe* lo, fe* hi) {
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
__global__ void k_bpoly_sum(const fe* __restrict__ lo, const fe* __restrict__ hi, unsigned B, unsigned L, unsigned H, fe* S, size_t len) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= len) return;
    const size_t jl = j & (((size_t)1 << L) - 1), jh = j >> L;
    fe acc = fe_zero();
    for (unsigned i = 0; i < B; i++)
        acc = fe_add<FS>(acc, fe_mul<FS>(load_fe_nc(lo + ((size_t)i << L) + jl), load_fe_nc(hi + ((size_t)i << H) + jh)));
    store_fe(S + j, acc);
}

// s[i][j] = lo[i][j mod 2^L] * hi[i][j >> L],  j < len, i = blockIdx.y: one vector of len entries per table pair, back to back
template <class FS>
__global__ void k_bpoly_expand(const fe* __restrict__ lo, const fe* __restrict__ hi, unsigned L, unsigned H, fe* s, size_t len) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= len) return;
    const size_t i = blockIdx.y;
    const size_t jl = j & (((size_t)1 << L) - 1), jh = j >> L;
    store_fe(s + i * len + j, fe_mul<FS>(load_fe_nc(lo + (i << L) + jl), load_fe_nc(hi + (i << H) + jh)));
}

}  // namespace zkb
