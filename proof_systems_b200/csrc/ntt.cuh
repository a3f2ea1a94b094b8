// ntt.cuh — radix-2 number-theoretic transform over the Pasta fields on sm_90a.
//
// Drop-in semantics of ark_poly::Radix2EvaluationDomain::<F>::{fft_in_place, ifft_in_place} as the reference calls
// them (kimchi/src/prover.rs:289,377,907,1163; kimchi/src/circuits/constraints.rs:494;
// poly-commitment/src/utils.rs:195-198 — SURVEY.md §8 row a8):
//     forward   out[i] = sum_j a[j] (g w^i)^j          inverse   a[j] = g^-j n^-1 sum_i out[i] w^-ij
// natural order in and out, w = (5^T)^(2^(32-log n)) (fp.rs:10,21-27), g = 1 (plain domain) or 5 (coset),
// elements in Montgomery form, inputs shorter than the domain zero-padded.
//
// H100 shape: a four-step decomposition n = n1 * n2 (n1, n2 <= 2^10) makes a transform of up to 2^20 elements exactly two kernel
// passes, n = n1 * n2 * n3 three (up to 2^30).  A pass is a batch of independent S-point column transforms; ONE column is one
// CTA's tile (32 KiB for S = 1024), so a 2^20 transform is 1024 tiles per pass — fine-grained enough to keep 132 SMs evenly
// loaded, and the 32-byte elements are exactly one DRAM sector each, so strided columns cost no bandwidth.  Inside a tile the
// transform is decimation in time: the load writes the column to shared memory in bit-reversed order, a warp runs the six
// layers of span <= 32 for a 64-row chunk entirely in REGISTERS (two elements per lane, partners exchanged with warp shuffles,
// one multiplication per lane and layer: ntt_butterfly.cuh), the remaining log2(S) - 6 layers go through shared memory
// (limb-major, padded: conflict-free), and the store — natural order, no permutation left — fuses the inter-pass twiddle
// (one multiplication against an n-entry table kept in HBM for the two-pass plan, n <= 2^20, or up to two against 1024-entry
// tables in the three-pass plan), the 1/n scaling
// (folded into the tables) and the transposition.  Work is 255-bit modular integer arithmetic: no tensor cores.
#pragma once
#include "common.cuh"

namespace zkb {

constexpr unsigned NTT_MAX_LOG_SUB = 10;   // sub-transform size limit (one column per tile, twiddles from a 512-entry table)
constexpr unsigned NTT_MAX_LOG_N = 30;     // three passes of <= 2^10

// device tables of one (field, log_n, direction), owned: lo .. chi are views into `block`
struct NttTables {
    DevScratch block;
    fe* lo = nullptr;    // [1024] w_n^(+-i)            (inverse: times n^-1)
    fe* ulo = nullptr;   // [1024] w_n^(+-i)            unscaled (the middle pass of a three-pass plan uses the tables of n2 * n3)
    fe* mid = nullptr;   // [1024] w_n^(+-1024 i)
    fe* hi2 = nullptr;   // [1024] w_n^(+-2^20 i)
    fe* clo = nullptr;   // [1024] g^(+-i)              coset powers
    fe* chi = nullptr;   // [1024] g^(+-1024 i)
    DevScratch full;     // [n]    w_n^(+-(col * k)) (inverse: times n^-1) at index col * n1 + k: contiguous per tile of pass 1; empty outside 2^10 < n <= 2^20
};

// w^e = lo[e & 1023] * mid[(e >> 10) & 1023] * hi2[e >> 20] from a transform's three 1024-entry tables (lo, or ulo for the
// unscaled powers), e < 2^30.  I: the index type of the caller's arithmetic.  e is taken by reference: taken by value, nvcc
// (12.9) tests the table indices in another form and the callers' SASS changes.
template <class F, class I> __device__ __forceinline__ fe domain_point(const fe* lo, const fe* mid, const fe* hi2, const I& e) {
    fe x = load_fe_nc(lo + (e & 1023));
    if ((e >> 10) & 1023) x = fe_mul<F>(x, load_fe_nc(mid + ((e >> 10) & 1023)));
    if (e >> 20) x = fe_mul<F>(x, load_fe_nc(hi2 + (e >> 20)));
    return x;
}

// One pass = independent S-point transforms of columns ("tiles").  Tile tau = (t_hi << split_log) | t_lo of polynomial b reads
//     in[b * in_bs + t_hi * in_hi + t_lo * in_lo + r * in_rs],  r < S        (zero where the position is >= in_len)
// and writes X[k] (natural order) times the pass twiddle to out[b * out_bs + t_hi * out_hi + t_lo * out_lo + k * out_rs].
struct NttPassParams {
    const fe* in;
    fe* out;
    const fe* small;       // [512] w_1024^(+-i)
    const fe* tw_full;     // pass twiddle: n-entry table, entry (tau << log_s) + k, or
    const fe* lo;          //               three 1024-entry tables, exponent e = (tw_by_lo ? t_lo : tau) * k,
    const fe* mid;         //               w^e = domain_point(lo, mid, hi2, e); all null: no twiddle
    const fe* hi2;
    const fe* scale;       // optional factor applied at the store (device pointer, e.g. n^-1), or null
    unsigned log_s;        // sub-transform size S = 2^log_s
    unsigned split_log;
    size_t in_hi, in_lo, in_rs, in_bs;
    size_t out_hi, out_lo, out_rs, out_bs;
    size_t in_len;         // input positions >= in_len read as zero
    int pos_is_row;        // 1: the position is the row index (every tile is a polynomial of its own), 0: the offset inside the polynomial
    int tw_by_lo;
};

template <class F> int ntt_build_small_table(fe* d_small, bool inverse, cudaStream_t st);
template <class F> int ntt_build_tables(NttTables& t, unsigned log_n, bool inverse, cudaStream_t st);
// log2(n2 * n3) of the three-pass plan for a transform of 2^log_n elements (0: one or two passes, no inner tables needed)
unsigned ntt_inner_log(unsigned log_n);

// Transform of `batch` polynomials of 2^log_n elements: polynomial b is read from d_in + b * in_bs (its first in_len elements;
// the rest is taken as zero) and written to d_out + b * 2^log_n.  d_in == d_out (in_bs == 2^log_n) transforms in place.
// d_tmp: scratch of batch * 2^log_n elements (used when log_n > NTT_MAX_LOG_SUB).  inner: the tables of the (n2 * n3)-point
// transform (log_n > 20 only).
template <class F>
int ntt_run(const fe* d_in, size_t in_bs, fe* d_out, fe* d_tmp, const fe* d_small, const NttTables& tabs, const NttTables* inner, unsigned log_n,
            size_t batch, size_t in_len, bool inverse, bool coset, cudaStream_t st, unsigned* launches);

}  // namespace zkb
