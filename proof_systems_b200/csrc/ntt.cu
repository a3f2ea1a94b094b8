// ntt.cu — kernels and launch plan of the Pasta-field NTT (see ntt.cuh for semantics and reference call sites).
#include "ntt.cuh"
#include "ntt_butterfly.cuh"

namespace zkb {

// ---------------------------------------------------------------------------------------------- table construction
// bases[0] = w      (n-th root of unity, or its inverse)        bases[1] = w^1024
// bases[2] = g      (coset generator 5, or its inverse)         bases[3] = g^1024
// bases[4] = scale  (1 forward, n^-1 inverse)                   bases[5] = 1            bases[6] = w^(2^20)
template <class F> __global__ void k_ntt_setup(fe* bases, unsigned log_n, int inverse) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    fe w;
#pragma unroll
    for (int i = 0; i < 8; i++) w.v[i] = F::ROOT(i);
    for (unsigned i = log_n; i < 32; i++) w = fe_sqr<F>(w);  // (5^T)^(2^(32-log_n)); kimchi/src/circuits/domains.rs:40-69
    fe five = fe_zero();
    five.v[0] = 5;
    fe g = fe_to_mont<F>(five);  // multiplicative generator (fp.rs:10 / fq.rs:10) = ark's default coset offset
    fe scale = fe_one<F>();
    if (inverse) {
        w = fe_inv<F>(w);
        g = fe_inv<F>(g);
        fe n = fe_zero();
        n.v[0] = 1u << log_n;  // log_n <= 30
        scale = fe_inv<F>(fe_to_mont<F>(n));
    }
    bases[0] = w;
    bases[1] = fe_pow_u64<F>(w, 1024);
    bases[2] = g;
    bases[3] = fe_pow_u64<F>(g, 1024);
    bases[4] = scale;
    bases[5] = fe_one<F>();
    bases[6] = fe_pow_u64<F>(w, (uint64_t)1 << 20);
}

// out[i] = base^i * scale, i < count
template <class F> __global__ void k_pow_table(fe* out, const fe* base, const fe* scale, unsigned count) {
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    fe b = *base;
    fe r = fe_mul<F>(fe_pow_u64<F>(b, i), *scale);
    store_fe(out + i, r);
}

// full[col * n1 + k] = w^(col * k) (* n^-1): the inter-pass twiddles of the two-pass plan, one contiguous run of n1 entries per
// tile (= column) of pass 1, so a tile streams its twiddles with fully coalesced loads
template <class F> __global__ void k_full_table(fe* full, const fe* __restrict__ lo, const fe* __restrict__ mid, unsigned log_n1, size_t n) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    const unsigned k = (unsigned)(idx & (((size_t)1 << log_n1) - 1)), col = (unsigned)(idx >> log_n1);
    const unsigned e = col * k;          // < n <= 2^20
    fe tw = load_fe_nc(lo + (e & 1023));
    if (e >> 10) tw = fe_mul<F>(tw, load_fe_nc(mid + (e >> 10)));
    store_fe(full + idx, tw);
}

template <class F> int ntt_build_small_table(fe* d_small, bool inverse, cudaStream_t st) {
    DevScratch tmp;
    if (int rc = tmp.ensure(8 * sizeof(fe))) return rc;
    fe* bases = tmp.at<fe>();
    k_ntt_setup<F><<<1, 32, 0, st>>>(bases, 10, inverse ? 1 : 0);
    k_pow_table<F><<<2, 256, 0, st>>>(d_small, bases + 0, bases + 5, 512);
    ZK_CUDA(cudaGetLastError());
    ZK_CUDA(cudaStreamSynchronize(st));
    return ZK_OK;
}

template <class F> int ntt_build_tables(NttTables& t, unsigned log_n, bool inverse, cudaStream_t st) {
    DevScratch tmp;
    if (int rc = tmp.ensure(8 * sizeof(fe))) return rc;
    fe* bases = tmp.at<fe>();
    if (int rc = t.block.ensure(6 * 1024 * sizeof(fe))) return rc;
    fe* blk = t.block.at<fe>();
    t.lo = blk; t.ulo = blk + 1024; t.mid = blk + 2048; t.hi2 = blk + 3072; t.clo = blk + 4096; t.chi = blk + 5120;
    k_ntt_setup<F><<<1, 32, 0, st>>>(bases, log_n, inverse ? 1 : 0);
    k_pow_table<F><<<4, 256, 0, st>>>(t.lo, bases + 0, bases + 4, 1024);   // w^i * (n^-1 if inverse)
    k_pow_table<F><<<4, 256, 0, st>>>(t.ulo, bases + 0, bases + 5, 1024);  // w^i
    k_pow_table<F><<<4, 256, 0, st>>>(t.mid, bases + 1, bases + 5, 1024);  // w^(1024 i)
    k_pow_table<F><<<4, 256, 0, st>>>(t.hi2, bases + 6, bases + 5, 1024);  // w^(2^20 i)
    k_pow_table<F><<<4, 256, 0, st>>>(t.clo, bases + 2, bases + 5, 1024);  // g^i
    k_pow_table<F><<<4, 256, 0, st>>>(t.chi, bases + 3, bases + 5, 1024);  // g^(1024 i)
    if (log_n > NTT_MAX_LOG_SUB && log_n <= 2 * NTT_MAX_LOG_SUB) {     // only the two-pass plan reads it (ntt_run)
        const size_t n = (size_t)1 << log_n;
        const unsigned log_n1 = (log_n + 1) / 2;
        if (int rc = t.full.ensure(n * sizeof(fe))) return rc;
        k_full_table<F><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(t.full.at<fe>(), t.lo, t.mid, log_n1, n);
    }
    ZK_CUDA(cudaGetLastError());
    ZK_CUDA(cudaStreamSynchronize(st));
    return ZK_OK;
}

// ---------------------------------------------------------------------------------------------- the tile pass
// Shared-memory tile of one column, limb-major and padded: word (limb l, row i) at sm[l * SP + i + (i >> 5)], SP = S + S / 32.
// Adjacent lanes touch adjacent rows in the register stage, in every shared-memory layer (span >= 64) and in the natural-order
// store; the bit-reversed write of the load hits rows S/32 apart, which the padding spreads over the 32 banks: conflict free.
__device__ __forceinline__ unsigned ntt_pad(unsigned i) { return i + (i >> 5); }

template <class F> __global__ void __launch_bounds__(128, 6) k_ntt_pass(NttPassParams p) {
    extern __shared__ uint32_t sm[];
    const unsigned S = 1u << p.log_s, SP = S + (S >> 5) + 1;
    const unsigned tid = threadIdx.x, nthr = blockDim.x;
    const size_t tau = blockIdx.x;
    const size_t t_hi = tau >> p.split_log, t_lo = tau & (((size_t)1 << p.split_log) - 1);
    const size_t in_off = t_hi * p.in_hi + t_lo * p.in_lo;
    const fe* in = p.in + (size_t)blockIdx.y * p.in_bs + in_off;
    const size_t out_off = t_hi * p.out_hi + t_lo * p.out_lo;
    fe* out = p.out + (size_t)blockIdx.y * p.out_bs + out_off;

    // load, zero-padded by position, written in bit-reversed row order; four independent loads in flight per thread
    for (unsigned r0 = tid; r0 < S; r0 += 4 * nthr) {
        fe v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const unsigned r = r0 + u * nthr;
            const size_t pos = p.pos_is_row ? (size_t)r : in_off + r * p.in_rs;
            v[u] = fe_zero();
            if (r < S && pos < p.in_len) v[u] = load_fe(in + r * p.in_rs);
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const unsigned r = r0 + u * nthr;
            if (r >= S) break;
            const unsigned i = p.log_s ? (__brev(r) >> (32 - p.log_s)) : 0;
            uint32_t* dst = sm + ntt_pad(i);
#pragma unroll
            for (int l = 0; l < 8; l++) dst[l * SP] = v[u].v[l];
        }
    }
    __syncthreads();

    unsigned l0 = 0;          // first layer that goes through shared memory
    if (p.log_s >= 6) {
        // register stage: layers 0..5 of one 64-row chunk per warp iteration (ntt_butterfly.cuh)
        const unsigned lane = tid & 31, warp = tid >> 5, nwarp = nthr >> 5;
        for (unsigned q = warp; q < (S >> 6); q += nwarp) {
            const unsigned ia = (q << 6) + lane, ib = (q << 6) + 32 + (lane ^ 31u);
            const uint32_t* pa = sm + ntt_pad(ia);
            const uint32_t* pb = sm + ntt_pad(ib);
            fe a, b;
#pragma unroll
            for (int k = 0; k < 8; k++) { a.v[k] = pa[k * SP]; b.v[k] = pb[k * SP]; }
#pragma unroll 1
            for (unsigned l = 0; l < 5; l++) {
                bool a_hi;
                fe tx, sa, sb;
                ntt_lane_pre<F>(lane, l, a, b, p.small, a_hi, tx, sa, sb);
                const fe ra = shfl_xor_fe(sa, 1u << l), rb = shfl_xor_fe(sb, 1u << l);
                ntt_lane_post<F>(a_hi, tx, ra, rb, a, b);
            }
            b = shfl_fe(b, (int)(lane ^ 31u));                    // block B back to natural order
            ntt_lane_last<F>(lane, a, b, p.small);
            __syncwarp();      // lane t read row 32 + (t ^ 31), which lane t ^ 31 writes below: order the warp's reads before its writes
            uint32_t* qa = sm + ntt_pad((q << 6) + lane);
            uint32_t* qb = sm + ntt_pad((q << 6) + 32 + lane);
#pragma unroll
            for (int k = 0; k < 8; k++) { qa[k * SP] = a.v[k]; qb[k * SP] = b.v[k]; }
        }
        __syncthreads();
        l0 = 6;
    }
    for (unsigned l = l0; l < p.log_s; l++) {
        for (unsigned bidx = tid; bidx < (S >> 1); bidx += nthr) {
            unsigned i0, tw;
            ntt_index2_dit(bidx, l, i0, tw);
            uint32_t* a0 = sm + ntt_pad(i0);
            uint32_t* a1 = sm + ntt_pad(i0 + (1u << l));
            fe u, v;
#pragma unroll
            for (int k = 0; k < 8; k++) { u.v[k] = a0[k * SP]; v.v[k] = a1[k * SP]; }
            if (l != 0) { const fe w = load_fe_nc(p.small + tw); ntt_bfly2_dit<F>(u, v, &w); }
            else ntt_bfly2_dit<F>(u, v, nullptr);
#pragma unroll
            for (int k = 0; k < 8; k++) { a0[k * SP] = u.v[k]; a1[k * SP] = v.v[k]; }
        }
        __syncthreads();
    }

    // store: natural order; inter-pass twiddle, scaling and transposition fused.  Four twiddle loads in flight per thread.
    const size_t tw_col = p.tw_by_lo ? t_lo : tau;
    for (unsigned k0 = tid; k0 < S; k0 += 4 * nthr) {
        fe tw[4];
        if (p.tw_full) {
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const unsigned k = k0 + u * nthr;
                if (k < S) tw[u] = load_fe_nc(p.tw_full + (tau << p.log_s) + k);
            }
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const unsigned k = k0 + u * nthr;
            if (k >= S) break;
            const uint32_t* src = sm + ntt_pad(k);
            fe v;
#pragma unroll
            for (int l = 0; l < 8; l++) v.v[l] = src[l * SP];
            if (p.tw_full) {
                v = fe_mul<F>(v, tw[u]);
            } else if (p.lo) {
                const unsigned e = (unsigned)tw_col * k;                  // < 2^30
                v = fe_mul<F>(v, domain_point<F>(p.lo, p.mid, p.hi2, e));
            }
            if (p.scale) v = fe_mul<F>(v, load_fe_nc(p.scale));
            store_fe(out + k * p.out_rs, v);
        }
    }
}

// x[j] *= g^(+-j) for j < len (forward coset: before the transform; inverse coset: after it)
template <class F> __global__ void k_coset_scale(fe* data, size_t n, size_t len, const fe* clo, const fe* chi, const fe* chi2) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= len) return;
    fe* p = data + (size_t)blockIdx.y * n + j;
    fe tw = load_fe_nc(clo + (j & 1023));
    if ((j >> 10) & 1023) tw = fe_mul<F>(tw, load_fe_nc(chi + ((j >> 10) & 1023)));
    if (j >> 20) tw = fe_mul<F>(tw, fe_pow_u64<F>(load_fe_nc(chi2), (uint64_t)(j >> 20) << 10));   // chi2 = g^(+-1024); domains beyond 2^20 only
    store_fe(p, fe_mul<F>(load_fe(p), tw));
}
// dst[b * n + j] = j < len ? src[b * src_bs + j] : 0   (coset transforms out of place: the input is scaled in the output buffer)
__global__ void k_copy_pad(fe* dst, const fe* __restrict__ src, size_t n, size_t src_bs, size_t len) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    store_fe(dst + (size_t)blockIdx.y * n + j, j < len ? load_fe_nc(src + (size_t)blockIdx.y * src_bs + j) : fe_zero());
}

unsigned ntt_inner_log(unsigned log_n) { return log_n <= 2 * NTT_MAX_LOG_SUB ? 0 : log_n - (log_n + 2) / 3; }

template <class F> static int launch_pass(const NttPassParams& p, size_t tiles, size_t batch_y, cudaStream_t st) {
    const unsigned S = 1u << p.log_s;
    const size_t smem = (size_t)8 * (S + (S >> 5) + 1) * sizeof(uint32_t);
    unsigned threads = S >> 1;                 // one shared-memory butterfly per thread and layer, one 64-row chunk per warp
    if (threads > 128) threads = 128;
    if (threads < 32) threads = 32;
    if (tiles > 0x7fffffffull || batch_y > 65535) { zk_set_error("ntt: %zu x %zu tiles exceed the grid limits", tiles, batch_y); return ZK_ERR_INVALID; }
    dim3 grid((unsigned)tiles, (unsigned)batch_y);
    k_ntt_pass<F><<<grid, threads, smem, st>>>(p);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}

template <class F>
int ntt_run(const fe* d_in, size_t in_bs, fe* d_out, fe* d_tmp, const fe* d_small, const NttTables& tabs, const NttTables* inner, unsigned log_n,
            size_t batch, size_t in_len, bool inverse, bool coset, cudaStream_t st, unsigned* launches) {
    if (log_n > NTT_MAX_LOG_N) { zk_set_error("ntt: log_n %u > %u not supported", log_n, NTT_MAX_LOG_N); return ZK_ERR_INVALID; }
    const size_t n = (size_t)1 << log_n;
    if (in_len == 0 || in_len > n) in_len = n;
    if (batch == 0) return ZK_OK;
    unsigned nl = 0;
    // batches beyond the grid's y limit run in slices
    if (batch > 65535) {
        for (size_t b0 = 0; b0 < batch; b0 += 32768) {
            const size_t cnt = std::min<size_t>(32768, batch - b0);
            int rc = ntt_run<F>(d_in + b0 * in_bs, in_bs, d_out + b0 * n, d_tmp ? d_tmp + b0 * n : nullptr, d_small, tabs, inner, log_n, cnt, in_len, inverse, coset, st, launches);
            if (rc) return rc;
        }
        return ZK_OK;
    }
    if (coset && !inverse) {
        // x[j] *= g^j first.  Out of place: the padded copy in the output buffer is scaled, and the transform runs in place there.
        if (d_in != d_out) {
            k_copy_pad<<<dim3((unsigned)((n + 255) / 256), (unsigned)batch), 256, 0, st>>>(d_out, d_in, n, in_bs, in_len);
            nl++;
            d_in = d_out;
            in_bs = n;
        }
        dim3 grid((unsigned)((in_len + 255) / 256), (unsigned)batch);
        k_coset_scale<F><<<grid, 256, 0, st>>>(d_out, n, in_len, tabs.clo, tabs.chi, tabs.chi + 1);
        nl++;
    }
    if (log_n == 0) {
        // n = 1: both transforms are the identity (n^-1 = 1)
        if (d_in != d_out) { k_copy_pad<<<dim3(1, (unsigned)batch), 32, 0, st>>>(d_out, d_in, 1, in_bs, in_len); nl++; }
    } else if (log_n <= NTT_MAX_LOG_SUB) {
        // one pass: every polynomial is one tile
        NttPassParams p{};
        p.in = d_in; p.out = d_out; p.small = d_small;
        p.log_s = log_n; p.split_log = 0;
        p.in_hi = in_bs; p.in_lo = 0; p.in_rs = 1; p.in_bs = 0;
        p.out_hi = n; p.out_lo = 0; p.out_rs = 1; p.out_bs = 0;
        p.in_len = in_len; p.pos_is_row = 1;
        p.scale = inverse ? tabs.lo : nullptr;  // entry 0 of the inverse lo table is n^-1
        // tiles along x (the batch may exceed the y limit of a grid)
        int rc = launch_pass<F>(p, batch, 1, st);
        if (rc) return rc;
        nl++;
    } else if (log_n <= 2 * NTT_MAX_LOG_SUB) {
        const unsigned log_n1 = (log_n + 1) / 2, log_n2 = log_n - log_n1;
        const size_t n1 = (size_t)1 << log_n1, n2 = (size_t)1 << log_n2;
        // pass 1: n2 column transforms of size n1 (stride n2), times w_n^(j2 k1); in -> tmp, layout [k1][j2]
        NttPassParams p{};
        p.in = d_in; p.out = d_tmp; p.small = d_small;
        p.tw_full = tabs.full.at<fe>();
        if (!tabs.full.p) { p.lo = tabs.lo; p.mid = tabs.mid; p.hi2 = tabs.hi2; }
        p.log_s = log_n1; p.split_log = 0;
        p.in_hi = 1; p.in_rs = n2; p.in_bs = in_bs;
        p.out_hi = 1; p.out_rs = n2; p.out_bs = n;
        p.in_len = in_len; p.pos_is_row = 0; p.tw_by_lo = 0;
        int rc = launch_pass<F>(p, n2, batch, st);
        if (rc) return rc;
        // pass 2: n1 row transforms of size n2 (contiguous), output transposed to natural order; tmp -> out
        NttPassParams q{};
        q.in = d_tmp; q.out = d_out; q.small = d_small;
        q.log_s = log_n2; q.split_log = 0;
        q.in_hi = n2; q.in_rs = 1; q.in_bs = n;
        q.out_hi = 1; q.out_rs = n1; q.out_bs = n;
        q.in_len = n; q.pos_is_row = 1;
        rc = launch_pass<F>(q, n1, batch, st);
        if (rc) return rc;
        nl += 2;
    } else {
        // three passes, n = n1 n2 n3:  j = j1 n2 n3 + j2 n3 + j3,  k = k1 + n1 k2 + n1 n2 k3
        if (!inner) { zk_set_error("ntt: the tables of the inner transform are missing"); return ZK_ERR_INVALID; }
        const unsigned log_rest = ntt_inner_log(log_n), log_n1 = log_n - log_rest, log_n2 = (log_rest + 1) / 2, log_n3 = log_rest - log_n2;
        const size_t n1 = (size_t)1 << log_n1, n2 = (size_t)1 << log_n2, n3 = (size_t)1 << log_n3, n23 = n2 * n3;
        // pass 1 (over j1): tiles (j2, j3), twiddle w_n^((j2 n3 + j3) k1); in -> out, layout [k1][j2][j3]
        NttPassParams p{};
        p.in = d_in; p.out = d_out; p.small = d_small;
        p.lo = tabs.lo; p.mid = tabs.mid; p.hi2 = tabs.hi2;
        p.log_s = log_n1; p.split_log = 0;
        p.in_hi = 1; p.in_rs = n23; p.in_bs = in_bs;
        p.out_hi = 1; p.out_rs = n23; p.out_bs = n;
        p.in_len = in_len; p.pos_is_row = 0; p.tw_by_lo = 0;
        int rc = launch_pass<F>(p, n23, batch, st);
        if (rc) return rc;
        // pass 2 (over j2): tiles (k1, j3), twiddle w_{n2 n3}^(j3 k2) (unscaled: 1/n went in with pass 1); out -> tmp, same layout
        NttPassParams q{};
        q.in = d_out; q.out = d_tmp; q.small = d_small;
        q.lo = inner->ulo; q.mid = inner->mid; q.hi2 = inner->hi2;
        q.log_s = log_n2; q.split_log = log_n3;
        q.in_hi = n23; q.in_lo = 1; q.in_rs = n3; q.in_bs = n;
        q.out_hi = n23; q.out_lo = 1; q.out_rs = n3; q.out_bs = n;
        q.in_len = n; q.pos_is_row = 1; q.tw_by_lo = 1;
        rc = launch_pass<F>(q, n1 * n3, batch, st);
        if (rc) return rc;
        // pass 3 (over j3): tiles (k1, k2), contiguous rows; output index k1 + n1 k2 + n1 n2 k3; tmp -> out
        NttPassParams r{};
        r.in = d_tmp; r.out = d_out; r.small = d_small;
        r.log_s = log_n3; r.split_log = log_n2;
        r.in_hi = n23; r.in_lo = n3; r.in_rs = 1; r.in_bs = n;
        r.out_hi = 1; r.out_lo = n1; r.out_rs = n1 * n2; r.out_bs = n;
        r.in_len = n; r.pos_is_row = 1;
        rc = launch_pass<F>(r, n1 * n2, batch, st);
        if (rc) return rc;
        nl += 3;
    }
    if (coset && inverse) {
        dim3 grid((unsigned)((n + 255) / 256), (unsigned)batch);
        k_coset_scale<F><<<grid, 256, 0, st>>>(d_out, n, n, tabs.clo, tabs.chi, tabs.chi + 1);
        nl++;
    }
    ZK_CUDA(cudaGetLastError());
    if (launches) *launches += nl;
    return ZK_OK;
}

template int ntt_build_small_table<FpParams>(fe*, bool, cudaStream_t);
template int ntt_build_small_table<FqParams>(fe*, bool, cudaStream_t);
template int ntt_build_tables<FpParams>(NttTables&, unsigned, bool, cudaStream_t);
template int ntt_build_tables<FqParams>(NttTables&, unsigned, bool, cudaStream_t);
template int ntt_run<FpParams>(const fe*, size_t, fe*, fe*, const fe*, const NttTables&, const NttTables*, unsigned, size_t, size_t, bool, bool, cudaStream_t, unsigned*);
template int ntt_run<FqParams>(const fe*, size_t, fe*, fe*, const fe*, const NttTables&, const NttTables*, unsigned, size_t, size_t, bool, bool, cudaStream_t, unsigned*);

}  // namespace zkb
