// msm.cu — kernels and pipeline of the Pallas/Vesta MSM (see msm.cuh for semantics and reference call sites).
#include "msm.cuh"
#include "quad.cuh"

#include <algorithm>

namespace zkb {

unsigned msm_num_windows(unsigned c) { return (256 + c - 1) / c; }  // top signed digit cannot carry out (scalars < 2^254 + 2^127)

int msm_default_window(size_t n, bool precomputed) {
    // accumulation costs ceil(256/c) * n mixed additions; the bucket side grows with 2^(c-1) (one bucket set with a
    // table, one per window without).  Measured on H100 (tools/sweep.py): with a table, 2^16 points -> c = 15 and 2^11 -> c = 10.
    unsigned l = 0;
    while (((size_t)1 << (l + 1)) <= n) l++;
    int c = (int)l - (precomputed ? 1 : 4);
    if (c < 4) c = 4;
    if (c > (int)MSM_MAX_WINDOW_BITS) c = MSM_MAX_WINDOW_BITS;
    return c;
}

// ---------------------------------------------------------------------------------------------- table of 2^(cw) P
template <class F> __global__ void k_build_table(affine_t* table, size_t n, unsigned c, unsigned nwin) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    affine_t p = load_affine_nc(table + i);
    xyzz_t acc = xyzz_from_affine<F>(p);
    for (unsigned w = 1; w < nwin; w++) {
        for (unsigned k = 0; k < c; k++) acc = xyzz_dbl<F>(acc);
        store_affine(table + (size_t)w * n + i, xyzz_to_affine<F>(acc));
    }
}

// The same table with ONE field inversion per point instead of one per row (Montgomery's trick over the rows of a point):
// ~255 doublings + 1 inversion + 8 multiplications per row, 3.4x less arithmetic than k_build_table.  nwin <= TABLE_MAX_ROWS.
constexpr unsigned TABLE_MAX_ROWS = 33;   // windows of >= 8 bits
template <class F> __global__ void __launch_bounds__(128) k_build_table_batched(affine_t* table, size_t n, unsigned c, unsigned nwin) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const affine_t p = load_affine_nc(table + i);
    if (affine_is_inf(p)) {
        for (unsigned w = 1; w < nwin; w++) store_affine(table + (size_t)w * n + i, p);
        return;
    }
    xyzz_t pts[TABLE_MAX_ROWS];
    fe pre[TABLE_MAX_ROWS];
    xyzz_t acc = xyzz_from_affine<F>(p);
    for (unsigned w = 1; w < nwin; w++) {
        for (unsigned k = 0; k < c; k++) acc = xyzz_dbl<F>(acc);
        pts[w] = acc;
        const fe z = fe_mul<F>(acc.ZZ, acc.ZZZ);        // never zero: the curve has prime order, doubling a finite point stays finite
        pre[w] = w == 1 ? z : fe_mul<F>(pre[w - 1], z);
    }
    if (nwin < 2) return;
    fe inv = fe_inv<F>(pre[nwin - 1]);
    for (unsigned w = nwin - 1; w >= 1; w--) {
        const fe zi = w == 1 ? inv : fe_mul<F>(inv, pre[w - 1]);          // 1 / (ZZ_w * ZZZ_w)
        inv = fe_mul<F>(inv, fe_mul<F>(pts[w].ZZ, pts[w].ZZZ));
        affine_t r;
        r.x = fe_mul<F>(pts[w].X, fe_mul<F>(zi, pts[w].ZZZ));              // X / ZZ
        r.y = fe_mul<F>(pts[w].Y, fe_mul<F>(zi, pts[w].ZZ));               // Y / ZZZ
        store_affine(table + (size_t)w * n + i, r);
    }
}

template <class F> int msm_bases_create(MsmBases& b, const affine_t* pts, bool pts_on_device, size_t n, unsigned c_table, cudaStream_t st) {
    if (c_table > MSM_MAX_WINDOW_BITS) { zk_set_error("msm: table window %u > %u", c_table, MSM_MAX_WINDOW_BITS); return ZK_ERR_INVALID; }
    b.n = n;
    b.c = c_table;
    b.nwin = c_table ? msm_num_windows(c_table) : 0;
    size_t rows = c_table ? b.nwin : 1;
    if (int rc = b.points.ensure(std::max<size_t>(rows * n, 1) * sizeof(affine_t))) return rc;
    b.d_points = b.points.at<affine_t>();
    if (n == 0) return ZK_OK;
    ZK_CUDA(cudaMemcpyAsync(b.d_points, pts, n * sizeof(affine_t), pts_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    if (c_table) {
        if (b.nwin <= TABLE_MAX_ROWS) k_build_table_batched<F><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(b.d_points, n, c_table, b.nwin);
        else k_build_table<F><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(b.d_points, n, c_table, b.nwin);
        ZK_CUDA(cudaGetLastError());
    }
    ZK_CUDA(cudaStreamSynchronize(st));
    return ZK_OK;
}

// ---------------------------------------------------------------------------------------------- recode + histogram
// One thread per scalar of one MSM of the batch (blockIdx.y): Montgomery -> canonical if asked (VariableBaseMSM::msm ==
// into_bigint + msm_bigint), then signed base-2^c digits d_w in (-2^(c-1), 2^(c-1)]; digit w of scalar i of MSM j at
// digits[(j*nwin + w)*n + i]; per-bucket counts.  Bucket group of (MSM j, window w): j*gpm + (per_window ? w : 0).
template <class FS>
__global__ void k_recode(MsmScalarSet sc, int scalars_mont, size_t n, unsigned c, unsigned nwin, unsigned gpm, int per_window,
                         int32_t* digits, uint32_t* counts, uint32_t* meta) {
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) meta[2] = 0;   // giant list of this run (k_plan)
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned j = blockIdx.y;
    fe s = load_fe_nc(sc.p[j] + i);
    if (scalars_mont) s = fe_from_mont<FS>(s);
    const uint32_t half = 1u << (c - 1), mask = (1u << c) - 1;
    const uint32_t B = half;
    uint32_t carry = 0;
    for (unsigned w = 0; w < nwin; w++) {
        unsigned off = w * c, limb = off >> 5, sh = off & 31;
        uint32_t v = 0;
        if (limb < 8) {
            v = s.v[limb] >> sh;
            if (sh + c > 32 && limb + 1 < 8) v |= s.v[limb + 1] << (32 - sh);
        }
        uint32_t d = (v & mask) + carry;
        int32_t sd;
        if (d > half) { sd = (int32_t)d - (int32_t)(1u << c); carry = 1; }
        else { sd = (int32_t)d; carry = 0; }
        digits[((size_t)j * nwin + w) * n + i] = sd;
        // warp-aggregated histogram update: lanes that hit the same bucket (kimchi's all-ones columns: all of them) elect
        // one lane to add their count — one atomic per distinct bucket per warp instead of one per lane
        const uint32_t mag = (uint32_t)(sd < 0 ? -sd : sd);
        const uint32_t key = sd != 0 ? (j * gpm + (per_window ? w : 0)) * B + (mag - 1) : 0xffffffffu;
        const uint32_t peers = __match_any_sync(__activemask(), key);
        if (sd != 0 && (threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicAdd(&counts[key], (uint32_t)__popc(peers));
    }
}

// Planning pass over the histogram: exclusive scans of the bucket counts (-> offsets of the sorted entry list) and of the
// per-bucket task counts s_b = ceil(n_b / K) (-> task_off).  One CTA per tile of 4096 buckets; the tiles are chained (tile t
// spins on tile t-1's published inclusive total — tiles are dispatched in order, so the predecessor is always resident), which
// keeps the scan a single launch for any batch size.  64-bit lanes carry (entry count << 32 | task count): one scan yields both.
// Buckets with more than smax tasks ("giant": the all-ones witness columns of kimchi put ~n entries in one bucket,
// SURVEY.md §3.1) are listed for k_giant_finish.  Clears counts (re-used as scatter cursors).
__device__ __forceinline__ uint64_t block_excl_scan_1024(uint64_t v, uint64_t* warp_sums, uint64_t* tile_total) {
    const unsigned tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    uint64_t x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint64_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= (unsigned)d) x += y;
    }
    if (lane == 31) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
        uint64_t ws = warp_sums[lane], z = ws;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            uint64_t y = __shfl_up_sync(0xffffffffu, z, d);
            if (lane >= (unsigned)d) z += y;
        }
        warp_sums[lane] = z - ws;
        if (lane == 31) *tile_total = z;
    }
    __syncthreads();
    uint64_t excl = warp_sums[wid] + (x - v);
    __syncthreads();
    return excl;
}

constexpr unsigned PLAN_PER_THREAD = 4, PLAN_TILE = 1024 * PLAN_PER_THREAD;
__global__ void __launch_bounds__(1024) k_plan(uint32_t* counts, uint32_t* offsets, uint32_t* task_off, uint32_t nb, uint32_t K, uint32_t smax,
                                                 uint32_t* meta, uint32_t* giants, uint64_t* chain, uint32_t* chain_flag, uint32_t epoch) {
    __shared__ uint64_t warp_sums[32];
    __shared__ uint64_t tile_total, prefix_s;
    const unsigned tid = threadIdx.x, tile = blockIdx.x;
    const uint32_t i0 = tile * PLAN_TILE + tid * PLAN_PER_THREAD;
    uint32_t v[PLAN_PER_THREAD];
    uint64_t pk[PLAN_PER_THREAD], sum = 0;
#pragma unroll
    for (unsigned k = 0; k < PLAN_PER_THREAD; k++) {
        v[k] = i0 + k < nb ? counts[i0 + k] : 0;
        if (i0 + k < nb) counts[i0 + k] = 0;
        pk[k] = ((uint64_t)v[k] << 32) | ((v[k] + K - 1) / K);
        sum += pk[k];
    }
    uint64_t ex = block_excl_scan_1024(sum, warp_sums, &tile_total);
    if (tid == 0) {
        uint64_t prefix = 0;
        if (tile > 0) {
            volatile uint32_t* f = chain_flag + (tile - 1);
            while (*f != epoch) { }
            __threadfence();
            prefix = *(volatile uint64_t*)(chain + (tile - 1));
        }
        *(volatile uint64_t*)(chain + tile) = prefix + tile_total;
        __threadfence();
        *(volatile uint32_t*)(chain_flag + tile) = epoch;
        prefix_s = prefix;
    }
    __syncthreads();
    ex += prefix_s;
#pragma unroll
    for (unsigned k = 0; k < PLAN_PER_THREAD; k++) {
        if (i0 + k < nb) {
            offsets[i0 + k] = (uint32_t)(ex >> 32);
            task_off[i0 + k] = (uint32_t)ex;
            if ((uint32_t)pk[k] > smax) {
                uint32_t gi = atomicAdd(&meta[2], 1u);
                if (gi < MSM_MAX_GIANTS) giants[gi] = i0 + k;
            }
        }
        ex += pk[k];
    }
    if (tile == gridDim.x - 1 && tid == 0) {
        const uint64_t tot = prefix_s + tile_total;
        offsets[nb] = (uint32_t)(tot >> 32); task_off[nb] = (uint32_t)tot;
        meta[0] = (uint32_t)(tot >> 32); meta[1] = (uint32_t)tot;
    }
}

// Counting-sort scatter: entry (point index | sign) of every non-zero digit goes to its bucket's range.
__global__ void k_scatter(const int32_t* digits, size_t n, unsigned c, unsigned nwin, unsigned batch, unsigned gpm, int per_window, MsmScalarSet sc,
                          size_t table_stride, int use_table, size_t n_main, size_t n_extra, uint32_t main_count, const uint32_t* offsets,
                          uint32_t* cursors, uint32_t* entries) {
    size_t id = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool in_range = id < n * nwin * batch;
    int32_t sd = in_range ? digits[id] : 0;
    const unsigned jw = (unsigned)(id / n), j = jw / nwin, w = jw - j * nwin;
    size_t i = id - (size_t)jw * n;
    const uint32_t B = 1u << (c - 1);
    uint32_t mag = (uint32_t)(sd < 0 ? -sd : sd);
    uint32_t key = sd != 0 ? (j * gpm + (per_window ? w : 0)) * B + (mag - 1) : 0xffffffffu;
    // warp-aggregated cursor bump (see k_recode): the leader reserves a run, every peer takes its rank inside it
    const uint32_t peers = __match_any_sync(0xffffffffu, key);
    const unsigned lane = threadIdx.x & 31, leader = (unsigned)(__ffs(peers) - 1);
    uint32_t base = 0;
    if (sd != 0 && lane == leader) base = atomicAdd(&cursors[key], (uint32_t)__popc(peers));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (sd == 0) return;
    uint32_t pos = offsets[key] + base + (uint32_t)__popc(peers & ((1u << lane) - 1));
    // scalars [0, n_main) belong to the resident bases, [n_main, n) to the call's extra points (their rows behind the table)
    size_t pidx = i < n_main ? (use_table ? (size_t)w * table_stride : 0) + sc.off[in_range ? j : 0] + i
                             : (size_t)main_count + (use_table ? (size_t)w * n_extra : 0) + (i - n_main);
    entries[pos] = (uint32_t)pidx | (sd < 0 ? 0x80000000u : 0u);
}

// ---------------------------------------------------------------------------------------------- accumulation
// Task t belongs to the bucket b with task_off[b] <= t < task_off[b+1]; the bucket's n_b sorted entries are cut into
// s_b = ceil(n_b / K) nearly equal parts, so no task crosses a bucket boundary and every thread sums <= K points with
// XYZZ mixed additions.  Single-task buckets are written directly, the others leave one partial per task.
template <class F>
__global__ void __launch_bounds__(128) k_accumulate(const affine_t* __restrict__ points, const uint32_t* __restrict__ entries,
                                                    const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ task_off, uint32_t nb,
                                                    uint32_t K, const uint32_t* __restrict__ meta, const affine_t* __restrict__ extra,
                                                    uint32_t main_count, xyzz_t* buckets, xyzz_t* partials) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= __ldg(meta + 1)) return;
    // upper_bound(task_off[0..nb], t) - 1
    uint32_t lo = 0, hi = nb;  // invariant: task_off[lo] <= t < task_off[hi]
    while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        if (__ldg(task_off + mid) <= t) lo = mid; else hi = mid;
    }
    const uint32_t b = lo;
    const uint32_t e0 = __ldg(offsets + b), nbk = __ldg(offsets + b + 1) - e0;
    const uint32_t sb = (nbk + K - 1) / K, sub = t - __ldg(task_off + b);
    const uint32_t base = nbk / sb, rem = nbk - base * sb;
    uint32_t i = e0 + sub * base + min(sub, rem);
    const uint32_t end = i + base + (sub < rem ? 1u : 0u);
    xyzz_t acc = xyzz_identity();
    // software pipeline: the gather of point i+1 is in flight while point i is added
    // (entries >= main_count address the call's extra points: h and U of an IPA round, ipa.rs:944,954)
    uint32_t e = __ldg(entries + i);
    uint32_t idx = e & 0x7fffffffu;
    affine_t p = load_affine_nc(idx < main_count ? points + idx : extra + (idx - main_count));
    for (; i < end; i++) {
        affine_t q = p;
        const uint32_t sign = e >> 31;
        if (i + 1 < end) {
            e = __ldg(entries + i + 1);
            idx = e & 0x7fffffffu;
            p = load_affine_nc(idx < main_count ? points + idx : extra + (idx - main_count));
        }
        if (sign) q.y = fe_neg<F>(q.y);
        acc = xyzz_madd<F>(acc, q);
    }
    store_xyzz(sb == 1 ? buckets + b : partials + t, acc);
}

// Balanced first level of the per-bucket sums.  The task partials lie in bucket order; thread u sums the RUN of `run`
// consecutive partials [u*run, (u+1)*run) segment by segment (a segment = the part of one bucket inside the run) and writes each
// segment sum back at the segment's first index.  Every thread executes at most run-1 additions whatever the bucket sizes, so a
// warp never waits for its longest bucket.  k_bucket_finish_serial then adds, per bucket, the partial at the bucket's first index
// and those at the multiples of `run` inside it.  (Slots of single-task buckets hold no partial — k_accumulate wrote the bucket
// itself — and are segments of their own: read and written back, never mixed.)
template <class F>
__global__ void __launch_bounds__(128, 4) k_run_sum(const uint32_t* __restrict__ task_off, uint32_t nb, const uint32_t* __restrict__ meta, uint32_t run,
                                                 uint32_t smax, xyzz_t* partials) {
    const uint32_t nt = meta[1];
    const uint64_t i0w = (uint64_t)(blockIdx.x * blockDim.x + threadIdx.x) * run;
    if (i0w >= nt) return;
    const uint32_t i0 = (uint32_t)i0w, i1 = min(nt, i0 + run);
    // largest b with task_off[b] <= i0 (skips the empty buckets that share a start)
    uint32_t lo = 0, hi = nb;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(task_off + mid) <= i0) lo = mid; else hi = mid;
    }
    uint32_t b = lo, nxt = __ldg(task_off + b + 1), seg = i0;
    // giant buckets were summed by k_giant_finish: their slots are skipped (a thread wholly inside one does nothing)
    const bool giants_done = meta[2] <= MSM_MAX_GIANTS;
    bool skip = giants_done && nxt - __ldg(task_off + b) > smax;
    if (skip && nxt >= i1) return;
    xyzz_t acc = load_xyzz(partials + i0);
    bool dirty = false;
    for (uint32_t i = i0 + 1; i < i1; i++) {
        if (skip && i != nxt) continue;
        const xyzz_t v = load_xyzz(partials + i);
        if (i == nxt) {
            if (dirty) store_xyzz(partials + seg, acc);
            // the bucket that starts at i: usually the next one; behind a stretch of empty buckets, found by bisection
            b++; nxt = __ldg(task_off + b + 1);
            if (nxt <= i) {
                uint32_t l2 = b, h2 = nb;
                while (h2 - l2 > 1) {
                    const uint32_t mid = (l2 + h2) >> 1;
                    if (__ldg(task_off + mid) <= i) l2 = mid; else h2 = mid;
                }
                b = l2; nxt = __ldg(task_off + b + 1);
            }
            skip = giants_done && nxt - i > smax;
            seg = i; acc = v; dirty = false;
        } else {
            acc = xyzz_add<F, true>(acc, v);
            dirty = true;
        }
    }
    if (dirty) store_xyzz(partials + seg, acc);
}

// Thread-per-bucket finish pass, for MANY buckets with few partials each: with more buckets than resident quads the pass is
// throughput-bound and the quad-cooperative variant below only adds work.  run == 0: the bucket's partials are summed one by
// one; run > 0: k_run_sum ran first and the bucket's value is spread over its first slot and the multiples of `run` inside it.
template <class F>
__global__ void __launch_bounds__(128, 4) k_bucket_finish_serial(const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ task_off, uint32_t nb,
                                                              uint32_t K, uint32_t smax, const uint32_t* __restrict__ meta, uint32_t run, xyzz_t* buckets,
                                                              const xyzz_t* __restrict__ partials) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    const uint32_t nbk = __ldg(offsets + b + 1) - __ldg(offsets + b);
    uint32_t sb = (nbk + K - 1) / K;
    if (sb > smax && meta[2] <= MSM_MAX_GIANTS) return;  // k_giant_finish
    if (sb < 2) return;                                  // 0: empty, 1: written by k_accumulate
    const uint32_t a = __ldg(task_off + b);
    xyzz_t acc = load_xyzz(partials + a);
    if (run == 0) {
        for (uint32_t j = 1; j < sb; j++) acc = xyzz_add<F, true>(acc, load_xyzz(partials + a + j));
    } else {
        for (uint32_t k = (a / run + 1) * run; k < a + sb; k += run) acc = xyzz_add<F, true>(acc, load_xyzz(partials + k));
    }
    store_xyzz(buckets + b, acc);
}

// Buckets with 2 <= s_b <= smax tasks: a group of G = 2^log_g QUADS (quad.cuh) sums the bucket's partials — strided serial
// part, then a shuffle tree over the quads of the group.  One quad per bucket when buckets hold only a few partials.
template <class F>
__global__ void __launch_bounds__(128) k_bucket_finish(const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ task_off, uint32_t nb,
                                                       uint32_t K, uint32_t smax, unsigned log_g, const uint32_t* __restrict__ meta,
                                                       xyzz_t* buckets, const xyzz_t* __restrict__ partials) {
    const uint32_t gq = (blockIdx.x * blockDim.x + threadIdx.x) >> 2;   // global quad
    const uint32_t G = 1u << log_g, b = gq >> log_g, gl = gq & (G - 1);
    uint32_t sb = 0, t0 = 0;
    if (b < nb) {
        const uint32_t nbk = __ldg(offsets + b + 1) - __ldg(offsets + b);
        sb = (nbk + K - 1) / K;
        t0 = __ldg(task_off + b);
        // giants are left to k_giant_finish — unless their list overflowed, then they are summed here (slow, correct)
        if (sb > smax && meta[2] <= MSM_MAX_GIANTS) sb = 0;
        if (sb < 2) sb = 0;
    }
    // warp-uniform trip count: every lane must take part in the quad additions' shuffles
    const unsigned my_trips = sb > gl ? (sb - gl + G - 1) / G : 0;
    const unsigned trips = __reduce_max_sync(0xffffffffu, my_trips);
    xyzz_t acc = xyzz_identity();
    for (unsigned k = 0; k < trips; k++) {
        const uint32_t j = gl + k * G;
        xyzz_t o = j < sb ? load_xyzz(partials + t0 + j) : xyzz_identity();
        acc = xyzz_add_quad<F>(acc, o);
    }
#pragma unroll 1
    for (unsigned d = G >> 1; d >= 1; d >>= 1) {
        xyzz_t o = shfl_down_xyzz(acc, 4 * d);
        if (gl >= d) o = xyzz_identity();
        acc = xyzz_add_quad<F>(acc, o);
    }
    if (gl == 0 && sb && (threadIdx.x & 3) == 0) store_xyzz(buckets + b, acc);
}

// ---------------------------------------------------------------------------------------------- bucket reduction
// sum_b (b+1) * B[b] = sum_t 2^t * T_t,  T_t = sum of B[b] over the b with bit t of (b+1) set.
// grid (blocks_per_bit, c, G); every CTA tree-sums its slice of one group's buckets for one bit.
constexpr unsigned TREE_THREADS = 256;              // 64 quads per CTA in the reduction kernels
constexpr unsigned TREE_QUADS = TREE_THREADS / 4;

// GIANT_SLICES CTAs per giant bucket: each sums a contiguous slice of the bucket's partial list (quads stride over it, then
// the block tree, quad.cuh); the last CTA to arrive (ticket counter) adds the slice sums and writes the bucket.
constexpr unsigned GIANT_SLICES = 16;
template <class F>
__global__ void __launch_bounds__(TREE_THREADS) k_giant_finish(const uint32_t* __restrict__ giants, const uint32_t* __restrict__ meta,
                                                               const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ task_off, uint32_t K,
                                                               xyzz_t* buckets, const xyzz_t* __restrict__ partials, xyzz_t* slice_sums,
                                                               uint32_t* tickets) {
    extern __shared__ xyzz_t sm_tree[];
    __shared__ uint32_t ticket_s;
    const uint32_t ng = meta[2];
    if (ng > MSM_MAX_GIANTS || blockIdx.x >= ng) return;  // overflow: k_bucket_finish took them
    const uint32_t b = giants[blockIdx.x];
    const uint32_t nbk = offsets[b + 1] - offsets[b], sb = (nbk + K - 1) / K, t0 = task_off[b];
    const uint32_t per = (sb + GIANT_SLICES - 1) / GIANT_SLICES;
    const uint32_t j_lo = blockIdx.y * per, j_hi = min(sb, j_lo + per);
    const unsigned qd = threadIdx.x >> 2, nq = blockDim.x >> 2;
    xyzz_t acc = xyzz_identity();
    for (uint32_t j0 = j_lo; j0 < j_hi; j0 += nq) {
        xyzz_t o = j0 + qd < j_hi ? load_xyzz(partials + t0 + j0 + qd) : xyzz_identity();
        acc = xyzz_add_quad<F>(acc, o);
    }
    acc = block_tree_sum_quad<F>(acc, sm_tree);
    xyzz_t* mine = slice_sums + (size_t)blockIdx.x * GIANT_SLICES;
    if (threadIdx.x == 0) {
        store_xyzz(mine + blockIdx.y, acc);
        __threadfence();
        ticket_s = atomicAdd(&tickets[blockIdx.x], 1u);
    }
    __syncthreads();
    if (ticket_s != GIANT_SLICES - 1) return;
    __threadfence();
    acc = qd < GIANT_SLICES ? load_xyzz(mine + qd) : xyzz_identity();
    acc = block_tree_sum_quad<F>(acc, sm_tree);
    if (threadIdx.x == 0) { store_xyzz(buckets + b, acc); tickets[blockIdx.x] = 0; }
}

// Two-level form of the same reduction (fewer additions, shorter dependency chains).  Split i = hi * W + lo, W = 2^w_lo:
//     sum_i i * B[i] = W * sum_hi hi * R[hi] + sum_lo lo * C[lo],   R[hi] = sum_lo B[hi W + lo],  C[lo] = sum_hi B[hi W + lo]
// k_gridsum: one CTA per row and per column of the (B/W + 1) x W bucket grid (row B/W holds the single bucket i = B);
// k_gridsum_final: one CTA per output bit: T_t = sum of C[lo] over bit t of lo (t < w_lo), of R[hi] over bit t - w_lo of hi
// (t >= w_lo).  Output layout and meaning are those of k_bitsum_final: c points per group, the MSM is sum_t 2^t T_t.
// About 2 B additions per group instead of (c - 1) B / 2.
template <class F>
__global__ void __launch_bounds__(128, 3) k_gridsum(const xyzz_t* __restrict__ buckets, uint32_t B, unsigned w_lo, xyzz_t* rc) {
    extern __shared__ xyzz_t sm_tree[];
    const uint32_t W = 1u << w_lo, nrows = (B >> w_lo) + 1;
    const unsigned g = blockIdx.z;
    const xyzz_t* bk = buckets + (size_t)g * B;
    const unsigned qd = threadIdx.x >> 2, nq = blockDim.x >> 2;
    const bool row = blockIdx.x < nrows;
    // a column holds B / W buckets — rows 0 .. B/W - 1, except column 0: rows 1 .. B/W (bucket 0 does not exist, bucket B closes
    // it) — so B / W trips cover every column: a power of two, no trip spent on the odd last row
    const uint32_t fixed = row ? blockIdx.x : blockIdx.x - nrows, count = row ? W : nrows - 1;
    const uint32_t shift = (!row && fixed == 0) ? 1u : 0u;
    xyzz_t acc = xyzz_identity();
    // The next trip's bucket is in flight while the current one is added (the additions are a dependent chain).  Each lane of the
    // quad fetches ONE coordinate (32 B) ahead — 8 registers instead of 32 — and the quad reassembles the point with shuffles.
    const unsigned lane = threadIdx.x & 31, base = lane & ~3u, coord = lane & 3;
    auto fetch = [&](uint32_t e) {
        fe part = fe_zero();
        if (e < count) {
            const uint32_t i = row ? fixed * W + e : (e + shift) * W + fixed;
            if (i >= 1 && i <= B) part = load_fe(reinterpret_cast<const fe*>(bk + (i - 1)) + coord);
        }
        return part;
    };
    fe nxt = fetch(qd);
    for (uint32_t e0 = 0; e0 < count; e0 += nq) {
        xyzz_t o;
        o.X = shfl_fe(nxt, base); o.Y = shfl_fe(nxt, base + 1); o.ZZ = shfl_fe(nxt, base + 2); o.ZZZ = shfl_fe(nxt, base + 3);
        if (e0 + nq < count) nxt = fetch(e0 + nq + qd);
        acc = xyzz_add_quad<F>(acc, o);
    }
    acc = block_tree_sum_quad<F>(acc, sm_tree);
    if (threadIdx.x == 0) store_xyzz(rc + (size_t)g * (nrows + W) + blockIdx.x, acc);
}

template <class F>
__global__ void __launch_bounds__(TREE_THREADS) k_gridsum_final(const xyzz_t* __restrict__ rc, uint32_t B, unsigned w_lo, unsigned c, xyzz_t* out) {
    extern __shared__ xyzz_t sm_tree[];
    const uint32_t W = 1u << w_lo, nrows = (B >> w_lo) + 1;
    const unsigned t = blockIdx.x, g = blockIdx.y;
    const bool cols = t < w_lo;
    const xyzz_t* src = rc + (size_t)g * (nrows + W) + (cols ? nrows : 0);
    const uint32_t count = cols ? W : nrows;
    const unsigned bit = cols ? t : t - w_lo;
    const unsigned qd = threadIdx.x >> 2, nq = blockDim.x >> 2;
    xyzz_t acc = xyzz_identity();
    // the j-th index with `bit` set: e = (j >> bit) << (bit + 1) | 1 << bit | (j & (2^bit - 1))
    for (uint32_t j0 = 0;; j0 += nq) {
        const uint32_t first = ((j0 >> bit) << (bit + 1)) | (1u << bit) | (j0 & ((1u << bit) - 1));
        if (first >= count) break;     // uniform over the block
        const uint32_t j = j0 + qd, e = ((j >> bit) << (bit + 1)) | (1u << bit) | (j & ((1u << bit) - 1));
        xyzz_t o = e < count ? load_xyzz(src + e) : xyzz_identity();
        acc = xyzz_add_quad<F>(acc, o);
    }
    acc = block_tree_sum_quad<F>(acc, sm_tree);
    if (threadIdx.x == 0) store_xyzz(out + (size_t)g * c + t, acc);
}

// ---------------------------------------------------------------------------------------------- pipeline
static unsigned pow2_ceil_log(uint64_t x) {
    unsigned l = 0;
    while (((uint64_t)1 << l) < x) l++;
    return l;
}

template <class F, class FS>
int msm_run(const MsmBases& b, const size_t* offs, size_t n_main, const fe* const* d_scalars, unsigned k, bool scalars_mont, unsigned c,
            const affine_t* d_extra, size_t n_extra, const MsmTuning& tune, int sm_count, bool profile, MsmWorkspace& ws, cudaStream_t st,
            xyzz_t* d_out, size_t out_cap, MsmResultShape* shape, unsigned* launches) {
    const size_t n = n_main + n_extra;                // scalars per MSM
    if (n_extra && !d_extra) { zk_set_error("msm: extra points missing"); return ZK_ERR_INVALID; }
    for (unsigned j = 0; j < k && j < MSM_MAX_BATCH; j++)
        if (offs[j] > b.n || n_main > b.n - offs[j]) { zk_set_error("msm: slice [%zu, %zu) outside the %zu resident bases", offs[j], offs[j] + n_main, b.n); return ZK_ERR_INVALID; }
    if (k == 0 || k > MSM_MAX_BATCH) { zk_set_error("msm: batch of %u outside [1, %u]", k, MSM_MAX_BATCH); return ZK_ERR_INVALID; }
    shape->c = 0; shape->groups = 0;
    if (n == 0) return ZK_OK;
    const bool use_table = b.c != 0;
    if (use_table) c = b.c;
    else if (c == 0) c = (unsigned)msm_default_window(n, false);
    if (c < 2 || c > MSM_MAX_WINDOW_BITS) { zk_set_error("msm: window bits %u outside [2, %u]", c, MSM_MAX_WINDOW_BITS); return ZK_ERR_INVALID; }
    const unsigned nwin = msm_num_windows(c);
    const unsigned gpm = use_table ? 1 : nwin;        // bucket groups per MSM
    const unsigned G = k * gpm;                       // bucket groups of the batch
    if (d_out && (size_t)G * c > out_cap) { zk_set_error("msm: %u slice sums do not fit the caller's buffer of %zu points", G * c, out_cap); return ZK_ERR_INVALID; }
    const uint32_t B = 1u << (c - 1);                 // buckets per group
    const size_t NB = (size_t)G * B;
    const size_t Mmax = n * nwin * (size_t)k;
    const size_t main_count = b.n * (size_t)std::max(1u, b.nwin);   // table entries; the extra points' rows are addressed behind them
    if (Mmax >= 0x7fffffffull || NB >= 0x7fffffffull || main_count + n_extra * nwin >= 0x7fffffffull) {
        zk_set_error("msm: %zu x %u x %u entries exceed the 31-bit index space", n, nwin, k);
        return ZK_ERR_INVALID;
    }
    // Entries per accumulation task: the accumulate kernel keeps `capacity` threads resident (4 CTAs of 128 per SM at
    // <= 128 registers); K is chosen so that the tasks fill a whole number of waves (a 1.02-wave grid costs two waves).
    // Short tasks keep the lanes of a warp balanced (a bucket of n_b entries is cut into ceil(n_b / K) equal parts: lengths lie
    // in (K s / (s + 1), K]): one wave of long tasks is slower than two waves of short ones for the same additions.
    const size_t capacity = (size_t)sm_count * (tune.wave_threads ? tune.wave_threads : 512);
    const size_t resident_quads = (size_t)sm_count * TREE_QUADS;
    const bool many_buckets = NB > resident_quads;    // many small buckets: throughput regime (see k_bucket_finish_serial)
    const bool serial_finish = many_buckets;
    uint32_t K = tune.chunk;
    if (K == 0) {
        // (1) lane balance: a bucket of n_b entries is cut into ceil(n_b / K) equal tasks, so task lengths lie in (K s / (s + 1), K];
        //     with s >= 8 tasks per average bucket the lanes of a warp differ by ~10%, whatever the batch size;
        // (2) small inputs: never fewer tasks than threads the machine holds at once.
        const size_t n_avg = std::max<size_t>(1, Mmax / NB);
        // (K >= 6 rather than 4: fewer partials for the finish pass; tools/msm_tune.py times the choices)
        size_t k_bal = many_buckets ? std::min<size_t>(64, std::max<size_t>(6, n_avg / 8)) : 64;
        const size_t slack = std::min<size_t>(NB / 2, capacity / 4);     // sum_b ceil(n_b/K) ~ M/K + (non-empty buckets)/2
        const size_t k_cap = std::max<size_t>(4, (Mmax + capacity - slack - 1) / (capacity - slack));
        K = (uint32_t)std::min(k_bal, k_cap);
    }
    const size_t NTmax = Mmax / K + NB + 1;           // sum_b ceil(n_b / K) <= M / K + (number of non-empty buckets)
    // lanes per bucket in the finish pass: ~a quarter of the expected partials per bucket
    const uint64_t s_avg = Mmax / ((uint64_t)K * NB) + 1;
    unsigned log_g = pow2_ceil_log((s_avg + 7) / 8);   // quads per bucket in the finish pass
    if (log_g > 3) log_g = 3;
    const uint32_t smax = 32u << log_g;               // more partials than this: the bucket is "giant"
    const uint32_t run = 4;                           // k_run_sum: consecutive partials summed per thread
    const unsigned w_lo = (c - 1) / 2;
    const uint32_t W = 1u << w_lo, nrows = (B >> w_lo) + 1;
    const size_t ntiles = (NB + PLAN_TILE - 1) / PLAN_TILE;

    static_assert(sizeof(xyzz_t) == 128 && sizeof(affine_t) == 64 && sizeof(fe) == 32, "layout");
    // scratch, grouped by what sizes it (MsmWorkspace)
    Layout le, lb, lf;
    const size_t o_digits = le.add(Mmax * sizeof(int32_t)), o_entries = le.add(Mmax * sizeof(uint32_t));
    const size_t o_counts = lb.add(NB * sizeof(uint32_t)), o_offsets = lb.add((NB + 1) * sizeof(uint32_t)),
                 o_task_off = lb.add((NB + 1) * sizeof(uint32_t)), o_buckets = lb.add(NB * sizeof(xyzz_t)), o_chain = lb.add(ntiles * sizeof(uint64_t));
    const size_t o_meta = lf.add(8 * sizeof(uint32_t)), o_giants = lf.add(MSM_MAX_GIANTS * sizeof(uint32_t)),
                 o_slices = lf.add((size_t)MSM_MAX_GIANTS * GIANT_SLICES * sizeof(xyzz_t)), o_tickets = lf.add(MSM_MAX_GIANTS * sizeof(uint32_t));
    if (int rc = ws.entries.ensure(le.total)) return rc;
    if (int rc = ws.partials.ensure(NTmax * sizeof(xyzz_t))) return rc;
    if (int rc = ws.buckets.ensure(lb.total)) return rc;
    const size_t flags_had = ws.chain_flags.cap;
    if (int rc = ws.chain_flags.ensure(ntiles * sizeof(uint32_t))) return rc;
    if (ws.chain_flags.cap != flags_had) {            // new flags: no stamps yet
        ZK_CUDA(cudaMemsetAsync(ws.chain_flags.p, 0, ntiles * sizeof(uint32_t), st));
        ws.epoch = 0;
    }
    if (int rc = ws.bitsums.ensure(((size_t)G * (nrows + W) + (size_t)G * c) * sizeof(xyzz_t))) return rc;
    if (!ws.fixed.p) {
        if (int rc = ws.fixed.ensure(lf.total)) return rc;
        ZK_CUDA(cudaMemsetAsync(ws.fixed.at<uint32_t>(o_tickets), 0, MSM_MAX_GIANTS * sizeof(uint32_t), st));
    }
    if (!d_out)
        if (int rc = ws.h_bitsums.ensure((size_t)G * c * sizeof(xyzz_t))) return rc;   // sized by G*c alone: few wide groups and many narrow ones differ
    int32_t* d_digits = ws.entries.at<int32_t>(o_digits);
    uint32_t* d_entries = ws.entries.at<uint32_t>(o_entries);
    xyzz_t* d_partials = ws.partials.at<xyzz_t>();
    uint32_t *d_counts = ws.buckets.at<uint32_t>(o_counts), *d_offsets = ws.buckets.at<uint32_t>(o_offsets), *d_task_off = ws.buckets.at<uint32_t>(o_task_off);
    xyzz_t* d_buckets = ws.buckets.at<xyzz_t>(o_buckets);
    uint64_t* d_chain = ws.buckets.at<uint64_t>(o_chain);
    uint32_t *d_meta = ws.fixed.at<uint32_t>(o_meta), *d_giants = ws.fixed.at<uint32_t>(o_giants), *d_giant_tickets = ws.fixed.at<uint32_t>(o_tickets);
    xyzz_t* d_giant_slices = ws.fixed.at<xyzz_t>(o_slices);
    unsigned nl = 0;
    if (profile)
        for (Event& ev : ws.ev) ZK_CUDA(ev.create(cudaEventDefault));
#define STAGE_MARK(s) do { if (profile) ZK_CUDA(cudaEventRecord(ws.ev[s].e, st)); } while (0)

    MsmScalarSet sc{};
    for (unsigned j = 0; j < k; j++) { sc.p[j] = d_scalars[j]; sc.off[j] = (uint32_t)offs[j]; }
    const uint32_t epoch = ++ws.epoch;
    ZK_CUDA(cudaMemsetAsync(d_counts, 0, NB * sizeof(uint32_t), st));
    ZK_CUDA(cudaMemsetAsync(d_buckets, 0, NB * sizeof(xyzz_t), st));  // all-zero XYZZ == identity
    STAGE_MARK(0);
    // 1. digits + histogram
    k_recode<FS><<<dim3((unsigned)((n + 127) / 128), k), 128, 0, st>>>(sc, scalars_mont ? 1 : 0, n, c, nwin, gpm, use_table ? 0 : 1, d_digits,
                                                                        d_counts, d_meta);
    STAGE_MARK(1);
    // 2. plan: bucket offsets, task offsets, giant list
    k_plan<<<(unsigned)ntiles, 1024, 0, st>>>(d_counts, d_offsets, d_task_off, (uint32_t)NB, K, smax, d_meta, d_giants, d_chain,
                                               ws.chain_flags.at<uint32_t>(), epoch);
    STAGE_MARK(2);
    // 3. scatter (counting sort by bucket)
    k_scatter<<<(unsigned)((Mmax + 255) / 256), 256, 0, st>>>(d_digits, n, c, nwin, k, gpm, use_table ? 0 : 1, sc, b.n, use_table ? 1 : 0,
                                                            n_main, n_extra, (uint32_t)main_count, d_offsets, d_counts, d_entries);
    STAGE_MARK(3);
    // 4. accumulation: one task per <= K sorted entries of one bucket
    k_accumulate<F><<<(unsigned)((NTmax + 127) / 128), 128, 0, st>>>(b.d_points, d_entries, d_offsets, d_task_off, (uint32_t)NB, K, d_meta,
                                                                   d_extra, (uint32_t)main_count, d_buckets, d_partials);
    STAGE_MARK(4);
    // 5. per-bucket sums of the task partials (+ giants)
    // giants first: k_giant_finish reads the untouched partial lists, k_run_sum then rewrites partials in place
    k_giant_finish<F><<<dim3(64, GIANT_SLICES), TREE_THREADS, TREE_QUADS * sizeof(xyzz_t), st>>>(
        d_giants, d_meta, d_offsets, d_task_off, K, d_buckets, d_partials, d_giant_slices, d_giant_tickets);
    if (serial_finish) {
        const size_t threads = (NTmax + run - 1) / run;
        k_run_sum<F><<<(unsigned)((threads + 127) / 128), 128, 0, st>>>(d_task_off, (uint32_t)NB, d_meta, run, smax, d_partials);
        nl += 1;
        k_bucket_finish_serial<F><<<(unsigned)((NB + 127) / 128), 128, 0, st>>>(d_offsets, d_task_off, (uint32_t)NB, K, smax, d_meta, run, d_buckets, d_partials);
    } else {
        k_bucket_finish<F><<<(unsigned)(((NB << (log_g + 2)) + 127) / 128), 128, 0, st>>>(d_offsets, d_task_off, (uint32_t)NB, K, smax, log_g, d_meta,
                                                                                  d_buckets, d_partials);
    }
    STAGE_MARK(5);
    // 6. two-level bucket reduction: row / column sums of the bucket grid, then their bit slices
    xyzz_t* d_rc = ws.bitsums.at<xyzz_t>();
    xyzz_t* d_T = d_rc + (size_t)G * (nrows + W);
    {
        // a quad per 1-4 elements of a row / column, but never more CTAs x threads than are resident at once (384 threads per
        // SM at the kernel's register budget), so that the whole grid of a single MSM — 385 CTAs at window 16 — runs as one wave
        unsigned gt = 128;                          // k_gridsum is built for 3 CTAs of 128 threads per SM (<= 168 registers)
        while (gt > 32 && (gt / 4 >= 2 * std::max(W, nrows) || (size_t)G * (nrows + W) * gt > (size_t)sm_count * 384)) gt /= 2;
        k_gridsum<F><<<dim3(nrows + W, 1, G), gt, (gt / 4) * sizeof(xyzz_t), st>>>(d_buckets, B, w_lo, d_rc);
        unsigned ft = TREE_THREADS;                 // half of the elements carry a given bit
        while (ft > 32 && ft / 4 >= std::max(W, nrows)) ft /= 2;
        k_gridsum_final<F><<<dim3(c, G), ft, (ft / 4) * sizeof(xyzz_t), st>>>(d_rc, B, w_lo, c, d_T);
    }
    nl += 8;
    STAGE_MARK(6);
#undef STAGE_MARK
    ZK_CUDA(cudaGetLastError());
    shape->c = c; shape->groups = gpm;
    if (launches) *launches += nl;
    if (d_out) {
        ZK_CUDA(cudaMemcpyAsync(d_out, d_T, (size_t)G * c * sizeof(xyzz_t), cudaMemcpyDeviceToDevice, st));
        return ZK_OK;
    }
    ZK_CUDA(cudaMemcpyAsync(ws.h_bitsums.p, d_T, (size_t)G * c * sizeof(xyzz_t), cudaMemcpyDeviceToHost, st));
    ZK_CUDA(cudaStreamSynchronize(st));
    if (profile)
        for (int s = 0; s < MSM_ST_COUNT; s++) ZK_CUDA(cudaEventElapsedTime(&ws.stage_ms[s], ws.ev[s].e, ws.ev[s + 1].e));
    // the O(c) serial tail (c doublings per group) is finished on the host from ws.h_bitsums (api.cu: msm_finish_t)
    return ZK_OK;
}

// one warp per output point: its 8 quads stride over the ranks, then a shuffle tree
template <class F> __global__ void __launch_bounds__(32) k_sum_partials(const xyzz_t* __restrict__ all, uint32_t world, uint32_t count, xyzz_t* out) {
    const unsigned i = blockIdx.x, qd = threadIdx.x >> 2;
    xyzz_t acc = xyzz_identity();
    for (uint32_t r0 = 0; r0 < world; r0 += 8) {
        const uint32_t r = r0 + qd;
        xyzz_t o = r < world ? load_xyzz(all + (size_t)r * count + i) : xyzz_identity();
        acc = xyzz_add_quad<F>(acc, o);
    }
#pragma unroll 1
    for (unsigned d = 4; d >= 1; d >>= 1) {
        xyzz_t o = shfl_down_xyzz(acc, 4 * d);
        if (qd >= d) o = xyzz_identity();
        acc = xyzz_add_quad<F>(acc, o);
    }
    if (threadIdx.x == 0) store_xyzz(out + i, acc);
}
template <class F> int msm_sum_partials(const xyzz_t* d_all, size_t world, size_t count, xyzz_t* d_out, cudaStream_t st) {
    if (count) k_sum_partials<F><<<(unsigned)count, 32, 0, st>>>(d_all, (uint32_t)world, (uint32_t)count, d_out);
    ZK_CUDA(cudaGetLastError());
    return ZK_OK;
}
template int msm_sum_partials<FpParams>(const xyzz_t*, size_t, size_t, xyzz_t*, cudaStream_t);
template int msm_sum_partials<FqParams>(const xyzz_t*, size_t, size_t, xyzz_t*, cudaStream_t);

#define INST(F, FS)                                                                                                             \
    template int msm_bases_create<F>(MsmBases&, const affine_t*, bool, size_t, unsigned, cudaStream_t);                          \
    template int msm_run<F, FS>(const MsmBases&, const size_t*, size_t, const fe* const*, unsigned, bool, unsigned, const affine_t*, size_t,          \
                                const MsmTuning&, int, bool, MsmWorkspace&, cudaStream_t, xyzz_t*, size_t, MsmResultShape*, unsigned*);
INST(FpParams, FqParams)  // Pallas: coordinates Fp, scalars Fq
INST(FqParams, FpParams)  // Vesta:  coordinates Fq, scalars Fp
#undef INST

}  // namespace zkb
