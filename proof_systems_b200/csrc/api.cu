// api.cu — the extern "C" boundary (include/zkb200.h): contexts, resident bases, MSM, NTT, diagnostics.
#include <cstdarg>
#include <cstring>
#include <map>
#include <mutex>
#include <vector>

#include "../../include/zkb200.h"
#include "ctx.hpp"
#include "msm.cuh"
#include "ntt.cuh"
#include "quad.cuh"

namespace zkb {

template <class F> int points_decompress(const uint8_t* d_in, affine_t* d_out, size_t n, unsigned* d_bad, cudaStream_t st);   // decompress.cu
template <class F> int points_from_uncompressed(const uint8_t* d_in, affine_t* d_out, size_t n, unsigned* d_bad, cudaStream_t st);
template <class F> int points_compress(const affine_t* d_in, uint8_t* d_out, size_t n, cudaStream_t st);
template <class F> int points_synthetic(affine_t* d_out, size_t n, uint64_t seed, cudaStream_t st);

static thread_local char g_err[512] = "";
void zk_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
}

// ---------------------------------------------------------------------------------------------- host tail of the MSM
template <class HP> static host::hxyzz msm_finish_t(const xyzz_t* T, unsigned c, unsigned G) {
    using namespace host;
    static_assert(sizeof(hxyzz) == sizeof(xyzz_t), "layout");
    hxyzz total = identity();
    for (int g = (int)G - 1; g >= 0; g--) {
        if (g != (int)G - 1)
            for (unsigned k = 0; k < c; k++) total = pdbl<HP>(total);
        hxyzz acc = identity();
        for (int t = (int)c - 1; t >= 0; t--) {
            hxyzz tt;
            memcpy(&tt, T + (size_t)g * c + t, sizeof tt);
            acc = padd<HP>(pdbl<HP>(acc), tt);
        }
        total = padd<HP>(total, acc);
    }
    return total;
}

static void xyzz_to_jac_out(int curve, const host::hxyzz& p, uint64_t out[12]) {
    const host::hjac j = with_curve(curve, [&](auto c) { return host::to_jacobian<typename decltype(c)::HP>(p); });
    memcpy(out, &j, sizeof j);
}

int ctx_msm_many(zk_ctx* ctx, const zk_bases* bases, size_t off, size_t n, const fe* const* d_scalars, size_t k, int mont, int window_bits,
                 uint64_t* out_xyz, const affine_t* d_extra, size_t n_extra) {
    std::vector<size_t> offs(k, off);
    return ctx_msm_many_offs(ctx, bases, offs.data(), n, d_scalars, k, mont, window_bits, out_xyz, d_extra, n_extra);
}

int ctx_msm_many_offs(zk_ctx* ctx, const zk_bases* bases, const size_t* offs, size_t n, const fe* const* d_scalars, size_t k, int mont, int window_bits,
                      uint64_t* out_xyz, const affine_t* d_extra, size_t n_extra) {
    if (window_bits < 0 || window_bits > (int)MSM_MAX_WINDOW_BITS) { zk_set_error("msm: window_bits %d outside [0, %u]", window_bits, MSM_MAX_WINDOW_BITS); return ZK_ERR_INVALID; }
    // MSMs per pipeline: the context's limit, and no more than keeps the sorted entry list below 2^28 entries (1 GiB of scratch)
    const unsigned c_eff = bases->b.c ? bases->b.c : (window_bits ? (unsigned)window_bits : (unsigned)msm_default_window(n, false));
    const size_t per_msm = std::max<size_t>(1, (n + n_extra) * msm_num_windows(std::max(2u, c_eff)));
    size_t fuse = std::min<size_t>((size_t)std::max(1, ctx->msm.batch), std::max<size_t>(1, ((size_t)1 << 28) / per_msm));
    if (ctx->profile) fuse = 1;   // stage times are those of ONE MSM (zk_ctx_last_stage_ms)
    for (size_t j0 = 0; j0 < k; j0 += fuse) {
        const unsigned cnt = (unsigned)std::min(fuse, k - j0);
        MsmResultShape shape;
        unsigned nl = 0;
        const int rc = with_curve(bases->b.curve, [&](auto c) {
            using C = decltype(c);
            if (int e = msm_run<typename C::F, typename C::FS>(bases->b, offs + j0, n, d_scalars + j0, cnt, mont != 0, (unsigned)window_bits, d_extra,
                                                               n_extra, ctx->msm, ctx->sm_count, ctx->profile, ctx->ws, ctx->stream, nullptr, 0,
                                                               &shape, &nl))
                return e;
            ctx->launches += nl;
            for (unsigned j = 0; j < cnt; j++) {
                host::hxyzz r = host::identity();
                if (shape.groups) r = msm_finish_t<typename C::HP>(ctx->ws.h_bitsums.at<xyzz_t>() + (size_t)j * shape.groups * shape.c, shape.c, shape.groups);
                xyzz_to_jac_out(bases->b.curve, r, out_xyz + 12 * (j0 + j));
            }
            return ZK_OK;
        });
        if (rc) return rc;
    }
    return ZK_OK;
}

int ctx_msm_device(zk_ctx* ctx, const zk_bases* bases, size_t off, size_t n, const fe* d_scalars, int mont, int window_bits,
                   uint64_t out_xyz[12]) {
    return ctx_msm_many(ctx, bases, off, n, &d_scalars, 1, mont, window_bits, out_xyz);
}

// The `count` scalars of a call where the recode kernel reads them.  Page-locked host memory (cudaHostAlloc / cudaHostRegister) is
// read in place over PCIe (unified addressing): no staging copy, the transfer is fused into the first kernel.  Device or managed
// memory is read in place when `device_ok`.  Anything else is staged in ctx->d_scalars.
static int msm_scalars_on_device(zk_ctx* ctx, const void* scalars, size_t count, bool device_ok, const fe** out) {
    cudaPointerAttributes attr;
    const bool known = cudaPointerGetAttributes(&attr, scalars) == cudaSuccess;
    if (!known) cudaGetLastError();   // clear the "invalid value" some drivers report for pageable pointers
    if (known && attr.type == cudaMemoryTypeHost && attr.devicePointer) {
        *out = (const fe*)attr.devicePointer;
    } else if (known && device_ok && (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged)) {
        *out = (const fe*)scalars;
    } else {
        if (int rc = ctx->d_scalars.ensure(std::max<size_t>(count, 1) * sizeof(fe))) return rc;
        *out = ctx->d_scalars.at<fe>();
        if (count) ZK_CUDA(cudaMemcpyAsync(ctx->d_scalars.p, scalars, count * sizeof(fe), cudaMemcpyHostToDevice, ctx->stream));
    }
    return ZK_OK;
}

// Multi-GPU sharding (SURVEY.md §8e): this rank's MSM is left on the device as its slice sums and nothing is synchronised, so
// the caller can enqueue the all-gather on the same stream while the kernels still run.
int ctx_msm_partial(zk_ctx* ctx, const zk_bases* bases, size_t off, size_t n, const void* scalars, int scalars_are_mont, int window_bits,
                    void* d_out, size_t capacity_points, unsigned* out_c, unsigned* out_groups) {
    if (!ctx || !bases || !d_out || !out_c || !out_groups || (!scalars && n)) { zk_set_error("msm_partial: null argument"); return ZK_ERR_INVALID; }
    if (ctx_root(bases->ctx) != ctx_root(ctx)) { zk_set_error("msm: bases belong to another context"); return ZK_ERR_INVALID; }
    if (window_bits < 0 || window_bits > (int)MSM_MAX_WINDOW_BITS) { zk_set_error("msm: window_bits %d outside [0, %u]", window_bits, MSM_MAX_WINDOW_BITS); return ZK_ERR_INVALID; }
    if (n == 0) { zk_set_error("msm_partial: empty slice"); return ZK_ERR_INVALID; }
    const fe* d_sc = nullptr;
    if (int rc = msm_scalars_on_device(ctx, scalars, n, true, &d_sc)) return rc;
    MsmResultShape shape;
    unsigned nl = 0;
    int rc = with_curve(bases->b.curve, [&](auto c) {
        using C = decltype(c);
        return msm_run<typename C::F, typename C::FS>(bases->b, &off, n, &d_sc, 1, scalars_are_mont != 0, (unsigned)window_bits, nullptr, 0, ctx->msm,
                                                      ctx->sm_count, ctx->profile, ctx->ws, ctx->stream, (xyzz_t*)d_out, capacity_points, &shape, &nl);
    });
    ctx->launches += nl;
    if (rc) return rc;
    *out_c = shape.c;
    *out_groups = shape.groups;
    return ZK_OK;
}

// d_all: `world` gathered partials of zk_msm_partial (device, world x groups*c points, same shape on every rank).  Sums them
// per slice on the device, copies groups*c points to the host and finishes the O(c) tail there.
int ctx_msm_finish_gathered(zk_ctx* ctx, int curve_id, const void* d_all, size_t world, unsigned c, unsigned groups, uint64_t out_xyz[12]) {
    if (!ctx || !d_all || !out_xyz || world == 0) { zk_set_error("msm_finish_gathered: null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_curve("msm_finish_gathered", curve_id)) return rc;
    const size_t count = (size_t)c * groups;
    if (count == 0 || count > 4096) { zk_set_error("msm_finish_gathered: bad shape c = %u, groups = %u", c, groups); return ZK_ERR_INVALID; }
    if (int rc = ctx->d_gather_sum.ensure(count * sizeof(xyzz_t))) return rc;
    if (int rc = ctx->h_gather.ensure(count * sizeof(xyzz_t))) return rc;
    xyzz_t *d_sum = ctx->d_gather_sum.at<xyzz_t>(), *h_sum = ctx->h_gather.at<xyzz_t>();
    return with_curve(curve_id, [&](auto cv) {
        using C = decltype(cv);
        if (int e = msm_sum_partials<typename C::F>((const xyzz_t*)d_all, world, count, d_sum, ctx->stream)) return e;
        ctx->launches += 1;
        ZK_CUDA(cudaMemcpyAsync(h_sum, d_sum, count * sizeof(xyzz_t), cudaMemcpyDeviceToHost, ctx->stream));
        ZK_CUDA(cudaStreamSynchronize(ctx->stream));
        xyzz_to_jac_out(curve_id, msm_finish_t<typename C::HP>(h_sum, c, groups), out_xyz);
        return ZK_OK;
    });
}

static int ctx_side_streams_init(zk_ctx* ctx) {
    for (Stream& s : ctx->side) ZK_CUDA(s.create(cudaStreamNonBlocking));
    ZK_CUDA(ctx->ev_fork.create(cudaEventDisableTiming));
    return ZK_OK;
}

// Tables are built in a local owner and enter the cache only once complete: a failed build leaves no entry behind.
static int ctx_ntt_tables(zk_ctx* lane, int field, unsigned log_n, bool inverse, const fe** small, const NttTables** tabs) {
    zk_ctx* ctx = ctx_root(lane);                      // one cache per pool; entries are immutable once built
    std::lock_guard<std::mutex> tl(ctx->tab_mu);
    DevScratch& sm = ctx->ntt_small[field][inverse ? 1 : 0];
    if (!sm.p) {
        DevScratch t;
        if (int rc = t.ensure(512 * sizeof(fe))) return rc;
        int rc = with_field(field, [&](auto f) { return ntt_build_small_table<typename decltype(f)::Dev>(t.at<fe>(), inverse, lane->stream); });
        if (rc) return rc;
        lane->launches += 2;
        sm = std::move(t);
    }
    unsigned key = (unsigned)field | (inverse ? 2u : 0u) | (log_n << 2);
    auto it = ctx->ntt_tables.find(key);
    if (it == ctx->ntt_tables.end()) {
        NttTables t;
        int rc = with_field(field, [&](auto f) { return ntt_build_tables<typename decltype(f)::Dev>(t, log_n, inverse, lane->stream); });
        if (rc) return rc;
        lane->launches += t.full.p ? 8 : 7;
        it = ctx->ntt_tables.emplace(key, std::move(t)).first;
    }
    *small = sm.at<fe>();
    *tabs = &it->second;
    return ZK_OK;
}

int ctx_ntt_table_ptrs(zk_ctx* ctx, int field, unsigned log_n, bool inverse, const fe** ulo, const fe** mid, const fe** hi2) {
    const fe* small;
    const NttTables* tabs;
    int rc = ctx_ntt_tables(ctx, field, log_n, inverse, &small, &tabs);
    if (rc) return rc;
    *ulo = tabs->ulo; *mid = tabs->mid; *hi2 = tabs->hi2;
    return ZK_OK;
}

// Transform of `batch` polynomials: polynomial b is read from d_in + b * in_bs (its first in_len elements) and written to
// d_out + b * 2^log_n; d_in == d_out (in_bs = 2^log_n) is the in-place form.
int ctx_ntt_device_oop(zk_ctx* ctx, int field, const fe* d_in, size_t in_bs, fe* d_out, unsigned log_n, size_t batch, size_t in_len, int inverse, int coset) {
    if (int rc = check_field("ntt", field)) return rc;
    if (log_n > NTT_MAX_LOG_N) { zk_set_error("ntt: log_n %u > %u not supported", log_n, NTT_MAX_LOG_N); return ZK_ERR_INVALID; }
    const fe* small;
    const NttTables* tabs;
    const NttTables* inner = nullptr;
    int rc = ctx_ntt_tables(ctx, field, log_n, inverse != 0, &small, &tabs);
    if (rc) return rc;
    if (const unsigned log_inner = ntt_inner_log(log_n)) {
        const fe* small2;
        rc = ctx_ntt_tables(ctx, field, log_inner, inverse != 0, &small2, &inner);
        if (rc) return rc;
    }
    size_t bytes = ((size_t)batch << log_n) * sizeof(fe);
    fe* tmp = nullptr;
    if (log_n > NTT_MAX_LOG_SUB) {
        rc = ctx->d_ntt_tmp.ensure(bytes);
        if (rc) return rc;
        tmp = ctx->d_ntt_tmp.at<fe>();
    }
    unsigned nl = 0;
    if (ctx->profile) {
        for (Event& ev : ctx->ev_ntt) ZK_CUDA(ev.create(cudaEventDefault));
        ZK_CUDA(cudaEventRecord(ctx->ev_ntt[0].e, ctx->stream));
    }
    rc = with_field(field, [&](auto f) {
        return ntt_run<typename decltype(f)::Dev>(d_in, in_bs, d_out, tmp, small, *tabs, inner, log_n, batch, in_len, inverse != 0, coset != 0, ctx->stream, &nl);
    });
    ctx->launches += nl;
    if (rc == ZK_OK && ctx->profile) {
        ZK_CUDA(cudaEventRecord(ctx->ev_ntt[1].e, ctx->stream));
        ZK_CUDA(cudaEventSynchronize(ctx->ev_ntt[1].e));
        ZK_CUDA(cudaEventElapsedTime(&ctx->ntt_ms, ctx->ev_ntt[0].e, ctx->ev_ntt[1].e));
    }
    return rc;
}

int ctx_ntt_device(zk_ctx* ctx, int field, fe* d_data, unsigned log_n, size_t batch, size_t in_len, int inverse, int coset) {
    return ctx_ntt_device_oop(ctx, field, d_data, (size_t)1 << (log_n > 62 ? 0 : log_n), d_data, log_n, batch, in_len, inverse, coset);
}

// ---------------------------------------------------------------------------------------------- lanes
static int ctx_init_lane(zk_ctx* c, int device_id) {
    c->device = device_id;
    cudaError_t se = c->own_stream.create(cudaStreamNonBlocking);
    if (se != cudaSuccess) { zk_set_error("cudaStreamCreate: %s", cudaGetErrorString(se)); return ZK_ERR_CUDA; }
    c->stream = c->own_stream.s;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device_id) == cudaSuccess) c->sm_count = prop.multiProcessorCount;
    return ZK_OK;
}

// host-pointer calls share the lane pool only on the own stream, unprofiled, with more than one lane (ctx->mu held)
static void ctx_update_pinned(zk_ctx* ctx) { ctx->pinned = ctx->stream != ctx->own_stream.s || ctx->profile || ctx->n_lanes <= 1; }

int ctx_acquire_lane(zk_ctx* ctx, LaneLock& out) {
    ctx = ctx_root(ctx);
    {
        // a free primary lane is taken whether or not calls are pinned to it; a busy one is waited for only when they are (a
        // blocking lock here would serialise the pool)
        std::unique_lock<std::mutex> root_lk(ctx->mu, std::try_to_lock);
        if (root_lk.owns_lock() || ctx->pinned.load()) {
            if (!root_lk.owns_lock()) root_lk.lock();
            out.lane = ctx;
            out.lk = std::move(root_lk);
            return ZK_OK;
        }
    }
    std::vector<zk_ctx*> lanes;
    unsigned start;
    {
        std::lock_guard<std::mutex> pl(ctx->pool_mu);
        while ((int)ctx->children.size() + 1 < ctx->n_lanes) {
            auto c = std::make_unique<zk_ctx>();
            c->parent = ctx;
            if (cudaSetDevice(ctx->device) != cudaSuccess || ctx_init_lane(c.get(), ctx->device) != ZK_OK) break;
            c->msm = ctx->msm;
            ctx->children.push_back(std::move(c));
        }
        lanes.push_back(ctx);
        for (auto& c : ctx->children) lanes.push_back(c.get());
        start = ctx->rr++;
    }
    // the primary lane first, then the children in order: a single-threaded caller always lands on the same (warm) lane, only
    // contention spills over; when every lane is busy the waiters spread round-robin
    for (size_t k = 0; k < lanes.size() && k < (size_t)ctx->n_lanes; k++) {
        zk_ctx* l = lanes[k];
        std::unique_lock<std::mutex> lk(l->mu, std::try_to_lock);
        if (lk.owns_lock()) { out.lane = l; out.lk = std::move(lk); return ZK_OK; }
    }
    zk_ctx* l = lanes[start % std::min<size_t>(lanes.size(), (size_t)ctx->n_lanes)];
    out.lane = l;
    out.lk = std::unique_lock<std::mutex>(l->mu);
    return ZK_OK;
}

// ---------------------------------------------------------------------------------------------- diagnostics kernels
template <class F> __global__ void k_field_op(int op, const fe* a, const fe* b, fe* out, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe x = load_fe(a + i), y = load_fe(b + i), r;
    if (op == 0) r = fe_mul<F>(x, y);
    else if (op == 1) r = fe_add<F>(x, y);
    else if (op == 2) r = fe_sub<F>(x, y);
    else r = fe_inv<F>(x);
    store_fe(out + i, r);
}
// ILP independent dependent-chains of fe_mul per thread (ILP = 1, 2, 4): latency vs throughput probe
template <class F, int ILP> __global__ void k_mul_chain(fe* out, unsigned iters) {
    fe x[ILP], y = fe_r2<F>();
    y.v[1] ^= blockIdx.x;
#pragma unroll
    for (int k = 0; k < ILP; k++) { x[k] = fe_one<F>(); x[k].v[0] ^= threadIdx.x + 977 * k; }
    for (unsigned i = 0; i < iters; i++) {
#pragma unroll
        for (int k = 0; k < ILP; k++) x[k] = fe_mul<F>(x[k], y);
    }
    uint32_t acc = 0;
#pragma unroll
    for (int k = 0; k < ILP; k++) acc ^= x[k].v[0] ^ x[k].v[7];
    if (acc == 0x12345678u) store_fe(out, x[0]);  // keep the chains alive
}
// chain of XYZZ mixed additions (the MSM inner loop) on register-resident operands
template <class F> __global__ void k_madd_chain(xyzz_t* out, unsigned iters) {
    affine_t q;
    q.x = fe_one<F>(); q.y = fe_r2<F>();
    q.x.v[0] ^= threadIdx.x; q.y.v[1] ^= blockIdx.x;
    xyzz_t acc = xyzz_from_affine<F>(q);
    acc.X.v[2] ^= 0x55u;
    for (unsigned i = 0; i < iters; i++) {
        acc = xyzz_madd<F>(acc, q);
        q.x.v[3] ^= acc.X.v[0];   // data-dependent operand so nothing is hoisted
    }
    if (acc.X.v[0] == 0x12345678u && acc.ZZ.v[7] == 0x9abcdef0u) store_xyzz(out, acc);
}

// chains of full XYZZ additions: serial formula (kind 102) and the quad-cooperative one (kind 101)
template <class F, int QUAD> __global__ void k_add_chain(xyzz_t* out, unsigned iters) {
    affine_t q;
    q.x = fe_one<F>(); q.y = fe_r2<F>();
    q.x.v[0] ^= QUAD ? (threadIdx.x >> 2) : threadIdx.x; q.y.v[1] ^= blockIdx.x;
    xyzz_t acc = xyzz_from_affine<F>(q), b = acc;
    b.X.v[2] ^= 0x55u; b.ZZ.v[1] ^= 0x3u;
    for (unsigned i = 0; i < iters; i++) {
        acc = QUAD ? xyzz_add_quad<F>(acc, b) : xyzz_add<F>(acc, b);
        b.X.v[3] ^= acc.X.v[0];
    }
    if (acc.X.v[0] == 0x12345678u && acc.ZZ.v[7] == 0x9abcdef0u) store_xyzz(out, acc);
}

}  // namespace zkb

using namespace zkb;

// ============================================================================================== extern "C"
extern "C" {

const char* zk_last_error(void) { return g_err; }

int zk_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

int zk_ctx_create(int device_id, zk_ctx** out) {
    if (!out) { zk_set_error("ctx_create: out is null"); return ZK_ERR_INVALID; }
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        zk_set_error("no CUDA device (%s): this library has no CPU fallback", e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
        return ZK_ERR_NO_DEVICE;
    }
    if (device_id < 0 || device_id >= n) { zk_set_error("ctx_create: device %d outside [0, %d)", device_id, n); return ZK_ERR_INVALID; }
    ZK_CUDA(cudaSetDevice(device_id));
    auto ctx = std::make_unique<zk_ctx>();
    if (int rc = ctx_init_lane(ctx.get(), device_id)) return rc;
    *out = ctx.release();
    return ZK_OK;
}

void zk_ctx_destroy(zk_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    delete ctx;                          // ~zk_ctx: the lanes wait for their streams, then everything they own is freed on this device
}

int zk_ctx_set_stream(zk_ctx* ctx, void* cuda_stream) {
    if (!ctx) { zk_set_error("set_stream: ctx is null"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    cudaStream_t next = cuda_stream ? (cudaStream_t)cuda_stream : ctx->own_stream.s;
    if (next == ctx->stream) return ZK_OK;
    // Several calls return with kernels still queued that read the context's scratch (the NTT's second buffer, the expression
    // program, the MSM workspace, ...).  The new stream waits for everything queued on the old one so far, without blocking the host.
    ZK_CUDA(cudaSetDevice(ctx->device));
    ZK_CUDA(ctx->ev_switch.create(cudaEventDisableTiming));
    ZK_CUDA(cudaEventRecord(ctx->ev_switch.e, ctx->stream));
    ZK_CUDA(cudaStreamWaitEvent(next, ctx->ev_switch.e, 0));
    ctx->stream = next;
    ctx_update_pinned(ctx);
    return ZK_OK;
}

uint64_t zk_ctx_launch_count(const zk_ctx* ctx) {
    if (!ctx) return 0;
    uint64_t n = ctx->launches;
    for (const auto& c : ctx->children) n += c->launches;
    return n;
}

int zk_ctx_set_profile(zk_ctx* ctx, int enabled) {
    if (!ctx) { zk_set_error("set_profile: ctx is null"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ctx->profile = enabled != 0;
    ctx_update_pinned(ctx);
    return ZK_OK;
}

int zk_ctx_set_option(zk_ctx* ctx, const char* name, long value) {
    if (!ctx || !name) { zk_set_error("set_option: null argument"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!strcmp(name, "ctx_lanes")) {
        if (value < 1 || value > 16) { zk_set_error("set_option: ctx_lanes %ld outside [1, 16]", value); return ZK_ERR_INVALID; }
        ctx->n_lanes = (int)value;       // lanes already created stay allocated; fewer are used from now on
        ctx_update_pinned(ctx);
        return ZK_OK;
    }
    if (!strcmp(name, "msm_chunk")) {
        if (value < 0 || value > 4096) { zk_set_error("set_option: msm_chunk %ld outside [0, 4096]", value); return ZK_ERR_INVALID; }
        ctx->msm.chunk = (uint32_t)value;
    } else if (!strcmp(name, "msm_batch")) {
        if (value < 1 || value > (long)MSM_MAX_BATCH) { zk_set_error("set_option: msm_batch %ld outside [1, %u]", value, MSM_MAX_BATCH); return ZK_ERR_INVALID; }
        ctx->msm.batch = (int)value;
    } else if (!strcmp(name, "msm_wave_threads")) {
        if (value < 0 || value > 2048) { zk_set_error("set_option: msm_wave_threads %ld outside [0, 2048]", value); return ZK_ERR_INVALID; }
        ctx->msm.wave_threads = (uint32_t)value;
    } else {
        zk_set_error("set_option: unknown option '%s'", name);
        return ZK_ERR_INVALID;
    }
    for (auto& c : ctx->children) c->msm = ctx->msm;
    return ZK_OK;
}

int zk_ctx_last_stage_ms(const zk_ctx* ctx, float* out, size_t capacity) {
    if (!ctx || !out || capacity < 8) { zk_set_error("last_stage_ms: need room for 8 floats"); return ZK_ERR_INVALID; }
    for (int k = 0; k < 6; k++) out[k] = ctx->ws.stage_ms[k];
    out[6] = ctx->ntt_ms;
    out[7] = 0;
    return ZK_OK;
}

// ---------------------------------------------------------------------------------------------- bases
int zk_bases_upload(zk_ctx* ctx, int curve_id, const uint64_t* xy_mont, size_t n, int window_bits, int points_on_device, zk_bases** out) {
    if (!ctx || !out || (!xy_mont && n)) { zk_set_error("bases_upload: null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_curve("bases_upload", curve_id)) return rc;
    if (window_bits < -1 || window_bits == 1 || window_bits > (int)MSM_MAX_WINDOW_BITS) { zk_set_error("bases_upload: window_bits %d not in {-1, 0, 2..%u}", window_bits, MSM_MAX_WINDOW_BITS); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    unsigned c = window_bits < 0 ? (unsigned)msm_default_window(n, true) : (unsigned)window_bits;
    auto bs = std::make_unique<zk_bases>();
    bs->ctx = ctx;
    bs->b.curve = curve_id;
    int rc = with_curve(curve_id, [&](auto cv) { return msm_bases_create<typename decltype(cv)::F>(bs->b, (const affine_t*)xy_mont, points_on_device != 0, n, c, ctx->stream); });
    if (rc) return rc;
    if (c) ctx->launches += 1;
    *out = bs.release();
    return ZK_OK;
}

void zk_bases_free(zk_bases* bases) {
    if (!bases) return;
    std::lock_guard<std::mutex> lk(bases->ctx->mu);
    cudaSetDevice(bases->ctx->device);
    delete bases;
}

size_t zk_bases_len(const zk_bases* bases) { return bases ? bases->b.n : 0; }
int zk_bases_window_bits(const zk_bases* bases) { return bases ? (int)bases->b.c : 0; }

// Point codecs between the reference's serialised forms and affine Montgomery points; host pointers.
//   mode 0: 33-byte compressed   -> affine   (decompression: one square root per point)
//   mode 1: 65-byte uncompressed -> affine   (unchecked, as SerdeAsUnchecked)
//   mode 2: affine -> 33-byte compressed
static int points_codec(zk_ctx* ctx, int curve_id, int mode, const void* in, size_t n, void* out, const char* what) {
    if (!ctx || (!in && n) || (!out && n)) { zk_set_error("%s: null argument", what); return ZK_ERR_INVALID; }
    if (int rc = check_curve(what, curve_id)) return rc;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    if (n == 0) return ZK_OK;
    const size_t in_bytes = (mode == 0 ? 33 : mode == 1 ? 65 : sizeof(affine_t)) * n, out_bytes = (mode == 2 ? 33 : sizeof(affine_t)) * n;
    DevScratch d_in, d_out, d_bad;       // transient: freed on every return
    int rc = d_in.ensure(in_bytes);
    if (rc || (rc = d_out.ensure(out_bytes)) || (rc = d_bad.ensure(sizeof(unsigned)))) return rc;
    ZK_CUDA(cudaMemsetAsync(d_bad.p, 0, sizeof(unsigned), ctx->stream));
    ZK_CUDA(cudaMemcpyAsync(d_in.p, in, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
    rc = with_curve(curve_id, [&](auto c) {
        using F = typename decltype(c)::F;
        if (mode == 0) return points_decompress<F>(d_in.at<uint8_t>(), d_out.at<affine_t>(), n, d_bad.at<unsigned>(), ctx->stream);
        if (mode == 1) return points_from_uncompressed<F>(d_in.at<uint8_t>(), d_out.at<affine_t>(), n, d_bad.at<unsigned>(), ctx->stream);
        return points_compress<F>(d_in.at<affine_t>(), d_out.at<uint8_t>(), n, ctx->stream);
    });
    if (rc) return rc;
    ctx->launches += 1;
    unsigned bad = 0;
    ZK_CUDA(cudaMemcpyAsync(out, d_out.p, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    ZK_CUDA(cudaMemcpyAsync(&bad, d_bad.p, sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    if (bad) {
        zk_set_error(mode == 0 ? "%s: %u of %zu encodings are invalid (x off the curve, x >= modulus, or unknown flag bits)" : "%s: %u of %zu points have a non-canonical coordinate", what, bad, n);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}

int zk_points_decompress(zk_ctx* ctx, int curve_id, const uint8_t* in33, size_t n, uint64_t* out_xy) {
    return points_codec(ctx, curve_id, 0, in33, n, out_xy, "points_decompress");
}
int zk_points_from_uncompressed(zk_ctx* ctx, int curve_id, const uint8_t* in65, size_t n, uint64_t* out_xy) {
    return points_codec(ctx, curve_id, 1, in65, n, out_xy, "points_from_uncompressed");
}
int zk_points_compress(zk_ctx* ctx, int curve_id, const uint64_t* xy_mont, size_t n, uint8_t* out33) {
    return points_codec(ctx, curve_id, 2, xy_mont, n, out33, "points_compress");
}

int zk_points_synthetic(zk_ctx* ctx, int curve_id, uint64_t seed, size_t n, uint64_t* out_xy) {
    if (!ctx || (!out_xy && n)) { zk_set_error("points_synthetic: null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_curve("points_synthetic", curve_id)) return rc;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    if (n == 0) return ZK_OK;
    DevScratch d;                        // transient: freed on every return
    if (int rc = d.ensure(n * sizeof(affine_t))) return rc;
    int rc = with_curve(curve_id, [&](auto c) { return points_synthetic<typename decltype(c)::F>(d.at<affine_t>(), n, seed, ctx->stream); });
    if (rc) return rc;
    ctx->launches += 1;
    ZK_CUDA(cudaMemcpyAsync(out_xy, d.p, n * sizeof(affine_t), cudaMemcpyDeviceToHost, ctx->stream));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}

// ---------------------------------------------------------------------------------------------- MSM
int zk_msm_dev(zk_ctx* ctx, const zk_bases* bases, size_t off, size_t n, const void* d_scalars, int scalars_are_mont, int window_bits, uint64_t out_xyz[12]) {
    if (!ctx || !bases || !out_xyz || (!d_scalars && n)) { zk_set_error("msm: null argument"); return ZK_ERR_INVALID; }
    if (ctx_root(bases->ctx) != ctx_root(ctx)) { zk_set_error("msm: bases belong to another context"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    return ctx_msm_device(ctx, bases, off, n, (const fe*)d_scalars, scalars_are_mont, window_bits, out_xyz);
}

int zk_msm_batch(zk_ctx* root, const zk_bases* bases, size_t off, size_t n, const uint64_t* scalars, size_t k, int scalars_are_mont, int window_bits, uint64_t* out_xyz) {
    if (!root || !bases || (!out_xyz && k) || (!scalars && n && k)) { zk_set_error("msm: null argument"); return ZK_ERR_INVALID; }
    if (ctx_root(bases->ctx) != ctx_root(root)) { zk_set_error("msm: bases belong to another context"); return ZK_ERR_INVALID; }
    LaneLock ll;                             // host pointers in, host result out: any free lane of the pool
    if (int rc = ctx_acquire_lane(root, ll)) return rc;
    zk_ctx* ctx = ll.lane;
    ZK_CUDA(cudaSetDevice(ctx->device));
    if (k == 0) return ZK_OK;
    const fe* d_sc = nullptr;
    if (int rc = msm_scalars_on_device(ctx, scalars, k * n, false, &d_sc)) return rc;
    std::vector<const fe*> scs(k);
    for (size_t j = 0; j < k; j++) scs[j] = d_sc + j * n;
    return ctx_msm_many(ctx, bases, off, n, scs.data(), k, scalars_are_mont, window_bits, out_xyz);
}

int zk_msm_partial(zk_ctx* ctx, const zk_bases* bases, size_t off, size_t n, const void* scalars, int scalars_are_mont, int window_bits,
                   void* d_out, size_t capacity_points, unsigned* out_c, unsigned* out_groups) {
    if (!ctx) { zk_set_error("msm_partial: null argument"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    return ctx_msm_partial(ctx, bases, off, n, scalars, scalars_are_mont, window_bits, d_out, capacity_points, out_c, out_groups);
}
int zk_msm_finish_gathered(zk_ctx* ctx, int curve_id, const void* d_all, size_t world, unsigned c, unsigned groups, uint64_t out_xyz[12]) {
    if (!ctx) { zk_set_error("msm_finish_gathered: null argument"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    return ctx_msm_finish_gathered(ctx, curve_id, d_all, world, c, groups, out_xyz);
}

int zk_msm(zk_ctx* ctx, const zk_bases* bases, size_t off, size_t n, const uint64_t* scalars, int scalars_are_mont, int window_bits, uint64_t out_xyz[12]) {
    return zk_msm_batch(ctx, bases, off, n, scalars, 1, scalars_are_mont, window_bits, out_xyz);
}

int zk_jacobian_to_affine(int curve_id, const uint64_t xyz[12], uint64_t out_xy[8]) {
    if (!xyz || !out_xy) { zk_set_error("null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_curve(nullptr, curve_id)) return rc;
    host::hjac j;
    memcpy(&j, xyz, sizeof j);
    const host::haffine a = with_curve(curve_id, [&](auto c) { using HP = typename decltype(c)::HP; return host::to_affine<HP>(host::from_jacobian<HP>(j)); });
    memcpy(out_xy, &a, sizeof a);
    return ZK_OK;
}

int zk_jacobian_sum(int curve_id, const uint64_t* xyz, size_t count, uint64_t out_xyz[12]) {
    if ((!xyz && count) || !out_xyz) { zk_set_error("null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_curve(nullptr, curve_id)) return rc;
    host::hxyzz acc = host::identity();
    for (size_t i = 0; i < count; i++) {
        host::hjac j;
        memcpy(&j, xyz + 12 * i, sizeof j);
        acc = with_curve(curve_id, [&](auto c) { using HP = typename decltype(c)::HP; return host::padd<HP>(acc, host::from_jacobian<HP>(j)); });
    }
    xyzz_to_jac_out(curve_id, acc, out_xyz);
    return ZK_OK;
}

int zk_jacobian_add(int curve_id, const uint64_t a_xyz[12], const uint64_t b_xyz[12], uint64_t out_xyz[12]) {
    if (!a_xyz || !b_xyz || !out_xyz) { zk_set_error("null argument"); return ZK_ERR_INVALID; }
    uint64_t both[24];
    memcpy(both, a_xyz, 96);
    memcpy(both + 12, b_xyz, 96);
    return zk_jacobian_sum(curve_id, both, 2, out_xyz);
}

// ---------------------------------------------------------------------------------------------- NTT
int zk_ntt_dev(zk_ctx* ctx, int field_id, void* d_data, unsigned log_n, size_t batch, size_t in_len, int inverse, int coset) {
    if (!ctx || (!d_data && batch)) { zk_set_error("ntt: null argument"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    return ctx_ntt_device(ctx, field_id, (fe*)d_data, log_n, batch, in_len, inverse, coset);
}

int zk_ntt_dev_oop(zk_ctx* ctx, int field_id, const void* d_in, size_t in_stride, size_t in_len, void* d_out, unsigned log_n, size_t batch, int inverse,
                   int coset) {
    if (!ctx || ((!d_in || !d_out) && batch)) { zk_set_error("ntt: null argument"); return ZK_ERR_INVALID; }
    if (log_n > NTT_MAX_LOG_N) { zk_set_error("ntt: log_n %u > %u not supported", log_n, NTT_MAX_LOG_N); return ZK_ERR_INVALID; }
    const size_t n = (size_t)1 << log_n;
    if (in_len == 0 || in_len > n) in_len = n;
    if (in_stride < in_len && batch > 1) { zk_set_error("ntt: input stride %zu shorter than the %zu elements read per polynomial", in_stride, in_len); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    return ctx_ntt_device_oop(ctx, field_id, (const fe*)d_in, in_stride, (fe*)d_out, log_n, batch, in_len, inverse, coset);
}

// ---------------------------------------------------------------------------------------------- device memory for the *_dev entry points
int zk_dev_alloc(zk_ctx* ctx, size_t bytes, void** out) {
    if (!ctx || !out) { zk_set_error("dev_alloc: null argument"); return ZK_ERR_INVALID; }
    *out = nullptr;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    ZK_CUDA(cudaMalloc(out, bytes ? bytes : 1));
    return ZK_OK;
}
int zk_dev_free(zk_ctx* ctx, void* d_ptr) {
    if (!ctx) { zk_set_error("dev_free: null argument"); return ZK_ERR_INVALID; }
    if (!d_ptr) return ZK_OK;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    ZK_CUDA(cudaFree(d_ptr));
    return ZK_OK;
}
int zk_dev_upload(zk_ctx* ctx, void* d_dst, const void* src, size_t bytes) {
    if (!ctx || ((!d_dst || !src) && bytes)) { zk_set_error("dev_upload: null argument"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    ZK_CUDA(cudaMemcpyAsync(d_dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));   // the source may be pageable and reused by the caller
    return ZK_OK;
}
int zk_dev_download(zk_ctx* ctx, void* dst, const void* d_src, size_t bytes) {
    if (!ctx || ((!dst || !d_src) && bytes)) { zk_set_error("dev_download: null argument"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    ZK_CUDA(cudaMemcpyAsync(dst, d_src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}

int zk_ntt_batch(zk_ctx* root, int field_id, uint64_t* data, unsigned log_n, size_t batch, size_t in_len, int inverse, int coset) {
    if (!root || (!data && batch)) { zk_set_error("ntt: null argument"); return ZK_ERR_INVALID; }
    if (log_n > NTT_MAX_LOG_N) { zk_set_error("ntt: log_n %u > %u not supported", log_n, NTT_MAX_LOG_N); return ZK_ERR_INVALID; }
    LaneLock ll;                             // host pointers in and out: any free lane of the pool
    if (int rc0 = ctx_acquire_lane(root, ll)) return rc0;
    zk_ctx* ctx = ll.lane;
    ZK_CUDA(cudaSetDevice(ctx->device));
    if (batch == 0) return ZK_OK;
    const size_t n = (size_t)1 << log_n, poly_bytes = n * sizeof(fe), bytes = batch * poly_bytes;
    if (in_len == 0 || in_len > n || inverse) in_len = n;
    // (Transforming page-locked memory in place over PCIe was measured and is slower than two staged copies: the tile loads
    //  are 64-128 B requests.  MSM scalars, read once in full lines, do take the zero-copy route — zk_msm_batch.)
    int rc = ctx->d_ntt.ensure(bytes);
    if (rc) return rc;
    fe* d_ntt = ctx->d_ntt.at<fe>();
    // Only the first in_len coefficients of every polynomial cross PCIe (the kernels zero-pad by position), and for batches in
    // page-locked memory the three stages are pipelined over chunks of polynomials: copy-in of chunk k+1, the transform of
    // chunk k and the copy-out of chunk k-1 run on three streams.  16 x FFT(8n) of kimchi's quotient step (in_len = n) moves
    // 32 MiB in and 256 MiB out: the call is bound by the copy-out alone instead of the sum of all three.
    cudaPointerAttributes attr;
    bool pinned = cudaPointerGetAttributes(&attr, data) == cudaSuccess && attr.type == cudaMemoryTypeHost;
    cudaGetLastError();
    size_t per = batch;                                  // polynomials per chunk
    if (pinned && !ctx->profile && batch >= 2 && bytes >= ((size_t)8 << 20)) {
        per = std::max<size_t>(1, ((size_t)16 << 20) / poly_bytes);
        if (per * 2 > batch) per = (batch + 1) / 2;
    }
    if (per == batch) {
        ZK_CUDA(cudaMemcpy2DAsync(d_ntt, poly_bytes, data, poly_bytes, in_len * sizeof(fe), batch, cudaMemcpyHostToDevice, ctx->stream));
        rc = ctx_ntt_device(ctx, field_id, d_ntt, log_n, batch, in_len, inverse, coset);
        if (rc) return rc;
        ZK_CUDA(cudaMemcpyAsync(data, d_ntt, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        ZK_CUDA(cudaStreamSynchronize(ctx->stream));
        return ZK_OK;
    }
    rc = ctx_side_streams_init(ctx);
    if (rc) return rc;
    cudaStream_t s_in = ctx->side[0].s, s_out = ctx->side[1].s;
    const size_t chunks = (batch + per - 1) / per;
    std::vector<Event> ev(2 * chunks);
    cudaError_t e = cudaEventRecord(ctx->ev_fork.e, ctx->stream);    // work already queued on the caller's stream comes first
    if (e == cudaSuccess) e = cudaStreamWaitEvent(s_in, ctx->ev_fork.e, 0);
    for (size_t k = 0; k < chunks && e == cudaSuccess && rc == ZK_OK; k++) {
        const size_t j0 = k * per, cnt = std::min(per, batch - j0);
        fe* d = d_ntt + j0 * n;
        const uint64_t* h = data + 4 * j0 * n;
        e = ev[2 * k].create(cudaEventDisableTiming);
        if (e == cudaSuccess) e = ev[2 * k + 1].create(cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaMemcpy2DAsync(d, poly_bytes, h, poly_bytes, in_len * sizeof(fe), cnt, cudaMemcpyHostToDevice, s_in);
        if (e == cudaSuccess) e = cudaEventRecord(ev[2 * k].e, s_in);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream, ev[2 * k].e, 0);
        if (e != cudaSuccess) break;
        rc = ctx_ntt_device(ctx, field_id, d, log_n, cnt, in_len, inverse, coset);
        if (rc) break;
        e = cudaEventRecord(ev[2 * k + 1].e, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(s_out, ev[2 * k + 1].e, 0);
        if (e == cudaSuccess) e = cudaMemcpyAsync((void*)h, d, cnt * poly_bytes, cudaMemcpyDeviceToHost, s_out);
    }
    cudaStreamSynchronize(s_in);
    cudaStreamSynchronize(ctx->stream);
    cudaError_t e2 = cudaStreamSynchronize(s_out);
    if (rc) return rc;
    if (e != cudaSuccess || e2 != cudaSuccess) { zk_set_error("ntt: %s", cudaGetErrorString(e != cudaSuccess ? e : e2)); return ZK_ERR_CUDA; }
    return ZK_OK;
}

int zk_ntt(zk_ctx* ctx, int field_id, uint64_t* data, unsigned log_n, int inverse, int coset) {
    return zk_ntt_batch(ctx, field_id, data, log_n, 1, 0, inverse, coset);
}

// ---------------------------------------------------------------------------------------------- diagnostics
int zk_debug_field_op(zk_ctx* ctx, int field_id, int op, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
    if (!ctx || !a || !b || !out) { zk_set_error("null argument"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    DevScratch da, db, dout;             // transient: freed on every return
    int rc = da.ensure(n * sizeof(fe));
    if (rc || (rc = db.ensure(n * sizeof(fe))) || (rc = dout.ensure(n * sizeof(fe)))) return rc;
    ZK_CUDA(cudaMemcpyAsync(da.p, a, n * sizeof(fe), cudaMemcpyHostToDevice, ctx->stream));
    ZK_CUDA(cudaMemcpyAsync(db.p, b, n * sizeof(fe), cudaMemcpyHostToDevice, ctx->stream));
    unsigned blocks = (unsigned)((n + 127) / 128);
    with_field(field_id, [&](auto f) { k_field_op<typename decltype(f)::Dev><<<blocks, 128, 0, ctx->stream>>>(op, da.at<fe>(), db.at<fe>(), dout.at<fe>(), n); });
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 1;
    ZK_CUDA(cudaMemcpyAsync(out, dout.p, n * sizeof(fe), cudaMemcpyDeviceToHost, ctx->stream));
    ZK_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZK_OK;
}

// kind: 1, 2, 4 = fe_mul chains with that many independent chains per thread; 100 = xyzz_madd chain.
// blocks == 0: 4 per SM.  Reports operations per second (fe_mul, or madd for kind 100).
int zk_debug_op_throughput(zk_ctx* ctx, int field_id, int kind, unsigned blocks, unsigned threads, unsigned iters, double* out_ops_per_s) {
    if (!ctx || !out_ops_per_s || threads == 0 || threads > 1024) { zk_set_error("op_throughput: bad argument"); return ZK_ERR_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    cudaDeviceProp prop;
    ZK_CUDA(cudaGetDeviceProperties(&prop, ctx->device));
    if (blocks == 0) blocks = prop.multiProcessorCount * 4;
    DevScratch dout;                     // transient, like the events: freed on every return
    if (int rc = dout.ensure(sizeof(xyzz_t))) return rc;
    xyzz_t* d = dout.at<xyzz_t>();
    Event e0, e1;
    ZK_CUDA(e0.create(cudaEventDefault));
    ZK_CUDA(e1.create(cudaEventDefault));
    for (int rep = 0; rep < 2; rep++) {  // first launch warms up
        ZK_CUDA(cudaEventRecord(e0.e, ctx->stream));
        with_field(field_id, [&](auto f) {
            using F = typename decltype(f)::Dev;
            if (kind == 1) k_mul_chain<F, 1><<<blocks, threads, 0, ctx->stream>>>((fe*)d, iters);
            else if (kind == 2) k_mul_chain<F, 2><<<blocks, threads, 0, ctx->stream>>>((fe*)d, iters);
            else if (kind == 4) k_mul_chain<F, 4><<<blocks, threads, 0, ctx->stream>>>((fe*)d, iters);
            else if (kind == 101) k_add_chain<F, 1><<<blocks, threads, 0, ctx->stream>>>(d, iters);
            else if (kind == 102) k_add_chain<F, 0><<<blocks, threads, 0, ctx->stream>>>(d, iters);
            else k_madd_chain<F><<<blocks, threads, 0, ctx->stream>>>(d, iters);
        });
        ZK_CUDA(cudaGetLastError());
        ZK_CUDA(cudaEventRecord(e1.e, ctx->stream));
        ZK_CUDA(cudaEventSynchronize(e1.e));
    }
    ctx->launches += 2;
    float ms = 0;
    ZK_CUDA(cudaEventElapsedTime(&ms, e0.e, e1.e));
    double per_thread = kind == 101 ? 0.25 : kind >= 100 ? 1.0 : (double)kind;
    *out_ops_per_s = per_thread * iters * (double)blocks * threads / (ms * 1e-3);
    return ZK_OK;
}

int zk_debug_mul_throughput(zk_ctx* ctx, int field_id, unsigned iters, double* out_mul_per_s) {
    return zk_debug_op_throughput(ctx, field_id, 2, 0, 256, iters, out_mul_per_s);
}

}  // extern "C"
