// ctx.hpp — the objects behind the opaque handles of include/zkb200.h, and the host-side helpers every entry point shares: the
// field_id / curve_id dispatch, the argument checks and the context's scratch memory.
#pragma once
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <vector>

#include "host_field.hpp"
#include "msm.cuh"
#include "ntt.cuh"

namespace zkb {
// a field: its device parameters (field.cuh) and its host arithmetic (host_field.hpp)
template <class D, class H, int ID> struct FieldTraits { using Dev = D; using Host = H; static constexpr int id = ID; };
using FpTraits = FieldTraits<FpParams, host::HFp, ZK_FP>;
using FqTraits = FieldTraits<FqParams, host::HFq, ZK_FQ>;

// a curve: the fields of its coordinates (F device, HP host) and of its scalars (FS, HS)
template <class B, class S> struct CurveTraits {
    using Base = B; using Scalar = S;
    using F = typename B::Dev; using HP = typename B::Host; using FS = typename S::Dev; using HS = typename S::Host;
    static constexpr int scalar_field = S::id;
};
using PallasTraits = CurveTraits<FpTraits, FqTraits>;
using VestaTraits = CurveTraits<FqTraits, FpTraits>;

// fn(traits of the id): ZK_FP / ZK_PALLAS select the first type, any other id the second (check_field / check_curve refuse bad ids)
template <class Fn> auto with_field(int field_id, Fn&& fn) { return field_id == ZK_FP ? fn(FpTraits{}) : fn(FqTraits{}); }
template <class Fn> auto with_curve(int curve_id, Fn&& fn) { return curve_id == ZK_PALLAS ? fn(PallasTraits{}) : fn(VestaTraits{}); }

inline int check_field(const char* what, int field_id) {
    if (field_id != ZK_FP && field_id != ZK_FQ) { zk_set_error("%s: unknown field_id %d", what, field_id); return ZK_ERR_INVALID; }
    return ZK_OK;
}
// what = null: the message has no prefix
inline int check_curve(const char* what, int curve_id) {
    if (curve_id == ZK_PALLAS || curve_id == ZK_VESTA) return ZK_OK;
    what ? zk_set_error("%s: unknown curve_id %d", what, curve_id) : zk_set_error("unknown curve_id %d", curve_id);
    return ZK_ERR_INVALID;
}
// domains of up to 2^30 points, the NTT's limit
inline int check_log_n(const char* what, unsigned log_n, const char* name = "log_n") {
    if (log_n > 30) { zk_set_error("%s: %s %u > 30", what, name, log_n); return ZK_ERR_INVALID; }
    return ZK_OK;
}
// x (4 little-endian u64 limbs) is below the field's modulus
inline bool canonical(int field_id, const uint64_t* x) {
    return with_field(field_id, [&](auto f) { return !host::geq_mod<typename decltype(f)::Host>(x); });
}

// a context's pinned slots for small read-backs (ctx_pinned), one per use
struct PinnedSlots {
    fe ip[2];                   // the IPA rounds' two inner products; zk_srs_open: the combined inner product, then a0
    fe s0[2];                   // s_0 = (1) of the IPA rounds per curve, by scalar field id: the source of host-to-device copies that
                                // nothing waits for, so it is only ever rewritten with the same value and never used for anything else
    unsigned remainder;         // zk_poly_divide_by_vanishing_dev: nonzero remainder flag
    unsigned long long ft_len;  // zk_prover_ft_dev: ft's length and ft(zeta omega)
    fe ft_eval1;
    unsigned agg_final;         // zk_perm_aggreg_dev / zk_lookup_aggreg_dev: z[n - zk_rows] == 1 / agg[n - zk_rows - 1] == 1
    unsigned lookup_sorted[2];  // zk_lookup_sorted_dev: the smallest row with a missing value (all ones: none), columns formed
    unsigned index_bad;         // zk_index_build: a gate coefficient is not a canonical field element
};

// [p, p + bytes) and [q, q + qbytes) share a byte
inline bool overlaps(const void* p, size_t bytes, const void* q, size_t qbytes) {
    const uintptr_t a = (uintptr_t)p, b = (uintptr_t)q;
    return a < b + qbytes && b < a + bytes;
}
}  // namespace zkb

struct zk_ctx {
    // Concurrency (SURVEY.md §8b "Threading": SRS is Sync + Send, 15 rayon workers commit at once, kimchi/src/prover.rs:329-351):
    // a context is a small POOL of lanes — itself plus up to n_lanes - 1 children, each a full context with its own stream,
    // scratch and mutex.  Host-pointer entry points (zk_msm*, zk_ntt / zk_ntt_batch, zk_srs_commit_*) take whichever lane is
    // free, so independent calls from different threads overlap on the device; the *_dev entry points (device pointers, caller
    // ordered) and handle-bound calls stay on the primary lane.  A caller-provided stream (zk_ctx_set_stream) or profiling mode
    // pins everything to the primary lane.  Resident bases and twiddle tables are shared, read-only.
    zk_ctx* parent = nullptr;                  // children point at the primary lane
    std::vector<std::unique_ptr<zk_ctx>> children;
    int n_lanes = 4;                           // zk_ctx_set_option("ctx_lanes")
    unsigned rr = 0;                           // round-robin start of the next acquisition (guarded by pool_mu)
    std::mutex pool_mu;                        // children list
    std::mutex tab_mu;                         // NTT table cache of the primary lane (shared by all lanes)
    int device = 0;
    int sm_count = 132;                        // SMs of the device (the MSM sizes its grids by them)
    zkb::Stream own_stream;
    cudaStream_t stream = nullptr;       // own_stream, or the caller's (zk_ctx_set_stream)
    std::mutex mu;                       // a context serialises its calls (SRS: Sync + Send, SURVEY.md §8b "Threading")
    zkb::MsmWorkspace ws;                // scratch of the MSM pipeline (runs on `stream`)
    static constexpr int SIDE_STREAMS = 2;   // copy-in / copy-out streams of the pipelined host-pointer NTT (zk_ntt_batch)
    zkb::Stream side[SIDE_STREAMS];
    zkb::MsmTuning msm;                  // zk_ctx_set_option("msm_batch", "msm_chunk", "msm_wave_threads")
    zkb::Event ev_fork;
    zkb::Event ev_switch;                // zk_ctx_set_stream: the new stream waits for the old one
    zkb::DevScratch d_scalars;           // staging for host-pointer MSM calls
    zkb::DevScratch d_ntt;               // staging for host-pointer NTT calls
    zkb::DevScratch d_ntt_tmp;           // second buffer of the two-pass plan
    // NTT table cache of the primary lane: an entry exists only once its build has succeeded
    zkb::DevScratch ntt_small[2][2];                   // [field][inverse] w_1024^(+-i), 512 entries
    std::map<unsigned, zkb::NttTables> ntt_tables;     // key: field | inverse << 1 | log_n << 2
    zkb::DevScratch d_gather_sum;        // zk_msm_finish_gathered: cross-rank sums of the slice sums
    zkb::PinnedScratch h_gather;         // ... and their pinned host copy
    zkb::PinnedScratch h_pinned_slots;   // zkb::PinnedSlots, through ctx_pinned
    zkb::DevScratch d_open;              // zk_srs_open: staged polynomials | evaluation part | descriptors | extra bases
    zkb::DevScratch d_flag;              // zk_poly_divide_by_vanishing_dev: remainder flag
    zkb::DevScratch d_expr;              // zk_expr_eval_dev: program | constants | column table
    zkb::DevScratch d_ipa;               // zk_srs_open: the rounds' state (a, b, challenge products, expanded scalars), kept between calls
    zkb::DevScratch d_verify;            // zk_srs_verify: s vector | challenge tables | proof points and their scalars
    zkb::DevScratch d_evals;             // zk_lagrange_evaluate_dev / zk_poly_evaluate_chunks_dev: descriptors | partial sums | results
    zkb::DevScratch d_ft;                // zk_prover_ft_dev: f over d1 | term descriptors | length counter
    zkb::DevScratch d_perm;              // zk_perm_aggreg_dev: den, then num / den over d1 | block products | final-value flag
    zkb::DevScratch d_lookup;            // zk_lookup_sorted_dev / zk_lookup_aggreg_dev: lowered lookup info | random rows | the
                                         // table's hash, counts and offsets, or the ratios and block products | flags
    uint64_t launches = 0;
    bool profile = false;                // per-stage device timing (zk_ctx_set_profile)
    std::atomic<bool> pinned{false};     // host-pointer calls stay on the primary lane (stream, profile, n_lanes; written under mu)
    zkb::Event ev_ntt[2];
    float ntt_ms = 0;                    // device time of the last profiled NTT call (all its kernels)
    // The child lanes go first (their work reads this lane's tables), then the lane waits for its streams; the members then free
    // themselves on the device zk_ctx_destroy made current.  Hidden like the library's other C++ symbols (zkb200.h gives the type
    // default visibility).
    __attribute__((visibility("hidden"))) ~zk_ctx() {
        children.clear();
        if (stream) cudaStreamSynchronize(stream);
        for (auto& s : side)
            if (s.s) cudaStreamSynchronize(s.s);
    }
};

// freed by zk_bases_free, which takes the context lock and makes its device current
struct zk_bases {
    zk_ctx* ctx = nullptr;
    zkb::MsmBases b;
};

namespace zkb {
// the lane a host-pointer call runs on, locked for the call's duration
struct LaneLock {
    zk_ctx* lane = nullptr;
    std::unique_lock<std::mutex> lk;
};
int ctx_acquire_lane(zk_ctx* ctx, LaneLock& out);
inline zk_ctx* ctx_root(zk_ctx* c) { return c && c->parent ? c->parent : c; }
inline const zk_ctx* ctx_root(const zk_ctx* c) { return c && c->parent ? c->parent : c; }
int ctx_msm_device(zk_ctx* ctx, const zk_bases* bases, size_t off, size_t n, const fe* d_scalars, int mont, int window_bits,
                   uint64_t out_xyz[12]);
// the context's pinned slots, allocated on first use; null (the error set) when that fails
inline PinnedSlots* ctx_pinned(zk_ctx* ctx) { return ctx->h_pinned_slots.ensure(sizeof(PinnedSlots)) ? nullptr : ctx->h_pinned_slots.at<PinnedSlots>(); }
// the unscaled twiddle tables of a forward / inverse transform (pointwise evaluators take x_i = w^i from them)
int ctx_ntt_table_ptrs(zk_ctx* ctx, int field, unsigned log_n, bool inverse, const fe** ulo, const fe** mid, const fe** hi2);
// the NTT of zk_ntt_dev without the context lock (the caller holds it)
int ctx_ntt_device(zk_ctx* ctx, int field, fe* d_data, unsigned log_n, size_t batch, size_t in_len, int inverse, int coset);
int ctx_ntt_device_oop(zk_ctx* ctx, int field, const fe* d_in, size_t in_bs, fe* d_out, unsigned log_n, size_t batch, size_t in_len, int inverse, int coset);
// k independent MSMs over the same bases slice [off, off + n), scalars j at d_scalars[j] (device memory, ordered after
// ctx->stream), fused into pipelines of up to ctx->msm.batch MSMs (msm.cuh).  Results (Jacobian) to out_xyz + 12 j.
// d_extra / n_extra: points of this call only, laid out like the table (msm.cuh); every scalar vector then has n + n_extra entries.
int ctx_msm_many(zk_ctx* ctx, const zk_bases* bases, size_t off, size_t n, const fe* const* d_scalars, size_t k, int mont, int window_bits,
                 uint64_t* out_xyz, const affine_t* d_extra = nullptr, size_t n_extra = 0);
// the same with one base offset per MSM (the chunks of a chunked Lagrange basis share their scalars, not their bases)
int ctx_msm_many_offs(zk_ctx* ctx, const zk_bases* bases, const size_t* offs, size_t n, const fe* const* d_scalars, size_t k, int mont, int window_bits,
                      uint64_t* out_xyz, const affine_t* d_extra = nullptr, size_t n_extra = 0);
// zk_msm_partial / zk_msm_finish_gathered without the context lock (the caller holds it)
int ctx_msm_partial(zk_ctx* ctx, const zk_bases* bases, size_t off, size_t n, const void* scalars, int scalars_are_mont, int window_bits,
                    void* d_out, size_t capacity_points, unsigned* out_c, unsigned* out_groups);
int ctx_msm_finish_gathered(zk_ctx* ctx, int curve_id, const void* d_all, size_t world, unsigned c, unsigned groups, uint64_t out_xyz[12]);
}  // namespace zkb

// host-side mirror of poly_commitment::ipa::SRS<G> (srs.cu); shared with the opening proof (open.cu)
struct zk_srs {
    zk_ctx* ctx = nullptr;
    int curve = 0;
    size_t n = 0;                       // |g| = max_poly_size
    zk_bases* g = nullptr;              // resident generators
    uint64_t h[8];                      // blinding base
    std::map<size_t, zk_bases*> lagrange;  // domain size -> resident Lagrange basis (one chunk per element: domain <= |g|)
};

// a prover index resident on the device: loaded from a cache file (index_cache.cu) or built from the gates (index_build.cu)
struct zk_index_cache {
    zk_ctx* ctx = nullptr;
    int field = -1;                   // scalar field of a built index; a loaded file does not record it (-1)
    zk_index_header hdr{};
    struct Section { uint32_t tag; uint64_t offset, length; uint32_t elem_domain_size; };
    std::vector<Section> sections;
    zkb::DevScratch payload;          // bytes [lo, hi) of the image (a loaded file) or every section back to back (lo = 0, built)
    uint64_t lo = 0, hi = 0;
};
