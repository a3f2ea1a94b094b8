// ctx.hpp — the objects behind the opaque handles of include/zkb200.h.
#pragma once
#include <map>
#include <memory>
#include <mutex>
#include <vector>

#include "msm.cuh"
#include "ntt.cuh"

struct zk_ctx {
    // Concurrency (SURVEY.md §8b "Threading": SRS is Sync + Send, 15 rayon workers commit at once, kimchi/src/prover.rs:329-351):
    // a context is a small POOL of lanes — itself plus up to n_lanes - 1 children, each a full context with its own stream,
    // scratch and mutex.  Host-pointer entry points (zk_msm*, zk_ntt / zk_ntt_batch, zk_srs_commit_*) take whichever lane is
    // free, so independent calls from different threads overlap on the device; the *_dev entry points (device pointers, caller
    // ordered) and handle-bound calls stay on the primary lane.  A caller-provided stream (zk_ctx_set_stream) or profiling mode
    // pins everything to the primary lane.  Resident bases and twiddle tables are shared, read-only.
    zk_ctx* parent = nullptr;                  // children point at the primary lane
    std::vector<zk_ctx*> children;
    int n_lanes = 4;                           // zk_ctx_set_option("ctx_lanes")
    unsigned rr = 0;                           // round-robin start of the next acquisition (guarded by pool_mu)
    std::mutex pool_mu;                        // children list
    std::mutex tab_mu;                         // NTT table cache of the primary lane (shared by all lanes)
    int device = 0;
    cudaStream_t own_stream = nullptr, stream = nullptr;
    std::mutex mu;                       // a context serialises its calls (SRS: Sync + Send, SURVEY.md §8b "Threading")
    zkb::MsmWorkspace ws;                // scratch of the MSM pipeline (runs on `stream`)
    static constexpr int SIDE_STREAMS = 2;   // copy-in / copy-out streams of the pipelined host-pointer NTT (zk_ntt_batch)
    cudaStream_t side[SIDE_STREAMS] = {};
    int batch = (int)zkb::MSM_MAX_BATCH; // zk_ctx_set_option("msm_batch"): MSMs of one call fused into one pipeline
    cudaEvent_t ev_fork = nullptr;
    zkb::fe* d_scalars = nullptr;        // staging for host-pointer MSM calls
    size_t cap_scalars = 0;
    zkb::fe* d_ntt = nullptr;            // staging for host-pointer NTT calls
    size_t cap_ntt = 0;
    zkb::fe* d_ntt_tmp = nullptr;        // second buffer of the two-pass plan
    size_t cap_ntt_tmp = 0;
    zkb::fe* ntt_small[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};  // [field][inverse] w_1024^(+-i)
    std::map<unsigned, zkb::NttTables> ntt_tables;                         // key: field | inverse << 1 | log_n << 2
    zkb::xyzz_t* d_gather_sum = nullptr; // zk_msm_finish_gathered: cross-rank sums of the slice sums
    size_t cap_gather_sum = 0;
    zkb::xyzz_t* h_gather = nullptr;     // ... and their pinned host copy
    size_t cap_h_gather = 0;
    void* h_scratch = nullptr;           // 256 pinned bytes for small read-backs
    void* d_open = nullptr;              // zk_srs_open: staged polynomials | evaluation part | descriptors | extra bases
    size_t cap_open = 0;
    unsigned* d_flag = nullptr;          // zk_poly_divide_by_vanishing_dev: remainder flag
    void* d_expr = nullptr;              // zk_expr_eval_dev: program | constants | column table
    size_t cap_expr = 0;
    void* d_ipa = nullptr;               // zk_srs_open: the rounds' state (a, b, challenge products, expanded scalars), kept between calls
    size_t cap_ipa = 0;
    void* d_verify = nullptr;            // zk_srs_verify: s vector | challenge tables | proof points and their scalars
    size_t cap_verify = 0;
    void* d_evals = nullptr;             // zk_lagrange_evaluate_dev / zk_poly_evaluate_chunks_dev: descriptors | partial sums | results
    size_t cap_evals = 0;
    void* d_ft = nullptr;                // zk_prover_ft_dev: f over d1 | term descriptors | length counter
    size_t cap_ft = 0;
    uint64_t launches = 0;
    bool profile = false;                // per-stage device timing (zk_ctx_set_profile)
    cudaEvent_t ev_ntt[2] = {nullptr, nullptr};
    float ntt_ms = 0;                    // device time of the last profiled NTT call (all its kernels)
};

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
int ctx_ensure(void** p, size_t* cap, size_t bytes);
// the NTT of zk_ntt_dev without the context lock (the caller holds it)
int ctx_ntt_device(zk_ctx* ctx, int field, fe* d_data, unsigned log_n, size_t batch, size_t in_len, int inverse, int coset);
int ctx_ntt_device_oop(zk_ctx* ctx, int field, const fe* d_in, size_t in_bs, fe* d_out, unsigned log_n, size_t batch, size_t in_len, int inverse, int coset);
// k independent MSMs over the same bases slice [off, off + n), scalars j at d_scalars[j] (device memory, ordered after
// ctx->stream), fused into pipelines of up to ctx->batch MSMs (msm.cuh).  Results (Jacobian) to out_xyz + 12 j.
// d_extra / n_extra: points of this call only, laid out like the table (msm.cuh); every scalar vector then has n + n_extra entries.
int ctx_msm_many(zk_ctx* ctx, const zk_bases* bases, size_t off, size_t n, const fe* const* d_scalars, size_t k, int mont, int window_bits,
                 uint64_t* out_xyz, const affine_t* d_extra = nullptr, size_t n_extra = 0);
// the same with one base offset per MSM (the chunks of a chunked Lagrange basis share their scalars, not their bases)
int ctx_msm_many_offs(zk_ctx* ctx, const zk_bases* bases, const size_t* offs, size_t n, const fe* const* d_scalars, size_t k, int mont, int window_bits,
                      uint64_t* out_xyz, const affine_t* d_extra = nullptr, size_t n_extra = 0);
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
