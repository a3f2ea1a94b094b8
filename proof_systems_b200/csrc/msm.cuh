// msm.cuh — variable-base multi-scalar multiplication on Pallas / Vesta for sm_90a.
//
// Drop-in semantics of ark_ec::VariableBaseMSM::{msm_bigint, msm} as the reference calls them
// (poly-commitment/src/ipa.rs:649-672,943,953,487,497; commitment.rs:382,387 — SURVEY.md §8 rows a1/a2):
//     result = sum_i s_i * P_i       bases affine (x, y Montgomery; identity allowed), scalars canonical 255-bit
// (or Montgomery, converted on the device first), min(len) semantics for msm_bigint.
//
// H100 shape (Pippenger with signed digits, bucket method):
//   * resident bases: an SRS (or a Lagrange basis) is uploaded once and kept in HBM — optionally as a
//     PRECOMPUTED table T[w][i] = 2^(c*w) * P_i (nwin * n affine points; 64 MiB for n = 2^16, c = 16).  With the table
//     all windows share ONE bucket set, so there is no per-window bucket reduction and no Horner doubling chain:
//     80 GB of HBM buys away ~half of the serial tail.  Without a table (one-shot bases) there is one bucket set per
//     window and the host combines the windows.
//   * scalars are recoded to signed base-2^c digits in (-2^(c-1), 2^(c-1)]; (digit != 0) entries are counting-sorted by
//     bucket (histogram -> scan -> scatter, all on device);
//   * accumulation is task based: the histogram is known before any point is touched, so every bucket's sorted entries
//     are cut into ceil(n_b / K) nearly equal tasks; a thread sums one task (<= K XYZZ mixed additions).  The task partials of
//     a bucket are summed thread-parallel in two balanced levels (runs of 4 consecutive partials, then <= 4 run sums per
//     bucket) — thread-serial additions have twice the throughput of the quad-cooperative ones (tools/microbench.py), so the
//     bulk of the reduction stays thread-serial and quads are kept for the short dependent tails.  The rare giant bucket (all
//     points in one bucket — the kimchi witness columns, SURVEY.md §3.1) gets 16 CTAs.  No atomics touch curve points;
//   * bucket reduction sum_b (b+1) B_b in two levels: with b+1 = hi * W + lo the sum is W * sum_hi hi R[hi] + sum_lo lo C[lo]
//     (row / column sums of the bucket grid, one CTA each), then bit slices T_t = sum of the rows / columns whose index has
//     bit t set, and the host finishes with c doublings;
//   * k MSMs over the same bases (the chunks of t, the 15 witness columns, the L/R pair of an IPA round) run as ONE pipeline
//     with k bucket groups: every latency-bound stage is paid once per batch, not once per MSM.
#pragma once
#include <vector>

#include "common.cuh"

namespace zkb {

constexpr unsigned MSM_MAX_WINDOW_BITS = 16;
constexpr uint32_t MSM_MAX_GIANTS = 64;       // buckets with > smax tasks get 16 CTAs each (k_giant_finish)
constexpr unsigned MSM_MAX_BATCH = 16;        // MSMs fused into one pipeline (scalar pointers travel as a kernel parameter)
struct MsmScalarSet {
    const fe* p[MSM_MAX_BATCH];
    uint32_t off[MSM_MAX_BATCH];              // first base of MSM j inside the resident set
};

// A resident set of bases on one device.
struct MsmBases {
    int curve = 0;             // 0 Pallas, 1 Vesta
    size_t n = 0;              // number of points
    unsigned c = 0;            // window bits of the precomputed table (0: no table)
    unsigned nwin = 0;         // windows in the table
    affine_t* d_points = nullptr;  // [max(1,nwin)][n]  row w holds 2^(c*w) * P_i: in `points`, or a view (zk_srs_verify's proof points)
    DevScratch points;
};

// Per-stage device timing of a profiled run (CUDA events on the launching stream).
enum MsmStage { MSM_ST_RECODE = 0, MSM_ST_PLAN, MSM_ST_SCATTER, MSM_ST_ACCUMULATE, MSM_ST_FINISH, MSM_ST_BITSUM, MSM_ST_COUNT };

// Device scratch of one lane's pipeline, sized for the largest call seen so far, grouped by what sizes it (M sorted entries, NB
// buckets in G groups of B, `tiles` scan tiles of k_plan, K entries per task).
struct MsmWorkspace {
    DevScratch entries;        // digits int32[M] | entries u32[M]: point index | sign << 31, sorted by bucket
    DevScratch partials;       // xyzz_t[M / K + NB + 1]: one partial sum per accumulation task
    DevScratch buckets;        // counts u32[NB]: histogram, then scatter cursors | offsets, task offsets u32[NB + 1]: exclusive scans
                               // of the counts and of ceil(count / K) | xyzz_t[NB] | chain u64[tiles]: inclusive (entries << 32 | tasks)
    DevScratch chain_flags;    // u32[tiles]: epoch stamps of the chain; an allocation of their own, so that no other array of a
                               // differently sized run ever lands on a stamp slot
    DevScratch bitsums;        // row/column sums xyzz_t[G][nrows + W], then the slice sums [G][c]
    DevScratch fixed;          // meta u32[8]: [0] sorted entries, [1] tasks, [2] giant buckets | giant bucket ids u32[MSM_MAX_GIANTS] |
                               // per-CTA slice sums of a giant's partials | arrival tickets u32[MSM_MAX_GIANTS] (self-resetting)
    PinnedScratch h_bitsums;   // host copy of the slice sums [G][c]
    uint32_t epoch = 0;        // stamp of the chain flags, bumped per run (no flag memset)
    Event ev[MSM_ST_COUNT + 1];         // stage boundaries of a profiled run
    float stage_ms[MSM_ST_COUNT] = {};  // duration of each stage in the last profiled call
};

// zk_ctx_set_option's MSM settings; every lane of a context runs with those of its primary lane
struct MsmTuning {
    int batch = (int)MSM_MAX_BATCH;   // "msm_batch": MSMs of one call fused into one pipeline
    uint32_t chunk = 0;               // "msm_chunk": entries per task (0: chosen per call so that the tasks fill the machine once)
    uint32_t wave_threads = 0;        // "msm_wave_threads": accumulation threads per SM the task count is sized for (0: built-in default)
};

int msm_default_window(size_t n, bool precomputed);
unsigned msm_num_windows(unsigned c);

// Upload n affine points (host or device memory, 16 u32 each) and optionally build the window table.
template <class F> int msm_bases_create(MsmBases& b, const affine_t* pts, bool pts_on_device, size_t n, unsigned c_table, cudaStream_t st);

// What msm_run leaves in ws.h_bitsums (or at d_out): k x groups x c XYZZ points T[j][g][t]; MSM j is sum_g 2^(c g) sum_t 2^t T[j][g][t].
struct MsmResultShape {
    unsigned c = 0, groups = 0;   // groups == 0: empty MSM (identity)
};

// out[i] = sum over r < world of all[r * count + i]   (the cross-rank sum of gathered slice sums, i < count)
template <class F> int msm_sum_partials(const xyzz_t* d_all, size_t world, size_t count, xyzz_t* d_out, cudaStream_t st);

// k <= MSM_MAX_BATCH MSMs in one pipeline, MSM j over bases[offs[j] .. offs[j]+n).  d_scalars[j]: the n scalars of MSM j, already on the device
// (8 u32 each).  window c: 0 = default (ignored when the bases carry a precomputed table).  The O(c) tail is finished by the caller.
// d_extra / n_extra: n_extra further points that belong to this call only (h and the fresh base U of an IPA round,
// poly-commitment/src/ipa.rs:944,954), laid out like the table — row w holds 2^(c*w) * E_e at d_extra[w * n_extra + e] (one row
// without a table); every scalar vector then carries n_main + n_extra scalars, the extras' last.
// d_out null: the slice sums are copied to ws.h_bitsums and the stream is synchronised (with `profile`, ws.stage_ms is filled).
// Otherwise they are copied to d_out (device, room for out_cap points; refused before anything runs when too small) and nothing
// is synchronised (multi-GPU exchange, zk_msm_partial).  sm_count: SMs of the device.
template <class F, class FS>
int msm_run(const MsmBases& b, const size_t* offs, size_t n_main, const fe* const* d_scalars, unsigned k, bool scalars_mont, unsigned c,
            const affine_t* d_extra, size_t n_extra, const MsmTuning& tune, int sm_count, bool profile, MsmWorkspace& ws, cudaStream_t st,
            xyzz_t* d_out, size_t out_cap, MsmResultShape* shape, unsigned* launches);

// group_ntt.cu: Lagrange-basis commitments of the domain of size 2^log_n from the resident generators (SRS::lagrange_basis)
template <class F, class FS> int lagrange_basis_build(const MsmBases& g, unsigned log_n, unsigned chunk, affine_t* d_out, cudaStream_t st, unsigned* launches);

}  // namespace zkb
