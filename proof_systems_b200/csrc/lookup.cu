// lookup.cu — kimchi's lookup argument on the device (kimchi/src/prover.rs:383-673): the joint lookup table, the snake-shaped
// sorted columns and the lookup aggregation polynomial, from the resident witness and lookup tables, so none of them is built on
// the host.  n = |d1|, L = n - zk_rows - 1 (lookup_rows), m = max_per_row.
//
// Joint table (one pointwise kernel over d8): T8[i] = sum_c jc^c col_c[i] + tic tid8[i], Horner over the reversed columns.
//
// Sorted columns (lookup/constraints.rs:90-201 and zk_patch), without a 256-bit sort:
//   k_lookup_insert   an open-addressing hash of T1[0 .. L) whose slots hold row indices: an empty slot is claimed with atomicCAS,
//                     a slot holding an equal value takes atomicMin, so each distinct value ends at its first row first(r)
//   k_lookup_count    one thread per (row, lookup slot): the joint value f, probed in the hash; count[first] += 1 (aggregated
//                     over the warp's lanes that hit the same row), a miss takes atomicMin(bad_row, i); padded slots are counted
//   k_lookup_pad      count[first(dummy)] += padding; whether the columns can be formed
//   k_lookup_offsets_block, k_scan_block_totals (scan.cuh), k_lookup_offsets_apply   offsets = exclusive sum of c_r = 1 + count[r]
//   k_lookup_place    one thread per output element: its position in the pre-snake sequence, a binary search of the offsets for
//                     the table row, T1[r] (or the caller's random value in the zk rows); nothing when a value was missing
// Aggregation (lookup/constraints.rs:233-338), aggreg.cuh with end = L + 1 and last = L (LookupRows): den over the m + 1 sorted
// columns, f and t recomputed from the witness and the table, ratio one at position L; the tail copies the zk_rows random rows.
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/zkb200.h"
#include "aggreg.cuh"

using namespace zkb;

namespace zkb {

constexpr unsigned LK_THREADS = 128;                        // every kernel below: 4 warps
constexpr unsigned LK_SCAN_ITEMS = 16;                      // table rows per thread of the offset scan
constexpr unsigned LK_SCAN_BLOCK = LK_THREADS * LK_SCAN_ITEMS;
constexpr unsigned LK_MAX_COLS = 16;                        // joint table columns
constexpr unsigned LK_MAX_M = 8;                            // max_per_row
constexpr unsigned LK_WITNESS = 15;                         // COLUMNS
constexpr uint32_t LK_EMPTY = 0xffffffffu;

// the lowered zk_lookup_info, as the kernels read it
struct DevTerm { fe coeff; uint32_t column, next; };
struct DevJoint {
    fe tid;                 // Constant(table_id) as a field element
    int32_t tid_column;     // -1: tid, else WitnessColumn(tid_column)
    uint32_t n_entries;
    uint32_t term_end[4];   // entry e: terms [e ? term_end[e - 1] : first_term, term_end[e])
    uint32_t first_term;
};
struct DevPattern { uint32_t first, count; };

struct LookupSpec {
    const fe* w[LK_WITNESS];
    const DevTerm* terms;
    const DevJoint* joints;
    const DevPattern* patterns;
    const uint8_t* row_pattern;    // L entries
    unsigned m;
    fe jc, tic;
};

// the joint lookup value of lookup `jl` at row i: sum_e jc^e entry_e + tic tid
template <class FS> __device__ __forceinline__ fe joint_value(const LookupSpec& s, const DevJoint& jl, size_t i) {
    fe acc = fe_zero();
    for (int e = (int)jl.n_entries - 1; e >= 0; e--) {
        fe ent = fe_zero();
        for (uint32_t t = e ? jl.term_end[e - 1] : jl.first_term; t < jl.term_end[e]; t++) {
            const DevTerm& tm = s.terms[t];
            ent = fe_add<FS>(ent, fe_mul<FS>(load_fe_nc(s.w[tm.column] + i + tm.next), tm.coeff));
        }
        acc = fe_add<FS>(fe_mul<FS>(acc, s.jc), ent);
    }
    const fe tid = jl.tid_column < 0 ? jl.tid : load_fe_nc(s.w[jl.tid_column] + i);
    return fe_add<FS>(acc, fe_mul<FS>(s.tic, tid));
}

// ------------------------------------------------------------------------------------------------------------ joint table
struct JointArgs {
    const fe* col[LK_MAX_COLS];
    const fe* tid8;     // null: table id 0
    const fe* rt8;      // null: no runtime table; else added to column 1
    fe* out8;
    fe* out1;           // null, or out1[i] = out8[8 i]
    size_t len;         // 8n
    unsigned n_cols;
    fe jc, tic;
};

template <class FS> __global__ void __launch_bounds__(LK_THREADS) k_lookup_joint_table(const __grid_constant__ JointArgs a) {
    const size_t i = (size_t)blockIdx.x * LK_THREADS + threadIdx.x;
    if (i >= a.len) return;
    fe acc = fe_zero();
    for (int c = (int)a.n_cols - 1; c >= 0; c--) {
        fe v = load_fe_nc(a.col[c] + i);
        if (c == 1 && a.rt8) v = fe_add<FS>(v, load_fe_nc(a.rt8 + i));
        acc = fe_add<FS>(fe_mul<FS>(acc, a.jc), v);
    }
    if (a.tid8) acc = fe_add<FS>(acc, fe_mul<FS>(a.tic, load_fe_nc(a.tid8 + i)));
    store_fe(a.out8 + i, acc);
    if (a.out1 && (i & 7) == 0) store_fe(a.out1 + (i >> 3), acc);
}

// ------------------------------------------------------------------------------------------------------------ sorted columns
// flags of the sorted call
enum { F_BAD_ROW = 0, F_OK = 1, F_PADDING = 2, F_PHANTOM = 3, F_COUNT = 4 };

__device__ __forceinline__ uint32_t slot_hash(const fe& v, unsigned log_h) {
    return ((v.v[0] ^ (v.v[1] * 0x85ebca6bu)) * 0x9e3779b1u) >> (32 - log_h);
}

// the first table row holding v, or LK_EMPTY
__device__ __forceinline__ uint32_t probe(const uint32_t* slots, unsigned log_h, const fe* T, size_t stride, const fe& v) {
    const uint32_t mask = (1u << log_h) - 1;
    for (uint32_t h = slot_hash(v, log_h);; h = (h + 1) & mask) {
        const uint32_t s = slots[h];
        if (s == LK_EMPTY || fe_eq(load_fe_nc(T + stride * s), v)) return s;
    }
}

__global__ void __launch_bounds__(LK_THREADS) k_lookup_insert(const fe* __restrict__ T, size_t stride, size_t L, uint32_t* slots, unsigned log_h) {
    const size_t r = (size_t)blockIdx.x * LK_THREADS + threadIdx.x;
    if (r >= L) return;
    const fe v = load_fe_nc(T + stride * r);
    const uint32_t mask = (1u << log_h) - 1;
    for (uint32_t h = slot_hash(v, log_h);; h = (h + 1) & mask) {
        const uint32_t s = atomicCAS(slots + h, LK_EMPTY, (uint32_t)r);
        if (s == LK_EMPTY) return;
        // a slot only ever moves between rows of one value, so this comparison does not depend on the atomics' order
        if (fe_eq(load_fe_nc(T + stride * s), v)) { atomicMin(slots + h, (uint32_t)r); return; }
    }
}

struct CountArgs {
    LookupSpec s;
    const fe* T;
    size_t stride, L;
    const uint32_t* slots;
    unsigned log_h;
    uint32_t* count;     // L, by first row
    uint32_t* flags;
    fe dummy;
};

// thread t = (row i, lookup slot j < m).  A value missing from the table is the reference's ValueNotInTable(i), except the dummy
// value at a row i >= 1: the reference has inserted the dummy into its counts after row 0 (its padding step), so that lookup
// succeeds there and only the columns come out malformed (F_PHANTOM, refused by k_lookup_pad).
template <class FS> __global__ void __launch_bounds__(LK_THREADS) k_lookup_count(const __grid_constant__ CountArgs a) {
    const size_t t = (size_t)blockIdx.x * LK_THREADS + threadIdx.x;
    uint32_t key = LK_EMPTY;
    bool pad = false, phantom = false;
    if (t < a.L * a.s.m) {
        const size_t i = t / a.s.m;
        const unsigned j = (unsigned)(t % a.s.m);
        const unsigned p = a.s.row_pattern[i];
        const DevPattern pat = p ? a.s.patterns[p - 1] : DevPattern{0, 0};
        if (j >= pat.count) {
            pad = true;
        } else {
            const fe f = joint_value<FS>(a.s, a.s.joints[pat.first + j], i);
            key = probe(a.slots, a.log_h, a.T, a.stride, f);
            if (key == LK_EMPTY) {
                if (i > 0 && fe_eq(f, a.dummy)) phantom = true;
                else atomicMin(a.flags + F_BAD_ROW, (uint32_t)i);
            }
        }
    }
    const unsigned same = __match_any_sync(0xffffffffu, key);
    if (key != LK_EMPTY && (threadIdx.x & 31) == (unsigned)__ffs(same) - 1) atomicAdd(a.count + key, (uint32_t)__popc(same));
    const int npad = __syncthreads_count(pad), nph = __syncthreads_count(phantom);
    if (threadIdx.x == 0) {
        if (npad) atomicAdd(a.flags + F_PADDING, (uint32_t)npad);
        if (nph) atomicAdd(a.flags + F_PHANTOM, (uint32_t)nph);
    }
}

// one thread: the padding goes to the dummy's first row; the columns are formed when no value was missing and every counted value
// is in the table (the dummy is, or nothing was padded)
__global__ void k_lookup_pad(const uint32_t* slots, unsigned log_h, const fe* T, size_t stride, const fe dummy, uint32_t* count, uint32_t* flags) {
    const uint32_t df = probe(slots, log_h, T, stride, dummy);
    if (df != LK_EMPTY) count[df] += flags[F_PADDING];
    const bool formed = df != LK_EMPTY || flags[F_PADDING] + flags[F_PHANTOM] == 0;
    flags[F_OK] = flags[F_BAD_ROW] == LK_EMPTY && formed ? 1u : 0u;
}

// off[r] = sum of c_q = 1 + count[q] over the block's q < r; btot[b] = the block's sum.  (m + 1) L < 2^32 bounds every sum.
__global__ void __launch_bounds__(LK_THREADS) k_lookup_offsets_block(const uint32_t* __restrict__ count, uint32_t* off, uint32_t* btot, size_t L) {
    const size_t r0 = ((size_t)blockIdx.x * LK_THREADS + threadIdx.x) * LK_SCAN_ITEMS;
    const size_t r1 = r0 + LK_SCAN_ITEMS < L ? r0 + LK_SCAN_ITEMS : L;
    uint32_t sum = 0;
    for (size_t r = r0; r < r1; r++) sum += 1 + count[r];
    uint32_t total;
    uint32_t run = block_exclusive_scan<AddU32, LK_THREADS>(sum, total);
    if (threadIdx.x == 0) btot[blockIdx.x] = total;
    for (size_t r = r0; r < r1; r++) {
        off[r] = run;
        run += 1 + count[r];
    }
}

__global__ void __launch_bounds__(LK_THREADS) k_lookup_offsets_apply(uint32_t* off, const uint32_t* __restrict__ btot, size_t L) {
    const size_t r = (size_t)blockIdx.x * LK_THREADS + threadIdx.x;
    if (r < L && r >= LK_SCAN_BLOCK) off[r] += btot[r / LK_SCAN_BLOCK];
}

struct PlaceArgs {
    fe* out[LK_MAX_M + 1];
    const fe* T;
    const fe* rand;       // (m + 1) zk_rows, column by column
    const uint32_t* off;  // L, strictly increasing from 0
    const uint32_t* flags;
    size_t stride, n, L, zk_rows;
    unsigned m;
};

// element (k, j) of the m + 1 columns.  Before the snake, column k holds seq[k L .. (k + 1) L) and then seq[(k + 1) L] (the last
// column: seq[(m + 1) L - 1] again); odd columns are reversed over their L + 1 entries; rows L + 1 .. n - 1 are random.
__global__ void __launch_bounds__(LK_THREADS) k_lookup_place(const __grid_constant__ PlaceArgs a) {
    const size_t t = (size_t)blockIdx.x * LK_THREADS + threadIdx.x;
    if (t >= (a.m + 1) * a.n || !a.flags[F_OK]) return;
    const unsigned k = (unsigned)(t / a.n);
    const size_t j = t % a.n;
    fe v;
    if (j > a.L) {
        v = load_fe_nc(a.rand + k * a.zk_rows + (j - a.L - 1));
    } else {
        const size_t jj = (k & 1) ? a.L - j : j;
        const uint32_t p = (uint32_t)(jj < a.L ? k * a.L + jj : k < a.m ? (k + 1) * a.L : (a.m + 1) * a.L - 1);
        size_t lo = 0, hi = a.L - 1;                // the last r with off[r] <= p
        while (lo < hi) {
            const size_t mid = (lo + hi + 1) >> 1;
            if (__ldg(a.off + mid) <= p) lo = mid;
            else hi = mid - 1;
        }
        v = load_fe_nc(a.T + a.stride * lo);
    }
    store_fe(a.out[k] + j, v);
}

// ------------------------------------------------------------------------------------------------------------ aggregation
template <class FS> struct LookupRows {
    LookupSpec s;
    const fe* T;
    const fe* sorted[LK_MAX_M + 1];
    size_t stride, L;
    fe beta, gamma, gb1; // gb1 = gamma (1 + beta)
    fe pad_pow[LK_MAX_M + 1];   // (1 + beta)^m (gamma + dummy)^k

    struct Cursor {};
    __device__ Cursor start(size_t) const { return {}; }
    // positions 0 .. L; position L: ratio one, it only receives agg[L]
    __device__ void row(Cursor&, size_t j, fe& num, fe& den) const {
        num = den = fe_one<FS>();
        if (j == L) return;
#pragma unroll 1
        for (unsigned k = 0; k <= s.m; k++) {
            const fe sa = load_fe_nc(sorted[k] + j + (k & 1)), sb = load_fe_nc(sorted[k] + j + 1 - (k & 1));
            den = fe_mul<FS>(den, fe_add<FS>(fe_add<FS>(gb1, sa), fe_mul<FS>(beta, sb)));
        }
        const unsigned p = s.row_pattern[j];
        const DevPattern pat = p ? s.patterns[p - 1] : DevPattern{0, 0};
        num = pad_pow[s.m - pat.count];
#pragma unroll 1
        for (unsigned q = 0; q < pat.count; q++)
            num = fe_mul<FS>(num, fe_add<FS>(gamma, joint_value<FS>(s, s.joints[pat.first + q], j)));
        const fe t0 = load_fe_nc(T + stride * j), t1 = load_fe_nc(T + stride * (j + 1));
        num = fe_mul<FS>(num, fe_add<FS>(fe_add<FS>(gb1, t0), fe_mul<FS>(beta, t1)));
    }
};

// agg[L + 1 + q] = rand[q], q < zk_rows
struct LookupTail {
    const fe* rand;
    size_t zk_rows;

    __device__ void operator()(fe* agg, size_t L, unsigned lane) const {
        for (size_t q = lane; q < zk_rows; q += 32) store_fe(agg + L + 1 + q, load_fe_nc(rand + q));
    }
};

// ------------------------------------------------------------------------------------------------------------ host side
// zk_lookup_info checked against a table of L lookup rows
static int check_info(const char* what, int field_id, size_t L, const zk_lookup_info* info) {
    if (!info->row_pattern || (info->n_terms && !info->terms) || (info->n_lookups && !info->lookups) ||
        (info->n_patterns && (!info->pattern_first || !info->pattern_count))) {
        zk_set_error("%s: null array in the lookup info", what);
        return ZK_ERR_INVALID;
    }
    const unsigned m = info->max_per_row;
    if (m < 1 || m > LK_MAX_M) { zk_set_error("%s: max_per_row %u is not in 1 .. %u", what, m, LK_MAX_M); return ZK_ERR_INVALID; }
    if ((uint64_t)(m + 1) * L >= ((uint64_t)1 << 32)) { zk_set_error("%s: (max_per_row + 1) * lookup rows >= 2^32", what); return ZK_ERR_INVALID; }
    if (info->n_patterns > 255) { zk_set_error("%s: %zu patterns, at most 255", what, info->n_patterns); return ZK_ERR_INVALID; }
    for (size_t p = 0; p < info->n_patterns; p++)
        if (info->pattern_count[p] > m || info->pattern_first[p] > info->n_lookups || info->pattern_count[p] > info->n_lookups - info->pattern_first[p]) {
            zk_set_error("%s: pattern %zu has more than max_per_row lookups or lies outside the lookups", what, p);
            return ZK_ERR_INVALID;
        }
    for (size_t q = 0; q < info->n_lookups; q++) {
        const zk_lookup_joint& jl = info->lookups[q];
        if (jl.n_entries > 4 || jl.table_id_column < -1 || jl.table_id_column >= (int)LK_WITNESS) {
            zk_set_error("%s: lookup %zu has more than 4 entries or a table id column outside -1 .. 14", what, q);
            return ZK_ERR_INVALID;
        }
        uint64_t end = jl.first_term;
        for (unsigned e = 0; e < jl.n_entries; e++) end += jl.entry_terms[e];
        if (end > info->n_terms) { zk_set_error("%s: lookup %zu reads terms past n_terms", what, q); return ZK_ERR_INVALID; }
    }
    for (size_t t = 0; t < info->n_terms; t++) {
        const zk_lookup_term& tm = info->terms[t];
        if (tm.column >= LK_WITNESS || tm.next > 1) { zk_set_error("%s: term %zu reads column %u, next %u", what, t, tm.column, tm.next); return ZK_ERR_INVALID; }
        if (!canonical(field_id, tm.coeff)) { zk_set_error("%s: term %zu has a non-canonical coefficient", what, t); return ZK_ERR_INVALID; }
    }
    for (size_t i = 0; i < L; i++)
        if (info->row_pattern[i] > info->n_patterns) {
            zk_set_error("%s: row %zu has pattern %u of %zu", what, i, (unsigned)info->row_pattern[i], info->n_patterns);
            return ZK_ERR_INVALID;
        }
    if (!canonical(field_id, info->joint_combiner) || !canonical(field_id, info->table_id_combiner) || !canonical(field_id, info->dummy)) {
        zk_set_error("%s: joint_combiner, table_id_combiner or dummy is not a canonical field element", what);
        return ZK_ERR_INVALID;
    }
    return ZK_OK;
}

// the arguments the sorted and aggregation calls share
static int check_common(const char* what, int field_id, unsigned log_n, size_t zk_rows, const void* const d_w[15], const void* d_table,
                        unsigned stride, const zk_lookup_info* info) {
    if (int rc = check_field(what, field_id)) return rc;
    if (int rc = check_log_n(what, log_n)) return rc;
    const size_t n = (size_t)1 << log_n;
    if (zk_rows < 1 || n < 3 || zk_rows > n - 2) { zk_set_error("%s: zk_rows %zu is not in [1, n - 2] for n = %zu", what, zk_rows, n); return ZK_ERR_INVALID; }
    for (unsigned c = 0; c < LK_WITNESS; c++)
        if (!d_w[c]) { zk_set_error("%s: witness column %u is null", what, c); return ZK_ERR_INVALID; }
    if (!d_table) { zk_set_error("%s: null table", what); return ZK_ERR_INVALID; }
    if (stride < 1 || stride > 8) { zk_set_error("%s: table stride %u is not in 1 .. 8", what, stride); return ZK_ERR_INVALID; }
    return check_info(what, field_id, n - zk_rows - 1, info);
}

// d_out (bytes) overlaps none of the witness columns and the table
static bool overlaps_inputs(const void* d_out, size_t bytes, const void* const d_w[15], const void* d_table, size_t table_bytes) {
    for (unsigned c = 0; c < LK_WITNESS; c++)
        if (overlaps(d_out, bytes, d_w[c], bytes)) return true;
    return overlaps(d_out, bytes, d_table, table_bytes);
}

// the lowered info, then `extra` (the random rows): the first buffers of a call's scratch layout `lay`
struct StagedInfo {
    std::vector<unsigned char> bytes;    // the staged part of the scratch, copied with one cudaMemcpyAsync
    size_t o_terms, o_joints, o_pats, o_rows, o_extra;
};

template <class T> static void lower_info(const zk_lookup_info* info, size_t L, const uint64_t* extra, size_t n_extra, Layout& lay, StagedInfo& st) {
    using namespace host;
    using HP = typename T::Host;
    std::vector<DevTerm> terms(info->n_terms);
    for (size_t t = 0; t < info->n_terms; t++) {
        memcpy(&terms[t].coeff, info->terms[t].coeff, 32);
        terms[t].column = info->terms[t].column;
        terms[t].next = info->terms[t].next;
    }
    hfe r2;
    memcpy(r2.l, HP::R2, 32);
    std::vector<DevJoint> joints(info->n_lookups);
    for (size_t q = 0; q < info->n_lookups; q++) {
        const zk_lookup_joint& jl = info->lookups[q];
        hfe id = zero();                                         // i32_to_field: a negative id gives -F(|id|)
        id.l[0] = jl.table_id < 0 ? (uint64_t)(-(int64_t)jl.table_id) : (uint64_t)jl.table_id;
        id = mul<HP>(id, r2);
        if (jl.table_id < 0) id = sub<HP>(zero(), id);
        memcpy(&joints[q].tid, id.l, 32);
        joints[q].tid_column = jl.table_id_column;
        joints[q].n_entries = jl.n_entries;
        joints[q].first_term = jl.first_term;
        uint32_t end = jl.first_term;
        for (unsigned e = 0; e < 4; e++) {
            if (e < jl.n_entries) end += jl.entry_terms[e];
            joints[q].term_end[e] = end;
        }
    }
    std::vector<DevPattern> pats(info->n_patterns);
    for (size_t p = 0; p < info->n_patterns; p++) pats[p] = DevPattern{info->pattern_first[p], info->pattern_count[p]};
    st.o_terms = lay.add(terms.size() * sizeof(DevTerm));
    st.o_joints = lay.add(joints.size() * sizeof(DevJoint));
    st.o_pats = lay.add(pats.size() * sizeof(DevPattern));
    st.o_rows = lay.add(L);
    st.o_extra = lay.add(n_extra * sizeof(fe));
    st.bytes.assign(lay.total, 0);
    memcpy(st.bytes.data() + st.o_terms, terms.data(), terms.size() * sizeof(DevTerm));
    memcpy(st.bytes.data() + st.o_joints, joints.data(), joints.size() * sizeof(DevJoint));
    memcpy(st.bytes.data() + st.o_pats, pats.data(), pats.size() * sizeof(DevPattern));
    memcpy(st.bytes.data() + st.o_rows, info->row_pattern, L);
    memcpy(st.bytes.data() + st.o_extra, extra, n_extra * sizeof(fe));
}

// the staged info copied to the start of ctx->d_lookup (already ensured) on stream st, and the kernels' view of it
static int upload_info(zk_ctx* ctx, cudaStream_t st, const StagedInfo& si, const zk_lookup_info* info, const void* const* d_w, LookupSpec& s) {
    ZK_CUDA(cudaMemcpyAsync(ctx->d_lookup.p, si.bytes.data(), si.bytes.size(), cudaMemcpyHostToDevice, st));
    for (unsigned c = 0; c < LK_WITNESS; c++) s.w[c] = (const fe*)d_w[c];
    s.terms = ctx->d_lookup.at<DevTerm>(si.o_terms);
    s.joints = ctx->d_lookup.at<DevJoint>(si.o_joints);
    s.patterns = ctx->d_lookup.at<DevPattern>(si.o_pats);
    s.row_pattern = ctx->d_lookup.at<uint8_t>(si.o_rows);
    s.m = info->max_per_row;
    memcpy(&s.jc, info->joint_combiner, 32);
    memcpy(&s.tic, info->table_id_combiner, 32);
    return ZK_OK;
}

static size_t blocks_for(size_t items, size_t per_block) { return (items + per_block - 1) / per_block; }

template <class T>
static int joint_table_impl(zk_ctx* ctx, unsigned log_n, const void* const* d_cols, size_t n_cols, const void* d_tid8, const void* d_rt8,
                            const uint64_t jc[4], const uint64_t tic[4], void* d_out8, void* d_out1) {
    JointArgs a{};
    for (size_t c = 0; c < n_cols; c++) a.col[c] = (const fe*)d_cols[c];
    a.tid8 = (const fe*)d_tid8; a.rt8 = (const fe*)d_rt8; a.out8 = (fe*)d_out8; a.out1 = (fe*)d_out1;
    a.len = (size_t)8 << log_n; a.n_cols = (unsigned)n_cols;
    memcpy(&a.jc, jc, 32);
    memcpy(&a.tic, tic, 32);
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    k_lookup_joint_table<typename T::Dev><<<(unsigned)blocks_for(a.len, LK_THREADS), LK_THREADS, 0, ctx->stream>>>(a);
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 1;
    return ZK_OK;
}

template <class T>
static int sorted_impl(zk_ctx* ctx, unsigned log_n, size_t zk_rows, const void* const d_w[15], const fe* T1, size_t stride,
                       const zk_lookup_info* info, const uint64_t* rand, void* const* d_sorted, int64_t* not_in_table_row) {
    using FS = typename T::Dev;
    const size_t n = (size_t)1 << log_n, L = n - zk_rows - 1;
    const unsigned m = info->max_per_row;
    unsigned log_h = 1;
    while (((size_t)1 << log_h) < 2 * L) log_h++;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    PinnedSlots* pin = ctx_pinned(ctx);
    if (!pin) return ZK_ERR_CUDA;
    // context scratch: lowered info | random rows | hash slots | counts | offsets | block sums | flags
    const size_t nb = blocks_for(L, LK_SCAN_BLOCK);
    Layout lay;
    StagedInfo si;
    lower_info<T>(info, L, rand, (m + 1) * zk_rows, lay, si);
    const size_t o_slots = lay.add((size_t)4 << log_h), o_count = lay.add(4 * L), o_off = lay.add(4 * L), o_btot = lay.add(4 * nb),
                 o_flags = lay.add(4 * F_COUNT);
    int rc = ctx->d_lookup.ensure(lay.total);
    if (rc) return rc;
    LookupSpec s{};
    rc = upload_info(ctx, st, si, info, d_w, s);
    if (rc) return rc;
    uint32_t* slots = ctx->d_lookup.at<uint32_t>(o_slots);
    uint32_t* count = ctx->d_lookup.at<uint32_t>(o_count);
    uint32_t* off = ctx->d_lookup.at<uint32_t>(o_off);
    uint32_t* btot = ctx->d_lookup.at<uint32_t>(o_btot);
    uint32_t* flags = ctx->d_lookup.at<uint32_t>(o_flags);
    ZK_CUDA(cudaMemsetAsync(slots, 0xff, (size_t)4 << log_h, st));
    ZK_CUDA(cudaMemsetAsync(count, 0, 4 * L, st));
    ZK_CUDA(cudaMemsetAsync(flags, 0, 4 * F_COUNT, st));
    ZK_CUDA(cudaMemsetAsync(flags + F_BAD_ROW, 0xff, 4, st));
    fe dummy;
    memcpy(&dummy, info->dummy, 32);

    k_lookup_insert<<<(unsigned)blocks_for(L, LK_THREADS), LK_THREADS, 0, st>>>(T1, stride, L, slots, log_h);
    ZK_CUDA(cudaGetLastError());
    CountArgs ca{s, T1, stride, L, slots, log_h, count, flags, dummy};
    k_lookup_count<FS><<<(unsigned)blocks_for(L * m, LK_THREADS), LK_THREADS, 0, st>>>(ca);
    ZK_CUDA(cudaGetLastError());
    k_lookup_pad<<<1, 1, 0, st>>>(slots, log_h, T1, stride, dummy, count, flags);
    ZK_CUDA(cudaGetLastError());
    k_lookup_offsets_block<<<(unsigned)nb, LK_THREADS, 0, st>>>(count, off, btot, L);
    ZK_CUDA(cudaGetLastError());
    k_scan_block_totals<AddU32, LK_THREADS><<<1, LK_THREADS, 0, st>>>(btot, nb);
    ZK_CUDA(cudaGetLastError());
    k_lookup_offsets_apply<<<(unsigned)blocks_for(L, LK_THREADS), LK_THREADS, 0, st>>>(off, btot, L);
    ZK_CUDA(cudaGetLastError());
    PlaceArgs pa{};
    for (unsigned k = 0; k <= m; k++) pa.out[k] = (fe*)d_sorted[k];
    pa.T = T1; pa.rand = ctx->d_lookup.at<fe>(si.o_extra); pa.off = off; pa.flags = flags;
    pa.stride = stride; pa.n = n; pa.L = L; pa.zk_rows = zk_rows; pa.m = m;
    k_lookup_place<<<(unsigned)blocks_for((m + 1) * n, LK_THREADS), LK_THREADS, 0, st>>>(pa);
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 7;
    ZK_CUDA(cudaMemcpyAsync(pin->lookup_sorted, flags, 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    ZK_CUDA(cudaStreamSynchronize(st));
    if (pin->lookup_sorted[F_BAD_ROW] != LK_EMPTY) {
        *not_in_table_row = pin->lookup_sorted[F_BAD_ROW];
        return ZK_OK;
    }
    if (!pin->lookup_sorted[F_OK]) {
        zk_set_error("lookup_sorted: the dummy value is not in the table's first %zu rows, but rows are padded with it", L);
        return ZK_ERR_INVALID;
    }
    *not_in_table_row = -1;
    return ZK_OK;
}

template <class T>
static int aggreg_impl(zk_ctx* ctx, unsigned log_n, size_t zk_rows, const void* const d_w[15], const fe* T1, size_t stride,
                       const zk_lookup_info* info, const void* const* d_sorted, const uint64_t beta[4], const uint64_t gamma[4],
                       const uint64_t* rand, fe* d_agg, int* final_is_one) {
    using namespace host;
    using FS = typename T::Dev; using HP = typename T::Host;
    const size_t n = (size_t)1 << log_n, L = n - zk_rows - 1;
    const unsigned m = info->max_per_row;
    LookupRows<FS> a{};
    for (unsigned k = 0; k <= m; k++) a.sorted[k] = (const fe*)d_sorted[k];
    a.T = T1; a.stride = stride; a.L = L;
    hfe hb, hg, hd;
    memcpy(hb.l, beta, 32);
    memcpy(hg.l, gamma, 32);
    memcpy(hd.l, info->dummy, 32);
    const hfe beta1 = add<HP>(one<HP>(), hb), gd = add<HP>(hg, hd);
    const hfe gb1 = mul<HP>(hg, beta1);
    hfe pw = pow_u64<HP>(beta1, m);
    for (unsigned k = 0; k <= m; k++) {
        memcpy(&a.pad_pow[k], pw.l, 32);
        pw = mul<HP>(pw, gd);
    }
    memcpy(&a.beta, beta, 32);
    memcpy(&a.gamma, gamma, 32);
    memcpy(&a.gb1, gb1.l, 32);

    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    PinnedSlots* pin = ctx_pinned(ctx);
    if (!pin) return ZK_ERR_CUDA;
    // context scratch: lowered info | random rows | ratios over positions 0 .. L | block products | final-value flag
    Layout lay;
    StagedInfo si;
    lower_info<T>(info, L, rand, zk_rows, lay, si);
    const size_t o_r = lay.add((L + 1) * sizeof(fe)), o_tot = lay.add(agg_blocks(L + 1) * sizeof(fe)), o_flag = lay.add(sizeof(unsigned));
    int rc = ctx->d_lookup.ensure(lay.total);
    if (rc) return rc;
    rc = upload_info(ctx, st, si, info, d_w, a.s);
    if (rc) return rc;
    unsigned* d_flag = ctx->d_lookup.at<unsigned>(o_flag);
    const LookupTail tail{ctx->d_lookup.at<fe>(si.o_extra), zk_rows};
    rc = agg_launch<FS>(ctx, a, tail, d_agg, ctx->d_lookup.at<fe>(o_r), ctx->d_lookup.at<fe>(o_tot), L + 1, L, d_flag);
    if (rc) return rc;
    ZK_CUDA(cudaMemcpyAsync(&pin->agg_final, d_flag, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    ZK_CUDA(cudaStreamSynchronize(st));
    *final_is_one = pin->agg_final ? 1 : 0;
    return ZK_OK;
}

}  // namespace zkb

extern "C" int zk_lookup_joint_table_dev(zk_ctx* ctx, int field_id, unsigned log_n, const void* const* d_cols, size_t n_cols, const void* d_table_ids8,
                                         const void* d_runtime8, const uint64_t joint_combiner[4], const uint64_t table_id_combiner[4], void* d_out8,
                                         void* d_out1) {
    const char* what = "lookup_joint_table";
    if (!ctx || !d_cols || !joint_combiner || !table_id_combiner || !d_out8) { zk_set_error("%s: null argument", what); return ZK_ERR_INVALID; }
    if (int rc = check_field(what, field_id)) return rc;
    if (int rc = check_log_n(what, log_n)) return rc;
    if (n_cols < 1 || n_cols > LK_MAX_COLS) { zk_set_error("%s: %zu columns, not 1 .. %u", what, n_cols, LK_MAX_COLS); return ZK_ERR_INVALID; }
    if (d_runtime8 && n_cols < 2) { zk_set_error("%s: a runtime table needs a second table column", what); return ZK_ERR_INVALID; }
    if (!canonical(field_id, joint_combiner) || !canonical(field_id, table_id_combiner)) {
        zk_set_error("%s: joint_combiner or table_id_combiner is not a canonical field element", what);
        return ZK_ERR_INVALID;
    }
    const size_t b8 = ((size_t)8 << log_n) * sizeof(fe), b1 = ((size_t)1 << log_n) * sizeof(fe);
    std::vector<const void*> ins(d_cols, d_cols + n_cols);
    for (size_t c = 0; c < n_cols; c++)
        if (!d_cols[c]) { zk_set_error("%s: column %zu is null", what, c); return ZK_ERR_INVALID; }
    if (d_table_ids8) ins.push_back(d_table_ids8);
    if (d_runtime8) ins.push_back(d_runtime8);
    for (const void* p : ins)
        if (overlaps(d_out8, b8, p, b8) || (d_out1 && overlaps(d_out1, b1, p, b8))) { zk_set_error("%s: an output overlaps an input", what); return ZK_ERR_INVALID; }
    if (d_out1 && overlaps(d_out1, b1, d_out8, b8)) { zk_set_error("%s: d_out1 overlaps d_out8", what); return ZK_ERR_INVALID; }
    return with_field(field_id, [&](auto f) {
        return joint_table_impl<decltype(f)>(ctx, log_n, d_cols, n_cols, d_table_ids8, d_runtime8, joint_combiner, table_id_combiner, d_out8, d_out1);
    });
}

extern "C" int zk_lookup_sorted_dev(zk_ctx* ctx, int field_id, unsigned log_n, size_t zk_rows, const void* const d_w[15], const void* d_table,
                                    unsigned table_stride, const zk_lookup_info* info, const uint64_t* rand, void* const* d_sorted,
                                    int64_t* not_in_table_row) {
    const char* what = "lookup_sorted";
    if (!ctx || !d_w || !info || !rand || !d_sorted || !not_in_table_row) { zk_set_error("%s: null argument", what); return ZK_ERR_INVALID; }
    if (int rc = check_common(what, field_id, log_n, zk_rows, d_w, d_table, table_stride, info)) return rc;
    const size_t n = (size_t)1 << log_n, bytes = n * sizeof(fe);
    const unsigned m = info->max_per_row;
    for (size_t q = 0; q < (m + 1) * zk_rows; q++)
        if (!canonical(field_id, rand + 4 * q)) { zk_set_error("%s: random value %zu is not a canonical field element", what, q); return ZK_ERR_INVALID; }
    for (unsigned k = 0; k <= m; k++) {
        if (!d_sorted[k]) { zk_set_error("%s: output %u is null", what, k); return ZK_ERR_INVALID; }
        if (overlaps_inputs(d_sorted[k], bytes, d_w, d_table, table_stride * bytes)) { zk_set_error("%s: output %u overlaps an input", what, k); return ZK_ERR_INVALID; }
        for (unsigned q = 0; q < k; q++)
            if (overlaps(d_sorted[k], bytes, d_sorted[q], bytes)) { zk_set_error("%s: outputs %u and %u overlap", what, q, k); return ZK_ERR_INVALID; }
    }
    return with_field(field_id, [&](auto f) {
        return sorted_impl<decltype(f)>(ctx, log_n, zk_rows, d_w, (const fe*)d_table, table_stride, info, rand, d_sorted, not_in_table_row);
    });
}

extern "C" int zk_lookup_aggreg_dev(zk_ctx* ctx, int field_id, unsigned log_n, size_t zk_rows, const void* const d_w[15], const void* d_table,
                                    unsigned table_stride, const zk_lookup_info* info, const void* const* d_sorted, const uint64_t beta[4],
                                    const uint64_t gamma[4], const uint64_t* rand, void* d_aggreg, int* final_is_one) {
    const char* what = "lookup_aggreg";
    if (!ctx || !d_w || !info || !d_sorted || !beta || !gamma || !rand || !d_aggreg || !final_is_one) {
        zk_set_error("%s: null argument", what);
        return ZK_ERR_INVALID;
    }
    if (int rc = check_common(what, field_id, log_n, zk_rows, d_w, d_table, table_stride, info)) return rc;
    const size_t n = (size_t)1 << log_n, bytes = n * sizeof(fe);
    if (!canonical(field_id, beta) || !canonical(field_id, gamma)) { zk_set_error("%s: beta or gamma is not a canonical field element", what); return ZK_ERR_INVALID; }
    for (size_t q = 0; q < zk_rows; q++)
        if (!canonical(field_id, rand + 4 * q)) { zk_set_error("%s: random value %zu is not a canonical field element", what, q); return ZK_ERR_INVALID; }
    if (overlaps_inputs(d_aggreg, bytes, d_w, d_table, table_stride * bytes)) { zk_set_error("%s: d_aggreg overlaps an input", what); return ZK_ERR_INVALID; }
    for (unsigned k = 0; k <= info->max_per_row; k++) {
        if (!d_sorted[k]) { zk_set_error("%s: sorted column %u is null", what, k); return ZK_ERR_INVALID; }
        if (overlaps(d_aggreg, bytes, d_sorted[k], bytes)) { zk_set_error("%s: d_aggreg overlaps sorted column %u", what, k); return ZK_ERR_INVALID; }
    }
    return with_field(field_id, [&](auto f) {
        return aggreg_impl<decltype(f)>(ctx, log_n, zk_rows, d_w, (const fe*)d_table, table_stride, info, d_sorted, beta, gamma, rand, (fe*)d_aggreg,
                                        final_is_one);
    });
}
