// lookup_index.cu — kimchi's lookup index built on the device from the circuit's gates and tables, and the lookup commitments of its
// verifier index.
//
// zk_lookup_index_build restates LookupConstraintSystem::create (kimchi/src/circuits/lookup/index.rs:202-482) with the pattern
// selectors of LookupInfo::selector_polynomials_and_tables (lookups.rs:235-283, LookupPattern::from_gate :541-553).  The host checks
// every argument and runs the reference's error checks in its order; then
//   k_lookup_index_columns   one thread per row writes the k x n d1 scratch: the w table columns and the table ids (the fixed tables
//                            as given, then the range-check and XOR tables computed in the kernel, then one [first_column, 0] table
//                            per runtime config, zero past them), the present pattern selectors from the tags of gates r and r - 1,
//                            and the runtime selector
//   iFFT(n)                  of all k columns in place (Evaluations::interpolate), batched
//   FFT(8n)                  out of place from the n coefficients straight into the handle's payload (evaluate_over_domain)
// The payload holds the sections back to back in the scratch's column order: 0x50 (w columns), 0x51, 0x52 .. 0x55, 0x56.
//
// zk_lookup_index_commitments restates the commitments of LookupVerifierIndex (verifier_index.rs:196-215) through index_commitments
// (index_build.cu): the table columns and the table ids masked (mask_fixed), the selectors and the runtime selector not.
#include <algorithm>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/zkb200.h"
#include "ctx.hpp"

using namespace zkb;

namespace {

constexpr unsigned GATE_BYTES = 60, MAX_TAG = 13, MAX_WIDTH = 16;   // MAX_WIDTH: the columns zk_lookup_joint_table_dev combines
constexpr size_t MAX_LOG_N = 27;                                   // d8 = 2^30, the NTT's limit
// gate_type_to_tag (cached_prover_index.rs:965-982)
enum : unsigned { TAG_LOOKUP = 7, TAG_RANGE_CHECK0 = 8, TAG_RANGE_CHECK1 = 9, TAG_FOREIGN_FIELD_MUL = 11, TAG_XOR16 = 12, TAG_ROT64 = 13 };
// the lookup patterns in the order of their sections 0x52 .. 0x55 and of LookupSelectorBits 1 .. 4 (cached_prover_index.rs:258-268)
enum : int { PAT_NONE = -1, PAT_XOR = 0, PAT_LOOKUP = 1, PAT_RANGE_CHECK = 2, PAT_FFMUL = 3 };
constexpr unsigned N_PATTERNS = 4;
constexpr uint32_t MAX_JOINT_SIZE[N_PATTERNS] = {3, 2, 1, 1};    // LookupPattern::max_joint_size (lookups.rs:435-441)
constexpr int32_t XOR_TABLE_ID = 0, RANGE_CHECK_TABLE_ID = 1;     // tables/mod.rs:15-18
constexpr uint64_t XOR_TABLE_LEN = 256, RANGE_CHECK_TABLE_LEN = 4096;
constexpr uint32_t BIT_TABLE_IDS8 = 1u << 0, BIT_RUNTIME_SELECTOR = 1u << 5;

// LookupPattern::from_gate (lookups.rs:541-553) for the current row and for the next row
__host__ __device__ inline int pattern_curr(unsigned tag) {
    switch (tag) {
        case TAG_LOOKUP: return PAT_LOOKUP;
        case TAG_RANGE_CHECK0: case TAG_RANGE_CHECK1: case TAG_ROT64: return PAT_RANGE_CHECK;
        case TAG_FOREIGN_FIELD_MUL: return PAT_FFMUL;
        case TAG_XOR16: return PAT_XOR;
        default: return PAT_NONE;
    }
}
__host__ __device__ inline int pattern_next(unsigned tag) {
    return tag == TAG_RANGE_CHECK1 ? PAT_RANGE_CHECK : tag == TAG_FOREIGN_FIELD_MUL ? PAT_FFMUL : PAT_NONE;
}

unsigned gate_tag(const uint8_t* gates, size_t r) { return (unsigned)gates[r * GATE_BYTES] | (unsigned)gates[r * GATE_BYTES + 1] << 8; }

// check_id_duplicates (index.rs:487-502): every id already seen, in order, as "msg: [a, b]"
std::string id_duplicates(const std::vector<int32_t>& ids, const char* msg) {
    std::vector<int32_t> seen, dups;
    for (int32_t id : ids) {
        if (std::find(seen.begin(), seen.end(), id) != seen.end()) dups.push_back(id);
        else seen.push_back(id);
    }
    if (dups.empty()) return {};
    std::string s = std::string(msg) + ": [";
    for (size_t i = 0; i < dups.size(); i++) s += (i ? ", " : "") + std::to_string(dups[i]);
    return s + "]";
}

}  // namespace

namespace zkb {

// one table of the concatenation: rows [start, start + len) of the d1 columns
enum : uint32_t { SEG_DATA = 0, SEG_RANGE_CHECK = 1, SEG_XOR = 2 };
struct LookupSegment {
    uint64_t start, len;
    uint64_t data;              // SEG_DATA: element offset of its columns (column-major, `width` x len) in the uploaded data
    uint32_t width, kind;       // width: uploaded columns (a runtime table: 1, its placeholder column is zero)
    int32_t id;
    uint32_t pad;
};

struct LookupIndexColumns {
    const uint8_t* gates;       // n_gates PrunedGate records
    const LookupSegment* segs;  // by start, none empty
    const fe* data;
    fe* cols;                   // the k x n scratch: table columns 0 .. width, then ids, selectors, runtime selector
    size_t n, n_gates;
    uint64_t total;             // rows the tables cover
    uint64_t rt_lo, rt_hi, zk_lo;   // the runtime selector is 0 on [rt_lo, rt_hi) and [zk_lo, n)
    unsigned n_segs, width, n_sel;
    int ids, runtime;
    int sel_pattern[N_PATTERNS];
};

template <class F> __device__ __forceinline__ fe small_fe(uint32_t x) {
    fe t = fe_zero();
    t.v[0] = x;
    return fe_to_mont<F>(t);
}

template <class F> __global__ void __launch_bounds__(256) k_lookup_index_columns(const LookupIndexColumns a) {
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.n) return;
    const size_t n = a.n;
    const fe zero = fe_zero(), one = fe_one<F>();
    // the table this row belongs to: the last segment starting at or before r
    uint64_t i = 0, len = 0, data = 0;
    uint32_t width = 0, kind = SEG_DATA;
    int32_t id = 0;
    if (r < a.total) {
        unsigned lo = 0, hi = a.n_segs;
        while (hi - lo > 1) {
            const unsigned mid = (lo + hi) / 2;
            if (a.segs[mid].start <= r) lo = mid;
            else hi = mid;
        }
        const LookupSegment* s = a.segs + lo;
        i = r - s->start, len = s->len, data = s->data, width = s->width, kind = s->kind, id = s->id;
    }
#pragma unroll 1
    for (unsigned c = 0; c < a.width; c++) {
        fe v = zero;
        if (r < a.total) {
            if (kind == SEG_DATA) {
                if (c < width) v = load_fe_nc(a.data + data + c * len + i);
            } else if (kind == SEG_RANGE_CHECK) {
                if (c == 0) v = small_fe<F>((uint32_t)i);           // range_check_table: 0 .. 4095
            } else if (c < 3) {                                     // xor_table, reversed: row i = (15 - i / 16, 15 - i % 16, xor)
                const uint32_t x = 15 - (uint32_t)(i >> 4), y = 15 - (uint32_t)(i & 15);
                v = small_fe<F>(c == 0 ? x : c == 1 ? y : x ^ y);
            }
        }
        store_fe(a.cols + c * n + r, v);
    }
    unsigned col = a.width;
    if (a.ids) {                                                    // i32_to_field, 0 past the tables
        fe v = zero;
        if (r < a.total && id != 0) {
            v = small_fe<F>(id < 0 ? (uint32_t)(-(int64_t)id) : (uint32_t)id);
            if (id < 0) v = fe_neg<F>(v);
        }
        store_fe(a.cols + (size_t)col++ * n + r, v);
    }
    const int cur = r < a.n_gates ? pattern_curr(*(const uint16_t*)(a.gates + r * GATE_BYTES)) : PAT_NONE;
    const int nxt = r >= 1 && r - 1 < a.n_gates ? pattern_next(*(const uint16_t*)(a.gates + (r - 1) * GATE_BYTES)) : PAT_NONE;
#pragma unroll
    for (unsigned k = 0; k < N_PATTERNS; k++)
        if (k < a.n_sel) store_fe(a.cols + (size_t)(col + k) * n + r, cur == a.sel_pattern[k] || nxt == a.sel_pattern[k] ? one : zero);
    col += a.n_sel;
    if (a.runtime) store_fe(a.cols + (size_t)col * n + r, (r >= a.rt_lo && r < a.rt_hi) || r >= a.zk_lo ? zero : one);
}

// the index's shape, fixed by the host before any device work
struct LookupPlan {
    size_t n, zk_rows, n_gates;
    std::vector<LookupSegment> segs;
    std::vector<const uint64_t*> seg_src;   // the host columns of each SEG_DATA segment (null for the gate tables)
    uint64_t data_elems = 0, total = 0, rt_lo = 0, rt_hi = 0;
    unsigned width = 0, n_sel = 0;
    int sel_pattern[N_PATTERNS] = {};
    bool ids = false, runtime = false;
    uint32_t bits = 0;
};

template <class T>
static int lookup_index_build_impl(zk_ctx* ctx, const LookupPlan& p, const uint8_t* gates, zk_index_cache** out) {
    using F = typename T::Dev;
    const size_t n = p.n;
    unsigned log_n = 0;
    while (((size_t)1 << log_n) < n) log_n++;
    const size_t k = p.width + p.ids + p.n_sel + p.runtime, b8 = 8 * n * sizeof(fe);
    auto c = std::make_unique<zk_index_cache>();
    c->ctx = ctx;
    c->field = T::id;
    // the sections in the reference writer's order (cached_prover_index.rs:1560-1620); 0x50's elem_domain_size is its column count
    c->sections.push_back({0x50, 0, p.width * b8, p.width});
    uint64_t off = p.width * b8;
    if (p.ids) { c->sections.push_back({0x51, off, b8, (uint32_t)(8 * n)}); off += b8; }
    for (unsigned s = 0; s < p.n_sel; s++) { c->sections.push_back({0x52u + p.sel_pattern[s], off, b8, (uint32_t)(8 * n)}); off += b8; }
    if (p.runtime) { c->sections.push_back({0x56, off, b8, (uint32_t)(8 * n)}); off += b8; }
    c->hdr.domain_d1_size = n;
    c->hdr.zk_rows = p.zk_rows;
    c->hdr.lookup_selectors_present = p.bits;
    c->hdr.num_sections = (uint32_t)c->sections.size();
    c->lo = 0;
    c->hi = off;

    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    if (int rc = c->payload.ensure(c->hi)) return rc;
    // inputs: gates | segments | table data, and the k x n column scratch (both freed on return)
    Layout in;
    const size_t o_g = in.add(p.n_gates * GATE_BYTES), o_s = in.add(p.segs.size() * sizeof(LookupSegment)),
                 o_d = in.add(p.data_elems * sizeof(fe));
    DevScratch d_in, d_cols;
    if (int rc = d_in.ensure(in.total)) return rc;
    if (int rc = d_cols.ensure(k * n * sizeof(fe))) return rc;
    if (p.n_gates) ZK_CUDA(cudaMemcpyAsync(d_in.at<uint8_t>(o_g), gates, p.n_gates * GATE_BYTES, cudaMemcpyHostToDevice, st));
    if (!p.segs.empty())
        ZK_CUDA(cudaMemcpyAsync(d_in.at<uint8_t>(o_s), p.segs.data(), p.segs.size() * sizeof(LookupSegment), cudaMemcpyHostToDevice, st));
    for (size_t j = 0; j < p.segs.size(); j++)
        if (p.seg_src[j])
            ZK_CUDA(cudaMemcpyAsync(d_in.at<fe>(o_d) + p.segs[j].data, p.seg_src[j], p.segs[j].width * p.segs[j].len * sizeof(fe),
                                    cudaMemcpyHostToDevice, st));
    LookupIndexColumns a{};
    a.gates = d_in.at<uint8_t>(o_g);
    a.segs = d_in.at<LookupSegment>(o_s);
    a.data = d_in.at<fe>(o_d);
    a.cols = d_cols.at<fe>();
    a.n = n;
    a.n_gates = p.n_gates;
    a.total = p.total;
    a.rt_lo = p.rt_lo;
    a.rt_hi = p.rt_hi;
    a.zk_lo = n - p.zk_rows;
    a.n_segs = (unsigned)p.segs.size();
    a.width = p.width;
    a.n_sel = p.n_sel;
    a.ids = p.ids;
    a.runtime = p.runtime;
    for (unsigned s = 0; s < N_PATTERNS; s++) a.sel_pattern[s] = p.sel_pattern[s];
    k_lookup_index_columns<F><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a);
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 1;
    fe* cols = d_cols.at<fe>();
    if (int rc = ntt_groups(ctx, T::id, cols, n, cols, log_n, k, 0, /* inverse = */ 1)) return rc;
    if (int rc = ntt_groups(ctx, T::id, cols, n, c->payload.at<fe>(), log_n + 3, k, n, 0)) return rc;
    ZK_CUDA(cudaStreamSynchronize(st));
    *out = c.release();
    return ZK_OK;
}

}  // namespace zkb

extern "C" {

int zk_lookup_index_build(zk_ctx* ctx, int field_id, uint64_t domain_d1_size, uint64_t zk_rows, const void* gates, size_t n_gates,
                          const zk_lookup_table* tables, size_t n_tables, const zk_runtime_table_cfg* runtime, size_t n_runtime,
                          int has_runtime, int* lookup_error, uint64_t* runtime_table_offset, zk_index_cache** out) {
    if (out) *out = nullptr;
    if (lookup_error) *lookup_error = ZK_LOOKUP_ERR_NONE;
    if (!ctx || !out || !lookup_error || (has_runtime && !runtime_table_offset) || (!gates && n_gates) || (!tables && n_tables) ||
        (!runtime && n_runtime)) {
        zk_set_error("lookup_index_build: null argument");
        return ZK_ERR_INVALID;
    }
    if (int rc = check_field("lookup_index_build", field_id)) return rc;
    const uint64_t n = domain_d1_size;
    if (n == 0 || (n & (n - 1)) || n > ((uint64_t)1 << MAX_LOG_N)) {
        zk_set_error("lookup_index_build: d1 size %llu is not a power of two up to 2^%zu", (unsigned long long)n, MAX_LOG_N);
        return ZK_ERR_INVALID;
    }
    if (zk_rows < 1 || zk_rows + 2 > n) { zk_set_error("lookup_index_build: zk_rows %llu is not in [1, %llu]", (unsigned long long)zk_rows, (unsigned long long)n - 2); return ZK_ERR_INVALID; }
    if (n_gates > n) { zk_set_error("lookup_index_build: %zu gates do not fit the domain of %llu rows", n_gates, (unsigned long long)n); return ZK_ERR_INVALID; }
    if (!has_runtime && n_runtime) { zk_set_error("lookup_index_build: %zu runtime tables without has_runtime", n_runtime); return ZK_ERR_INVALID; }
    const uint8_t* g = (const uint8_t*)gates;
    for (size_t r = 0; r < n_gates; r++)
        if (gate_tag(g, r) > MAX_TAG) { zk_set_error("lookup_index_build: gate %zu has tag %u > %u", r, gate_tag(g, r), MAX_TAG); return ZK_ERR_INVALID; }
    // selector_polynomials_and_tables sets row i + 1 for a Next pattern: on the last row the reference indexes past the domain
    if (n_gates == n && pattern_next(gate_tag(g, n - 1)) != PAT_NONE) {
        zk_set_error("lookup_index_build: gate %zu on the last row looks up the next row", n_gates - 1);
        return ZK_ERR_INVALID;
    }
    for (size_t t = 0; t < n_tables; t++) {
        const zk_lookup_table& tb = tables[t];
        if (tb.width == 0 || tb.width > MAX_WIDTH) { zk_set_error("lookup_index_build: table %zu has width %u, not in [1, %u]", t, tb.width, MAX_WIDTH); return ZK_ERR_INVALID; }
        if (tb.len && !tb.data) { zk_set_error("lookup_index_build: table %zu has no data", t); return ZK_ERR_INVALID; }
        for (uint64_t e = 0; e < (uint64_t)tb.width * tb.len; e++)
            if (!canonical(field_id, tb.data + 4 * e)) { zk_set_error("lookup_index_build: table %zu entry %llu is not a canonical field element", t, (unsigned long long)e); return ZK_ERR_INVALID; }
    }
    for (size_t t = 0; t < n_runtime; t++) {
        const zk_runtime_table_cfg& rt = runtime[t];
        if (rt.len && !rt.first_column) { zk_set_error("lookup_index_build: runtime table %zu has no first column", t); return ZK_ERR_INVALID; }
        for (uint64_t e = 0; e < rt.len; e++)
            if (!canonical(field_id, rt.first_column + 4 * e)) { zk_set_error("lookup_index_build: runtime table %zu entry %llu is not a canonical field element", t, (unsigned long long)e); return ZK_ERR_INVALID; }
    }

    // LookupInfo::create_from_gates: no pattern, no lookup index
    bool present[N_PATTERNS] = {};
    for (size_t r = 0; r < n_gates; r++) {
        const unsigned tag = gate_tag(g, r);
        if (pattern_curr(tag) != PAT_NONE) present[pattern_curr(tag)] = true;
        if (pattern_next(tag) != PAT_NONE) present[pattern_next(tag)] = true;
    }
    LookupPlan p;
    p.n = n;
    p.zk_rows = zk_rows;
    p.n_gates = n_gates;
    uint32_t max_joint = 0;
    for (unsigned s = 0; s < N_PATTERNS; s++)
        if (present[s]) {
            p.sel_pattern[p.n_sel++] = (int)s;
            p.bits |= 1u << (1 + s);
            max_joint = std::max(max_joint, MAX_JOINT_SIZE[s]);
        }
    if (!p.n_sel) return ZK_OK;

    auto lookup_err = [&](int kind, const std::string& msg) {
        *lookup_error = kind;
        zk_set_error("%s", msg.c_str());
        return ZK_ERR_INVALID;
    };
    // the gate tables in GateLookupTable's order: RangeCheck before Xor (tables/mod.rs:36-46)
    const bool rc_table = present[PAT_RANGE_CHECK] || present[PAT_FFMUL], xor_table = present[PAT_XOR];
    std::vector<int32_t> ids;
    for (size_t t = 0; t < n_tables; t++) ids.push_back(tables[t].id);
    if (rc_table) ids.push_back(RANGE_CHECK_TABLE_ID);
    if (xor_table) ids.push_back(XOR_TABLE_ID);
    std::string dup = id_duplicates(ids, "duplicates between fixed given and fixed from-gate tables");
    if (dup.empty() && has_runtime) {
        std::vector<int32_t> rids;
        for (size_t t = 0; t < n_runtime; t++) rids.push_back(runtime[t].id);
        dup = id_duplicates(rids, "runtime table duplicates");
    }
    if (!dup.empty())
        return lookup_err(ZK_LOOKUP_ERR_ID_COLLISION, "Cannot create a combined table since ids for sub-tables are colliding. The collision type is: " + dup);

    // the concatenation: fixed tables, gate tables, runtime tables (index.rs:239-406)
    uint64_t total = 0;
    bool has_id0 = false, id0_zero_entry = false, nonzero_id = false;
    unsigned width = max_joint;
    auto add = [&](uint32_t kind, int32_t id, uint64_t len, uint32_t w, uint32_t data_width, const uint64_t* src) {
        if (len) {
            p.segs.push_back({total, len, p.data_elems, data_width, kind, id, 0});
            p.seg_src.push_back(src);
            if (src) p.data_elems += (uint64_t)data_width * len;
        }
        total += len;
        width = std::max(width, w);
        if (id == 0) has_id0 = true;
        else nonzero_id = true;
    };
    auto zero_row = [&](const uint64_t* cols, uint32_t w, uint64_t len) {   // LookupTable::has_zero_entry
        for (uint64_t i = 0; i < len; i++) {
            bool all = true;
            for (uint32_t c = 0; c < w && all; c++) {
                const uint64_t* x = cols + 4 * (c * len + i);
                all = !(x[0] | x[1] | x[2] | x[3]);
            }
            if (all) return true;
        }
        return false;
    };
    for (size_t t = 0; t < n_tables; t++) {
        add(SEG_DATA, tables[t].id, tables[t].len, tables[t].width, tables[t].width, tables[t].data);
        if (tables[t].id == 0 && zero_row(tables[t].data, tables[t].width, tables[t].len)) id0_zero_entry = true;
    }
    if (rc_table) add(SEG_RANGE_CHECK, RANGE_CHECK_TABLE_ID, RANGE_CHECK_TABLE_LEN, 1, 0, nullptr);
    if (xor_table) { add(SEG_XOR, XOR_TABLE_ID, XOR_TABLE_LEN, 3, 0, nullptr); id0_zero_entry = true; }   // its last row is zero
    if (has_runtime) {
        uint64_t runtime_len = 0;
        for (size_t t = 0; t < n_runtime; t++) runtime_len += runtime[t].len;
        // the runtime selector is built before the length check: the reference's `d1_size - offset - runtime_len` underflows
        if (total > n || runtime_len > n - total) {
            zk_set_error("lookup_index_build: %llu table rows and %llu runtime rows exceed the domain of %llu rows", (unsigned long long)total,
                         (unsigned long long)runtime_len, (unsigned long long)n);
            return ZK_ERR_INVALID;
        }
        p.runtime = true;
        p.rt_lo = total;
        p.rt_hi = total + runtime_len;
        p.bits |= BIT_RUNTIME_SELECTOR;
        for (size_t t = 0; t < n_runtime; t++) {
            add(SEG_DATA, runtime[t].id, runtime[t].len, 2, 1, runtime[t].first_column);
            if (runtime[t].id == 0 && zero_row(runtime[t].first_column, 1, runtime[t].len)) id0_zero_entry = true;
        }
    }
    if (has_id0 && !id0_zero_entry) return lookup_err(ZK_LOOKUP_ERR_TABLE_ID_ZERO, "The table with id 0 must have an entry of all zeros");
    const uint64_t max_num_entries = n - zk_rows - 1;
    if (total >= max_num_entries)
        return lookup_err(ZK_LOOKUP_ERR_TOO_LONG, "The combined lookup table is larger than allowed by the domain size. Observed: " +
                                                      std::to_string(total) + ", expected: " + std::to_string(max_num_entries - 1));
    p.total = total;
    p.width = width;
    p.ids = nonzero_id;
    if (p.ids) p.bits |= BIT_TABLE_IDS8;
    if (has_runtime) *runtime_table_offset = p.rt_lo;
    return with_field(field_id, [&](auto f) { return lookup_index_build_impl<decltype(f)>(ctx, p, g, out); });
}

int zk_lookup_index_commitments(zk_srs* srs, const zk_index_cache* index, uint64_t* out_xy, size_t capacity_points, size_t* out_points) {
    if (!srs || !index || !out_xy || !out_points) { zk_set_error("lookup_index_commitments: null argument"); return ZK_ERR_INVALID; }
    const int sf = with_curve(srs->curve, [](auto c) { return decltype(c)::scalar_field; });
    if (index->field >= 0 && index->field != sf) { zk_set_error("lookup_index_commitments: the index is over field %d, the SRS's scalars over %d", index->field, sf); return ZK_ERR_INVALID; }
    const uint64_t n = index->hdr.domain_d1_size;
    auto find = [&](uint32_t t) -> const zk_index_cache::Section* {
        for (const auto& o : index->sections)
            if (o.tag == t) return &o;
        return nullptr;
    };
    // verifier_index.rs:196-215: lookup_table (masked), table_ids (masked), lookup_selectors (xor, lookup, range_check, ffmul),
    // runtime_tables_selector; the header's bits say which of the optional ones the index has
    std::vector<IndexCommitment> cols;
    const zk_index_cache::Section* t50 = find(0x50);
    if (!t50) { zk_set_error("lookup_index_commitments: section 0x50 missing"); return ZK_ERR_INVALID; }
    const uint64_t w = t50->elem_domain_size, len50 = t50->length / sizeof(fe);
    if (w == 0 || len50 == 0 || len50 % w || (len50 / w) % n || (len50 / w) / n > UINT32_MAX) {
        zk_set_error("lookup_index_commitments: section 0x50 has %llu elements, not %llu columns of a multiple of %llu", (unsigned long long)len50,
                     (unsigned long long)w, (unsigned long long)n);
        return ZK_ERR_INVALID;
    }
    for (uint64_t c = 0; c < w; c++) cols.push_back({index->payload.at<fe>(t50->offset - index->lo) + c * (len50 / w), (uint32_t)(len50 / w / n), true});
    const uint32_t bits = index->hdr.lookup_selectors_present;
    for (unsigned b = 0; b < 6; b++) {
        if (!((bits >> b) & 1)) continue;
        const uint32_t t = b == 0 ? 0x51 : b == 5 ? 0x56 : 0x51 + b;
        const zk_index_cache::Section* s = find(t);
        if (!s) { zk_set_error("lookup_index_commitments: section %#x missing", t); return ZK_ERR_INVALID; }
        const uint64_t len = s->length / sizeof(fe);
        if (len == 0 || len % n || len / n > UINT32_MAX) { zk_set_error("lookup_index_commitments: section %#x has %llu elements, not a multiple of %llu", t, (unsigned long long)len, (unsigned long long)n); return ZK_ERR_INVALID; }
        cols.push_back({index->payload.at<fe>(s->offset - index->lo), (uint32_t)(len / n), b == 0});
    }
    const size_t chunks = zk_srs_lagrange_basis_chunks(srs, n);
    *out_points = cols.size() * chunks;
    if (capacity_points < *out_points) { zk_set_error("lookup_index_commitments: %zu points do not fit the capacity %zu", *out_points, capacity_points); return ZK_ERR_INVALID; }
    return index_commitments(srs, n, cols, out_xy);
}

}  // extern "C"
