// index_build.cu — kimchi's prover index built on the device from the circuit's gates, and the commitments of its verifier index.
//
// zk_index_build restates ConstraintSystem::evaluated_column_coefficients and column_evaluations (kimchi/src/circuits/constraints.rs:
// 510-760, selector_polynomial at :334-362) with the gates in the cache file's own encoding (PrunedGate records and GateCoeffs,
// cached_prover_index.rs:270-300, :1007-1015, :1472-1479):
//   k_index_columns     one thread per row: decodes the gate (a self-wired zero gate past the list, constraints.rs:1010-1020) and
//                       writes sid[r] = omega^r, sigma_k[r] = shift[col] omega^row of wire k (zero on rows n + 2 - zk_rows .. n - 2),
//                       the 15 coefficients and the selectors into a k x n scratch; a non-canonical coefficient sets a flag
//   iFFT(n)             of all k columns in place (Evaluations::interpolate), batched
//   FFT(8n) / FFT(4n)   out of place from the n coefficients straight into the handle's payload (evaluate_over_domain_by_ref)
// The payload holds the d8 sections back to back in the scratch's column order, then the two d4 sections, then sid, so every
// transform group is one batched call.  With zero_selectors, selector_polynomial's columns are not built: their sections are zeroed.
//
// zk_index_commitments restates the commitment fields of ProverIndex::verifier_index (kimchi/src/verifier_index.rs:221-300):
// k_index_gather sub-samples every section to d1 (commit_evaluations_non_hiding, poly-commitment/src/ipa.rs:706-728), the MSMs run
// as fused batches over the resident Lagrange basis (one per chunk of a chunked basis), and the host adds h to each chunk of the six
// masked commitments (mask_fixed, verifier_index.rs:179-185).  ntt_groups and index_commitments also serve the lookup index
// (lookup_index.cu).
#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/zkb200.h"
#include "ctx.hpp"

using namespace zkb;

namespace {

constexpr unsigned PERMUTS = 7, COLUMNS = 15, GATE_BYTES = 2 + 2 + 2 * 4 * PERMUTS, MAX_TAG = 13, OPTIONAL_BITS = 6;
constexpr unsigned MAX_SELECTORS = 12;       // poseidon, VarBaseMul, EndoMul, EndoMulScalar, 6 optional; generic, CompleteAdd
constexpr size_t MAX_LOG_N = 27;             // d8 = 2^30, the NTT's limit
constexpr size_t NTT_GROUP_BYTES = (size_t)1 << 30;   // elements per batched transform, bounding the NTT's second buffer
// gate_type_to_tag (cached_prover_index.rs:965-982)
enum : uint8_t { TAG_GENERIC = 1, TAG_POSEIDON = 2, TAG_COMPLETE_ADD = 3, TAG_VAR_BASE_MUL = 4, TAG_ENDO_MUL = 5, TAG_ENDO_MUL_SCALAR = 6,
                 TAG_RANGE_CHECK0 = 8 };

uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }

}  // namespace

namespace zkb {

struct IndexColumns {
    const uint8_t* gates;       // n_gates PrunedGate records
    const uint8_t* coeffs;      // the GateCoeffs records
    const uint64_t* coeff_off;  // byte offset of gate r's u32 count in coeffs
    const fe* shift;            // the 7 shifts
    const fe* ulo;              // omega^e of d1 (domain_point, ntt.cuh)
    const fe* mid;
    const fe* hi2;
    fe* cols;                   // column c at cols + c n: sigma 0..6, coefficients 7..21, then the selectors
    fe* sid;
    size_t n, n_gates, zero_lo, zero_hi;   // sigma is zero on rows [zero_lo, zero_hi)
    unsigned n_sel;
    uint8_t sel_tag[MAX_SELECTORS];        // selector column 22 + s is 1 where the gate's tag is sel_tag[s]
    unsigned* bad;              // set when a coefficient is not a canonical field element
};

template <class F> __global__ void __launch_bounds__(256) k_index_columns(const IndexColumns a) {
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.n) return;
    const size_t n = a.n;
    store_fe(a.sid + r, domain_point<F>(a.ulo, a.mid, a.hi2, r));
    const bool real = r < a.n_gates;
    const uint8_t* g = a.gates + r * GATE_BYTES;             // 4-byte aligned: 60 r
    const unsigned typ = real ? *(const uint16_t*)g : 0u;
    const bool zeroed = r >= a.zero_lo && r < a.zero_hi;
#pragma unroll 1
    for (unsigned k = 0; k < PERMUTS; k++) {
        fe s = fe_zero();
        if (!zeroed) {
            const uint32_t* w = (const uint32_t*)(g + 4 + 8 * k);
            const size_t row = real ? w[0] : r;
            const unsigned col = real ? w[1] : k;
            s = fe_mul<F>(load_fe_nc(a.shift + col), domain_point<F>(a.ulo, a.mid, a.hi2, row));
        }
        store_fe(a.cols + k * n + r, s);
    }
    unsigned cnt = 0;
    const uint32_t* ce = nullptr;
    if (real) {
        const uint8_t* rec = a.coeffs + a.coeff_off[r];     // u32 count, then the elements: 4-byte aligned
        cnt = *(const uint32_t*)rec;
        ce = (const uint32_t*)(rec + 4);
    }
    bool ok = true;
#pragma unroll 1
    for (unsigned i = 0; i < COLUMNS; i++) {
        fe c = fe_zero();
        if (i < cnt) {
#pragma unroll
            for (int j = 0; j < 8; j++) c.v[j] = __ldg(ce + 8 * i + j);
            ok &= fe_lt_modulus<F>(c);
        }
        store_fe(a.cols + (PERMUTS + i) * n + r, c);
    }
    if (!ok) *a.bad = 1;
    const fe one = fe_one<F>(), zero = fe_zero();
#pragma unroll
    for (unsigned s = 0; s < MAX_SELECTORS; s++)
        if (s < a.n_sel) store_fe(a.cols + (PERMUTS + COLUMNS + s) * n + r, typ == a.sel_tag[s] ? one : zero);
}

// up to MAX_GATHER sections sub-sampled to d1: out[j n + i] = sec_j[stride_j i]
constexpr unsigned MAX_GATHER = 40;
struct IndexGather {
    const fe* src[MAX_GATHER];
    uint32_t stride[MAX_GATHER];
    fe* out;
    size_t n;
};

__global__ void __launch_bounds__(256) k_index_gather(const __grid_constant__ IndexGather a) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned j = blockIdx.y;
    if (i < a.n) store_fe(a.out + j * a.n + i, load_fe_nc(a.src[j] + (size_t)a.stride[j] * i));
}

// the library's NTT over `count` polynomials in groups, so its second buffer stays within NTT_GROUP_BYTES
int ntt_groups(zk_ctx* ctx, int field, const fe* in, size_t in_bs, fe* out, unsigned log_n, size_t count, size_t in_len, int inverse) {
    const size_t per = std::max<size_t>(1, NTT_GROUP_BYTES / (sizeof(fe) << log_n));
    for (size_t c0 = 0; c0 < count; c0 += per) {
        const size_t b = std::min(per, count - c0);
        if (int rc = ctx_ntt_device_oop(ctx, field, in + c0 * in_bs, in_bs, out + (c0 << log_n), log_n, b, in_len, inverse, 0)) return rc;
    }
    return ZK_OK;
}

template <class T>
static int index_build_impl(zk_ctx* ctx, const zk_index_header* hdr, const uint8_t* gates, size_t n_gates, const uint8_t* gate_coeffs,
                            size_t gate_coeffs_len, const std::vector<uint64_t>& coeff_off, bool zero_selectors, zk_index_cache** out) {
    using F = typename T::Dev;
    const size_t n = hdr->domain_d1_size;
    unsigned log_n = 0;
    while (((size_t)1 << log_n) < n) log_n++;
    const uint32_t opt = hdr->optional_selectors_present;
    unsigned n_opt = 0;
    for (unsigned b = 0; b < OPTIONAL_BITS; b++) n_opt += (opt >> b) & 1;

    // selector columns after sigma and the coefficients: the d8 ones, then the d4 ones; selector_polynomial's are built only when
    // they are not all zero
    IndexColumns a{};
    a.sel_tag[a.n_sel++] = TAG_POSEIDON;
    if (!zero_selectors) {
        for (uint8_t t : {TAG_VAR_BASE_MUL, TAG_ENDO_MUL, TAG_ENDO_MUL_SCALAR}) a.sel_tag[a.n_sel++] = t;
        for (unsigned b = 0; b < OPTIONAL_BITS; b++)
            if ((opt >> b) & 1) a.sel_tag[a.n_sel++] = (uint8_t)(TAG_RANGE_CHECK0 + b);
    }
    const size_t built8 = PERMUTS + COLUMNS + a.n_sel;        // d8 columns that are transformed
    a.sel_tag[a.n_sel++] = TAG_GENERIC;
    if (!zero_selectors) a.sel_tag[a.n_sel++] = TAG_COMPLETE_ADD;
    const size_t k = PERMUTS + COLUMNS + a.n_sel, built4 = k - built8;

    // payload: d8 sections (sigma, coefficients, poseidon, VarBaseMul, EndoMul, EndoMulScalar, optional), d4 (generic, CompleteAdd), sid
    const size_t n8 = PERMUTS + COLUMNS + 4 + n_opt, b8 = 8 * n * sizeof(fe), b4 = 4 * n * sizeof(fe);
    auto c = std::make_unique<zk_index_cache>();
    c->ctx = ctx;
    c->field = T::id;
    std::vector<uint32_t> tags8;
    for (unsigned i = 0; i < PERMUTS; i++) tags8.push_back(0x30 + i);
    for (unsigned i = 0; i < COLUMNS; i++) tags8.push_back(0x10 + i);
    for (uint32_t t : {0x21u, 0x23u, 0x24u, 0x25u}) tags8.push_back(t);
    for (unsigned b = 0; b < OPTIONAL_BITS; b++)
        if ((opt >> b) & 1) tags8.push_back(0x40 + b);
    // the section table in the order of the reference's writer (sid, coefficients8, permutation_coefficients8, selectors, optional)
    auto off8 = [&](uint32_t tag) { return (uint64_t)(std::find(tags8.begin(), tags8.end(), tag) - tags8.begin()) * b8; };
    const uint64_t o4 = n8 * b8, o_sid = o4 + 2 * b4;
    c->sections.push_back({0x01, o_sid, n * sizeof(fe), (uint32_t)n});
    for (unsigned i = 0; i < COLUMNS; i++) c->sections.push_back({0x10 + i, off8(0x10 + i), b8, (uint32_t)(8 * n)});
    for (unsigned i = 0; i < PERMUTS; i++) c->sections.push_back({0x30 + i, off8(0x30 + i), b8, (uint32_t)(8 * n)});
    c->sections.push_back({0x20, o4, b4, (uint32_t)(4 * n)});
    c->sections.push_back({0x21, off8(0x21), b8, (uint32_t)(8 * n)});
    c->sections.push_back({0x22, o4 + b4, b4, (uint32_t)(4 * n)});
    for (uint32_t t : {0x23u, 0x24u, 0x25u}) c->sections.push_back({t, off8(t), b8, (uint32_t)(8 * n)});
    for (unsigned b = 0; b < OPTIONAL_BITS; b++)
        if ((opt >> b) & 1) c->sections.push_back({0x40 + b, off8(0x40 + b), b8, (uint32_t)(8 * n)});
    c->hdr = *hdr;
    c->hdr.num_sections = (uint32_t)c->sections.size();
    c->hdr.identifier[sizeof(c->hdr.identifier) - 1] = 0;
    c->lo = 0;
    c->hi = o_sid + n * sizeof(fe);

    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    PinnedSlots* pin = ctx_pinned(ctx);
    if (!pin) return ZK_ERR_CUDA;
    if (int rc = ctx_ntt_table_ptrs(ctx, T::id, log_n, false, &a.ulo, &a.mid, &a.hi2)) return rc;
    if (int rc = c->payload.ensure(c->hi)) return rc;
    // inputs: gates | coefficient records | their offsets | shifts | flag, and the k x n column scratch (both freed on return)
    Layout in;
    const size_t o_g = in.add(n_gates * GATE_BYTES), o_c = in.add(gate_coeffs_len), o_off = in.add(n_gates * sizeof(uint64_t)),
                 o_sh = in.add(PERMUTS * sizeof(fe)), o_bad = in.add(sizeof(unsigned));
    DevScratch d_in, d_cols;
    if (int rc = d_in.ensure(in.total)) return rc;
    if (int rc = d_cols.ensure(k * n * sizeof(fe))) return rc;
    if (n_gates) {
        ZK_CUDA(cudaMemcpyAsync(d_in.at<uint8_t>(o_g), gates, n_gates * GATE_BYTES, cudaMemcpyHostToDevice, st));
        ZK_CUDA(cudaMemcpyAsync(d_in.at<uint64_t>(o_off), coeff_off.data(), n_gates * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
    }
    if (gate_coeffs_len) ZK_CUDA(cudaMemcpyAsync(d_in.at<uint8_t>(o_c), gate_coeffs, gate_coeffs_len, cudaMemcpyHostToDevice, st));
    ZK_CUDA(cudaMemcpyAsync(d_in.at<fe>(o_sh), hdr->shift, PERMUTS * sizeof(fe), cudaMemcpyHostToDevice, st));
    ZK_CUDA(cudaMemsetAsync(d_in.at<unsigned>(o_bad), 0, sizeof(unsigned), st));
    a.gates = d_in.at<uint8_t>(o_g);
    a.coeffs = d_in.at<uint8_t>(o_c);
    a.coeff_off = d_in.at<uint64_t>(o_off);
    a.shift = d_in.at<fe>(o_sh);
    a.cols = d_cols.at<fe>();
    a.sid = c->payload.at<fe>(o_sid);
    a.n = n;
    a.n_gates = n_gates;
    a.zero_lo = n + 2 - hdr->zk_rows;                      // constraints.rs:516-530
    a.zero_hi = n - 1;
    a.bad = d_in.at<unsigned>(o_bad);
    k_index_columns<F><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a);
    ZK_CUDA(cudaGetLastError());
    ctx->launches += 1;
    fe* cols = d_cols.at<fe>();
    fe* p8 = c->payload.at<fe>();
    fe* p4 = c->payload.at<fe>(o4);
    if (int rc = ntt_groups(ctx, T::id, cols, n, cols, log_n, k, 0, /* inverse = */ 1)) return rc;
    if (int rc = ntt_groups(ctx, T::id, cols, n, p8, log_n + 3, built8, n, 0)) return rc;
    if (int rc = ntt_groups(ctx, T::id, cols + built8 * n, n, p4, log_n + 2, built4, n, 0)) return rc;
    if (zero_selectors) {                                   // selector_polynomial: DP::zero().evaluate_over_domain_by_ref
        ZK_CUDA(cudaMemsetAsync(c->payload.at<uint8_t>(built8 * b8), 0, (n8 - built8) * b8, st));
        ZK_CUDA(cudaMemsetAsync(c->payload.at<uint8_t>(o4 + b4), 0, b4, st));
    }
    ZK_CUDA(cudaMemcpyAsync(&pin->index_bad, a.bad, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    ZK_CUDA(cudaStreamSynchronize(st));
    if (pin->index_bad) { zk_set_error("index_build: a gate coefficient is not a canonical field element"); return ZK_ERR_INVALID; }
    *out = c.release();
    return ZK_OK;
}

template <class C>
static int index_commitments_impl(zk_srs* srs, size_t n, const std::vector<IndexCommitment>& cols, size_t chunks, uint64_t* out_xy) {
    using namespace host;
    using HP = typename C::HP;
    const size_t k = cols.size();
    zk_ctx* ctx = srs->ctx;
    const zk_bases* basis = srs->lagrange.at(n);
    std::vector<uint64_t> jac(12 * k * chunks);
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        ZK_CUDA(cudaSetDevice(ctx->device));
        DevScratch d_sc;                                    // the d1 sub-samples, k x n (freed on return)
        if (int rc = d_sc.ensure(k * n * sizeof(fe))) return rc;
        for (size_t j0 = 0; j0 < k; j0 += MAX_GATHER) {
            IndexGather g{};
            const unsigned cnt = (unsigned)std::min<size_t>(MAX_GATHER, k - j0);
            for (unsigned j = 0; j < cnt; j++) {
                g.src[j] = cols[j0 + j].evals;
                g.stride[j] = cols[j0 + j].stride;
            }
            g.out = d_sc.at<fe>() + j0 * n;
            g.n = n;
            k_index_gather<<<dim3((unsigned)((n + 255) / 256), cnt), 256, 0, ctx->stream>>>(g);
            ZK_CUDA(cudaGetLastError());
            ctx->launches += 1;
        }
        // PolyComm::multi_scalar_mul (commitment.rs:350-394): chunk c of a commitment is the MSM of its scalars over chunk c of the basis
        std::vector<const fe*> sc(k * chunks);
        std::vector<size_t> offs(k * chunks);
        for (size_t j = 0; j < k; j++)
            for (size_t c = 0; c < chunks; c++) { sc[j * chunks + c] = d_sc.at<fe>() + j * n; offs[j * chunks + c] = c * n; }
        if (int rc = ctx_msm_many_offs(ctx, basis, offs.data(), n, sc.data(), k * chunks, /* mont = */ 1, 0, jac.data())) return rc;
    }
    haffine h;
    memcpy(&h, srs->h, sizeof(h));
    for (size_t j = 0; j < k; j++) {
        for (size_t c = 0; c < chunks; c++) {
            hjac q;
            memcpy(&q, jac.data() + 12 * (j * chunks + c), sizeof(q));
            hxyzz p = from_jacobian<HP>(q);
            if (cols[j].masked) p = padd<HP>(p, from_affine<HP>(h));     // mask_fixed: blinder one, every chunk + h
            const haffine r = to_affine<HP>(p);
            memcpy(out_xy + 8 * (j * chunks + c), &r, sizeof(r));
        }
    }
    return ZK_OK;
}

int index_commitments(zk_srs* srs, size_t n, const std::vector<IndexCommitment>& cols, uint64_t* out_xy) {
    if (int rc = zk_srs_lagrange_basis(srs, n, -1)) return rc;      // get_lagrange_basis (ipa.rs:780-795)
    const size_t chunks = zk_srs_lagrange_basis_chunks(srs, n);
    return with_curve(srs->curve, [&](auto c) { return index_commitments_impl<decltype(c)>(srs, n, cols, chunks, out_xy); });
}

}  // namespace zkb

extern "C" {

int zk_index_build(zk_ctx* ctx, int field_id, const zk_index_header* hdr, const void* gates, size_t n_gates, const void* gate_coeffs,
                   size_t gate_coeffs_len, int zero_selectors, zk_index_cache** out) {
    if (out) *out = nullptr;
    if (!ctx || !hdr || !out || (!gates && n_gates) || (!gate_coeffs && gate_coeffs_len)) { zk_set_error("index_build: null argument"); return ZK_ERR_INVALID; }
    if (int rc = check_field("index_build", field_id)) return rc;
    const uint64_t n = hdr->domain_d1_size;
    if (n == 0 || (n & (n - 1)) || n > ((uint64_t)1 << MAX_LOG_N)) {
        zk_set_error("index_build: d1 size %llu is not a power of two up to 2^%zu", (unsigned long long)n, MAX_LOG_N);
        return ZK_ERR_INVALID;
    }
    if (hdr->zk_rows < 3 || hdr->zk_rows >= n) { zk_set_error("index_build: zk_rows %llu is not in [3, %llu)", (unsigned long long)hdr->zk_rows, (unsigned long long)n); return ZK_ERR_INVALID; }
    if (n_gates > n) { zk_set_error("index_build: %zu gates do not fit the domain of %llu rows", n_gates, (unsigned long long)n); return ZK_ERR_INVALID; }
    if (hdr->optional_selectors_present >> OPTIONAL_BITS) { zk_set_error("index_build: optional selector bits %#x beyond bit 5", hdr->optional_selectors_present); return ZK_ERR_INVALID; }
    for (unsigned k = 0; k < PERMUTS; k++)
        if (!canonical(field_id, hdr->shift[k])) { zk_set_error("index_build: shift %u is not a canonical field element", k); return ZK_ERR_INVALID; }
    const uint8_t* g = (const uint8_t*)gates;
    for (size_t r = 0; r < n_gates; r++) {
        const uint8_t* rec = g + r * GATE_BYTES;
        const unsigned tag = (unsigned)rec[0] | (unsigned)rec[1] << 8;
        if (tag > MAX_TAG) { zk_set_error("index_build: gate %zu has tag %u > %u", r, tag, MAX_TAG); return ZK_ERR_INVALID; }
        for (unsigned k = 0; k < PERMUTS; k++) {
            const uint32_t row = rd32(rec + 4 + 8 * k), col = rd32(rec + 8 + 8 * k);
            if (row >= n || col >= PERMUTS) { zk_set_error("index_build: gate %zu wire %u points at (%u, %u), outside %llu x 7", r, k, row, col, (unsigned long long)n); return ZK_ERR_INVALID; }
        }
    }
    // the coefficient records are variable-length: one walk over the counts gives each gate's offset
    const uint8_t* gc = (const uint8_t*)gate_coeffs;
    std::vector<uint64_t> off(n_gates);
    size_t pos = 0;
    for (size_t r = 0; r < n_gates; r++) {
        if (gate_coeffs_len - pos < 4) { zk_set_error("index_build: gate_coeffs ends inside record %zu of %zu", r, n_gates); return ZK_ERR_INVALID; }
        const uint64_t cnt = rd32(gc + pos);
        if ((gate_coeffs_len - pos - 4) / 32 < cnt) { zk_set_error("index_build: gate_coeffs ends inside record %zu of %zu", r, n_gates); return ZK_ERR_INVALID; }
        off[r] = pos;
        pos += 4 + 32 * cnt;
    }
    if (pos != gate_coeffs_len) { zk_set_error("index_build: gate_coeffs holds %zu bytes past the %zu records", gate_coeffs_len - pos, n_gates); return ZK_ERR_INVALID; }
    return with_field(field_id, [&](auto f) {
        return index_build_impl<decltype(f)>(ctx, hdr, g, n_gates, gc, gate_coeffs_len, off, zero_selectors != 0, out);
    });
}

int zk_index_commitments(zk_srs* srs, const zk_index_cache* index, uint64_t* out_xy, size_t capacity_points, size_t* out_points) {
    if (!srs || !index || !out_xy || !out_points) { zk_set_error("index_commitments: null argument"); return ZK_ERR_INVALID; }
    const int sf = with_curve(srs->curve, [](auto c) { return decltype(c)::scalar_field; });
    if (index->field >= 0 && index->field != sf) { zk_set_error("index_commitments: the index is over field %d, the SRS's scalars over %d", index->field, sf); return ZK_ERR_INVALID; }
    const uint64_t n = index->hdr.domain_d1_size;
    // verifier_index.rs:221-300: sigma_comm, coefficients_comm, generic, psm, complete_add, mul, emul, endomul_scalar, optional selectors
    std::vector<uint32_t> tags;
    for (unsigned i = 0; i < PERMUTS; i++) tags.push_back(0x30 + i);
    for (unsigned i = 0; i < COLUMNS; i++) tags.push_back(0x10 + i);
    for (uint32_t t = 0x20; t <= 0x25; t++) tags.push_back(t);
    for (unsigned b = 0; b < 32; b++)
        if ((index->hdr.optional_selectors_present >> b) & 1) tags.push_back(0x40 + b);
    std::vector<IndexCommitment> cols;
    for (uint32_t t : tags) {
        const zk_index_cache::Section* s = nullptr;
        for (const auto& o : index->sections)
            if (o.tag == t) s = &o;
        if (!s) { zk_set_error("index_commitments: section %#x missing", t); return ZK_ERR_INVALID; }
        const uint64_t len = s->length / sizeof(fe);
        if (len == 0 || len % n || len / n > UINT32_MAX) { zk_set_error("index_commitments: section %#x has %llu elements, not a multiple of %llu", t, (unsigned long long)len, (unsigned long long)n); return ZK_ERR_INVALID; }
        // the six fixed selectors (generic .. endomul_scalar) are masked
        cols.push_back({index->payload.at<fe>(s->offset - index->lo), (uint32_t)(len / n), cols.size() >= PERMUTS + COLUMNS && cols.size() < PERMUTS + COLUMNS + 6});
    }
    const size_t chunks = zk_srs_lagrange_basis_chunks(srs, n);
    *out_points = cols.size() * chunks;
    if (capacity_points < *out_points) { zk_set_error("index_commitments: %zu points do not fit the capacity %zu", *out_points, capacity_points); return ZK_ERR_INVALID; }
    return index_commitments(srs, n, cols, out_xy);
}

}  // extern "C"
