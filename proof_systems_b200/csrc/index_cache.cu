// index_cache.cu — device-side ingestion of kimchi's mmap-backed proving-key cache (SURVEY.md §8f row 4, second half).
//
// kimchi/src/cached_prover_index.rs:26-56 ("MINAPK01", format version 3) stores every big array of the prover index — the 15
// coefficient columns and the 7 permutation-coefficient columns over d8, the gate selectors over d4 / d8, sid, the lookup
// tables — as raw MONTGOMERY limbs, four little-endian u64 per field element, 32-byte aligned, precisely so that the reader can
// point `Vec<F>` into the mapping without touching the data (:41-49, :486-530).  That is also this library's device format, so
// ingestion is a parse of the fixed header and the section table on the host and ONE host-to-device copy of the payload as it
// lies in the mapping: no per-element decoding anywhere.  The sections then serve as resident operands of the pointwise
// evaluators (zk_perm_quotient_dev takes permutation_coefficients8 from here).
//
// Layout restated from the reference's writer (:560-760):
//   preamble       magic[8] "MINAPK01" | format_version u32 | reserved u32 | ark-ff version[32] | identifier_len u32 |
//                  identifier[512] | num_sections u32
//   ScalarHeader   public u32 | prev_challenges u32 | zk_rows u64 | max_poly_size u64 | disable_gates_checks u8 | pad[7] |
//                  domain_d1_size u64 | feature_flags u32 | optional_selectors_present u32 | lookup_selectors_present u32 |
//                  has_verifier_index_digest u8 | pad[3] | endo[4 u64] | shift[7][4 u64] | verifier_index_digest[4 u64]
//   section table  num_sections x { tag u32 | offset u64 | length u64 | elem_domain_size u32 | reserved u32 }
//   payload        sections at their offsets (from the start of the file), each 32-byte aligned
#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/zkb200.h"
#include "ctx.hpp"

using namespace zkb;

namespace {

constexpr size_t ARK_FF_VERSION_MAX_LEN = 32, IDENTIFIER_MAX_LEN = 512, PERMUTS = 7;
constexpr size_t PREAMBLE_SIZE = 8 + 4 + 4 + ARK_FF_VERSION_MAX_LEN + 4 + IDENTIFIER_MAX_LEN + 4;
constexpr size_t SCALAR_HEADER_SIZE = 4 + 4 + 8 + 8 + 1 + 7 + 8 + 4 + 4 + 4 + 1 + 3 + 32 + 32 * PERMUTS + 32;
constexpr size_t SECTION_ENTRY_SIZE = 4 + 8 + 8 + 4 + 4;
constexpr uint32_t FORMAT_VERSION = 3;

uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
uint64_t rd64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }

// sections whose payload is an array of field elements (SectionTag, cached_prover_index.rs:74-140)
bool is_field_section(uint32_t tag) {
    return tag == 0x01 || (tag >= 0x10 && tag <= 0x1E) || (tag >= 0x20 && tag <= 0x25) || (tag >= 0x30 && tag <= 0x36) ||
           (tag >= 0x40 && tag <= 0x45) || (tag >= 0x50 && tag <= 0x56);
}

}  // namespace

extern "C" {

int zk_index_cache_load(zk_ctx* ctx, const void* image, size_t image_len, const char* expect_identifier, zk_index_cache** out) {
    if (!ctx || !image || !out) { zk_set_error("index_cache_load: null argument"); return ZK_ERR_INVALID; }
    *out = nullptr;
    const uint8_t* p = (const uint8_t*)image;
    if (image_len < PREAMBLE_SIZE + SCALAR_HEADER_SIZE) { zk_set_error("index_cache: cache file truncated before end of declared payload"); return ZK_ERR_INVALID; }
    if (memcmp(p, "MINAPK01", 8) != 0) { zk_set_error("index_cache: bad file magic"); return ZK_ERR_INVALID; }
    const uint32_t version = rd32(p + 8);
    if (version != FORMAT_VERSION) { zk_set_error("index_cache: unsupported cache format version %u (this build supports %u)", version, FORMAT_VERSION); return ZK_ERR_INVALID; }
    const uint8_t* ark = p + 16;
    if (strncmp((const char*)ark, "ark-ff-0.5", ARK_FF_VERSION_MAX_LEN) != 0) {
        zk_set_error("index_cache: ark-ff version mismatch: file declares %.32s, expected ark-ff-0.5", (const char*)ark);
        return ZK_ERR_INVALID;
    }
    const uint32_t id_len = rd32(p + 16 + ARK_FF_VERSION_MAX_LEN);
    const uint8_t* id = p + 16 + ARK_FF_VERSION_MAX_LEN + 4;
    if (id_len > IDENTIFIER_MAX_LEN) { zk_set_error("index_cache: identifier length %u exceeds maximum %zu", id_len, IDENTIFIER_MAX_LEN); return ZK_ERR_INVALID; }
    if (expect_identifier && (strlen(expect_identifier) != id_len || memcmp(expect_identifier, id, id_len) != 0)) {
        zk_set_error("index_cache: cache file identifier mismatch");
        return ZK_ERR_INVALID;
    }
    const uint32_t num_sections = rd32(id + IDENTIFIER_MAX_LEN);
    const uint8_t* h = p + PREAMBLE_SIZE;
    auto c = std::make_unique<zk_index_cache>();
    c->ctx = ctx;
    zk_index_header& H = c->hdr;
    H.public_inputs = rd32(h); H.prev_challenges = rd32(h + 4); H.zk_rows = rd64(h + 8); H.max_poly_size = rd64(h + 16);
    H.disable_gates_checks = h[24] != 0;
    H.domain_d1_size = rd64(h + 32);
    H.feature_flags = rd32(h + 40); H.optional_selectors_present = rd32(h + 44); H.lookup_selectors_present = rd32(h + 48);
    H.has_verifier_index_digest = h[52] != 0;
    memcpy(H.endo, h + 56, 32);
    memcpy(H.shift, h + 88, 32 * PERMUTS);
    memcpy(H.verifier_index_digest, h + 88 + 32 * PERMUTS, 32);
    H.num_sections = num_sections;
    memcpy(H.identifier, id, id_len);
    H.identifier[id_len < IDENTIFIER_MAX_LEN ? id_len : IDENTIFIER_MAX_LEN - 1] = 0;
    if (H.domain_d1_size == 0 || (H.domain_d1_size & (H.domain_d1_size - 1)) || H.domain_d1_size > ((uint64_t)1 << 29)) {
        zk_set_error("index_cache: stored d1 domain size %llu is not a valid evaluation domain", (unsigned long long)H.domain_d1_size);
        return ZK_ERR_INVALID;
    }
    const size_t table_off = PREAMBLE_SIZE + SCALAR_HEADER_SIZE;
    if (image_len < table_off + (size_t)num_sections * SECTION_ENTRY_SIZE) { zk_set_error("index_cache: cache file truncated before end of declared payload"); return ZK_ERR_INVALID; }
    uint64_t lo = UINT64_MAX, hi = 0;
    for (uint32_t s = 0; s < num_sections; s++) {
        const uint8_t* e = p + table_off + (size_t)s * SECTION_ENTRY_SIZE;
        zk_index_cache::Section sec{rd32(e), rd64(e + 4), rd64(e + 12), rd32(e + 20)};
        for (const auto& o : c->sections)
            if (o.tag == sec.tag) { zk_set_error("index_cache: duplicate section tag %#x in section table", sec.tag); return ZK_ERR_INVALID; }
        if (sec.offset % 32) { zk_set_error("index_cache: section %#x offset %llu is not 32-byte aligned", sec.tag, (unsigned long long)sec.offset); return ZK_ERR_INVALID; }
        if (sec.offset > image_len || sec.length > image_len - sec.offset) { zk_set_error("index_cache: cache file truncated before end of declared payload"); return ZK_ERR_INVALID; }
        if (is_field_section(sec.tag)) {
            if (sec.length % 32) { zk_set_error("index_cache: section %#x payload length %llu is not a multiple of 32", sec.tag, (unsigned long long)sec.length); return ZK_ERR_INVALID; }
            if (sec.elem_domain_size && sec.tag != 0x50 && sec.length != (uint64_t)sec.elem_domain_size * 32) {
                zk_set_error("index_cache: section %#x length mismatch: expected %llu, found %llu", sec.tag, (unsigned long long)sec.elem_domain_size * 32, (unsigned long long)sec.length);
                return ZK_ERR_INVALID;
            }
            if (sec.length) { lo = std::min(lo, sec.offset); hi = std::max(hi, sec.offset + sec.length); }
        }
        c->sections.push_back(sec);
    }
    // the 7 permutation-coefficient columns and the 15 coefficient columns are required (cached_prover_index.rs: MissingSection)
    for (uint32_t tag : {0x30u, 0x31u, 0x32u, 0x33u, 0x34u, 0x35u, 0x36u}) {
        bool found = false;
        for (const auto& o : c->sections) found |= o.tag == tag;
        if (!found) { zk_set_error("index_cache: required section tag %#x missing from section table", tag); return ZK_ERR_INVALID; }
    }
    std::lock_guard<std::mutex> lk(ctx->mu);
    ZK_CUDA(cudaSetDevice(ctx->device));
    if (hi > lo) {
        c->lo = lo; c->hi = hi;
        if (int rc = c->payload.ensure(hi - lo)) return rc;
        // ONE copy of the payload as it lies in the mapping: the bytes are already the device's field-element format
        cudaError_t e = cudaMemcpyAsync(c->payload.p, p + lo, hi - lo, cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) { zk_set_error("index_cache: %s", cudaGetErrorString(e)); return ZK_ERR_CUDA; }
    }
    *out = c.release();
    return ZK_OK;
}

void zk_index_cache_free(zk_index_cache* c) {
    if (!c) return;
    std::lock_guard<std::mutex> lk(c->ctx->mu);
    cudaSetDevice(c->ctx->device);
    cudaStreamSynchronize(c->ctx->stream);
    delete c;
}

int zk_index_cache_header(const zk_index_cache* c, zk_index_header* out) {
    if (!c || !out) { zk_set_error("index_cache_header: null argument"); return ZK_ERR_INVALID; }
    *out = c->hdr;
    return ZK_OK;
}

// Device pointer, element count and declared evaluation-domain size of a field-element section; ZK_ERR_INVALID if the file has none
// with this tag (optional selectors) or the section is not an array of field elements (gates, runtime-table specs).
int zk_index_cache_section(const zk_index_cache* c, uint32_t tag, const void** d_ptr, size_t* n_elems, uint32_t* elem_domain_size) {
    if (!c || !d_ptr || !n_elems) { zk_set_error("index_cache_section: null argument"); return ZK_ERR_INVALID; }
    for (const auto& s : c->sections) {
        if (s.tag != tag) continue;
        if (!is_field_section(tag)) { zk_set_error("index_cache_section: section %#x does not hold field elements", tag); return ZK_ERR_INVALID; }
        *d_ptr = s.length ? c->payload.at<uint8_t>(s.offset - c->lo) : nullptr;
        *n_elems = s.length / 32;
        if (elem_domain_size) *elem_domain_size = s.elem_domain_size;
        return ZK_OK;
    }
    zk_set_error("index_cache_section: required section tag %#x missing from section table", tag);
    return ZK_ERR_INVALID;
}

}  // extern "C"
