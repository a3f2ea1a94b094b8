// ipa.hpp — state of the device-resident IPA folding rounds (ipa.cu), shared with the opening proof (open.cu).
#pragma once
#include "ctx.hpp"

struct zk_ipa {
    using fe = zkb::fe;
    using affine_t = zkb::affine_t;
    zk_ctx* ctx = nullptr;
    int curve = 0;
    size_t n = 0;           // current length (halves every fold)
    size_t n0 = 0;          // original (padded) length
    const zk_bases* bases = nullptr;
    fe* d_s[2] = {nullptr, nullptr};   // b_poly_coefficients of the challenges so far (ping-pong), Montgomery
    int cur = 0;
    fe* d_sc = nullptr;     // expanded MSM scalars of L and of R, 2 x n0 entries, Montgomery
    fe* d_a = nullptr;      // a | b | s0 | s1 | sc_L | sc_R | partials (ipa_storage_bytes): in `storage`, or in a buffer of the context
                            // (zk_srs_open reuses it call after call)
    fe* d_b = nullptr;
    fe* d_part = nullptr;   // inner-product partials
    fe* h_ip = nullptr;     // the context's pinned PinnedSlots::ip: two field elements
    // SRS::open (open.cu): h and the fresh base U travel as extra points of every round's MSMs (ipa.rs:944,954), their scalars
    // (rand_l | rand_r of the round, and the round's two inner products) are appended on the device
    affine_t* d_extra = nullptr;   // [max(1, nwin)][2] rows of (h, U); null for the bare rounds of zk_ipa_*
    fe* d_rand = nullptr;          // [2 * rounds] rand_l, rand_r per round (Montgomery)
    unsigned round = 0;
    zkb::DevScratch storage;
};


namespace zkb {
constexpr unsigned IP_THREADS = 256, IP_BLOCKS = 64;
// the calls below assume the context lock is held and the device is current (so does `delete` of a zk_ipa)
// a, b uninitialised device vectors of n elements; storage: null (own allocation) or ipa_storage_bytes(n) bytes of device memory
int ipa_create(zk_ctx* ctx, const zk_bases* bases, size_t n, zk_ipa** out, void* storage = nullptr);
size_t ipa_storage_bytes(size_t n);
int ipa_round_lr(zk_ipa* s, uint64_t out_l_xyz[12], uint64_t out_r_xyz[12], uint64_t out_ip_l[4], uint64_t out_ip_r[4]);
int ipa_round_fold(zk_ipa* s, const uint64_t u_mont[4], const uint64_t u_inv_mont[4]);
template <class FS> int ipa_inner_product(zk_ipa* s, const fe* x, const fe* y, size_t m, fe* d_out);
}  // namespace zkb
