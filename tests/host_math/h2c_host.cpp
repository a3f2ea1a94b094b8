// tests/host_math/h2c_host.cpp — compiles hash_to_curve.cuh (Blake2b-512, the digest packing, the BW group map and the shared
// Tonelli-Shanks square root) for the host, so that the code k_srs_generate runs can be checked without a GPU
// (tests/test_h2c_host.py).  Test infrastructure only.
#include <cstring>

#include "../../proof_systems_b200/csrc/hash_to_curve.cuh"
using namespace zkb;

static void pack_message(const uint8_t* msg, unsigned len, uint64_t (&m)[16]) {
    memset(m, 0, sizeof m);
    for (unsigned i = 0; i < len; i++) m[i / 8] |= (uint64_t)msg[i] << (8 * (i % 8));
}

extern "C" int h2c_blake2b(const uint8_t* msg, unsigned len, uint8_t* out64) {
    if (len > 128) return -1;
    uint64_t m[16], h[8];
    pack_message(msg, len, m);
    blake2b_512(m, len, h);
    for (int i = 0; i < 64; i++) out64[i] = (uint8_t)(h[i / 8] >> (8 * (i % 8)));
    return 0;
}

// digest (64 bytes) -> t, canonical 8 x u32
extern "C" void h2c_digest_to_field(const uint8_t* d64, uint32_t* t) {
    uint64_t h[8] = {};
    for (int i = 0; i < 64; i++) h[i / 8] |= (uint64_t)d64[i] << (8 * (i % 8));
    const fe r = digest_to_field(h);
    memcpy(t, r.v, 32);
}

// to_group(t): t canonical in, x and y Montgomery out; 1 on success
extern "C" int h2c_to_group(int fid, const uint32_t* t_canon, uint32_t* x, uint32_t* y) {
    fe t, rx, ry;
    memcpy(t.v, t_canon, 32);
    const bool ok = fid == 0 ? bw_to_group<FpParams>(fe_to_mont<FpParams>(t), rx, ry) : bw_to_group<FqParams>(fe_to_mont<FqParams>(t), rx, ry);
    memcpy(x, rx.v, 32);
    memcpy(y, ry.v, 32);
    return ok;
}

// point_of_random_bytes(Blake2b512(msg)): x and y Montgomery; 1 on success
extern "C" int h2c_point_of_message(int fid, const uint8_t* msg, unsigned len, uint32_t* x, uint32_t* y) {
    if (len > 128) return -1;
    uint64_t m[16];
    pack_message(msg, len, m);
    fe rx, ry;
    const bool ok = fid == 0 ? point_of_message<FpParams>(m, len, rx, ry) : point_of_message<FqParams>(m, len, rx, ry);
    memcpy(x, rx.v, 32);
    memcpy(y, ry.v, 32);
    return ok;
}

// fe_sqrt (field_sqrt.cuh): a and the root Montgomery; 1 when a is a square
extern "C" int h2c_sqrt(int fid, const uint32_t* a_mont, uint32_t* out) {
    fe a, r = fe_zero();
    memcpy(a.v, a_mont, 32);
    const bool ok = fid == 0 ? fe_sqrt<FpParams>(a, r) : fe_sqrt<FqParams>(a, r);
    memcpy(out, r.v, 32);
    return ok;
}

// the four BW constants (BW_FU, BW_INV_THREE_U2, BW_SQRT_NEG_THREE_U2, BW_SQRT_NEG_THREE_U2_MINUS_U_OVER_2), Montgomery, 4 x 8 u32
extern "C" void h2c_bw_consts(int fid, uint32_t* out) {
    for (int c = 0; c < 4; c++) {
        const fe r = fid == 0 ? bw_const<FpParams>(c) : bw_const<FqParams>(c);
        memcpy(out + 8 * c, r.v, 32);
    }
}
