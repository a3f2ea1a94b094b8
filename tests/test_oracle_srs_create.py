"""`SRS::create(depth)` restated in Python (tests/srs_create_replay.py) against the generators the reference ships: every
g[i] of srs/{pallas,vesta}.srs (the fixtures' g_cmp) and h (h_xy).  The reference's own heavy_test_srs_serialization
(precomputed_srs.rs:156-234) asserts SRS::create(2^16) == srs/*.srs, so these bytes are create's output."""
import random

import pytest

import srs_create_replay as rp
from kimchi_transcript import FP, FQ, BWGroupMap, sqrt_ark

CURVES = [("pallas_srs", rp.PALLAS), ("vesta_srs", rp.VESTA)]


def sample_indices(n=65536):
    rng = random.Random(2024)
    return list(range(256)) + list(range(256, n, 997)) + rng.sample(range(256, n), 40) + [n - 1]


@pytest.mark.parametrize("name,curve", CURVES)
def test_generators_and_h_equal_the_shipped_srs(request, name, curve):
    G = request.getfixturevalue(name)
    for i in sample_indices(G.g_cmp.shape[0]):
        assert rp.compress(curve, rp.generator(curve, i)) == G.g_cmp[i].tobytes(), i
    assert rp.xy_bytes(rp.blinder(curve)) == G.h_xy_canon.tobytes()


@pytest.mark.parametrize("p", [FP, FQ])
def test_bw_constants_are_what_setup_derives(p):
    """BWParameters::setup (groupmap/src/lib.rs) for y^2 = x^3 + 5: u is the first u >= 1 with u^3 + 5 != 0, and the three
    derived constants satisfy their defining equations; the root is the one ark's Tonelli-Shanks returns."""
    m = BWGroupMap(p)
    assert (m.u, m.fu) == (1, 6)
    three_u2 = 3 * m.u * m.u % p
    assert m.inv_three_u_squared * three_u2 % p == 1
    assert m.sqrt_neg_three_u_squared ** 2 % p == (-three_u2) % p
    assert m.sqrt_neg_three_u_squared == sqrt_ark(-three_u2, p)
    assert (2 * m.sqrt_neg_three_u_squared_minus_u_over_2 + m.u) % p == m.sqrt_neg_three_u_squared


@pytest.mark.parametrize("name,curve", CURVES)
def test_packing_is_bit_reversed_big_endian(request, name, curve):
    """Only the reading the reference uses reproduces g[0]: a little-endian reading of the same 31 bytes, or big-endian bytes
    without the bit reversal, gives another point."""
    G = request.getfixturevalue(name)
    d = rp.digest((0).to_bytes(4, "big"))
    m = rp.group_map(curve)
    assert rp.compress(curve, m.to_group(rp.pack(d))) == G.g_cmp[0].tobytes()
    assert rp.pack(d) == int("".join(format(b, "08b")[::-1] for b in d[:31]), 2)      # bits[8i + j] = (d[i] >> j) & 1, MSB first
    for wrong in (int.from_bytes(d[:31], "little"), int.from_bytes(d[:31], "big")):
        assert rp.compress(curve, m.to_group(wrong)) != G.g_cmp[0].tobytes()

