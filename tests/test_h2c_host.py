"""The code k_srs_generate runs (proof_systems_b200/csrc/hash_to_curve.cuh and field_sqrt.cuh), compiled for the host with the
PTX carry chains emulated (field.cuh), against hashlib and the Python restatement of `SRS::create` (tests/srs_create_replay.py):
Blake2b-512, the digest packing, the BW constants and group map, and the shared Tonelli-Shanks square root."""
import ctypes
import hashlib
import os
import random
import subprocess

import pytest

import srs_create_replay as rp
from kimchi_transcript import FP, FQ, BWGroupMap, sqrt_ark

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_math", "h2c_host.cpp")
SO = os.path.join(HERE, "host_math", "libh2c_host.so")
CSRC = os.path.join(os.path.dirname(HERE), "proof_systems_b200", "csrc")
MOD = {0: FP, 1: FQ}                      # field id: Fp (Pallas base field), Fq (Vesta base field)
R = 1 << 256


@pytest.fixture(scope="module")
def h2c():
    deps = [SRC] + [os.path.join(CSRC, f) for f in ("field.cuh", "field_sqrt.cuh", "hash_to_curve.cuh")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", SO, SRC])
    return ctypes.CDLL(SO)


def limbs(x: int):
    return (ctypes.c_uint32 * 8)(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(8)])


def value(a) -> int:
    return sum(int(w) << (32 * i) for i, w in enumerate(a))


def from_mont(a, fid) -> int:
    return value(a) * pow(R, -1, MOD[fid]) % MOD[fid]


def device_to_group(h2c, fid, t):
    x, y = limbs(0), limbs(0)
    assert h2c.h2c_to_group(fid, limbs(t), x, y) == 1
    return from_mont(x, fid), from_mont(y, fid)


def test_blake2b_equals_hashlib(h2c):
    rng = random.Random(3)
    msgs = [(0).to_bytes(4, "big"), (65535).to_bytes(4, "big"), ((1 << 32) - 1).to_bytes(4, "big"), b"srs_misc" + bytes(4), b"",
            b"\x00", b"abc"] + [rng.randbytes(n) for n in (1, 8, 31, 64, 100, 127, 128)]
    for msg in msgs:
        out = (ctypes.c_uint8 * 64)()
        assert h2c.h2c_blake2b(msg, len(msg), out) == 0
        assert bytes(out) == hashlib.blake2b(msg, digest_size=64).digest(), msg


def test_digest_packing_equals_the_restatement(h2c):
    rng = random.Random(4)
    digests = [rp.digest(i.to_bytes(4, "big")) for i in range(64)] + [rng.randbytes(64) for _ in range(64)] + [bytes(64), b"\xff" * 64]
    for d in digests:
        t = limbs(0)
        h2c.h2c_digest_to_field(d, t)
        assert value(t) == rp.pack(d), d.hex()


@pytest.mark.parametrize("fid", [0, 1])
def test_bw_constants_equal_setup(h2c, fid):
    m = BWGroupMap(MOD[fid])
    out = (ctypes.c_uint32 * 32)()
    h2c.h2c_bw_consts(fid, out)
    got = [from_mont(out[8 * c:8 * c + 8], fid) for c in range(4)]
    assert got == [m.fu, m.inv_three_u_squared, m.sqrt_neg_three_u_squared, m.sqrt_neg_three_u_squared_minus_u_over_2]


@pytest.mark.parametrize("fid", [0, 1])
def test_square_root_is_arks_root(h2c, fid):
    p = MOD[fid]
    rng = random.Random(5 + fid)
    for a in [0, 1, 2, 3, 4, 5, p - 1, p - 3] + [rng.randrange(p) for _ in range(200)]:
        out = limbs(0)
        ok = h2c.h2c_sqrt(fid, limbs(a * R % p), out)
        want = sqrt_ark(a, p)
        assert bool(ok) == (want is not None), a
        if ok:
            assert from_mont(out, fid) == want, a


@pytest.mark.parametrize("fid", [0, 1])
def test_group_map_equals_the_restatement_at_hashed_t(h2c, fid):
    """Every candidate is reached: the sample includes t whose first and whose second candidate are off the curve."""
    m = BWGroupMap(MOD[fid])
    used = set()
    for i in list(range(96)) + [40000, 65535, 1 << 20, (1 << 32) - 1]:
        t = rp.pack(rp.digest(i.to_bytes(4, "big")))
        want = m.to_group(t)
        assert device_to_group(h2c, fid, t) == want, i
        x, y = limbs(0), limbs(0)
        assert h2c.h2c_point_of_message(fid, i.to_bytes(4, "big"), 4, x, y) == 1
        assert (from_mont(x, fid), from_mont(y, fid)) == want, i
        t2 = t * t % m.p
        alpha = pow(t2 * (t2 + m.fu) % m.p, -1, m.p)
        x1 = (m.sqrt_neg_three_u_squared_minus_u_over_2 - t2 * t2 % m.p * alpha % m.p * m.sqrt_neg_three_u_squared) % m.p
        used.add(0 if want[0] == x1 else 1 if want[0] == (-m.u - x1) % m.p else 2)
    assert used == {0, 1, 2}
    x, y = limbs(0), limbs(0)
    assert h2c.h2c_point_of_message(fid, b"srs_misc" + bytes(4), 12, x, y) == 1
    assert (from_mont(x, fid), from_mont(y, fid)) == rp.blinder(fid)


@pytest.mark.parametrize("fid", [0, 1])
def test_group_map_where_alpha_is_zero(h2c, fid):
    """t^2 (t^2 + fu) = 0 makes alpha zero (the reference's unwrap_or_else(zero)); no hashed t reaches it.  t = 0 always does,
    and so does a root of t^2 = -fu where -6 is a square."""
    m = BWGroupMap(MOD[fid])
    ts = [0]
    r = sqrt_ark(-m.fu, m.p)
    if r is not None:
        ts += [r, m.p - r]
    for t in ts:
        assert device_to_group(h2c, fid, t) == m.to_group(t), t
