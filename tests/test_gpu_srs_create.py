"""`SRS::create(depth)` on the device (zk_srs_generate, zk.SRS.create) against the generators the reference ships and against the
Python restatement (tests/srs_create_replay.py):
  heavy_test_srs_serialization (precomputed_srs.rs:156-234)   SRS::create(2^16) == srs/{pallas,vesta}.srs, byte for byte
  ser_regression_canonical_polycomm (commitment.rs:345-385)   starts from SRS::<Vesta>::create(1 << 7)
and the handle it returns is a working SRS: commitments, the 2^16 Lagrange basis of srs/test_vesta.srs, the optional host copies,
argument refusals and the caller's stream."""
import ctypes
import hashlib
import json
import os
import random

import numpy as np
import pytest
import torch

import proof_systems_b200 as zk
import srs_create_replay as rp

pytestmark = pytest.mark.gpu

SPIN = 20_000_000          # cycles of the spin kernel: about 10 ms at the H100's 1.6 to 2 GHz


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def created(ctx):
    """SRS.create(2^16) of each curve, made once for the module"""
    out = {cid: zk.SRS.create(ctx, cid, 1 << 16) for cid in (zk.PALLAS, zk.VESTA)}
    yield out
    for s in out.values():
        s.close()


def mont_of(orc, base, pt):
    """(x, y) canonical integers -> affine Montgomery [8]"""
    return orc.to_mont(base, orc.ints_to_limbs(list(pt))).reshape(8)


@pytest.mark.parametrize("name", ["pallas_srs", "vesta_srs"])
def test_create_2_16_is_the_shipped_srs(ctx, request, created, name):
    """heavy_test_srs_serialization: every one of the 65 536 generators, compressed on the device, equals srs/*.srs; h equals
    the file's h"""
    G = request.getfixturevalue(name)
    srs = created[G.cid]
    assert srs.max_poly_size() == 1 << 16 and srs.g.shape == (1 << 16, 8)
    assert np.array_equal(ctx.compress_points(G.cid, srs.g), G.g_cmp)
    assert np.array_equal(srs.h, G.mont_points(G.h_xy_canon)[0])


@pytest.mark.parametrize("name", ["pallas_srs", "vesta_srs"])
def test_small_depths_are_prefixes(ctx, request, name):
    """create(depth) for depths that are and are not powers of two: g is the first `depth` generators, h does not depend on depth"""
    G = request.getfixturevalue(name)
    h = G.mont_points(G.h_xy_canon)[0]
    for depth in (1, 2, 3, 20, 127, 128, 129, 1000):
        with zk.SRS.create(ctx, G.cid, depth) as srs:
            assert srs.max_poly_size() == depth
            assert np.array_equal(srs.g, G.g[:depth]), depth
            assert np.array_equal(srs.h, h), depth


def test_create_2_20_vesta(ctx, orc, vesta_srs):
    """Past the shipped 2^16: the prefix equals the file, seeded indices above it equal the restatement, every point is on the curve"""
    G = vesta_srs
    n = 1 << 20
    with zk.SRS.create(ctx, G.cid, n, window_bits=0) as srs:
        g = srs.g
    assert np.array_equal(g[: 1 << 16], G.g)
    idx = sorted(random.Random(20).sample(range(1 << 16, n), 512)) + [n - 1]
    for i in idx:
        assert np.array_equal(g[i], mont_of(orc, G.base, rp.generator(G.cid, i))), i
    assert all(orc.on_curve(G.cid, p) for p in g)


def test_create_128_reproduces_the_polycomm_regression(ctx, orc):
    """ser_regression_canonical_polycomm (commitment.rs:345-385) on SRS::<Vesta>::create(1 << 7) with no fixture points: the
    generators, commit_non_hiding, mask_custom and the compression all from the device"""
    from test_ser_regression import GOLDEN, msgpack_points, padded, polycomm_inputs
    coeffs, blinders = polycomm_inputs(orc)
    with zk.SRS.create(ctx, zk.VESTA, 128) as srs:
        com = srs.commit_custom(coeffs, 6, blinders)
    assert len(com) == 6
    raw = msgpack_points([bytes(p) for p in ctx.compress_points(zk.VESTA, com.chunks)], struct_prefix=b"\x91")
    want = json.load(open(GOLDEN))["polycomm_vesta_srs128_deg300_chunks6"]
    assert padded(raw, len(want)) == want


def test_lagrange_basis_of_the_created_srs(orc, created, vesta_srs):
    """get_lagrange_basis_from_domain_size(2^16) on a created 2^16 SRS is the basis stored in srs/test_vesta.srs (its sha256)"""
    G = vesta_srs
    lag = created[G.cid].get_lagrange_basis_from_domain_size(1 << 16)
    canon = orc.from_mont(G.base, np.ascontiguousarray(lag).reshape(-1, 4)).reshape(-1, 8)
    want = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vesta_srs.npz"))["lag_65536_sha256"]
    assert hashlib.sha256(canon.astype("<u8").tobytes()).digest() == want.tobytes()
    assert np.array_equal(canon[G.lag_65536_idx].view(np.uint8).reshape(-1, 64), G.lag_65536_canon)


@pytest.mark.parametrize("name", ["pallas_srs", "vesta_srs"])
def test_commitments_equal_those_on_the_fixture_points(ctx, orc, request, created, name):
    G = request.getfixturevalue(name)
    n = 1 << 16
    coeffs = orc.to_mont(G.scalar, orc.random_scalars(G.scalar, n + 5000, seed=31))
    with zk.SRS(ctx, G.cid, G.g, G.mont_points(G.h_xy_canon)[0]) as ref:
        assert np.array_equal(created[G.cid].commit_non_hiding(coeffs, 1).chunks, ref.commit_non_hiding(coeffs, 1).chunks)


@pytest.mark.parametrize("window_bits", [-1, 0])
def test_host_copies_are_what_the_handle_holds(ctx, orc, pallas_srs, window_bits):
    """g_xy_out / h_xy_out equal the resident points: an MSM over the handle's generators and mask_custom with blinder 1 (which
    adds h) agree with the host copies.  NULL outputs give the same handle; launches: the generation, plus the table if any."""
    G = pallas_srs
    n = 3000
    sc = orc.random_scalars(G.scalar, n, seed=32)
    one = orc.to_mont(G.scalar, orc.ints_to_limbs([1]))
    for with_copies in (True, False):
        before = ctx.launch_count
        if with_copies:
            srs = zk.SRS.create(ctx, G.cid, n, window_bits=window_bits)
            g, h = srs.g, srs.h
            assert np.array_equal(g, G.g[:n]) and np.array_equal(h, G.mont_points(G.h_xy_canon)[0])
        else:
            srs = zk.SRS(ctx, G.cid, np.zeros((n, 8), dtype=np.uint64), np.zeros(8, dtype=np.uint64), _create=lambda g_, h_, out: zk.lib().zk_srs_generate(
                ctx._h, G.cid, n, window_bits, None, None, out))
        assert ctx.launch_count - before == (1 if window_bits == 0 else 2)
        with srs:
            com = srs.commit_non_hiding(orc.to_mont(G.scalar, sc), 1)
            assert np.array_equal(com.chunks[0], orc.msm(G.cid, g, sc))
            masked = srs.mask_custom(zk.PolyComm(np.zeros((1, 8), dtype=np.uint64)), one)
            assert np.array_equal(masked.chunks[0], h)


def test_refusals(ctx):
    """ZK_ERR_INVALID, before anything is allocated, for depth 0, depth past 2^32 (the reference's u32 index), a bad curve and a
    NULL out; a depth whose points could not fit in memory would otherwise fail in cudaMalloc with ZK_ERR_CUDA"""
    L = zk.lib()
    h = ctypes.c_void_p()
    for curve, depth, out in ((zk.VESTA, 0, ctypes.byref(h)), (zk.VESTA, (1 << 32) + 1, ctypes.byref(h)), (7, 16, ctypes.byref(h)),
                              (-1, 16, ctypes.byref(h)), (zk.VESTA, 16, None)):
        assert L.zk_srs_generate(ctx._h, curve, depth, -1, None, None, out) == -1, (curve, depth)
        assert not h.value
        if depth != 16:
            assert b"depth" in L.zk_last_error()
    assert L.zk_srs_generate(ctx._h, zk.VESTA, 16, 1, None, None, ctypes.byref(h)) == -1      # window_bits 1: no such table
    assert not h.value
    with pytest.raises(zk.ZkError):
        zk.SRS.create(ctx, zk.VESTA, 0)


def test_on_the_callers_stream(orc, pallas_srs):
    """The call queued on a caller's stream held back by a spin kernel (the pattern of test_gpu_streams.py): nothing runs on
    another stream, so the result is the same"""
    G = pallas_srs
    stream = torch.cuda.Stream()
    with zk.Context(0) as c:
        c.set_stream(stream.cuda_stream)
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(SPIN)
            srs = zk.SRS.create(c, G.cid, 4096)
        stream.synchronize()
        with srs:
            assert np.array_equal(srs.g, G.g[:4096]) and np.array_equal(srs.h, G.mont_points(G.h_xy_canon)[0])
            sc = orc.random_scalars(G.scalar, 4096, seed=33)
            assert np.array_equal(srs.commit_non_hiding(orc.to_mont(G.scalar, sc), 1).chunks[0], orc.msm(G.cid, G.g[:4096], sc))
