"""Batch verification of IPA opening proofs on the device (zk_srs_verify behind proof_systems_b200.srs_verify) against the oracle
restatement of SRS::verify (poly-commitment/src/ipa.rs:301-502, tests/verify_replay.py): the reference's randomised 7-proof batch
with the Poseidon transcript, tampered batches (the accumulated point equal to the oracle's bit for bit), both curves at the full
2^16-point SRS with every table layout, the edge cases of the scalar bookkeeping, errors, and two threads on one context."""
import threading

import numpy as np
import pytest

import proof_systems_b200 as zk
from verify_replay import (TAMPERINGS, Entry, HashTranscript, device_open, oracle_verify, reference_batch, tamper, to_device)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def ints(orc, fid, n, seed):
    return orc.limbs_to_ints(orc.random_scalars(fid, n, seed=seed))


def mont(orc, fid, xs):
    return orc.to_mont(fid, orc.ints_to_limbs(list(xs))) if len(xs) else np.zeros((0, 4), dtype=np.uint64)


def mont1(orc, fid, x):
    return mont(orc, fid, [x])[0]


def device_verify(orc, G, srs, entries, rand_base, sg_rand_base):
    batch = [to_device(zk, orc, G.scalar, e) for e in entries]
    return zk.srs_verify(srs, batch, mont1(orc, G.scalar, rand_base), mont1(orc, G.scalar, sg_rand_base), return_sum=True)


# ---------------------------------------------------------------------------------------------- the reference's batch
@pytest.fixture(scope="module")
def ref(ctx, orc, vesta_srs):
    g, h = vesta_srs.g[:128], vesta_srs.mont_points(vesta_srs.h_xy_canon)[0]
    srs = zk.SRS(ctx, zk.VESTA, g, h)
    m = lambda xs: mont(orc, orc.FP, xs)

    def opener(polys, elm, ps, es, draws, tr):
        return device_open(zk, orc, srs, orc.FP, [(m(c), m(bl)) for c, bl in polys], elm, ps, es, draws, tr)[0]

    entries, rb, sgb, g, h = reference_batch(orc, vesta_srs, opener)
    yield srs, entries, rb, sgb, g, h
    srs.close()


def test_the_reference_batch_verifies(orc, vesta_srs, ref):
    srs, entries, rb, sgb, _, _ = ref
    ok, pt = device_verify(orc, vesta_srs, srs, entries, rb, sgb)
    assert ok and not pt.any()


@pytest.mark.parametrize("kind", TAMPERINGS)
def test_a_tampered_reference_batch_fails_with_the_oracle_sum(orc, vesta_srs, ref, kind):
    srs, entries, rb, sgb, g, h = ref
    bad = tamper(entries, kind, orc.FP_MODULUS, g[5])
    ok, pt = device_verify(orc, vesta_srs, srs, bad, rb, sgb)
    assert not ok
    assert np.array_equal(pt, oracle_verify(orc, orc.VESTA, g, h, bad, rb, sgb))


# ---------------------------------------------------------------------------------------------- batches with the hash transcript
def hash_entries(orc, G, srs, g, h, n_proofs, seed, poly_lens, zero_poly=False, empty_comm=False):
    """n_proofs openings on `srs` (device) of random polynomials of the given lengths, each with its own HashTranscript; a zero
    polynomial with a zero blinder gives an identity commitment chunk, an empty PolyComm is an evaluation without chunks"""
    m, n = orc.MODULUS[G.scalar], g.shape[0]
    u_points = G.g[200:232]
    polys, comms = [], []
    for j, ln in enumerate(poly_lens):
        coeffs = mont(orc, G.scalar, ints(orc, G.scalar, ln, seed * 100 + j))
        bl = mont(orc, G.scalar, ints(orc, G.scalar, max(1, -(-ln // n)), seed * 100 + 50 + j))
        polys.append((coeffs, bl))
        comms.append(srs.commit_custom(coeffs, 1, bl).chunks)
    if zero_poly:
        polys.append((np.zeros((0, 4), dtype=np.uint64), np.zeros((1, 4), dtype=np.uint64)))
        comms.append(np.zeros((1, 8), dtype=np.uint64))
    if empty_comm:
        comms.append(np.zeros((0, 8), dtype=np.uint64))
    k = (n - 1).bit_length()
    entries = []
    for i in range(n_proofs):
        sc = ints(orc, G.scalar, 2 * k + 6, seed * 1000 + i)
        elm, ps, es, draws = sc[:2], sc[2], sc[3], sc[4:]
        make = lambda s=seed * 1000 + i: HashTranscript(m, u_points, s)
        op, cip = device_open(zk, orc, srs, G.scalar, polys, elm, ps, es, draws, make())
        entries.append(Entry(op, elm, ps, es, comms, cip, make))
    return entries


def scales(orc, G, seed):
    return tuple(ints(orc, G.scalar, 2, seed))


@pytest.fixture(scope="module", params=["pallas_srs", "vesta_srs"])
def full(request, ctx, orc):
    """16 proofs at |g| = 2^16 on the fixture's generators"""
    G = request.getfixturevalue(request.param)
    g, h = G.g[: 1 << 16], G.mont_points(G.h_xy_canon)[0]
    srs = zk.SRS(ctx, G.cid, g, h)
    entries = hash_entries(orc, G, srs, g, h, 16, 7, [1 << 16])
    srs.close()
    return G, g, h, entries


@pytest.mark.parametrize("window_bits", [15, 16, 0])
def test_full_srs_batches_verify(ctx, orc, full, window_bits):
    G, g, h, entries = full
    rb, sgb = scales(orc, G, 3)
    with zk.SRS(ctx, G.cid, g, h, window_bits=window_bits) as srs:
        for B in (1, 16):
            ok, pt = device_verify(orc, G, srs, entries[:B], rb, sgb)
            assert ok and not pt.any(), B
        if window_bits == 15:
            bad = tamper(entries, "z1", orc.MODULUS[G.scalar], g[9])
            ok, pt = device_verify(orc, G, srs, bad, rb, sgb)
            assert not ok
            assert np.array_equal(pt, oracle_verify(orc, G.cid, g, h, bad, rb, sgb))


@pytest.mark.parametrize("n", [48, 128])
def test_non_power_of_two_srs_chunked_zero_and_empty_commitments(ctx, orc, vesta_srs, n):
    """a 48-point SRS (padded to 64), chunked commitments (polynomials longer than |g|), an identity chunk and an empty PolyComm"""
    G = vesta_srs
    g, h = G.g[:n], G.mont_points(G.h_xy_canon)[0]
    with zk.SRS(ctx, G.cid, g, h) as srs:
        entries = hash_entries(orc, G, srs, g, h, 3, n, [n // 2 + 1, 2 * n + 17], zero_poly=True, empty_comm=True)
        assert max(c.shape[0] for c in entries[0].comms) == 3 and entries[0].comms[-1].shape[0] == 0
        rb, sgb = scales(orc, G, 5)
        ok, pt = device_verify(orc, G, srs, entries, rb, sgb)
        assert ok and not pt.any()
        assert not oracle_verify(orc, G.cid, g, h, entries, rb, sgb).any()
        bad = tamper(entries, "z2", orc.FP_MODULUS, g[3], at=1)
        ok, pt = device_verify(orc, G, srs, bad, rb, sgb)
        assert not ok and np.array_equal(pt, oracle_verify(orc, G.cid, g, h, bad, rb, sgb))


def test_fewer_rounds_zero_challenge_and_empty_batch(ctx, orc, vesta_srs):
    G = vesta_srs
    g, h = G.g[:128], G.mont_points(G.h_xy_canon)[0]
    with zk.SRS(ctx, G.cid, g[:32], h) as small:
        with zk.SRS(ctx, G.cid, g, h) as srs:
            short = hash_entries(orc, G, small, g[:32], h, 1, 11, [20])          # 5 rounds: its s covers the first 32 generators
            full = hash_entries(orc, G, srs, g, h, 2, 12, [100])
            assert len(short[0].opening.lr) == 5 and len(full[0].opening.lr) == 7
            rb, sgb = scales(orc, G, 6)
            batch = [full[0], short[0], full[1]]
            ok, pt = device_verify(orc, G, srs, batch, rb, sgb)
            assert ok and not pt.any()
            assert not oracle_verify(orc, G.cid, g, h, batch, rb, sgb).any()
            # a transcript that answers 0 in round 2: chal_inv stays 0 (batch_inversion), the proof fails, the sum is the oracle's
            zero = list(batch)
            e = zero[0]
            zero[0] = Entry(e.opening, e.elm, e.polyscale, e.evalscale, e.comms, e.cip,
                            lambda: HashTranscript(orc.FP_MODULUS, G.g[200:232], 12000, zero_round=2))
            ok, pt = device_verify(orc, G, srs, zero, rb, sgb)
            assert not ok and np.array_equal(pt, oracle_verify(orc, G.cid, g, h, zero, rb, sgb))
            ok, pt = zk.srs_verify(srs, [], mont1(orc, G.scalar, rb), mont1(orc, G.scalar, sgb), return_sum=True)
            assert ok and not pt.any()
            assert zk.srs_verify(srs, [], mont1(orc, G.scalar, rb), mont1(orc, G.scalar, sgb)) is True


class CallbackFailure(Exception):
    pass


def test_errors(ctx, orc, vesta_srs):
    G = vesta_srs
    g, h = G.g[:128], G.mont_points(G.h_xy_canon)[0]
    with zk.SRS(ctx, G.cid, g, h) as srs:
        with zk.SRS(ctx, G.cid, g[:64], h) as small:
            entries = hash_entries(orc, G, srs, g, h, 2, 21, [50])
            rb, sgb = (mont1(orc, G.scalar, x) for x in scales(orc, G, 8))
            with pytest.raises(zk.ZkError) as e:                                   # 7 rounds against a 64-point SRS
                zk.srs_verify(small, [to_device(zk, orc, G.scalar, x) for x in entries], rb, sgb)
            assert e.value.code == -4
            batch = [to_device(zk, orc, G.scalar, x) for x in entries]

            def boom(j, l, r):
                raise CallbackFailure("round %d" % j)
            batch[1].round_challenge = boom
            with pytest.raises(CallbackFailure):
                zk.srs_verify(srs, batch, rb, sgb)
            assert b"round callback failed" in zk.lib().zk_last_error()
            assert zk.srs_verify(srs, [to_device(zk, orc, G.scalar, x) for x in entries], rb, sgb) is True    # the context still works


def test_two_threads_on_one_context(ctx, orc, vesta_srs):
    G = vesta_srs
    g, h = G.g[:128], G.mont_points(G.h_xy_canon)[0]
    with zk.SRS(ctx, G.cid, g, h) as srs:
        good = hash_entries(orc, G, srs, g, h, 4, 31, [90])
        bad = tamper(hash_entries(orc, G, srs, g, h, 4, 32, [70]), "sg", orc.FP_MODULUS, g[1], at=0)
        rb, sgb = scales(orc, G, 9)
        want_bad = oracle_verify(orc, G.cid, g, h, bad, rb, sgb)
        results, errors = {"good": [], "bad": []}, []

        def run(name, entries):
            try:
                for _ in range(4):
                    results[name].append(device_verify(orc, G, srs, entries, rb, sgb))
            except Exception as e:
                errors.append(e)
        threads = [threading.Thread(target=run, args=("good", good)), threading.Thread(target=run, args=("bad", bad))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors
        assert all(ok and not pt.any() for ok, pt in results["good"]) and len(results["good"]) == 4
        assert all(not ok and np.array_equal(pt, want_bad) for ok, pt in results["bad"]) and len(results["bad"]) == 4
