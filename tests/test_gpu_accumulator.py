"""The recursion accumulators on the device (zk_srs_accumulator_check / zk_srs_accumulator_generate behind
proof_systems_b200.batch_dlog_accumulator_check / _generate) against the CPU restatement of poly-commitment/src/utils.rs:204-312
(tests/accumulator_replay.py): kimchi's regression on the basis i G, generate bit for bit on both curves at |g| = 2^16 with every
table layout, the check on honest and perturbed batches (the sum equal to the restatement's), openings made by zk_srs_open, every
refusal, a caller's stream and two threads on one context."""
import ctypes
import threading

import numpy as np
import pytest

import accumulator_replay as acc
import proof_systems_b200 as zk
from open_replay import GENERATOR_Y_VESTA, Points
from verify_replay import device_open, reference_batch

pytestmark = pytest.mark.gpu

EX = 3756288960823668761746459900985719106126835112055076922409498125279524024429
EY = 7540929664328976141648477194277016811781677917189411360504995258251130097840
R = 0x1234567890ABCDEF1234567890ABCDEF        # the check's r (the reference draws it from OsRng)


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def generate(orc, G, srs, k, chals):
    return zk.batch_dlog_accumulator_generate(srs, k, acc.mont(orc, G.scalar, chals))


def check(orc, G, srs, comms, chals, r=R):
    """(ok, affine sum)"""
    return zk.batch_dlog_accumulator_check(srs, comms, acc.mont(orc, G.scalar, chals), acc.mont(orc, G.scalar, [r])[0], return_sum=True)


def test_recursion_challenge_commitment_regression(ctx, orc):
    """kimchi/src/proof.rs:1164-1204 through the device: g = (i G)_{i = 1..16} on Vesta, challenges [2, 3, 5, 7]"""
    P = Points(orc)
    gen = P.from_xy(1, GENERATOR_Y_VESTA)
    basis = np.stack([P.mul(gen, i) for i in range(1, 17)])
    with zk.SRS(ctx, zk.VESTA, basis, gen) as srs:
        out = zk.batch_dlog_accumulator_generate(srs, 1, acc.mont(orc, orc.FP, [2, 3, 5, 7]))
        assert out.shape == (1, 8)
        assert orc.fe_int(orc.FQ, out[0, :4]) == EX and orc.fe_int(orc.FQ, out[0, 4:]) == EY
        assert zk.batch_dlog_accumulator_check(srs, out, acc.mont(orc, orc.FP, [2, 3, 5, 7]))       # r from the OS


# ---------------------------------------------------------------------------------------------- |g| = 2^16, both curves
CASES = {                                       # name: (num_comms, number of challenges, seed)
    "rounds5": (3, 15, 5), "rounds11": (3, 33, 11), "rounds17": (3, 51, 17), "four_for_three": (3, 8, 4),
}


@pytest.fixture(scope="module", params=["pallas_srs", "vesta_srs"])
def full(request, orc):
    """the fixture's 2^16 generators, 33 accumulators of 16 rounds and the CASES, all from the restatement"""
    G = request.getfixturevalue(request.param)
    g, h = G.g[: 1 << 16], G.mont_points(G.h_xy_canon)[0]
    chals = acc.random_chals(orc, G.scalar, 33 * 16, seed=100 + G.cid)
    want = acc.generate(orc, G.cid, g, 33, chals)
    cases = {}
    for name, (k, n, seed) in CASES.items():
        c = acc.random_chals(orc, G.scalar, n, seed=seed)
        cases[name] = (k, c, acc.generate(orc, G.cid, g, k, c))
    return G, g, h, chals, want, cases


@pytest.mark.parametrize("window_bits", [0, -1, 16])
def test_generate_is_bit_exact(ctx, orc, full, window_bits):
    G, g, h, chals, want, cases = full
    with zk.SRS(ctx, G.cid, g, h, window_bits=window_bits) as srs:
        for k in (1, 2, 16, 17, 33):
            got = generate(orc, G, srs, k, chals[: 16 * k])
            assert np.array_equal(got, want[:k]), k
        for name, (k, c, w) in cases.items():
            got = generate(orc, G, srs, k, c)
            assert got.shape == w.shape and np.array_equal(got, w), name
        assert cases["four_for_three"][2].shape == (4, 8)
        got = generate(orc, G, srs, 2, [0] * 32)                       # b_poly_coefficients of zeros: (1, 0, ...)
        assert np.array_equal(got, np.stack([g[0], g[0]]))


@pytest.mark.parametrize("k", [1, 2, 16, 17, 100])
def test_honest_accumulators_pass(ctx, orc, full, k):
    G, g, h, chals, want, _ = full
    with zk.SRS(ctx, G.cid, g, h) as srs:
        ch = chals[: 16 * k] if k <= 33 else acc.random_chals(orc, G.scalar, 16 * k, seed=300 + k)
        if k <= 33:
            ok, pt = check(orc, G, srs, want[:k], ch)                  # the restatement's accumulators
            assert ok and not pt.any()
        comms = generate(orc, G, srs, k, ch)                           # the device's
        ok, pt = check(orc, G, srs, comms, ch)
        assert ok and not pt.any()


@pytest.mark.parametrize("kind", acc.PERTURBATIONS)
def test_each_perturbation_fails_with_the_restatement_sum(ctx, orc, full, kind):
    G, g, h, chals, want, _ = full
    bad_comms, bad_chals = acc.perturb(orc, G.cid, want[:16], chals[: 16 * 16], 16, kind, g[7], at=3)
    with zk.SRS(ctx, G.cid, g, h) as srs:
        ok, pt = check(orc, G, srs, bad_comms, bad_chals)
    assert not ok
    assert np.array_equal(pt, acc.check_sum(orc, G.cid, g, bad_comms, bad_chals, R))


def test_r_zero_checks_only_the_first_accumulator(ctx, orc, full):
    G, g, h, chals, want, _ = full
    with zk.SRS(ctx, G.cid, g, h) as srs:
        late, _ = acc.perturb(orc, G.cid, want[:16], chals, 16, "replace", g[7], at=5)
        ok, pt = check(orc, G, srs, late, chals[:256], r=0)
        assert ok and not pt.any()
        first, _ = acc.perturb(orc, G.cid, want[:16], chals, 16, "replace", g[7], at=0)
        ok, pt = check(orc, G, srs, first, chals[:256], r=0)
        assert not ok and np.array_equal(pt, acc.check_sum(orc, G.cid, g, first, chals[:256], 0))


def test_a_thousand_accumulators(ctx, orc, full):
    """k = 1024 (16 384 challenges): device accumulators pass, one tampered commitment fails"""
    G, g, h, *_ = full
    chals = acc.random_chals(orc, G.scalar, 1024 * 16, seed=400)
    with zk.SRS(ctx, G.cid, g, h) as srs:
        comms = generate(orc, G, srs, 1024, chals)
        assert comms.shape == (1024, 8)
        assert np.array_equal(comms[1023], acc.generate(orc, G.cid, g, 1, chals[-16:])[0])
        ok, pt = check(orc, G, srs, comms, chals)
        assert ok and not pt.any()
        comms[700] = g[1]
        ok, pt = check(orc, G, srs, comms, chals)
        assert not ok and pt.any()


# ---------------------------------------------------------------------------------------------- openings of zk_srs_open
def test_the_openings_of_the_reference_batch(ctx, orc, vesta_srs):
    """commitment.rs:119-257's seven openings, made on the device: their sg and the round challenges their transcripts return are
    honest accumulators of the 128-point SRS; a swapped pair fails"""
    g, h = vesta_srs.g[:128], vesta_srs.mont_points(vesta_srs.h_xy_canon)[0]
    m = lambda xs: acc.mont(orc, orc.FP, xs)
    with zk.SRS(ctx, zk.VESTA, g, h) as srs:
        def opener(polys, elm, ps, es, draws, tr):
            return device_open(zk, orc, srs, orc.FP, [(m(c), m(bl)) for c, bl in polys], elm, ps, es, draws, tr)[0]
        entries, *_ = reference_batch(orc, vesta_srs, opener)
        comms, chals = [], []
        for e in entries:
            tr = e.transcript()
            tr.u_base(e.cip)
            chals += [tr.round(j, l, r) for j, (l, r) in enumerate(e.opening.lr)]
            comms.append(e.opening.sg)
        comms = np.stack(comms)
        assert len(chals) == 7 * 7
        ok, pt = check(orc, vesta_srs, srs, comms, chals)
        assert ok and not pt.any()
        assert np.array_equal(generate(orc, vesta_srs, srs, 7, chals), comms)
        swapped, _ = acc.perturb(orc, orc.VESTA, comms, chals, 7, "swap", None, at=2)
        ok, pt = check(orc, vesta_srs, srs, swapped, chals)
        assert not ok and np.array_equal(pt, acc.check_sum(orc, orc.VESTA, g, swapped, chals, R))


# ---------------------------------------------------------------------------------------------- refusals, streams, threads
def test_every_refusal(ctx, orc, vesta_srs):
    G = vesta_srs
    g, h = G.g[:1 << 16], G.mont_points(G.h_xy_canon)[0]
    chals = acc.random_chals(orc, G.scalar, 64, seed=500)
    with zk.SRS(ctx, G.cid, g, h) as srs, zk.SRS(ctx, G.cid, g[:96], h) as odd:
        honest = generate(orc, G, srs, 4, chals)
        cases = [                                                     # (comms / num_comms, challenges, srs, code, message)
            (0, chals[:3], srs, -1, "3 challenges for no accumulators"),
            (3, chals[:2], srs, -1, "2 challenges for 3 accumulators leave 0 rounds"),
            (3, [], srs, -1, "0 challenges for 3 accumulators leave 0 rounds"),
            (2, chals[:7], srs, -1, "7 challenges are not a multiple of 3 rounds"),
        ]
        for k, ch, s, code, msg in cases:
            for call in (lambda: check(orc, G, s, honest[:k], ch), lambda: generate(orc, G, s, k, ch)):
                with pytest.raises(zk.ZkError) as e:
                    call()
                assert e.value.code == code and msg in str(e.value), (k, len(ch), str(e.value))
        for s, k, ch in ((srs, 2, chals[:30]), (srs, 2, chals[:34]), (odd, 2, chals[:14])):    # 2^rounds != |g| (96 is no power of two)
            with pytest.raises(zk.ZkError) as e:
                check(orc, G, s, honest[:k], ch)
            assert e.value.code == -4 and "coefficients per accumulator" in str(e.value)
        # more points than the capacity: the count is set first (4 for num_comms = 3 and 8 challenges)
        c8 = acc.mont(orc, G.scalar, chals[:8])
        out, got = np.zeros((3, 8), dtype=np.uint64), ctypes.c_size_t(0)
        rc = zk.lib().zk_srs_accumulator_generate(srs._h, 3, c8.ctypes.data, 8, out.ctypes.data, 3, ctypes.byref(got))
        assert rc == -1 and got.value == 4 and b"do not fit the capacity" in zk.lib().zk_last_error()
        # empty batches, then the context still works
        ok, pt = check(orc, G, srs, np.zeros((0, 8), dtype=np.uint64), [])
        assert ok and not pt.any()
        assert generate(orc, G, srs, 0, []).shape == (0, 8)
        ok, pt = check(orc, G, srs, honest, chals)
        assert ok and not pt.any()
        assert np.array_equal(generate(orc, G, srs, 4, chals), honest)


def test_on_a_callers_stream(orc, vesta_srs):
    import torch
    G = vesta_srs
    g, h = G.g[:1 << 16], G.mont_points(G.h_xy_canon)[0]
    chals = acc.random_chals(orc, G.scalar, 5 * 16, seed=600)
    want = acc.generate(orc, G.cid, g, 5, chals)
    stream = torch.cuda.Stream()
    with zk.Context(0) as c, zk.SRS(c, G.cid, g, h) as srs:
        c.set_stream(stream.cuda_stream)
        try:
            assert np.array_equal(generate(orc, G, srs, 5, chals), want)
            ok, pt = check(orc, G, srs, want, chals)
            assert ok and not pt.any()
        finally:
            c.set_stream(None)


def test_two_threads_on_one_context(ctx, orc, vesta_srs):
    G = vesta_srs
    g, h = G.g[:1 << 16], G.mont_points(G.h_xy_canon)[0]
    chals = acc.random_chals(orc, G.scalar, 3 * 16, seed=700)
    want = acc.generate(orc, G.cid, g, 3, chals)
    bad, _ = acc.perturb(orc, G.cid, want, chals, 16, "swap", None, at=0)
    want_bad = acc.check_sum(orc, G.cid, g, bad, chals, R)
    with zk.SRS(ctx, G.cid, g, h) as srs:
        results, errors = {"gen": [], "check": []}, []

        def run(name, fn):
            try:
                for _ in range(4):
                    results[name].append(fn())
            except Exception as e:
                errors.append(e)
        threads = [threading.Thread(target=run, args=("gen", lambda: generate(orc, G, srs, 3, chals))),
                   threading.Thread(target=run, args=("check", lambda: check(orc, G, srs, bad, chals)))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors
        assert len(results["gen"]) == 4 and all(np.array_equal(x, want) for x in results["gen"])
        assert len(results["check"]) == 4 and all(not ok and np.array_equal(pt, want_bad) for ok, pt in results["check"])
