"""The CPU restatement of batch_dlog_accumulator_check / batch_dlog_accumulator_generate (tests/accumulator_replay.py) against the
reference's own regression (kimchi/src/proof.rs:1164-1204) and the behaviour of poly-commitment/src/utils.rs:204-312: honest
accumulators pass, perturbed ones fail, and every edge case (empty batches, the asserts, trailing chunks, truncation) behaves as
the reference's code does."""
import numpy as np
import pytest

import accumulator_replay as acc
from open_replay import GENERATOR_Y_VESTA, Points

EX = 3756288960823668761746459900985719106126835112055076922409498125279524024429
EY = 7540929664328976141648477194277016811781677917189411360504995258251130097840


def test_generate_reproduces_the_recursion_challenge_commitment_regression(orc):
    """proof.rs:1164-1204: U = <b_poly_coefficients([2, 3, 5, 7]), (i G)_{i = 1..16}> over Vesta"""
    P = Points(orc)
    G = P.from_xy(1, GENERATOR_Y_VESTA)
    basis = np.stack([P.mul(G, i) for i in range(1, 17)])
    out = acc.generate(orc, orc.VESTA, basis, 1, [2, 3, 5, 7])
    assert out.shape == (1, 8)
    assert orc.fe_int(orc.FQ, out[0, :4]) == EX and orc.fe_int(orc.FQ, out[0, 4:]) == EY
    assert acc.check(orc, orc.VESTA, basis, out, [2, 3, 5, 7], 12345)


@pytest.fixture(scope="module")
def g128(vesta_srs):
    return vesta_srs.g[:128]


@pytest.mark.parametrize("k", [1, 2, 7])
def test_honest_accumulators_pass(orc, g128, k):
    chals = acc.random_chals(orc, orc.FP, 7 * k, seed=k)
    comms = acc.generate(orc, orc.VESTA, g128, k, chals)
    assert comms.shape == (k, 8)
    assert acc.check(orc, orc.VESTA, g128, comms, chals, 987654321)


@pytest.mark.parametrize("kind", acc.PERTURBATIONS)
def test_each_perturbation_fails(orc, g128, kind):
    k = 3
    chals = acc.random_chals(orc, orc.FP, 7 * k, seed=40)
    comms = acc.generate(orc, orc.VESTA, g128, k, chals)
    bad_comms, bad_chals = acc.perturb(orc, orc.VESTA, comms, chals, 7, kind, g128[5], at=1)
    assert not acc.check(orc, orc.VESTA, g128, bad_comms, bad_chals, 31337)


def test_r_zero_checks_only_the_first_accumulator(orc, g128):
    chals = acc.random_chals(orc, orc.FP, 14, seed=41)
    comms = acc.generate(orc, orc.VESTA, g128, 2, chals)
    bad_comms, _ = acc.perturb(orc, orc.VESTA, comms, chals, 7, "replace", g128[3], at=1)
    assert acc.check(orc, orc.VESTA, g128, bad_comms, chals, 0)
    bad_comms, _ = acc.perturb(orc, orc.VESTA, comms, chals, 7, "replace", g128[3], at=0)
    assert not acc.check(orc, orc.VESTA, g128, bad_comms, chals, 0)


def test_empty_batches(orc, g128):
    assert acc.check(orc, orc.VESTA, g128, np.zeros((0, 8), dtype=np.uint64), [], 5)
    assert not acc.check_sum(orc, orc.VESTA, g128, np.zeros((0, 8), dtype=np.uint64), [], 5).any()
    assert acc.generate(orc, orc.VESTA, g128, 0, []).shape == (0, 8)


@pytest.mark.parametrize("k, n_chals", [(0, 3), (3, 2), (3, 0), (2, 7)])
def test_the_asserts_panic(orc, g128, k, n_chals):
    """k = 0 with challenges, rounds = 0 (fewer challenges than accumulators), and a remainder: 7 challenges, k = 2, rounds 3"""
    chals = acc.random_chals(orc, orc.FP, n_chals, seed=42)
    comms = g128[:k]
    with pytest.raises(acc.Panic):
        acc.check(orc, orc.VESTA, g128, comms, chals, 1)
    with pytest.raises(acc.Panic):
        acc.generate(orc, orc.VESTA, g128, k, chals)


@pytest.mark.parametrize("n, rounds", [(128, 6), (128, 8), (96, 7), (96, 6)])
def test_check_panics_unless_2_to_the_rounds_is_g(orc, vesta_srs, n, rounds):
    g = vesta_srs.g[:n]
    chals = acc.random_chals(orc, orc.FP, 2 * rounds, seed=43)
    with pytest.raises(acc.Panic):
        acc.check(orc, orc.VESTA, g, g[:2], chals, 1)


def test_trailing_chunks(orc, g128):
    """k = 3 with 24 challenges: rounds 8, 3 chunks; k = 3 with 8 challenges at |g| = 4: rounds 2, 4 chunks — the check reads the
    first 3, generate returns 4 points"""
    g4 = g128[:4]
    chals = acc.random_chals(orc, orc.FP, 8, seed=44)
    out = acc.generate(orc, orc.VESTA, g4, 3, chals)
    assert out.shape == (4, 8)
    for i in range(4):
        assert np.array_equal(out[i], acc.generate(orc, orc.VESTA, g4, 1, chals[2 * i:2 * i + 2])[0])
    assert acc.check(orc, orc.VESTA, g4, out[:3], chals, 77)
    wrong_tail = list(chals[:6]) + [1, 2]                          # the fourth chunk is never read
    assert acc.check(orc, orc.VESTA, g4, out[:3], wrong_tail, 77)


def test_generate_truncates_both_ways(orc, g128):
    """rounds < log |g|: the coefficients cover g[..2^rounds]; rounds > log |g|: the first |g| coefficients, which depend on the
    last log |g| challenges only"""
    m = orc.FP_MODULUS
    short = acc.random_chals(orc, orc.FP, 5, seed=45)
    s = acc.generate(orc, orc.VESTA, g128, 1, short)[0]
    assert np.array_equal(s, orc.msm(orc.VESTA, g128[:32], orc.ints_to_limbs(acc.b_poly_coefficients(short, m))))
    long = acc.random_chals(orc, orc.FP, 9, seed=46)
    s = acc.generate(orc, orc.VESTA, g128, 1, long)[0]
    assert np.array_equal(s, acc.generate(orc, orc.VESTA, g128, 1, long[2:])[0])


def test_zero_challenges_are_allowed(orc, g128):
    """b_poly_coefficients of zeros is (1, 0, 0, ...): the accumulator is g[0]; batch_inversion leaves the zeros alone"""
    out = acc.generate(orc, orc.VESTA, g128, 2, [0] * 14)
    assert np.array_equal(out, np.stack([g128[0], g128[0]]))
    assert acc.check(orc, orc.VESTA, g128, out, [0] * 14, 3)
