"""The reference's unit tests of LagrangeBasisEvaluations (kimchi/src/lagrange_basis_evaluations.rs:274-375) replayed on the Python
restatement (tests/evals_replay.py) for log n = 1..9 and both fields, plus the identities the device code relies on: the chunked basis
evaluates the coefficient chunks of a polynomial given in evaluation form, a point of the domain gives the all-zero basis, and
evaluate_chunks pads with zero chunks and refuses too many."""
import random

import pytest

import evals_replay as ev

LOGS = range(1, 10)


def rand_field(rng, P, k):
    return [rng.randrange(P) for _ in range(k)]


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n", LOGS)
def test_lagrange_evaluations(orc, fid, log_n):
    """test_lagrange_evaluations: l_i(x) == interpolate(e_i).evaluate(x) for every unit vector e_i"""
    P, n = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(100 * fid + log_n)
    x = rng.randrange(P)
    got = ev.lagrange_basis(orc, fid, n, log_n, x)
    assert len(got) == 1 and len(got[0]) == n
    for i in range(n):
        e = [0] * n
        e[i] = 1
        assert got[0][i] == ev.interpolate_then_evaluate(orc, fid, e, x), i


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n", LOGS)
def test_new_with_chunked_segments(orc, fid, log_n):
    """test_new_with_chunked_segments: with max_poly_size = n the chunked construction gives the unchunked basis"""
    P, n = orc.MODULUS[fid], 1 << log_n
    x = random.Random(200 * fid + log_n).randrange(P)
    assert ev.basis_chunked(orc, fid, n, log_n, x) == ev.lagrange_basis(orc, fid, n, log_n, x)


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n", LOGS)
def test_evaluation(orc, fid, log_n):
    """test_evaluation: evaluate(p) == [p.interpolate().evaluate(x)]"""
    P, n = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(300 * fid + log_n)
    p, x = rand_field(rng, P, n), rng.randrange(P)
    basis = ev.lagrange_basis(orc, fid, n, log_n, x)
    assert ev.evaluate(basis, p, P) == [ev.interpolate_then_evaluate(orc, fid, p, x)]


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n", LOGS)
def test_evaluation_boolean(orc, fid, log_n):
    """test_evaluation_boolean: on a 0/1 column evaluate_boolean(p) == [p.interpolate().evaluate(x)]"""
    P, n = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(400 * fid + log_n)
    p, x = [rng.randrange(2) for _ in range(n)], rng.randrange(P)
    basis = ev.lagrange_basis(orc, fid, n, log_n, x)
    assert ev.evaluate_boolean(basis, p, P) == [ev.interpolate_then_evaluate(orc, fid, p, x)]
    assert ev.evaluate_boolean(basis, p, P) == ev.evaluate(basis, p, P)


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,c", [(1, 2), (3, 2), (5, 4), (8, 8), (9, 2)])
def test_chunked_basis_evaluates_the_coefficient_chunks(orc, fid, log_n, c):
    """f of degree < n = c m in evaluation form: evaluate(f)[i] == the Horner value of coefficient chunk i"""
    P, n = orc.MODULUS[fid], 1 << log_n
    m = n // c
    rng = random.Random(500 * fid + log_n)
    f, x = rand_field(rng, P, n), rng.randrange(P)
    coeffs = ev.ints(orc, fid, orc.ntt(fid, ev.mont(orc, fid, f), inverse=True))
    basis = ev.lagrange_basis(orc, fid, m, log_n, x)
    assert len(basis) == c
    assert ev.evaluate(basis, f, P) == [ev.horner(coeffs[i * m:(i + 1) * m], x, P) for i in range(c)]
    assert ev.evaluate(basis, f, P) == ev.evaluate_chunks(coeffs, c, m, x, P)


@pytest.mark.parametrize("fid", [0, 1])
def test_a_point_of_the_domain_gives_the_zero_basis(orc, fid):
    """x = w^i: the numerator x^n - 1 is zero and batch_inversion_and_mul skips the zero denominator, so every l_i is 0"""
    log_n = 4
    w = ev.omega(orc, fid, log_n)
    for x in (1, w, pow(w, 3, orc.MODULUS[fid])):
        assert ev.lagrange_basis(orc, fid, 16, log_n, x) == [[0] * 16]


def test_batch_inversion_skips_zeros():
    P = 101
    assert ev.batch_inversion_and_mul([0, 2, 0, 5], 3, P) == [0, 3 * pow(2, -1, P) % P, 0, 3 * pow(5, -1, P) % P]
    assert ev.batch_inversion_and_mul([0, 0], 7, P) == [0, 0]


def test_evaluate_boolean_counts_any_nonzero_as_one(orc):
    fid, log_n = 0, 3
    P = orc.MODULUS[fid]
    basis = ev.lagrange_basis(orc, fid, 8, log_n, 12345)
    p = [0, 1, 7, 0, P - 1, 1, 0, 2]
    assert ev.evaluate_boolean(basis, p, P) == ev.evaluate(basis, [1 if v else 0 for v in p], P)
    assert ev.evaluate_boolean(basis, p, P) != ev.evaluate(basis, p, P)


def test_evaluate_chunks_pads_and_refuses_too_many_chunks():
    P = 101
    assert ev.evaluate_chunks([1, 2, 3], 3, 2, 5, P) == [1 + 2 * 5, 3, 0]
    assert ev.evaluate_chunks([], 2, 4, 5, P) == [0, 0]
    with pytest.raises(ValueError):
        ev.evaluate_chunks([1, 2, 3], 1, 2, 5, P)
