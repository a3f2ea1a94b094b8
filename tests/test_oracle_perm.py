"""The restatement of perm_aggreg (tests/perm_replay.py) on its own: wired instances pass the final-value check, a broken cell fails it,
a zero denominator is skipped like ark_ff::batch_inversion does, the tail restarts from the two random values, and the coefficients
interpolate z."""
import random

import pytest

import evals_replay as ev
import perm_replay as pr


def horner(coeffs, x, P):
    acc = 0
    for c in reversed(coeffs):
        acc = (acc * x + c) % P
    return acc


def run(orc, fid, log_n, zk_rows, inst):
    return pr.perm_aggreg(orc, fid, log_n, zk_rows, inst.w, inst.sigma, inst.shifts, inst.beta, inst.gamma, inst.rand)


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,zk_rows", [(2, 3), (4, 3), (4, 5), (4, 15), (7, 3), (7, 16), (9, 127)])
def test_wired_instances_pass_the_final_value_check(orc, fid, log_n, zk_rows):
    P, n = orc.MODULUS[fid], 1 << log_n
    inst = pr.wired_instance(orc, fid, log_n, zk_rows, seed=log_n * 100 + zk_rows + fid)
    z, coeffs, ok = run(orc, fid, log_n, zk_rows, inst)
    assert ok and z[0] == 1 and z[n - zk_rows] == 1
    # the coefficients interpolate z over d1
    omega = ev.omega(orc, fid, log_n)
    for j in (0, 1, n - zk_rows, n - 1):
        assert horner(coeffs, pow(omega, j, P), P) == z[j]
    # the zk rows are fixed by the permutation: every tail ratio is one, so z stays at the second random value
    assert z[n - zk_rows + 1:] == [inst.rand[0]] + [inst.rand[1]] * (zk_rows - 2)


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,zk_rows", [(4, 3), (7, 5), (7, 100)])
def test_one_changed_wired_cell_fails_with_final_value(orc, fid, log_n, zk_rows):
    P, n = orc.MODULUS[fid], 1 << log_n
    inst = pr.wired_instance(orc, fid, log_n, zk_rows, seed=7 + log_n + fid)
    rng = random.Random(fid + log_n)
    for _ in range(4):
        bad = inst.copy()
        k, j = rng.choice(inst.wired)
        bad.w[k][j] = (bad.w[k][j] + rng.randrange(1, P)) % P
        z, _, ok = run(orc, fid, log_n, zk_rows, bad)
        assert not ok and z[n - zk_rows] != 1        # ProverError::Permutation("final value")
    # wiring a zk row leaves the check alone but moves the tail off the second random value
    if zk_rows > 3:
        bad = inst.copy()
        bad.sigma[2][n - zk_rows + 2] = rng.randrange(P)
        z, _, ok = run(orc, fid, log_n, zk_rows, bad)
        assert ok and z[n - zk_rows + 3] not in (0, inst.rand[1])


@pytest.mark.parametrize("fid", [0, 1])
def test_zero_denominator_zeroes_z_from_the_next_row(orc, fid):
    """ark_ff::batch_inversion skips a zero entry and leaves it zero, so num / den is 0 there: no error, z = 0 from j + 1 on,
    up to the random rows; the other inverses are unaffected"""
    P, log_n, zk_rows = orc.MODULUS[fid], 6, 5
    n = 1 << log_n
    last = n - zk_rows
    for j in (0, 17, last - 1):
        inst = pr.wired_instance(orc, fid, log_n, zk_rows, seed=j + fid)
        pr.zero_denominator(inst, P, 3, j)
        z, _, ok = run(orc, fid, log_n, zk_rows, inst)
        assert not ok
        assert all(v != 0 for v in z[:j + 1]) and all(v == 0 for v in z[j + 1:last + 1])
        assert z[last + 1:last + 3] == inst.rand
    # a zero denominator in the tail zeroes the rest of the tail only
    inst = pr.wired_instance(orc, fid, log_n, zk_rows, seed=99 + fid)
    pr.zero_denominator(inst, P, 0, last + 2)
    z, _, ok = run(orc, fid, log_n, zk_rows, inst)
    assert ok and z[last + 2] == inst.rand[1] and z[last + 3:] == [0] * (zk_rows - 3)
    # ... and in a row whose ratio the random values replace, it changes nothing
    inst = pr.wired_instance(orc, fid, log_n, zk_rows, seed=5 + fid)
    want, _, _ = run(orc, fid, log_n, zk_rows, inst)
    pr.zero_denominator(inst, P, 6, last)
    z, _, ok = run(orc, fid, log_n, zk_rows, inst)
    assert ok and z == want


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("zk_rows", [3, 4, 9])
def test_tail_follows_the_two_random_values(orc, fid, zk_rows):
    P, log_n = orc.MODULUS[fid], 5
    n = 1 << log_n
    last = n - zk_rows
    rng = random.Random(zk_rows + fid)
    inst = pr.Instance([[rng.randrange(P) for _ in range(n)] for _ in range(7)], [[rng.randrange(P) for _ in range(n)] for _ in range(7)],
                       [rng.randrange(P) for _ in range(7)], rng.randrange(P), rng.randrange(P), [rng.randrange(P), rng.randrange(P)])
    z, _, ok = run(orc, fid, log_n, zk_rows, inst)
    assert not ok
    num, den = pr.ratio_factors(inst.w, inst.sigma, inst.shifts, inst.beta, inst.gamma, ev.omega(orc, fid, log_n), P)
    assert z[0] == 1
    for j in range(last):
        assert z[j + 1] == z[j] * num[j] * pow(den[j], P - 2, P) % P
    assert z[last + 1] == inst.rand[0] and z[last + 2] == inst.rand[1]
    for j in range(last + 2, n - 1):
        assert z[j + 1] == z[j] * num[j] * pow(den[j], P - 2, P) % P
    # other draws move only the tail
    inst.rand = [rng.randrange(P), rng.randrange(P)]
    z2, _, _ = run(orc, fid, log_n, zk_rows, inst)
    assert z2[:last + 1] == z[:last + 1] and z2[last + 1] == inst.rand[0] and z2[last + 1:] != z[last + 1:]
