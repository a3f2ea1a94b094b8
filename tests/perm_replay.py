"""The permutation aggregation polynomial z (ProverIndex::perm_aggreg, kimchi/src/circuits/polynomials/permutation.rs:447-574) restated
with Python integers, and generators of wired instances for it.  Field elements are canonical ints; `evals_replay.ints` / `mont`
convert from / to the library's Montgomery limbs.  The interpolation takes its inverse FFT from the CPU oracle (orc.ntt)."""
import random

import numpy as np

import evals_replay as ev

COLS = 7     # PERMUTS


def ratio_factors(w, sigma, shifts, beta, gamma, omega, P):
    """num[j] = prod_k (w_k[j] + omega^j beta shift_k + gamma), den[j] = prod_k (w_k[j] + sigma_k[j] beta + gamma), j < n - 1;
    sigma: the 7 columns at the points of d1 (permutation_coefficients8[k][8 j])"""
    n = len(w[0])
    num, den, x = [], [], 1
    for j in range(n - 1):
        a = b = 1
        for k in range(COLS):
            a = a * (w[k][j] + x * beta % P * shifts[k] + gamma) % P
            b = b * (w[k][j] + sigma[k][j] * beta + gamma) % P
        num.append(a)
        den.append(b)
        x = x * omega % P
    return num, den


def z_evaluations(num, den, zk_rows, rand, P):
    """the reference's loop over d1: z[0] = 1, batch_inversion(den) (zeros skipped and left zero), then
    z[j + 1] = z[j] num[j] / den[j], except the two random values at j = n - zk_rows and n - zk_rows + 1.
    Returns (z, z[n - zk_rows] == 1)."""
    n = len(num) + 1
    inv = ev.batch_inversion_and_mul(den, 1, P)
    draws = iter(rand)
    z = [1] + [0] * (n - 1)
    for j in range(n - 1):
        if j == n - zk_rows or j == n - zk_rows + 1:
            z[j + 1] = next(draws)
        else:
            z[j + 1] = z[j] * num[j] % P * inv[j] % P
    return z, z[n - zk_rows] == 1


def perm_aggreg(orc, fid, log_n, zk_rows, w, sigma, shifts, beta, gamma, rand):
    """-> (z over d1, z's n coefficients (Evaluations::interpolate, untrimmed), final value ok)"""
    P = orc.MODULUS[fid]
    assert len(w[0]) == 1 << log_n and 3 <= zk_rows < 1 << log_n
    num, den = ratio_factors(w, sigma, shifts, beta, gamma, ev.omega(orc, fid, log_n), P)
    z, ok = z_evaluations(num, den, zk_rows, rand, P)
    return z, interpolate(orc, fid, z), ok


def interpolate(orc, fid, evals):
    return ev.ints(orc, fid, orc.ntt(fid, ev.mont(orc, fid, evals), inverse=True))


# ------------------------------------------------------------------------------------------------------------ instances
class Instance:
    """w, sigma (at the points of d1), shifts, beta, gamma, rand: canonical ints"""

    def __init__(self, w, sigma, shifts, beta, gamma, rand, wired=()):
        self.w, self.sigma, self.shifts, self.beta, self.gamma, self.rand = w, sigma, shifts, beta, gamma, rand
        self.wired = list(wired)        # (k, j) of the cells on cycles of two or more: changing one breaks the permutation

    def copy(self):
        return Instance([list(c) for c in self.w], [list(c) for c in self.sigma], list(self.shifts), self.beta, self.gamma, list(self.rand),
                        self.wired)


def wired_instance(orc, fid, log_n, zk_rows, seed):
    """A permutation of the 7 n cells that maps the cells of rows < n - zk_rows among themselves (random cycles of 1 to 4 cells)
    and fixes the others; w constant on each cycle and random in the zk rows; sigma_k[j] = shift_k' omega^j' for
    (k', j') = pi(k, j); random distinct shifts."""
    P, n = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(seed)
    last = n - zk_rows
    shifts = []
    while len(shifts) < COLS:
        s = rng.randrange(1, P)
        if s not in shifts:
            shifts.append(s)
    omega = ev.omega(orc, fid, log_n)
    pw = [1] * n
    for j in range(1, n):
        pw[j] = pw[j - 1] * omega % P
    w = [[rng.randrange(P) for _ in range(n)] for _ in range(COLS)]
    sigma = [[shifts[k] * pw[j] % P for j in range(n)] for k in range(COLS)]
    cells = list(range(COLS * last))                    # cell c = (k, j) = (c % 7, c // 7)
    rng.shuffle(cells)
    wired = []
    i = 0
    while i < len(cells):
        cyc = cells[i:i + rng.randint(1, 4)]
        i += len(cyc)
        v = rng.randrange(P)
        if len(cyc) > 1:
            wired += [(a % COLS, a // COLS) for a in cyc]
        for a, b in zip(cyc, cyc[1:] + cyc[:1]):           # pi(a) = b
            w[a % COLS][a // COLS] = v
            sigma[a % COLS][a // COLS] = shifts[b % COLS] * pw[b // COLS] % P
    beta, gamma = rng.randrange(P), rng.randrange(P)
    rand = [rng.randrange(P), rng.randrange(P)]
    return Instance(w, sigma, shifts, beta, gamma, rand, wired)


def zero_denominator(inst, P, k, j):
    """w_k[j] = -(beta sigma_k[j] + gamma): den[j] = 0"""
    inst.w[k][j] = (-(inst.beta * inst.sigma[k][j] + inst.gamma)) % P


def sigma_strided(orc, fid, sigma_k, stride, seed):
    """one sigma column as the device reads it: Montgomery [stride n, 4], sigma_k[j] at stride j and random elements elsewhere"""
    n = len(sigma_k)
    out = orc.to_mont(fid, orc.random_scalars(fid, stride * n, seed=seed))
    out[::stride] = ev.mont(orc, fid, sigma_k)
    return np.ascontiguousarray(out)


def sigma_d8(orc, fid, sigma_k):
    """one sigma column as permutation_coefficients8 holds it: Montgomery [8 n, 4], the evaluations over d8 of its interpolation"""
    n = len(sigma_k)
    c = orc.ntt(fid, ev.mont(orc, fid, sigma_k), inverse=True)
    pad = np.zeros((8 * n, 4), dtype=np.uint64)
    pad[:n] = c
    return orc.ntt(fid, pad)
