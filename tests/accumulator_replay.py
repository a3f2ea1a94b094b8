"""batch_dlog_accumulator_check and batch_dlog_accumulator_generate (poly-commitment/src/utils.rs:204-312, the same code as
kimchi-stubs/src/urs_utils.rs:10-101) restated on the CPU oracle, quirks included, and the accumulators the tests feed them.

Scalars are canonical Python integers, points affine Montgomery arrays (identity = zeros).  Where the reference panics the
restatement raises `Panic`: k = 0 with challenges, fewer challenges than accumulators (`% 0`), a remainder, and for the check
2^rounds != |g|.  The check uses only the first k chunks of challenges (`zip(rs)`); generate makes one point per chunk, so 8
challenges for k = 3 give rounds 2 and 4 points; msm_bigint truncates the coefficients to g[..2^rounds].  Test infrastructure only."""
import numpy as np

from verify_replay import b_poly_coefficients

ZERO_PT = np.zeros(8, dtype=np.uint64)


class Panic(Exception):
    """the reference panics here"""


def rounds_of(k: int, chals: list) -> int:
    """rounds = chals.len() / k with the reference's asserts; 0 for k = 0 without challenges"""
    if k == 0:
        if chals:
            raise Panic("assert_eq!(chals.len(), 0)")
        return 0
    rounds = len(chals) // k
    if rounds == 0:
        raise Panic("chals.len() % 0")
    if len(chals) % rounds:
        raise Panic("assert_eq!(chals.len() % rounds, 0)")
    return rounds


def chunks(chals: list, rounds: int) -> list:
    return [chals[o:o + rounds] for o in range(0, len(chals), rounds)]


def check_sum(orc, cid, g, comms, chals, r):
    """the point batch_dlog_accumulator_check compares with zero, affine [8]: MSM(g || comms, (-sum_i r^i s_i) || (r^0 .. r^(k-1)))"""
    m = orc.MODULUS[orc.SCALAR_FIELD[cid]]
    k, n = len(comms), g.shape[0]
    rounds = rounds_of(k, chals)
    if k == 0:
        return ZERO_PT.copy()
    if rounds >= 64 or (1 << rounds) != n:                      # assert_eq!(terms.len(), n), before any term is used
        raise Panic("assert_eq!(terms.len(), n)")
    rs = [1] * k
    for i in range(1, k):
        rs[i] = r * rs[i - 1] % m
    scalars = [0] * n + rs
    for chunk, ri in zip(chunks(chals, rounds), rs):             # the first k chunks only
        for j, v in enumerate(b_poly_coefficients(chunk, m)):
            scalars[j] -= ri * v
    points = np.concatenate([g, np.asarray(comms, dtype=np.uint64).reshape(-1, 8)])
    return orc.msm(cid, points, orc.ints_to_limbs([x % m for x in scalars]))


def check(orc, cid, g, comms, chals, r) -> bool:
    return not check_sum(orc, cid, g, comms, chals, r).any()


def generate(orc, cid, g, num_comms, chals) -> np.ndarray:
    """batch_dlog_accumulator_generate: uint64 [len(chals) / rounds, 8]"""
    m = orc.MODULUS[orc.SCALAR_FIELD[cid]]
    rounds = rounds_of(num_comms, chals)
    if num_comms == 0:
        return np.zeros((0, 8), dtype=np.uint64)
    n = g.shape[0]
    out = []
    for chunk in chunks(chals, rounds):
        s = b_poly_coefficients(chunk, m)[:n]                    # msm_bigint over min(|g|, 2^rounds) pairs
        out.append(orc.msm(cid, g[:len(s)], orc.ints_to_limbs(s)))
    return np.stack(out)


def random_chals(orc, fid, n, seed) -> list:
    return orc.limbs_to_ints(orc.random_scalars(fid, n, seed=seed)) if n else []


def mont(orc, fid, xs) -> np.ndarray:
    """canonical integers -> Montgomery limbs [n, 4]"""
    return orc.to_mont(fid, orc.ints_to_limbs(list(xs))) if len(xs) else np.zeros((0, 4), dtype=np.uint64)


PERTURBATIONS = ["replace", "swap", "challenge"]


def perturb(orc, cid, comms, chals, rounds, kind, other_point, at=0):
    """(comms, chals) with one change: commitment `at` replaced by other_point, commitments at and at + 1 swapped, or the first
    challenge of accumulator `at` changed"""
    comms, chals = np.array(comms, dtype=np.uint64, copy=True), list(chals)
    if kind == "replace":
        comms[at] = other_point
    elif kind == "swap":
        comms[[at, at + 1]] = comms[[at + 1, at]]
    elif kind == "challenge":
        chals[at * rounds] = (chals[at * rounds] + 1) % orc.MODULUS[orc.SCALAR_FIELD[cid]]
    else:
        raise ValueError(kind)
    return comms, chals
