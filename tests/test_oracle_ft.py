"""The restatement of ft (tests/ft_replay.py) against the reference's own unit tests for chunked polynomials, Maller's identity
ft(zeta) = f(zeta) - (zeta^n - 1) t(zeta), and the trimming rules of linearize and the subtraction."""
import random

import pytest

import evals_replay as ev
import ft_replay as fr


def test_chunk_poly():
    """utils/tests/chunked_polynomials.rs::test_chunk_poly"""
    P = 28948022309329048855892746252171976963363056481941560715954676764349967630337
    zeta = 2
    zeta_n = zeta * zeta % P
    res = (1 + zeta) * (1 + zeta_n + zeta_n * zeta**2 + zeta_n * zeta**4) % P
    lin = fr.linearize(fr.to_chunked_polynomial([1] * 8, 4, 2), 2, zeta_n, P)
    assert fr.evaluate(lin, zeta, P) == res


def test_chunk():
    """utils/tests/dense_polynomial.rs::test_chunk"""
    P = 28948022309329048855892746252171976963363056481941560715954676764349967630337
    chunks = fr.to_chunked_polynomial([1] * 8, 4, 2)
    evals = [fr.evaluate(c, 2, P) for c in chunks]
    assert evals == [3] * 4


def test_chunked_polynomial_assert():
    with pytest.raises(ValueError):
        fr.to_chunked_polynomial([1] * 9, 4, 2)
    assert fr.to_chunked_polynomial([], 3, 4) == [[], [], []]


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,m", [(6, 64), (6, 128), (7, 32), (8, 64)])
def test_maller_identity(orc, fid, log_n, m):
    """unchunked, n < m and chunked shapes; random f (one stride-8 term and a stride-1 term) and a full-length t"""
    P, n = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(100 * fid + 10 * log_n + m)
    nc = fr.num_chunks(n, m)
    terms = [([rng.randrange(P) for _ in range(8 * n)], rng.randrange(P)), ([rng.randrange(P) for _ in range(n)], rng.randrange(P))]
    t = [rng.randrange(P) for _ in range(7 * nc * m - rng.randrange(3))]
    zeta = rng.randrange(P)
    f, ft, ft_eval1 = fr.ft(orc, fid, log_n, m, terms, t, zeta)
    assert len(f) <= n and len(ft) <= m
    zh = (pow(zeta, n, P) - 1) % P
    assert fr.evaluate(ft, zeta, P) == (fr.evaluate(f, zeta, P) - zh * fr.evaluate(t, zeta, P)) % P
    assert ft_eval1 == fr.evaluate(ft, zeta * ev.omega(orc, fid, log_n) % P, P)
    # f is the interpolation of the combined evaluations: it reproduces them on d1
    w = ev.omega(orc, fid, log_n)
    f_eval = fr.combine_terms(terms, n, P)
    assert all(fr.evaluate(f, pow(w, i, P), P) == f_eval[i] for i in range(0, n, 7))
    with pytest.raises(ValueError):
        fr.ft(orc, fid, log_n, m, terms, t + [0] * (m + 1), zeta)


def test_trimming(orc):
    """top coefficients that cancel shorten ft; complete cancellation gives the empty polynomial; zeta^n = 1 keeps f's length"""
    fid = 0
    P, log_n, m = orc.MODULUS[fid], 5, 32
    n = 1 << log_n
    rng = random.Random(5)
    terms = [([rng.randrange(P) for _ in range(n)], 1)]
    zeta = rng.randrange(P)
    zh = (pow(zeta, n, P) - 1) % P
    f = fr.interpolate(orc, fid, fr.combine_terms(terms, n, P))
    inv = pow(zh, P - 2, P)
    t_full = [c * inv % P for c in f]                 # zh * t = f: ft = 0
    _, ft, e1 = fr.ft(orc, fid, log_n, m, terms, t_full, zeta)
    assert ft == [] and e1 == 0
    t_part = t_full[:n - 5]                           # the top 5 coefficients remain
    _, ft, _ = fr.ft(orc, fid, log_n, m, terms, t_part, zeta)
    assert len(ft) == len(f) and ft[:n - 5] == [0] * (n - 5)
    t_low = list(t_full)
    t_low[3] = (t_low[3] + 1) % P                     # only coefficient 3 survives
    _, ft, _ = fr.ft(orc, fid, log_n, m, terms, t_low, zeta)
    assert len(ft) == 4 and ft[:3] == [0, 0, 0]
    _, ft, _ = fr.ft(orc, fid, log_n, m, terms, [rng.randrange(P) for _ in range(40)], 1)     # zeta^n - 1 = 0
    assert ft == f
    assert fr.sub([], [1, 2], P) == [P - 1, P - 2] and fr.sub([1, 2], [0, 0], P) == [1, 2] and fr.sub([1, 2], [1, 2], P) == []


def test_chunk_blinding():
    P = 101
    assert fr.chunk_blinding([3, 5, 7], 10, P) == (3 + 5 * 10 + 7 * 100) % P
    assert fr.chunk_blinding([], 10, P) == 0
