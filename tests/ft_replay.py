"""The ft polynomial of Maller's optimisation (kimchi/src/prover.rs:1147-1206) restated with Python integers: the terms' sum with
perm_lnrz's stride (permutation.rs:359-386), the interpolation over d1 (the CPU oracle's inverse NTT), to_chunked_polynomial
(utils/src/dense_polynomial.rs:50-69), linearize with its trim and evaluate_chunks (chunked_polynomial.rs:21-51), scale
(dense_polynomial.rs:34-38), ark-poly's trimmed subtraction, evaluate, and PolyComm::chunk_blinding (commitment.rs:79-89).
Field elements are canonical ints; polynomials are coefficient lists."""
import evals_replay as ev


def num_chunks(n: int, m: int) -> int:
    """prover.rs:208-212"""
    return 1 if n < m else n // m


def combine_terms(terms, n: int, P: int) -> list:
    """f_eval[i] = sum_k coeff_k * evals_k[(len_k / n) i]: perm_lnrz (sigma_6 over d8 scaled by perm_scalar) plus the
    linearisation's column terms; terms = [(evals, coeff)]"""
    out = [0] * n
    for evals, c in terms:
        assert len(evals) % n == 0
        s = len(evals) // n
        for i in range(n):
            out[i] = (out[i] + c * evals[s * i]) % P
    return out


def interpolate(orc, fid, evals: list) -> list:
    """Evaluations::interpolate over D(len(evals)), then DensePolynomial::from_coefficients_vec's trim"""
    return trim(ev.ints(orc, fid, orc.ntt(fid, ev.mont(orc, fid, evals), inverse=True)))


def trim(coeffs: list) -> list:
    c = list(coeffs)
    while c and c[-1] == 0:
        c.pop()
    return c


def to_chunked_polynomial(coeffs: list, n_chunks: int, size: int) -> list:
    """the chunks of `size` coefficients, padded with empty polynomials; more chunks than asked is the reference's assert_eq!"""
    chunks = [coeffs[k:k + size] for k in range(0, len(coeffs), size)]
    chunks += [[] for _ in range(n_chunks - len(chunks))]
    if len(chunks) != n_chunks:
        raise ValueError(f"{len(chunks)} chunks, expected {n_chunks}")
    return chunks


def linearize(chunks: list, size: int, zeta_n: int, P: int) -> list:
    """sum_k zeta_n^k chunk_k in a vector of `size` coefficients, trailing zeros trimmed"""
    coeffs, scale = [0] * size, 1
    for poly in chunks:
        for i, c in enumerate(poly[:size]):
            coeffs[i] = (coeffs[i] + scale * c) % P
        scale = scale * zeta_n % P
    return trim(coeffs)


def scale(coeffs: list, elm: int, P: int) -> list:
    """every coefficient times elm; no trim (scaling by 0 keeps the length)"""
    return [c * elm % P for c in coeffs]


def is_zero(p: list) -> bool:
    return all(c == 0 for c in p)


def degree(p: list) -> int:
    if is_zero(p):
        return 0
    assert p[-1] != 0
    return len(p) - 1


def sub(a: list, b: list, P: int) -> list:
    """&a - &b for ark-poly DensePolynomials: the branches of its Sub impl, then truncate_leading_zeros"""
    if is_zero(a):
        r = [(-c) % P for c in b]
    elif is_zero(b):
        r = list(a)
    elif degree(a) >= degree(b):
        r = list(a)
        for i, c in enumerate(b):
            r[i] = (r[i] - c) % P
    else:
        r = list(a) + [0] * (len(b) - len(a))
        for i, c in enumerate(b):
            r[i] = (r[i] - c) % P
    return trim(r)


def evaluate(coeffs: list, x: int, P: int) -> int:
    return ev.horner(coeffs, x, P)


def chunk_blinding(chunks: list, zeta_n: int, P: int) -> int:
    """chunk[0] + zeta_n chunk[1] + zeta_n^2 chunk[2] + ..., by Horner from the last chunk"""
    res = 0
    for c in reversed(chunks):
        res = (res * zeta_n + c) % P
    return res


def ft(orc, fid, log_n: int, m: int, terms, t: list, zeta: int):
    """(f, ft, ft_eval1) of prover.rs:1147-1206; terms = [(evals, coeff)], t the quotient's coefficients"""
    P, n = orc.MODULUS[fid], 1 << log_n
    nc = num_chunks(n, m)
    zeta_m, zh = pow(zeta, m, P), (pow(zeta, n, P) - 1) % P
    f = interpolate(orc, fid, combine_terms(terms, n, P)) if terms else []
    f_chunked = linearize(to_chunked_polynomial(f, nc, m), m, zeta_m, P)
    t_chunked = linearize(to_chunked_polynomial(t, 7 * nc, m), m, zeta_m, P)
    out = sub(f_chunked, scale(t_chunked, zh, P), P)
    return f, out, evaluate(out, zeta * ev.omega(orc, fid, log_n) % P, P)


def blinding_ft(t_blinders: list, zeta: int, log_n: int, m: int, P: int) -> int:
    """prover.rs:1192-1203: blinding_f - (zeta^n - 1) * t_comm.blinders.chunk_blinding(zeta^m), blinding_f = 0"""
    return -(pow(zeta, 1 << log_n, P) - 1) * chunk_blinding(t_blinders, pow(zeta, m, P), P) % P
