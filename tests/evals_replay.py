"""The prover's evaluation step at zeta and zeta*omega (kimchi/src/prover.rs:1009-1058) restated with Python integers:
LagrangeBasisEvaluations::{new, evaluate, evaluate_boolean} (kimchi/src/lagrange_basis_evaluations.rs:72-258), with ark_ff's
batch_inversion_and_mul, and DensePolynomial::to_chunked_polynomial(..).evaluate_chunks (utils/src/dense_polynomial.rs:50-69,
chunked_polynomial.rs:21-28).  Field elements are canonical ints here; `ints` / `mont` convert from / to the library's Montgomery limbs.
The chunked basis takes its inverse FFT from the CPU oracle (orc.ntt)."""
import numpy as np


def ints(orc, fid, a) -> list:
    """Montgomery limbs [..., 4] -> canonical ints (flattened)"""
    raw = np.ascontiguousarray(orc.from_mont(fid, np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4))).tobytes()
    return [int.from_bytes(raw[k:k + 32], "little") for k in range(0, len(raw), 32)]


def mont(orc, fid, xs) -> np.ndarray:
    """canonical ints -> Montgomery limbs [len, 4]"""
    raw = b"".join(int(x).to_bytes(32, "little") for x in xs)
    return orc.to_mont(fid, np.frombuffer(raw, dtype="<u8").reshape(-1, 4).copy())


def omega(orc, fid, log_n) -> int:
    return ints(orc, fid, orc.root_of_unity(fid, log_n))[0]


def batch_inversion_and_mul(v: list, coeff: int, P: int) -> list:
    """ark_ff::batch_inversion_and_mul (serial form): every NONZERO entry becomes coeff / entry, zeros are skipped and stay zero"""
    prod, tmp = [], 1
    for f in v:
        if f:
            tmp = tmp * f % P
            prod.append(tmp)
    tmp = pow(tmp, P - 2, P) * coeff % P
    out = list(v)
    nz = [i for i, f in enumerate(v) if f]
    prev = [1] + prod[:-1]
    for k in reversed(range(len(nz))):
        i = nz[k]
        f = v[i]
        out[i] = tmp * prev[k] % P
        tmp = tmp * f % P
    return out


def basis_segment_size_1(orc, fid, log_n: int, x: int) -> list:
    """new_with_segment_size_1 (:126-198): l_i = (x^n - 1) / (w^-i t_0 (x - w^i)) through batch_inversion_and_mul"""
    P, n = orc.MODULUS[fid], 1 << log_n
    w = omega(orc, fid, log_n)
    omegas = [1] * n
    for i in range(1, n):
        omegas[i] = omegas[i - 1] * w % P
    t0 = 1
    for wi in omegas[1:]:
        t0 = t0 * (1 - wi) % P
    denoms = [omegas[(n - i) % n] * t0 % P * ((x - omegas[i]) % P) % P for i in range(n)]
    return batch_inversion_and_mul(denoms, (pow(x, n, P) - 1) % P, P)


def basis_chunked(orc, fid, max_poly_size: int, log_n: int, x: int) -> list:
    """new_with_chunked_segments (:203-240): vector i = iFFT(n) of x^0 .. x^{m-1} at positions i m .. (i+1) m - 1"""
    P, n, m = orc.MODULUS[fid], 1 << log_n, max_poly_size
    assert n % m == 0
    out = []
    for i in range(n // m):
        v = [0] * n
        xp = 1
        for j in range(m):
            v[i * m + j] = xp
            xp = xp * x % P
        out.append(ints(orc, fid, orc.ntt(fid, mont(orc, fid, v), inverse=True)))
    return out


def lagrange_basis(orc, fid, max_poly_size: int, log_n: int, x: int) -> list:
    """LagrangeBasisEvaluations::new (:242-258): a list of chunks, each a list of n ints"""
    if (1 << log_n) <= max_poly_size:
        return [basis_segment_size_1(orc, fid, log_n, x)]
    return basis_chunked(orc, fid, max_poly_size, log_n, x)


def evaluate(basis: list, p: list, P: int) -> list:
    """evaluate (:72-109): chunk j is sum_i p[stride i] l_j[i]"""
    n = len(basis[0])
    assert len(p) % n == 0
    stride = len(p) // n
    return [sum(p[stride * i] * e for i, e in enumerate(l)) % P for l in basis]


def evaluate_boolean(basis: list, p: list, P: int) -> list:
    """evaluate_boolean (:116-131): chunk j is the sum of l_j[i] over every i with p[stride i] != 0"""
    n = len(basis[0])
    assert len(p) % n == 0
    stride = len(p) // n
    return [sum(e for i, e in enumerate(l) if p[stride * i] != 0) % P for l in basis]


def horner(coeffs: list, x: int, P: int) -> int:
    acc = 0
    for c in reversed(coeffs):
        acc = (acc * x + c) % P
    return acc


def evaluate_chunks(coeffs: list, num_chunks: int, chunk_size: int, x: int, P: int) -> list:
    """to_chunked_polynomial(num_chunks, chunk_size).evaluate_chunks(x): chunks past the end are zero polynomials; more chunks
    than num_chunks is the reference's assert_eq! (ValueError here)"""
    chunks = [coeffs[k:k + chunk_size] for k in range(0, len(coeffs), chunk_size)]
    chunks += [[]] * (num_chunks - len(chunks))
    if len(chunks) != num_chunks:
        raise ValueError(f"{len(chunks)} chunks, expected {num_chunks}")
    return [horner(c, x, P) for c in chunks]


def interpolate_then_evaluate(orc, fid, evals: list, x: int) -> int:
    """Evaluations::interpolate().evaluate(&x)"""
    return horner(ints(orc, fid, orc.ntt(fid, mont(orc, fid, evals), inverse=True)), x, orc.MODULUS[fid])
