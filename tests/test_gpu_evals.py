"""The prover's evaluations at zeta and zeta*omega on the device (kimchi/src/prover.rs:1009-1058): zk_lagrange_evals_dev,
zk_lagrange_evaluate_dev and zk_poly_evaluate_chunks_dev, every result compared bit for bit with the Python restatement of
LagrangeBasisEvaluations / evaluate_chunks (tests/evals_replay.py)."""
import random
import threading

import numpy as np
import pytest

import evals_replay as ev
import proof_systems_b200 as zk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def put(ctx, bufs, a):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    p = ctx.dev_alloc(max(a.nbytes, 32))
    bufs.append(p)
    ctx.dev_upload(p, a)
    return p


def free_all(ctx, bufs):
    for p in bufs:
        ctx.dev_free(p)


def device_basis(ctx, orc, fid, m, log_n, x):
    lb = zk.LagrangeBasisEvaluations.new(ctx, fid, m, log_n, ev.mont(orc, fid, [x])[0])
    try:
        return lb.chunks, lb.evals()
    finally:
        lb.close()


def expected_basis(orc, fid, m, log_n, x):
    return np.stack([ev.mont(orc, fid, v) for v in ev.lagrange_basis(orc, fid, m, log_n, x)])


# ---------------------------------------------------------------------------------------------------------------- basis values
@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n", [0, 1, 2, 5, 10, 16])
@pytest.mark.parametrize("mult", [1, 2, 3])
def test_unchunked_basis(ctx, orc, fid, log_n, mult):
    n = 1 << log_n
    x = random.Random(10 * log_n + fid + 1000 * mult).randrange(orc.MODULUS[fid])
    chunks, got = device_basis(ctx, orc, fid, mult * n, log_n, x)
    assert chunks == 1
    assert np.array_equal(got, expected_basis(orc, fid, mult * n, log_n, x))


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,div", [(10, 2), (10, 4), (10, 64), (17, 2)])
def test_chunked_basis(ctx, orc, fid, log_n, div):
    n = 1 << log_n
    x = random.Random(log_n + div + 7 * fid).randrange(orc.MODULUS[fid])
    chunks, got = device_basis(ctx, orc, fid, n // div, log_n, x)
    assert chunks == div == zk.Context.lagrange_evals_chunks(n, n // div)
    assert np.array_equal(got, expected_basis(orc, fid, n // div, log_n, x))


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n", [5, 10])
def test_special_points(ctx, orc, fid, log_n):
    """x = 0; x = 1 and x = w^3 lie in the domain: the whole unchunked basis is zero (batch_inversion_and_mul skips the zero
    denominator and the numerator is zero); x random"""
    P, n = orc.MODULUS[fid], 1 << log_n
    w3 = pow(ev.omega(orc, fid, log_n), 3, P)
    for x in (0, 1, w3, random.Random(log_n).randrange(P)):
        _, got = device_basis(ctx, orc, fid, n, log_n, x)
        want = expected_basis(orc, fid, n, log_n, x)
        assert np.array_equal(got, want), x
        if x in (1, w3):
            assert not want.any()
    _, got = device_basis(ctx, orc, fid, n // 4, log_n, 0)                       # chunked at x = 0
    assert np.array_equal(got, expected_basis(orc, fid, n // 4, log_n, 0))


# ---------------------------------------------------------------------------------------------------------------- evaluate
@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("chunks", [1, 2, 4])
def test_evaluate_two_points_in_one_call(ctx, orc, fid, chunks):
    """strides 1, 4 and 8 against the bases of zeta and zeta*omega in one call"""
    P, log_n = orc.MODULUS[fid], 10
    n = 1 << log_n
    rng = random.Random(fid * 10 + chunks)
    zeta = rng.randrange(P)
    pts = [zeta, zeta * ev.omega(orc, fid, log_n) % P]
    cols = {s: [rng.randrange(P) for _ in range(s * n)] for s in (1, 4, 8)}
    bufs, lbs = [], [zk.LagrangeBasisEvaluations(ctx, fid, n // chunks, log_n, ev.mont(orc, fid, [x])[0]) for x in pts]
    try:
        d = {s: put(ctx, bufs, ev.mont(orc, fid, c)) for s, c in cols.items()}
        got = zk.LagrangeBasisEvaluations.evaluate_all(lbs, [(d[s], s * n, False) for s in (1, 4, 8)])
        assert got.shape == (3, 2, chunks, 4)
        for j, s in enumerate((1, 4, 8)):
            for t, x in enumerate(pts):
                want = ev.evaluate(ev.lagrange_basis(orc, fid, n // chunks, log_n, x), cols[s], P)
                assert np.array_equal(got[j, t], ev.mont(orc, fid, want)), (s, t)
        assert np.array_equal(lbs[1].evaluate((d[4], 4 * n)), got[1, 1])
    finally:
        for lb in lbs:
            lb.close()
        free_all(ctx, bufs)


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("chunks", [1, 2])
def test_evaluate_boolean(ctx, orc, fid, chunks):
    """0/1 columns, and a column with other values: a nonzero value counts as one (the reference's rule)"""
    P, log_n = orc.MODULUS[fid], 9
    n = 1 << log_n
    rng = random.Random(77 + fid + chunks)
    x = rng.randrange(P)
    bits = [rng.randrange(2) for _ in range(4 * n)]
    other = [rng.choice([0, 1, 2, P - 1, rng.randrange(P)]) for _ in range(n)]
    basis = ev.lagrange_basis(orc, fid, n // chunks, log_n, x)
    bufs, lb = [], zk.LagrangeBasisEvaluations(ctx, fid, n // chunks, log_n, ev.mont(orc, fid, [x])[0])
    try:
        d_bits, d_other = put(ctx, bufs, ev.mont(orc, fid, bits)), put(ctx, bufs, ev.mont(orc, fid, other))
        assert np.array_equal(lb.evaluate_boolean((d_bits, 4 * n)), ev.mont(orc, fid, ev.evaluate_boolean(basis, bits, P)))
        got = lb.evaluate_boolean((d_other, n))
        assert np.array_equal(got, ev.mont(orc, fid, ev.evaluate_boolean(basis, other, P)))
        assert not np.array_equal(got, lb.evaluate((d_other, n)))
        both = ctx.lagrange_evaluate_dev(fid, [lb.ptr], log_n, lb.chunks, [(d_other, n, True), (d_other, n, False)])
        assert np.array_equal(both[0, 0], got) and np.array_equal(both[1, 0], ev.mont(orc, fid, ev.evaluate(basis, other, P)))
    finally:
        lb.close()
        free_all(ctx, bufs)


# ---------------------------------------------------------------------------------------------------------------- evaluate_chunks
@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("num_chunks,chunk_size", [(3, 1000), (1, 4096), (2, 1 << 16)])
def test_evaluate_chunks(ctx, orc, fid, num_chunks, chunk_size):
    P = orc.MODULUS[fid]
    rng = random.Random(fid + num_chunks + chunk_size)
    lens = [0, 1, chunk_size - 3, num_chunks * chunk_size, max(0, (num_chunks - 1) * chunk_size - 5)]
    polys = [[rng.randrange(P) for _ in range(k)] for k in lens]
    pts = [0, 1, rng.randrange(P)]
    bufs = []
    try:
        desc = [(put(ctx, bufs, ev.mont(orc, fid, p)) if p else 0, len(p)) for p in polys]
        got = ctx.poly_evaluate_chunks_dev(fid, desc, num_chunks, chunk_size, ev.mont(orc, fid, pts))
        assert got.shape == (len(polys), len(pts), num_chunks, 4)
        for j, p in enumerate(polys):
            for t, x in enumerate(pts):
                assert np.array_equal(got[j, t], ev.mont(orc, fid, ev.evaluate_chunks(p, num_chunks, chunk_size, x, P))), (lens[j], t)
        with pytest.raises(zk.ZkError) as e:
            ctx.poly_evaluate_chunks_dev(fid, desc[3:4], num_chunks - 1, chunk_size, ev.mont(orc, fid, pts))
        assert e.value.code == -4                                                   # ZK_ERR_LENGTH
    finally:
        free_all(ctx, bufs)


# ---------------------------------------------------------------------------------------------------------------- the prover's step
def test_prover_step_at_zeta_and_zeta_omega(ctx, orc):
    """d1 = 2^16, max_poly_size = 2^16: witness, z and public made resident as in the quotient pipeline (iFFT(n) in place, FFT(8n) out
    of place), index columns uploaded once; ONE lagrange_evaluate_dev call (7 s + 15 coefficients over d8, 6 selectors over d4 / d8,
    the 15 witness columns over d8) and ONE poly_evaluate_chunks_dev call (15 w, z, public) give every evaluation at zeta and
    zeta*omega; no column is downloaded.  The witness evaluated both ways (coefficient chunks at zeta, Lagrange basis over d8) agrees."""
    fid, log_n = zk.FP, 16
    P, n = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(2024)
    rnd = lambda k, seed: orc.to_mont(fid, orc.random_scalars(fid, k, seed=seed))
    cols = rnd(17 * n, 31).reshape(17, n, 4)                   # w_0..w_14, z, public as evaluations over d1
    s8, c8 = rnd(7 * 8 * n, 32).reshape(7, 8 * n, 4), rnd(15 * 8 * n, 33).reshape(15, 8 * n, 4)
    one = orc.fe(fid, 1)
    bits = np.random.default_rng(7)
    sel = [np.where(bits.integers(0, 2, size=(k * n, 1)) == 1, one, np.uint64(0)).astype(np.uint64) for k in (4, 4, 8, 8, 8, 8)]
    zeta = rng.randrange(P)
    pts = [zeta, zeta * ev.omega(orc, fid, log_n) % P]
    # ---------------------------------------------------------------- oracle
    coeffs = [ev.ints(orc, fid, orc.ntt(fid, cols[j], inverse=True)) for j in range(17)]
    bases = [ev.lagrange_basis(orc, fid, n, log_n, x) for x in pts]
    host = [ev.ints(orc, fid, a[::len(a) // n]) for a in list(s8) + list(c8) + sel]    # only the entries evaluate reads
    want_l = [[ev.evaluate(b, h, P) if k < 22 else ev.evaluate_boolean(b, h, P) for b in bases] for k, h in enumerate(host)]
    want_c = [[ev.evaluate_chunks(c, 1, n, x, P) for x in pts] for c in coeffs]
    # ---------------------------------------------------------------- device
    bufs = []
    lbs = []
    try:
        d_cols = put(ctx, bufs, cols)
        d_s8, d_c8 = put(ctx, bufs, s8), put(ctx, bufs, c8)
        d_sel = [put(ctx, bufs, s) for s in sel]
        d_w8 = ctx.dev_alloc(15 * 8 * n * 32); bufs.append(d_w8)
        ctx.ntt_dev(fid, d_cols, log_n, batch=17, inverse=True)                      # prover.rs:370-381: the columns' coefficients
        ctx.ntt_dev_oop(fid, d_cols, n, n, d_w8, log_n + 3, batch=15)                 # constraints.rs:488-507: witness over d8
        lbs = [zk.LagrangeBasisEvaluations(ctx, fid, n, log_n, ev.mont(orc, fid, [x])[0]) for x in pts]
        columns = [(d_s8 + k * 8 * n * 32, 8 * n, False) for k in range(7)] + [(d_c8 + k * 8 * n * 32, 8 * n, False) for k in range(15)]
        columns += [(d, s.shape[0], True) for d, s in zip(d_sel, sel)]
        columns += [(d_w8 + k * 8 * n * 32, 8 * n, False) for k in range(15)]
        got_l = zk.LagrangeBasisEvaluations.evaluate_all(lbs, columns)
        got_c = ctx.poly_evaluate_chunks_dev(fid, [(d_cols + j * n * 32, n) for j in range(17)], 1, n, ev.mont(orc, fid, pts))
    finally:
        for lb in lbs:
            lb.close()
        free_all(ctx, bufs)
    for k in range(28):
        for t in range(2):
            assert np.array_equal(got_l[k, t], ev.mont(orc, fid, want_l[k][t])), (k, t)
    for j in range(17):
        for t in range(2):
            assert np.array_equal(got_c[j, t], ev.mont(orc, fid, want_c[j][t])), (j, t)
    for k in range(15):                                                               # two device paths agree
        assert np.array_equal(got_l[28 + k, :, 0], got_c[k, :, 0]), k


# ---------------------------------------------------------------------------------------------------------------- errors, threads
def test_errors(ctx, orc):
    L, h, fid = zk.lib(), ctx._h, zk.FP
    P = orc.MODULUS[fid]
    x = ev.mont(orc, fid, [5])[0]
    bad_x = np.array([P & (2**64 - 1), (P >> 64) & (2**64 - 1), (P >> 128) & (2**64 - 1), P >> 192], dtype=np.uint64)
    bufs = []
    try:
        d = ctx.dev_alloc(64 * 32); bufs.append(d)
        inv = lambda f: pytest.raises(zk.ZkError, match="error -1")
        with inv(0): ctx.lagrange_basis_evals_dev(7, 4, 16, x, d)                     # unknown field
        with inv(0): ctx.lagrange_basis_evals_dev(fid, 31, 16, x, d)                  # log_n > 30
        with inv(0): ctx.lagrange_basis_evals_dev(fid, 4, 0, x, d)                    # max_poly_size == 0
        with inv(0): ctx.lagrange_basis_evals_dev(fid, 4, 3, x, d)                    # 16 % 3 != 0
        with inv(0): ctx.lagrange_basis_evals_dev(fid, 4, 16, bad_x, d)               # not a canonical element
        with inv(0): ctx.lagrange_basis_evals_dev(fid, 4, 16, x, 0)                   # null output
        assert L.zk_lagrange_evals_dev(h, fid, 4, 16, None, d) == -1                  # null point
        assert zk.Context.lagrange_evals_chunks(16, 3) == 0 and zk.Context.lagrange_evals_chunks(16, 0) == 0
        assert zk.Context.lagrange_evals_chunks(16, 32) == 1 and zk.Context.lagrange_evals_chunks(16, 4) == 4
        assert ctx.lagrange_basis_evals_dev(fid, 4, 16, x, d) == 1
        with inv(0): ctx.lagrange_evaluate_dev(fid, [d], 4, 1, [(d, 0, False)])       # empty column
        with inv(0): ctx.lagrange_evaluate_dev(fid, [d], 4, 1, [(d, 24, False)])      # not a multiple of n
        with inv(0): ctx.lagrange_evaluate_dev(fid, [d], 4, 3, [(d, 16, False)])      # no basis of D(16) has 3 chunks
        with inv(0): ctx.lagrange_evaluate_dev(fid, [d], 4, 32, [(d, 16, False)])
        with inv(0): ctx.lagrange_evaluate_dev(fid, [0], 4, 1, [(d, 16, False)])      # null basis
        with inv(0): ctx.lagrange_evaluate_dev(fid, [d], 4, 1, [(0, 16, False)])      # null column
        with inv(0): ctx.lagrange_evaluate_dev(9, [d], 4, 1, [(d, 16, False)])
        with inv(0): ctx.lagrange_evaluate_dev(fid, [d], 31, 1, [(d, 16, False)])
        with inv(0): ctx.poly_evaluate_chunks_dev(fid, [(d, 16)], 1, 0, [x])         # chunk_size == 0
        with inv(0): ctx.poly_evaluate_chunks_dev(fid, [(0, 16)], 1, 16, [x])        # null polynomial
        with inv(0): ctx.poly_evaluate_chunks_dev(fid, [(d, 16)], 1, 16, [bad_x])    # not a canonical point
        with inv(0): ctx.poly_evaluate_chunks_dev(3, [(d, 16)], 1, 16, [x])
        with pytest.raises(zk.ZkError) as e:
            ctx.poly_evaluate_chunks_dev(fid, [(d, 17)], 1, 16, [x])
        assert e.value.code == -4 and "more than 1 chunks of 16" in str(e.value)
        assert ctx.poly_evaluate_chunks_dev(fid, [(d, 16)], 1, 16, [x]).shape == (1, 1, 1, 4)
    finally:
        free_all(ctx, bufs)


def test_two_threads_share_a_context(ctx, orc):
    fid, log_n = zk.FQ, 12
    P, n = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(9)
    col = [rng.randrange(P) for _ in range(4 * n)]
    coeffs = [rng.randrange(P) for _ in range(n)]
    xs = [rng.randrange(P) for _ in range(2)]
    want = [(ev.evaluate(ev.lagrange_basis(orc, fid, n // 2, log_n, x), col, P), ev.evaluate_chunks(coeffs, 2, n // 2, x, P)) for x in xs]
    bufs = []
    d_col, d_coeffs = put(ctx, bufs, ev.mont(orc, fid, col)), put(ctx, bufs, ev.mont(orc, fid, coeffs))
    errors = []

    def work(t):
        try:
            xm = ev.mont(orc, fid, [xs[t]])
            for _ in range(6):
                lb = zk.LagrangeBasisEvaluations(ctx, fid, n // 2, log_n, xm[0])
                try:
                    got = lb.evaluate((d_col, 4 * n))
                finally:
                    lb.close()
                assert np.array_equal(got, ev.mont(orc, fid, want[t][0]))
                got = ctx.poly_evaluate_chunks_dev(fid, [(d_coeffs, n)], 2, n // 2, xm)[0, 0]
                assert np.array_equal(got, ev.mont(orc, fid, want[t][1]))
        except Exception as e:                    # reported by the main thread
            errors.append(e)

    try:
        th = [threading.Thread(target=work, args=(t,)) for t in range(2)]
        for t in th:
            t.start()
        for t in th:
            t.join()
    finally:
        free_all(ctx, bufs)
    assert not errors, errors
