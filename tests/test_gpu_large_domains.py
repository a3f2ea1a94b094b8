"""The size regimes the per-kernel files stop short of.  Several code paths only turn on above fixed sizes: omega^i and g^j take a
third table factor past 2^20 (evals.cu, perm.cu, quotient.cu, the coset scaling in ntt.cu), the three-pass NTT plan runs past 2^20,
the scan over block totals in perm.cu loops from 2^19, zk_ntt_batch pipelines page-locked batches of 8 MiB and more over chunks, and
ntt_run slices batches past the grid's y limit.  Kimchi's d8 for a 2^18-gate circuit is 2^21 (kimchi/src/circuits/domains.rs:40-69).
Every result is compared bit for bit with the CPU oracle or the Python restatements (tests/evals_replay.py, tests/perm_replay.py).
Each test stays below about 2.5 GiB of device memory and 6 GiB of host memory, on a context of its own so that the scratch a large
transform grows is freed when the test ends."""
import random

import numpy as np
import pytest

import evals_replay as ev
import perm_replay as pr
import proof_systems_b200 as zk

pytestmark = pytest.mark.gpu


@pytest.fixture
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def rnd(orc, fid, k, seed):
    return orc.to_mont(fid, orc.random_scalars(fid, k, seed=seed))


def zero_past(a, in_len):
    """a copy of the polynomials a [..., n, 4] with every coefficient from in_len on set to zero"""
    p = a.copy()
    p[..., in_len:, :] = 0
    return p


def canonical_ints(a) -> list:
    """canonical limbs [k, 4] (orc.random_scalars) -> ints"""
    raw = np.ascontiguousarray(a, dtype=np.uint64).tobytes()
    return [int.from_bytes(raw[k:k + 32], "little") for k in range(0, len(raw), 32)]


# ---------------------------------------------------------------------------------------------------------------- three-pass NTT
@pytest.mark.parametrize("fid,log_n", [(0, 21), (1, 23)])
def test_coset_transforms(ctx, orc, fid, log_n):
    """coset forward and inverse vs the oracle, and the forward coset transform of in_len = 3n/4 + 3 coefficients (odd, past 2^20)
    with garbage after them: g^j for j >= 2^20 takes k_coset_scale's third factor, on a zero-padded input"""
    n = 1 << log_n
    a = rnd(orc, fid, n, 100 + log_n)
    assert np.array_equal(ctx.ntt(fid, a, coset=True), orc.ntt(fid, a, coset=True))
    assert np.array_equal(ctx.ntt(fid, a, inverse=True, coset=True), orc.ntt(fid, a, inverse=True, coset=True))
    in_len = 3 * n // 4 + 3
    assert np.array_equal(ctx.ntt(fid, a, coset=True, in_len=in_len), orc.ntt(fid, zero_past(a, in_len), coset=True))


def test_out_of_place_2_18_gates_to_d8(ctx, orc):
    """constraints.rs:488-507 for a 2^18-gate circuit: the 15 witness polynomials, 2^18 coefficients each packed at in_stride = 2^18,
    evaluated over d8 = 2^21 and over its coset by zk_ntt_dev_oop (a batch of 15 three-pass transforms reading a strided source);
    every column vs the oracle, and the source left untouched"""
    fid, log_n, k = zk.FP, 18, 15
    n, m = 1 << log_n, 8 << log_n
    coeffs = rnd(orc, fid, k * n, 110).reshape(k, n, 4)
    with ctx.buffers() as bufs:
        d_c = bufs.put(coeffs)
        d_8 = bufs.alloc(k * m * 32)
        pad = np.zeros((m, 4), dtype=np.uint64)
        for coset in (False, True):
            ctx.ntt_dev_oop(fid, d_c, n, n, d_8, log_n + 3, batch=k, coset=coset)
            assert np.array_equal(ctx.dev_download(d_c, (k, n, 4)), coeffs), coset
            got = ctx.dev_download(d_8, (k, m, 4))
            for j in range(k):
                pad[:n] = coeffs[j]
                assert np.array_equal(got[j], orc.ntt(fid, pad, coset=coset)), (coset, j)
            del got


def test_in_place_batch_of_3_at_2_22(ctx, orc):
    """zk_ntt_dev in place, three polynomials of 2^22 in one call: forward vs the oracle, then the inverse gives the input back"""
    fid, log_n, k = zk.FQ, 22, 3
    n = 1 << log_n
    a = rnd(orc, fid, k * n, 120).reshape(k, n, 4)
    with ctx.buffers() as bufs:
        d = bufs.put(a)
        ctx.ntt_dev(fid, d, log_n, batch=k)
        got = ctx.dev_download(d, (k, n, 4))
        for j in range(k):
            assert np.array_equal(got[j], orc.ntt(fid, a[j])), j
        del got
        ctx.ntt_dev(fid, d, log_n, batch=k, inverse=True)
        assert np.array_equal(ctx.dev_download(d, (k, n, 4)), a)


def test_three_pass_sizes_build_no_full_table(ctx, orc):
    """The n-entry inter-pass table serves the two-pass plan only (2^10 < n <= 2^20).  On a fresh context whose 2^14 tables are
    built (those of the inner transform of 2^21 = 2^7 x 2^14), the first 2^21 transform launches the seven kernels of its
    1024-entry tables and its three passes: no 64 MiB table is built that nothing reads."""
    fid = zk.FP
    a = rnd(orc, fid, 1 << 21, 125)
    ctx.ntt(fid, a[:1 << 14])
    before = ctx.launch_count
    assert np.array_equal(ctx.ntt(fid, a), orc.ntt(fid, a))
    assert ctx.launch_count - before == 7 + 3


# ---------------------------------------------------------------------------------------------------------------- zk_ntt_batch, host memory
@pytest.mark.parametrize("fid,log_n,batch,inverse,in_len,chunks", [
    (0, 17, 5, True, 0, 2),                    # 4 MiB polynomials, 16 MiB chunks and at least two of them: 3 + 2, the last one shorter
    (1, 17, 5, False, 3 * (1 << 15) + 1, 2),   # forward, zero-padded past in_len: only in_len coefficients per polynomial are copied in
    (1, 21, 3, False, 0, 3),                   # 64 MiB polynomials: one per chunk
])
def test_pinned_batch_is_pipelined(ctx, orc, fid, log_n, batch, inverse, in_len, chunks):
    """A page-locked batch of 8 MiB or more is copied in, transformed and copied out in chunks of polynomials on three streams.
    Every polynomial vs the oracle; the launch count shows that the batch ran as `chunks` transforms."""
    import torch
    n = 1 << log_n
    a = rnd(orc, fid, batch * n, 130 + log_n + in_len).reshape(batch, n, 4)
    ctx.ntt(fid, a[0], inverse=inverse)                        # the tables, built once, are not part of the count below
    t = torch.from_numpy(a.view(np.int64).copy()).pin_memory()
    view = t.numpy().view(np.uint64)
    before = ctx.launch_count
    ctx.ntt_inplace(fid, view, inverse=inverse, in_len=in_len)
    assert ctx.launch_count - before == chunks * (2 if log_n <= 20 else 3)
    want = a if not in_len else zero_past(a, in_len)
    for j in range(batch):
        assert np.array_equal(view[j], orc.ntt(fid, want[j], inverse=inverse)), j


def test_batches_beyond_the_grid_y_limit(ctx, orc):
    """ntt_run runs a batch of more than 65535 polynomials in slices of 32768: 2^3 x 70001 in place through zk_ntt_batch, the same
    out of place from a source at in_stride 13 (5 coefficients each), and 2^0 x 65537 out of place at in_stride 3; every
    polynomial vs the oracle"""
    fid = zk.FQ
    n, batch = 8, 70001
    a = rnd(orc, fid, batch * n, 140).reshape(batch, n, 4)
    got = ctx.ntt(fid, a)
    for j in range(batch):
        assert np.array_equal(got[j], orc.ntt(fid, a[j])), j
    del got
    src = rnd(orc, fid, batch * 13, 141).reshape(batch, 13, 4)
    one = rnd(orc, fid, 65537 * 3, 142).reshape(65537, 3, 4)
    with ctx.buffers() as bufs:
        d_src, d_one = bufs.put(src), bufs.put(one)
        d_out = bufs.alloc(batch * n * 32)
        ctx.ntt_dev_oop(fid, d_src, 13, 5, d_out, 3, batch=batch)
        got = ctx.dev_download(d_out, (batch, n, 4))
        pad = np.zeros((n, 4), dtype=np.uint64)
        for j in range(batch):
            pad[:5] = src[j, :5]
            assert np.array_equal(got[j], orc.ntt(fid, pad)), j
        ctx.ntt_dev_oop(fid, d_one, 3, 1, d_out, 0, batch=65537)
        assert np.array_equal(ctx.dev_download(d_out, (65537, 4)), one[:, 0])


# ---------------------------------------------------------------------------------------------------------------- Lagrange basis
@pytest.mark.parametrize("fid,max_poly_size", [(0, 1 << 21), (1, 1 << 19)])
def test_lagrange_basis_and_evaluate_at_2_21(ctx, orc, fid, max_poly_size):
    """LagrangeBasisEvaluations over D(2^21): unchunked (w^-i of i >= 2^20 takes the third table factor) and chunked with
    max_poly_size = 2^19 (four vectors through one batched three-pass inverse NTT).  The basis vs evals_replay.lagrange_basis, and
    evaluate of a random column vs evals_replay.evaluate."""
    log_n = 21
    P, n = orc.MODULUS[fid], 1 << log_n
    x = random.Random(150 + fid).randrange(P)
    col = orc.random_scalars(fid, n, seed=151 + fid)
    basis = ev.lagrange_basis(orc, fid, max_poly_size, log_n, x)
    want_eval = ev.mont(orc, fid, ev.evaluate(basis, canonical_ints(col), P))
    with ctx.buffers() as bufs:
        with zk.LagrangeBasisEvaluations(ctx, fid, max_poly_size, log_n, ev.mont(orc, fid, [x])[0]) as lb:
            assert lb.chunks == len(basis) == max(1, n // max_poly_size)
            got = lb.evals()
            for k, v in enumerate(basis):
                assert np.array_equal(got[k], ev.mont(orc, fid, v)), k
            del got
            d_col = bufs.put(orc.to_mont(fid, col))
            assert np.array_equal(lb.evaluate((d_col, n)), want_eval)


# ---------------------------------------------------------------------------------------------------------------- permutation
def device_z(ctx, orc, fid, log_n, zk_rows, w, sigma, beta, gamma, shifts, rand):
    """zk_perm_aggreg_dev on w [7, n, 4] and sigma [7, s n, 4] (Montgomery; sigma read at stride s); scalars as canonical ints
    -> (z's coefficients, final-value flag)"""
    n = 1 << log_n
    m = lambda xs: ev.mont(orc, fid, xs)
    with ctx.buffers() as bufs:
        d_w, d_s = bufs.put(w), bufs.put(sigma)
        d_z = bufs.alloc(n * 32)
        ok = ctx.perm_aggreg_dev(fid, log_n, zk_rows, [d_w + k * n * 32 for k in range(7)],
                                 [d_s + k * sigma.shape[1] * 32 for k in range(7)], sigma.shape[1], m([beta])[0], m([gamma])[0],
                                 m(shifts), m(rand), d_z)
        return ctx.dev_download(d_z, (n, 4)), ok


def draw_scalars(P, seed):
    rng = random.Random(seed)
    return rng.randrange(P), rng.randrange(P), [rng.randrange(1, P) for _ in range(7)], [rng.randrange(P), rng.randrange(P)]


@pytest.mark.parametrize("fid,log_n,zk_rows,stride", [(0, 19, 3, 8), (1, 21, 9, 1)])
def test_perm_aggreg_random_instance(ctx, orc, fid, log_n, zk_rows, stride):
    """random, unwired witness and sigma columns: z's coefficients and the final-value flag vs perm_replay.  At 2^19 the scan over
    256 block totals gives each thread of k_scan_block_totals two of them; at 2^21 omega^j takes its third table factor past 2^20."""
    P, n = orc.MODULUS[fid], 1 << log_n
    beta, gamma, shifts, rand = draw_scalars(P, 160 + log_n)
    w = orc.random_scalars(fid, 7 * n, seed=161).reshape(7, n, 4)
    sigma = orc.random_scalars(fid, 7 * stride * n, seed=162).reshape(7, stride * n, 4)
    num, den = pr.ratio_factors([canonical_ints(w[k]) for k in range(7)], [canonical_ints(sigma[k, ::stride]) for k in range(7)],
                                shifts, beta, gamma, ev.omega(orc, fid, log_n), P)
    z, want_ok = pr.z_evaluations(num, den, zk_rows, rand, P)
    del num, den
    want = orc.ntt(fid, ev.mont(orc, fid, z), inverse=True)
    del z
    got, ok = device_z(ctx, orc, fid, log_n, zk_rows, orc.to_mont(fid, w), orc.to_mont(fid, sigma), beta, gamma, shifts, rand)
    assert ok == want_ok
    assert np.array_equal(got, want)


@pytest.mark.parametrize("fid,log_n,zk_rows", [(0, 21, 3), (1, 22, 7)])
def test_perm_aggreg_identity_wiring(ctx, orc, fid, log_n, zk_rows):
    """sigma_k = shift_k omega^j, every cell wired to itself: num[j] = den[j] on every row, so z = 1 up to row n - zk_rows, then
    rand0, then rand1 to the end, and the final-value flag is set.  sigma_k is the oracle's transform of the polynomial shift_k X;
    a wrong omega^j on the device breaks num = den."""
    P, n = orc.MODULUS[fid], 1 << log_n
    last = n - zk_rows
    beta, gamma, shifts, rand = draw_scalars(P, 170 + log_n)
    sigma = np.empty((7, n, 4), dtype=np.uint64)
    x = np.zeros((n, 4), dtype=np.uint64)
    for k in range(7):
        x[1] = ev.mont(orc, fid, [shifts[k]])[0]
        sigma[k] = orc.ntt(fid, x)
    del x
    z = np.empty((n, 4), dtype=np.uint64)
    z[:last + 1] = ev.mont(orc, fid, [1])[0]
    z[last + 1], z[last + 2:] = ev.mont(orc, fid, rand)
    want = orc.ntt(fid, z, inverse=True)
    del z
    got, ok = device_z(ctx, orc, fid, log_n, zk_rows, rnd(orc, fid, 7 * n, 171).reshape(7, n, 4), sigma, beta, gamma, shifts, rand)
    assert ok is True
    assert np.array_equal(got, want)
