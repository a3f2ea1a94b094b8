"""SURVEY.md §8f row 3, first slice: witness polynomials stay on the device from interpolation (kimchi/src/prover.rs:370-381) through
the evaluation over d8 (kimchi/src/circuits/constraints.rs:488-507) into the first pointwise evaluator — the permutation part of
the quotient (kimchi/src/circuits/polynomials/permutation.rs:223-357) — and back through iFFT(8n) (prover.rs:907).  Every stage is
compared bit-exactly with the oracle's restatement computed from the same host inputs."""
import numpy as np
import pytest

import proof_systems_b200 as zk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("fid,log_m", [(0, 10), (1, 13), (0, 21), (1, 22)])
def test_permutation_quotient_kernel_vs_oracle(ctx, orc, fid, log_m):
    m = 1 << log_m
    rnd = lambda k, seed: orc.to_mont(fid, orc.random_scalars(fid, k, seed=seed))
    w, sigma = rnd(7 * m, 1).reshape(7, m, 4), rnd(7 * m, 2).reshape(7, m, 4)
    z, zkpm = rnd(m, 3), rnd(m, 4)
    beta, gamma, alpha0, shifts = rnd(1, 5)[0], rnd(1, 6)[0], rnd(1, 7)[0], rnd(7, 8)
    want = orc.perm_quot(fid, w, z, sigma, zkpm, beta, gamma, alpha0, shifts)
    bufs = {k: ctx.dev_alloc(v.nbytes) for k, v in (("w", w), ("sigma", sigma), ("z", z), ("zkpm", zkpm), ("out", z))}
    try:
        for k, v in (("w", w), ("sigma", sigma), ("z", z), ("zkpm", zkpm)):
            ctx.dev_upload(bufs[k], v)
        cols = lambda base: [base + k * m * 32 for k in range(7)]
        ctx.perm_quotient_dev(fid, log_m, cols(bufs["w"]), bufs["z"], cols(bufs["sigma"]), bufs["zkpm"], beta, gamma, alpha0, shifts, bufs["out"])
        assert np.array_equal(ctx.dev_download(bufs["out"], (m, 4)), want)
    finally:
        for p in bufs.values():
            ctx.dev_free(p)


def test_device_resident_d8_pipeline(ctx, orc):
    """evaluations over d1 (host) -> [device: iFFT(n) of 7 columns + z, FFT(8n) out of place from the packed coefficients, permutation
    quotient over d8, iFFT(8n)] -> quotient-part coefficients (host): ONE upload and ONE download, equal to the oracle's
    interpolate / evaluate_over_domain / perm / interpolate chain."""
    fid, log_n = zk.FP, 9
    n, m = 1 << log_n, 8 << log_n
    rnd = lambda k, seed: orc.to_mont(fid, orc.random_scalars(fid, k, seed=seed))
    cols = rnd(8 * n, 11).reshape(8, n, 4)                       # w_0..w_6 and z as evaluations over d1
    sigma8, zkpm = rnd(7 * m, 12).reshape(7, m, 4), rnd(m, 13)   # per-index precomputations, resident in a real prover
    beta, gamma, alpha0, shifts = rnd(1, 14)[0], rnd(1, 15)[0], rnd(1, 16)[0], rnd(7, 17)
    # ---- oracle
    coeffs = np.stack([orc.ntt(fid, cols[j], inverse=True) for j in range(8)])
    ev8 = []
    for j in range(8):
        pad = np.zeros((m, 4), dtype=np.uint64)
        pad[:n] = coeffs[j]
        ev8.append(orc.ntt(fid, pad))
    ev8 = np.stack(ev8)
    perm = orc.perm_quot(fid, ev8[:7], ev8[7], sigma8, zkpm, beta, gamma, alpha0, shifts)
    want = orc.ntt(fid, perm, inverse=True)
    # ---- device
    d_cols, d_ev8 = ctx.dev_alloc(cols.nbytes), ctx.dev_alloc(8 * m * 32)
    d_sigma, d_zkpm, d_out = ctx.dev_alloc(sigma8.nbytes), ctx.dev_alloc(zkpm.nbytes), ctx.dev_alloc(m * 32)
    try:
        launches0 = ctx.launch_count
        ctx.dev_upload(d_cols, cols)
        ctx.dev_upload(d_sigma, sigma8)
        ctx.dev_upload(d_zkpm, zkpm)
        ctx.ntt_dev(fid, d_cols, log_n, batch=8, inverse=True)                 # prover.rs:370-381
        ctx.ntt_dev_oop(fid, d_cols, n, n, d_ev8, log_n + 3, batch=8)           # constraints.rs:488-507
        ctx.perm_quotient_dev(fid, log_n + 3, [d_ev8 + k * m * 32 for k in range(7)], d_ev8 + 7 * m * 32, [d_sigma + k * m * 32 for k in range(7)], d_zkpm,
                              beta, gamma, alpha0, shifts, d_out)
        ctx.ntt_dev(fid, d_out, log_n + 3, inverse=True)                        # prover.rs:907
        got = ctx.dev_download(d_out, (m, 4))
        assert np.array_equal(got, want)
        assert ctx.launch_count - launches0 >= 6
    finally:
        for p in (d_cols, d_ev8, d_sigma, d_zkpm, d_out):
            ctx.dev_free(p)
