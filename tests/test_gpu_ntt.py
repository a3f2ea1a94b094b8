"""NTT parity: CUDA path (through the C ABI) vs the CPU oracle, bit-exact, plus size-independent properties at the
BASELINE sizes.  Mirrors what the reference checks about its FFTs (SURVEY.md §4: no numeric vectors; cross-checks):
kimchi/src/lagrange_basis_evaluations.rs:274-375, poly-commitment/tests/ipa_commitment.rs:27-119."""
import numpy as np
import pytest

import proof_systems_b200 as zk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n", [0, 1, 2, 3, 5, 8, 10, 11, 12, 13, 16])
def test_forward_and_inverse_match_oracle(ctx, orc, fid, log_n):
    n = 1 << log_n
    a = orc.to_mont(fid, orc.random_scalars(fid, n, seed=40 + log_n))
    assert np.array_equal(ctx.ntt(fid, a), orc.ntt(fid, a))
    assert np.array_equal(ctx.ntt(fid, a, inverse=True), orc.ntt(fid, a, inverse=True))


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n", [17, 18, 19])
def test_prover_domain_sizes_match_oracle(ctx, orc, fid, log_n):
    """The d2 / d4 / d8 transforms of a 2^16-gate proof (kimchi/src/circuits/domains.rs:40-69): forward and inverse at full length,
    the forward transform of n = 2^16 coefficients zero-padded to the larger domain (evaluate_over_domain_by_ref(d8),
    kimchi/src/circuits/constraints.rs:488-507), and the inverse that follows the quotient (prover.rs:907), vs the oracle."""
    n = 1 << log_n
    a = orc.to_mont(fid, orc.random_scalars(fid, n, seed=60 + log_n))
    assert np.array_equal(ctx.ntt(fid, a), orc.ntt(fid, a))
    assert np.array_equal(ctx.ntt(fid, a, inverse=True), orc.ntt(fid, a, inverse=True))
    padded = a.copy()
    padded[1 << 16:] = 0
    assert np.array_equal(ctx.ntt(fid, a, in_len=1 << 16), orc.ntt(fid, padded))


@pytest.mark.parametrize("log_n", [17, 19])
def test_batch_16_zero_padded_prover_shape(ctx, orc, log_n):
    """constraints.rs:488-507: 15 witness columns + z, each n = 2^16 coefficients, evaluated over d2 / d8 in ONE batch call;
    every polynomial of the batch must equal its own oracle transform (sampled columns at d8 to bound the CPU time)."""
    fid, n, m, batch = zk.FP, 1 << log_n, 1 << 16, 16
    a = np.zeros((batch, n, 4), dtype=np.uint64)
    a[:, :m] = orc.to_mont(fid, orc.random_scalars(fid, batch * m, seed=71)).reshape(batch, m, 4)
    garbage = a.copy()
    garbage[:, m:] = orc.to_mont(fid, orc.random_scalars(fid, n - m, seed=72))      # beyond in_len: must be ignored
    got = ctx.ntt(fid, garbage, in_len=m)
    for j in (range(batch) if log_n == 17 else (0, 7, 15)):
        assert np.array_equal(got[j], orc.ntt(fid, a[j])), j
    back = ctx.ntt(fid, got, inverse=True)
    assert np.array_equal(back, a)


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n", [4, 10, 14])
def test_coset_transforms_match_oracle(ctx, orc, fid, log_n):
    n = 1 << log_n
    a = orc.to_mont(fid, orc.random_scalars(fid, n, seed=7))
    assert np.array_equal(ctx.ntt(fid, a, coset=True), orc.ntt(fid, a, coset=True))
    assert np.array_equal(ctx.ntt(fid, a, inverse=True, coset=True), orc.ntt(fid, a, inverse=True, coset=True))


@pytest.mark.parametrize("log_n,batch", [(3, 5), (9, 15), (12, 3), (16, 2)])
def test_batched_matches_per_polynomial(ctx, orc, log_n, batch):
    """prover.rs:370-381 issues 15 independent iFFTs; the batch call must equal 15 single calls."""
    fid = zk.FP
    n = 1 << log_n
    a = orc.to_mont(fid, orc.random_scalars(fid, n * batch, seed=3)).reshape(batch, n, 4)
    got = ctx.ntt(fid, a, inverse=True)
    for j in range(batch):
        assert np.array_equal(got[j], orc.ntt(fid, a[j], inverse=True)), j


@pytest.mark.parametrize("log_n,in_len", [(6, 8), (13, 1024), (16, 8192), (10, 1)])
def test_zero_padded_input(ctx, orc, log_n, in_len):
    """evaluate_over_domain of a short polynomial (constraints.rs:490-495: degree < n evaluated over d8)."""
    fid = zk.FQ
    n = 1 << log_n
    coeffs = orc.to_mont(fid, orc.random_scalars(fid, in_len, seed=5))
    padded = np.zeros((n, 4), dtype=np.uint64)
    padded[:in_len] = coeffs
    garbage = padded.copy()
    garbage[in_len:] = orc.to_mont(fid, orc.random_scalars(fid, n - in_len, seed=6))   # must be ignored
    assert np.array_equal(ctx.ntt(fid, garbage, in_len=in_len), orc.ntt(fid, padded))


def test_radix2_domain_mirror(ctx, orc):
    d = zk.Radix2EvaluationDomain(ctx, zk.FP, 1000)     # new(1000) -> size 1024
    assert d.size == 1024 and d.log_size_of_group == 10
    c = orc.to_mont(zk.FP, orc.random_scalars(zk.FP, 700, seed=8))
    ev = d.fft(c)
    padded = np.zeros((1024, 4), dtype=np.uint64)
    padded[:700] = c
    assert np.array_equal(ev, orc.ntt(zk.FP, padded))
    assert np.array_equal(d.ifft(ev), padded)
    assert np.array_equal(d.coset_ifft(d.coset_fft(c)), padded)


@pytest.mark.parametrize("fid", [0, 1])
def test_config3_2_20_roundtrip_and_forward(ctx, orc, fid):
    """BASELINE config 3: 2^20 elements, forward then inverse == input; forward == oracle; delta and linearity."""
    log_n = 20
    n = 1 << log_n
    a = orc.to_mont(fid, orc.random_scalars(fid, n, seed=2))
    f = ctx.ntt(fid, a)
    assert np.array_equal(ctx.ntt(fid, f, inverse=True), a)
    assert np.array_equal(f, orc.ntt(fid, a))
    # linearity: NTT(a + b) = NTT(a) + NTT(b) on a sample of positions
    b = orc.to_mont(fid, orc.random_scalars(fid, n, seed=9))
    idx = [0, 1, 12345, n // 2, n - 1]
    fb = ctx.ntt(fid, b)
    ab = np.stack([orc.fe_add(fid, a[i], b[i]) for i in range(n)]) if False else None
    s = a.copy()
    # build a+b with the device op (already validated in test_gpu_field)
    s = ctx.field_op(fid, "add", a, b)
    fs = ctx.ntt(fid, s)
    for i in idx:
        assert np.array_equal(fs[i], orc.fe_add(fid, f[i], fb[i]))


def test_domain_chain_d1_in_d8(ctx, orc):
    """kimchi/src/circuits/domains.rs:64-66 + ipa.rs:717-722: evaluations over d8, sub-sampled by 8, are those over d1."""
    fid = zk.FP
    n = 1 << 12
    c = orc.to_mont(fid, orc.random_scalars(fid, n, seed=12))
    big = np.zeros((8 * n, 4), dtype=np.uint64)
    big[:n] = c
    ev8 = ctx.ntt(fid, big, in_len=n)
    assert np.array_equal(ev8[::8], ctx.ntt(fid, c))


def test_pinned_host_memory_is_transformed_in_place(ctx, orc):
    """zero-copy path of zk_ntt_batch / zk_msm: page-locked buffers are read and written over PCIe by the kernels"""
    import torch
    for log_n, batch in ((9, 3), (14, 2)):
        n = 1 << log_n
        a = orc.to_mont(zk.FQ, orc.random_scalars(zk.FQ, n * batch, seed=77)).reshape(batch, n, 4)
        t = torch.from_numpy(a.view(np.int64).copy()).pin_memory()
        view = t.numpy().view(np.uint64)
        ctx.ntt_inplace(zk.FQ, view, inverse=True)
        for j in range(batch):
            assert np.array_equal(view[j], orc.ntt(zk.FQ, a[j], inverse=True)), (log_n, j)


@pytest.mark.parametrize("fid,log_n", [(0, 21), (1, 22), (0, 23), (1, 24), (0, 25)])
def test_three_pass_plan_beyond_2_20(ctx, orc, fid, log_n):
    """kimchi's d8 for a 2^18-gate circuit is 2^21 (kimchi/src/circuits/domains.rs:40-69): transforms beyond 2^20 run as three
    passes (n = n1 n2 n3; log2 of the factors 7.7.7, 8.7.7, 8.8.7, 8.8.8 and 9.8.8 from 2^21 to 2^25).  Forward vs the oracle,
    inverse(forward) == input, and the zero-padded form."""
    n = 1 << log_n
    a = orc.to_mont(fid, orc.random_scalars(fid, n, seed=80 + log_n))
    f = ctx.ntt(fid, a)
    assert np.array_equal(f, orc.ntt(fid, a))
    assert np.array_equal(ctx.ntt(fid, f, inverse=True), a)
    padded = a.copy()
    padded[n // 8:] = 0
    assert np.array_equal(ctx.ntt(fid, a, in_len=n // 8), orc.ntt(fid, padded))


def test_out_of_place_device_pipeline(ctx, orc):
    """zk_ntt_dev_oop + zk_dev_*: witness columns stay on the device from interpolation to evaluation over d8 (prover.rs:370-381 ->
    constraints.rs:488-507): iFFT(n) in place on 5 columns, then FFT(8n) reading the n coefficients of each column straight from the
    packed coefficient array (in_stride = n) — no zero-padded copy, no host round trip — equals the oracle's two-step result."""
    fid, log_n, k = zk.FP, 10, 5
    n, m = 1 << log_n, 8 << log_n
    ev = orc.to_mont(fid, orc.random_scalars(fid, k * n, seed=90)).reshape(k, n, 4)
    d_w = ctx.dev_alloc(ev.nbytes)
    d_8 = ctx.dev_alloc(k * m * 32)
    try:
        ctx.dev_upload(d_w, ev)
        ctx.ntt_dev(fid, d_w, log_n, batch=k, inverse=True)
        coeffs = ctx.dev_download(d_w, (k, n, 4))
        ctx.ntt_dev_oop(fid, d_w, n, n, d_8, log_n + 3, batch=k)
        got = ctx.dev_download(d_8, (k, m, 4))
        # the source is untouched by the out-of-place transform
        assert np.array_equal(ctx.dev_download(d_w, (k, n, 4)), coeffs)
        for j in range(k):
            c = orc.ntt(fid, ev[j], inverse=True)
            assert np.array_equal(coeffs[j], c)
            pad = np.zeros((m, 4), dtype=np.uint64)
            pad[:n] = c
            assert np.array_equal(got[j], orc.ntt(fid, pad)), j
            assert np.array_equal(got[j][::8], ev[j])                       # d1 sits inside d8 (domains.rs:64-66)
        # coset variant out of place: the input stays intact as well
        ctx.ntt_dev_oop(fid, d_w, n, n, d_8, log_n + 1, batch=k, coset=True)
        got2 = ctx.dev_download(d_8, (k, 2 * n, 4))
        pad = np.zeros((2 * n, 4), dtype=np.uint64)
        pad[:n] = coeffs[2]
        assert np.array_equal(got2[2], orc.ntt(fid, pad, coset=True))
        assert np.array_equal(ctx.dev_download(d_w, (k, n, 4)), coeffs)
    finally:
        ctx.dev_free(d_w)
        ctx.dev_free(d_8)
