"""The library on a caller's CUDA stream (zk_ctx_set_stream), on torch's default stream, across stream switches and in profiled
runs: every result compared bit for bit with the CPU oracle or the Python restatements.

Ordering is made to show up as wrong values.  Each call's device inputs start out as zeros; a spin kernel (torch.cuda._sleep) is
queued on the caller's stream, then torch copies the real inputs in on that same stream, then the library is called, then torch
clones the outputs on the stream, and the host synchronises once at the end.  A library call that launched anything on another
stream would run while the spin holds the copies back, read zeros and produce a wrong result."""
import random
import threading

import numpy as np
import pytest
import torch

import evals_replay as ev
import ft_replay as fr
import gate_programs as gp
import perm_replay as pr
import proof_systems_b200 as zk
from open_replay import opening_proof_bytes_product_level
from test_gpu_perm_aggreg import scalars as perm_scalars
from test_gpu_quotient_pipeline import QuotientCase
from test_gpu_verify import device_verify, hash_entries, scales
from verify_replay import oracle_verify, tamper

pytestmark = pytest.mark.gpu

SPIN = 20_000_000          # cycles of the spin kernel: about 10 ms at the H100's 1.6 to 2 GHz
STALE = 0x0123456789ABCDEF


@pytest.fixture(scope="module")
def stream():
    return torch.cuda.Stream()


@pytest.fixture(scope="module")
def ctx(stream):
    c = zk.Context(0)
    c.set_stream(stream.cuda_stream)
    yield c
    c.close()


def dev(a) -> torch.Tensor:
    """uint64 numpy -> a device tensor with the same bytes"""
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).cuda()


def host(t: torch.Tensor) -> np.ndarray:
    return t.cpu().numpy().view(np.uint64)


def stale(*shape) -> torch.Tensor:
    """an output buffer holding a recognisable pattern: nothing of it may survive where the library writes"""
    return torch.full(shape, STALE, dtype=torch.int64, device="cuda")


class Inputs:
    """Device copies of the inputs (ready before anything is queued) and the zeroed buffers the library reads, which only the
    caller's stream fills, behind the spin"""

    def __init__(self):
        self.pairs = []

    def __call__(self, a) -> int:
        src = dev(a)
        dst = torch.zeros_like(src)
        self.pairs.append((dst, src))
        return dst.data_ptr()


def on_stream(stream, inputs, call, outputs=()):
    """Queues on `stream`: the spin, the copies of `inputs`, call(), clones of `outputs`; one synchronisation at the end.
    Returns (call's value, the clones as uint64 numpy arrays)."""
    torch.cuda.synchronize()                 # the sources and the zeroed / stale buffers are in place before anything is queued
    with torch.cuda.stream(stream):
        torch.cuda._sleep(SPIN)
        for dst, src in (inputs.pairs if inputs else []):
            dst.copy_(src)
        r = call()
        got = [o.clone() for o in outputs]
    stream.synchronize()
    return r, [host(g) for g in got]


def mont_rnd(orc, fid, k, seed):
    return orc.to_mont(fid, orc.random_scalars(fid, k, seed=seed))


def zero_past(a, in_len):
    a = a.copy()
    a[..., in_len:, :] = 0
    return a


def add_mont(orc, fid, a, b):
    P = orc.MODULUS[fid]
    s = [(x + y) % P for x, y in zip(orc.limbs_to_ints(orc.from_mont(fid, a)), orc.limbs_to_ints(orc.from_mont(fid, b)))]
    return orc.to_mont(fid, orc.ints_to_limbs(s))


# ---------------------------------------------------------------------------------------------------------------- device entry points
def test_ntt_dev_in_place_coset_zero_padded(ctx, stream, orc):
    """2^12 (two passes through the context's second buffer), a batch of two, a coset and the first 3000 coefficients read"""
    fid, log_n, in_len = zk.FP, 12, 3000
    a = mont_rnd(orc, fid, 2 << log_n, 1).reshape(2, 1 << log_n, 4)
    inp = Inputs()
    d = inp(a)
    _, (got,) = on_stream(stream, inp, lambda: ctx.ntt_dev(fid, d, log_n, batch=2, in_len=in_len, coset=True), [inp.pairs[0][0]])
    want = zero_past(a, in_len)
    for b in range(2):
        assert np.array_equal(got.reshape(2, -1, 4)[b], orc.ntt(fid, want[b], coset=True)), b


def test_ntt_dev_oop_d1_to_d8(ctx, stream, orc):
    fid, log_n, batch = zk.FQ, 9, 3
    n, m = 1 << log_n, 8 << log_n
    a = mont_rnd(orc, fid, batch * n, 2).reshape(batch, n, 4)
    inp = Inputs()
    d_in = inp(a)
    out = stale(batch, m, 4)
    _, (got,) = on_stream(stream, inp, lambda: ctx.ntt_dev_oop(fid, d_in, n, n, out.data_ptr(), log_n + 3, batch=batch), [out])
    for b in range(batch):
        pad = np.zeros((m, 4), dtype=np.uint64); pad[:n] = a[b]
        assert np.array_equal(got.reshape(batch, m, 4)[b], orc.ntt(fid, pad)), b


def test_msm_dev(ctx, stream, orc, vesta_srs):
    G, n = vesta_srs, 2048
    sc = orc.random_scalars(G.scalar, n, seed=3)
    with ctx.upload_bases(G.cid, G.g[:n]) as bases:
        inp = Inputs()
        d = inp(sc)
        r, _ = on_stream(stream, inp, lambda: ctx.msm_dev(bases, d, n))
        assert np.array_equal(zk.jacobian_to_affine(G.cid, r), orc.msm(G.cid, G.g[:n], sc))


def test_msm_partial_and_finish_gathered(ctx, stream, orc, vesta_srs):
    G, n = vesta_srs, 2048
    sc = orc.random_scalars(G.scalar, n, seed=4)
    with ctx.upload_bases(G.cid, G.g[:n]) as bases:
        inp = Inputs()
        d = inp(sc)
        d_all = torch.zeros((4096, 16), dtype=torch.int64, device="cuda")

        def call():
            c, g = ctx.msm_partial(bases, d, n, d_all.data_ptr(), 4096)
            return ctx.msm_finish_gathered(G.cid, d_all.data_ptr(), 1, c, g)
        r, _ = on_stream(stream, inp, call)
        assert np.array_equal(zk.jacobian_to_affine(G.cid, r), orc.msm(G.cid, G.g[:n], sc))


def test_poly_add_and_divide_by_vanishing(ctx, stream, orc):
    fid, log_n = zk.FQ, 10
    n = 1 << log_n
    f, g = mont_rnd(orc, fid, 8 * n, 5), mont_rnd(orc, fid, 4 * n, 6)
    fg = f.copy()
    fg[:4 * n] = add_mont(orc, fid, f[:4 * n], g)
    want_q, want_r = orc.divide_by_vanishing(fid, fg, log_n)
    inp = Inputs()
    d_f, d_g = inp(f), inp(g)
    q = stale(7 * n, 4)

    def call():
        ctx.poly_add_dev(fid, d_f, d_g, 4 * n)
        return ctx.poly_divide_by_vanishing_dev(fid, d_f, 8 * n, log_n, q.data_ptr())
    zero_rem, (got_f, got_q) = on_stream(stream, inp, call, [inp.pairs[0][0], q])
    assert want_r.any() and zero_rem is False
    assert np.array_equal(got_f.reshape(-1, 4), fg)
    assert np.array_equal(got_q.reshape(-1, 4), want_q)


def test_expr_eval_generic_then_accumulate(ctx, stream, orc):
    """the generic gate over d4, then the poseidon gate accumulated into a d8 buffer the stream also fills"""
    fid, log_n = zk.FP, 8
    n, m = 1 << log_n, 8 << log_n
    cols = mont_rnd(orc, fid, 30 * m, 7).reshape(30, m, 4)
    sel4, sel8, acc = mont_rnd(orc, fid, 4 * n, 8), mont_rnd(orc, fid, m, 9), mont_rnd(orc, fid, m, 10)
    alphas, mds = mont_rnd(orc, fid, 17, 11), mont_rnd(orc, fid, 9, 12).reshape(3, 3, 4)
    gen, pos = gp.generic_gate(gp.Recorder(), alphas[:2]), gp.poseidon_gate(gp.Recorder(), alphas[2:], mds)
    base = [(cols[k], 8) for k in range(30)]
    want4 = orc.expr_eval(fid, gen.ops, gen.args, gen.literals, base + [(sel4, 4)], 4 * n)
    want8 = orc.expr_eval(fid, pos.ops, pos.args, pos.literals, base + [(sel8, 8)], m, acc=acc)
    inp = Inputs()
    d_cols, d_sel4, d_sel8, d_acc = inp(cols), inp(sel4), inp(sel8), inp(acc)
    t4 = stale(4 * n, 4)
    dc = [(d_cols + k * m * 32, m, 8) for k in range(30)]

    def call():
        gp.generic_gate(zk.ExprProgram(), alphas[:2]).evaluations(ctx, fid, dc + [(d_sel4, 4 * n, 4)], 4 * n, 4, t4.data_ptr())
        gp.poseidon_gate(zk.ExprProgram(), alphas[2:], mds).evaluations(ctx, fid, dc + [(d_sel8, m, 8)], m, 8, d_acc, accumulate=True)
    _, (got4, got8) = on_stream(stream, inp, call, [t4, inp.pairs[3][0]])
    assert np.array_equal(got4.reshape(-1, 4), want4)
    assert np.array_equal(got8.reshape(-1, 4), want8)


def test_perm_quotient_dev(ctx, stream, orc):
    fid, log_m = zk.FQ, 11
    m = 1 << log_m
    w, sigma = mont_rnd(orc, fid, 7 * m, 13).reshape(7, m, 4), mont_rnd(orc, fid, 7 * m, 14).reshape(7, m, 4)
    z, zkpm = mont_rnd(orc, fid, m, 15), mont_rnd(orc, fid, m, 16)
    beta, gamma, alpha0, shifts = mont_rnd(orc, fid, 1, 17)[0], mont_rnd(orc, fid, 1, 18)[0], mont_rnd(orc, fid, 1, 19)[0], mont_rnd(orc, fid, 7, 20)
    want = orc.perm_quot(fid, w, z, sigma, zkpm, beta, gamma, alpha0, shifts)
    inp = Inputs()
    d_w, d_s, d_z, d_zkpm = inp(w), inp(sigma), inp(z), inp(zkpm)
    out = stale(m, 4)
    call = lambda: ctx.perm_quotient_dev(fid, log_m, [d_w + k * m * 32 for k in range(7)], d_z, [d_s + k * m * 32 for k in range(7)], d_zkpm,
                                         beta, gamma, alpha0, shifts, out.data_ptr())
    _, (got,) = on_stream(stream, inp, call, [out])
    assert np.array_equal(got.reshape(-1, 4), want)


def test_perm_aggreg_dev(ctx, stream, orc):
    fid, log_n, zk_rows, stride = zk.FP, 10, 3, 8
    n = 1 << log_n
    inst = pr.wired_instance(orc, fid, log_n, zk_rows, seed=21)
    _, coeffs, want_ok = pr.perm_aggreg(orc, fid, log_n, zk_rows, inst.w, inst.sigma, inst.shifts, inst.beta, inst.gamma, inst.rand)
    inp = Inputs()
    d_w = [inp(ev.mont(orc, fid, inst.w[k])) for k in range(7)]
    d_s = [inp(pr.sigma_strided(orc, fid, inst.sigma[k], stride, 30 + k)) for k in range(7)]
    z = stale(n, 4)
    ok, (got,) = on_stream(stream, inp, lambda: ctx.perm_aggreg_dev(fid, log_n, zk_rows, d_w, d_s, stride * n, *perm_scalars(orc, fid, inst), z.data_ptr()),
                           [z])
    assert want_ok and ok
    assert np.array_equal(got.reshape(-1, 4), ev.mont(orc, fid, coeffs))


@pytest.mark.parametrize("chunks", [1, 4])
def test_lagrange_basis_then_evaluate(ctx, stream, orc, chunks):
    """the basis of LagrangeBasisEvaluations (unchunked and in four chunks) into a stale buffer, then evaluate of a stride-4 column"""
    fid, log_n = zk.FQ, 10
    P, n = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(chunks)
    x = rng.randrange(P)
    col = [rng.randrange(P) for _ in range(4 * n)]
    basis = ev.lagrange_basis(orc, fid, n // chunks, log_n, x)
    inp = Inputs()
    d_col = inp(ev.mont(orc, fid, col))
    d_basis = stale(chunks, n, 4)

    def call():
        assert ctx.lagrange_basis_evals_dev(fid, log_n, n // chunks, ev.mont(orc, fid, [x])[0], d_basis.data_ptr()) == chunks
        return ctx.lagrange_evaluate_dev(fid, [d_basis.data_ptr()], log_n, chunks, [(d_col, 4 * n, False)])
    r, (got_basis,) = on_stream(stream, inp, call, [d_basis])
    assert np.array_equal(got_basis.reshape(chunks, n, 4), np.stack([ev.mont(orc, fid, v) for v in basis]))
    assert np.array_equal(r[0, 0], ev.mont(orc, fid, ev.evaluate(basis, col, P)))


def test_poly_evaluate_chunks_dev(ctx, stream, orc):
    fid, log_n = zk.FP, 8
    P, size = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(5)
    coeffs = [rng.randrange(P) for _ in range(3 * size + 5)]
    zeta = rng.randrange(P)
    pts = [zeta, zeta * ev.omega(orc, fid, log_n) % P]
    inp = Inputs()
    d = inp(ev.mont(orc, fid, coeffs))
    r, _ = on_stream(stream, inp, lambda: ctx.poly_evaluate_chunks_dev(fid, [(d, len(coeffs))], 4, size, ev.mont(orc, fid, pts)))
    for t, x in enumerate(pts):
        assert np.array_equal(r[0, t], ev.mont(orc, fid, ev.evaluate_chunks(coeffs, 4, size, x, P))), t


def test_prover_ft_dev(ctx, stream, orc):
    fid, log_n, m = zk.FQ, 8, 128
    P, n = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(6)
    terms = [([rng.randrange(P) for _ in range(s * n)], rng.randrange(P)) for s in (1, 4, 8)]
    t = [rng.randrange(P) for _ in range(7 * fr.num_chunks(n, m) * m - 5)]
    zeta = rng.randrange(P)
    _, want, want_e1 = fr.ft(orc, fid, log_n, m, terms, t, zeta)
    inp = Inputs()
    d_terms = [(inp(ev.mont(orc, fid, e)), len(e), ev.mont(orc, fid, [c])[0]) for e, c in terms]
    d_t = inp(ev.mont(orc, fid, t))
    ft = stale(m, 4)
    (ft_len, e1), (got,) = on_stream(stream, inp, lambda: ctx.prover_ft_dev(fid, log_n, m, d_terms, d_t, len(t), ev.mont(orc, fid, [zeta])[0],
                                                                             ft.data_ptr()), [ft])
    got = got.reshape(m, 4)
    assert ft_len == len(want)
    assert np.array_equal(got[:ft_len], ev.mont(orc, fid, want).reshape(-1, 4)[:ft_len]) and not got[ft_len:].any()
    assert np.array_equal(e1, ev.mont(orc, fid, [want_e1])[0])


def test_points_fold_dev(ctx, stream, orc, pallas_srs):
    G, h = pallas_srs, 37
    g = G.g[: 2 * h]
    u = orc.limbs_to_ints(orc.random_scalars(G.scalar, 1, seed=8))[0]
    inp = Inputs()
    d_g = inp(g)
    out = stale(h, 8)
    _, (got,) = on_stream(stream, inp, lambda: ctx.points_fold_dev(G.cid, d_g, h, orc.to_mont(G.scalar, orc.ints_to_limbs([u]))[0], out.data_ptr()),
                          [out])
    got = got.reshape(h, 8)
    for i in range(h):
        assert np.array_equal(got[i], orc.affine_add(G.cid, g[i], orc.scalar_mul(G.cid, g[h + i], u))), i


def test_bases_from_device_points(ctx, stream, orc, pallas_srs):
    """Bases(..., device_ptr=...): the points are read (and the window table built) on the caller's stream"""
    G, n = pallas_srs, 1024
    sc = orc.random_scalars(G.scalar, n, seed=9)
    inp = Inputs()
    d_pts, d_sc = inp(G.g[:n]), inp(sc)
    made = []

    def call():
        made.append(zk.Bases(ctx, G.cid, None, device_ptr=d_pts, n=n))
        return ctx.msm_dev(made[0], d_sc, n)
    try:
        r, _ = on_stream(stream, inp, call)
        assert np.array_equal(zk.jacobian_to_affine(G.cid, r), orc.msm(G.cid, G.g[:n], sc))
    finally:
        for b in made:
            b.free()


def test_one_quotient_polynomial_never_leaving_the_stream(ctx, stream, orc, vesta_srs):
    """the sequence of test_gpu_quotient_pipeline on the caller's stream: inputs copied in behind the spin, no host read in between"""
    case = QuotientCase(orc, vesta_srs)
    n = 1 << case.log_n
    inp = Inputs()
    d = {name: inp(getattr(case, name)) for name in QuotientCase.INPUTS}
    scratch = {name: stale(nb // 8) for name, nb in case.scratch_bytes().items()}
    d.update({name: t.data_ptr() for name, t in scratch.items()})
    with ctx.upload_bases(vesta_srs.cid, vesta_srs.g[:n]) as bases:
        got, (q,) = on_stream(stream, inp, lambda: case.run_on_device(ctx, d, bases), [scratch["q"]])
        assert np.array_equal(q.reshape(-1, 4), case.quot)
        for c in range(7):
            assert np.array_equal(got[c], case.want_comm[c]), c


# ---------------------------------------------------------------------------------------------------------------- host pointers and handles
def behind_spin(stream, call):
    """call() with the caller's stream held back by the spin: a result read back on any other stream would be read too early"""
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(SPIN)
        r = call()
    stream.synchronize()
    return r


def pinned(a) -> np.ndarray:
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).pin_memory().numpy().view(np.uint64)


def test_host_pointer_msm_and_msm_batch(ctx, stream, orc, vesta_srs):
    G, n, k = vesta_srs, 2048, 5
    sc = orc.random_scalars(G.scalar, k * n, seed=10).reshape(k, n, 4)
    want = [orc.msm(G.cid, G.g[:n], sc[j]) for j in range(k)]
    with ctx.upload_bases(G.cid, G.g[:n]) as bases:
        assert np.array_equal(behind_spin(stream, lambda: ctx.msm_affine(bases, sc[0])), want[0])
        assert np.array_equal(behind_spin(stream, lambda: ctx.msm_affine(bases, pinned(sc[1]))), want[1])
        out = behind_spin(stream, lambda: ctx.msm_batch(bases, sc))
        for j in range(k):
            assert np.array_equal(zk.jacobian_to_affine(G.cid, out[j]), want[j]), j


def check_pinned_ntt_batch(ctx, stream, orc):
    """20 x 2^14 in page-locked memory (10 MiB): the pipelined path, its side streams forked from the caller's stream"""
    fid, log_n, batch = zk.FQ, 14, 20
    a = mont_rnd(orc, fid, batch << log_n, 11).reshape(batch, 1 << log_n, 4)
    buf = pinned(a)
    behind_spin(stream, lambda: ctx.ntt_inplace(fid, buf))
    for b in range(batch):
        assert np.array_equal(buf[b], orc.ntt(fid, a[b])), b


def test_host_pointer_pipelined_ntt_batch(ctx, stream, orc):
    check_pinned_ntt_batch(ctx, stream, orc)


def commit_batch_case(orc, G, n=2048):
    ev15 = orc.to_mont(G.scalar, orc.random_scalars(G.scalar, 15 * n, seed=12)).reshape(15, n, 4)
    lag = G.mont_points(G.lag_2048_canon)
    return ev15, lag, [orc.msm_mont(G.cid, lag, ev15[j]) for j in range(15)]


def test_commit_evaluations_batch(ctx, stream, orc, pallas_srs):
    G, n = pallas_srs, 2048
    ev15, lag, want = commit_batch_case(orc, G, n)
    with zk.SRS(ctx, G.cid, G.g[:n], G.mont_points(G.h_xy_canon)[0]) as srs:
        srs.add_lagrange_basis(n, lag)
        got = behind_spin(stream, lambda: srs.commit_evaluations_non_hiding_batch(n, ev15))
        for j in range(15):
            assert np.array_equal(got[j].chunks[0], want[j]), j
        # the basis built on the device and read back (zk_srs_get_lagrange_basis) on the same stream
        assert np.array_equal(behind_spin(stream, lambda: srs.get_lagrange_basis_from_domain_size(n)), lag)


def opening_bytes_want():
    import json

    from test_ser_regression import GOLDEN
    return json.load(open(GOLDEN))["opening_proof_vesta_srs128"]


def test_srs_open_regression_bytes(ctx, stream, orc, vesta_srs):
    from test_ser_regression import padded
    want = opening_bytes_want()
    raw = behind_spin(stream, lambda: opening_proof_bytes_product_level(orc, zk, ctx, vesta_srs))
    assert padded(raw, len(want)) == want


def test_srs_verify(ctx, stream, orc, vesta_srs):
    G, n = vesta_srs, 1024
    g, h = G.g[:n], G.mont_points(G.h_xy_canon)[0]
    with zk.SRS(ctx, G.cid, g, h) as srs:
        entries = hash_entries(orc, G, srs, g, h, 2, 31, [n - 3])
        rb, sgb = scales(orc, G, 7)
        ok, pt = behind_spin(stream, lambda: device_verify(orc, G, srs, entries, rb, sgb))
        assert ok and not pt.any()
        bad = tamper(entries, "z1", orc.FP_MODULUS, g[3], at=1)
        ok, pt = behind_spin(stream, lambda: device_verify(orc, G, srs, bad, rb, sgb))
        assert not ok and np.array_equal(pt, oracle_verify(orc, G.cid, g, h, bad, rb, sgb))


@pytest.mark.parametrize("lanes", [4, 1])
def test_eight_threads_on_a_caller_stream(ctx, stream, orc, vesta_srs, lanes):
    """a context with a caller's stream pins every call to its primary lane, whatever the lane count"""
    G, n = vesta_srs, 1024
    scs = [orc.random_scalars(G.scalar, n, seed=200 + t) for t in range(8)]
    want = [orc.msm(G.cid, G.g[:n], s) for s in scs]
    bases = ctx.upload_bases(G.cid, G.g[:n])
    got, errs = [None] * 8, []

    def work(t):
        try:
            for _ in range(3):
                got[t] = ctx.msm_affine(bases, scs[t])
        except Exception as e:  # pragma: no cover
            errs.append(e)
    try:
        ctx.set_option("ctx_lanes", lanes)
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(SPIN)
        th = [threading.Thread(target=work, args=(t,)) for t in range(8)]
        [t.start() for t in th]
        [t.join() for t in th]
        assert not errs
        for t in range(8):
            assert np.array_equal(got[t], want[t]), t
    finally:
        ctx.set_option("ctx_lanes", 4)
        bases.free()


# ---------------------------------------------------------------------------------------------------------------- stream switches
def slow_program(orc, fid, k0, k1):
    """(k0 cell0 + k1 cell1)^(2^32 - 1), twice: about 130 field products a row, and the same tokens for every (k0, k1)"""
    def build(p):
        p.literal(k0).cell(0).mul().literal(k1).cell(1).mul().add().pow(0xFFFFFFFF).pow(0xFFFFFFFF)
        return p
    return build(gp.Recorder()), build(zk.ExprProgram())


def test_switch_while_an_expression_still_runs(ctx, stream, orc):
    """A long evaluation (2^20 rows of d8) is queued on stream A; set_stream(B) follows at once, then a program with the same tokens
    but other constants and columns on B.  B's staging copy rewrites the program, constants and column table the kernel on A reads
    from, so B must wait for A."""
    fid, rows = zk.FP, 1 << 20
    a_stream, b_stream = torch.cuda.Stream(), torch.cuda.Stream()
    ks = mont_rnd(orc, fid, 4, 40)
    cols = [mont_rnd(orc, fid, rows, 41 + j) for j in range(4)]
    progs = [slow_program(orc, fid, ks[0], ks[1]), slow_program(orc, fid, ks[2], ks[3])]
    want = [orc.expr_eval(fid, progs[i][0].ops, progs[i][0].args, progs[i][0].literals, [(cols[2 * i], 8), (cols[2 * i + 1], 8)], rows)
            for i in range(2)]
    d_cols = [dev(c) for c in cols]
    outs = [stale(rows, 4), stale(rows, 4)]
    torch.cuda.synchronize()
    try:
        for i, s in enumerate((a_stream, b_stream)):
            ctx.set_stream(s.cuda_stream)
            progs[i][1].evaluations(ctx, fid, [(d_cols[2 * i].data_ptr(), rows, 8), (d_cols[2 * i + 1].data_ptr(), rows, 8)], rows, 8, outs[i].data_ptr())
        torch.cuda.synchronize()
    finally:
        ctx.set_stream(stream.cuda_stream)
    for i in range(2):
        assert np.array_equal(host(outs[i]).reshape(-1, 4), want[i]), "AB"[i]


def test_switch_while_a_transform_still_runs(ctx, stream, orc):
    """two 2^20 transforms of the same shape on different buffers, the first on A, the second on B right after set_stream(B): both
    use the context's second buffer"""
    fid, log_n, batch = zk.FQ, 20, 2
    a_stream, b_stream = torch.cuda.Stream(), torch.cuda.Stream()
    data = [mont_rnd(orc, fid, batch << log_n, 50 + i).reshape(batch, 1 << log_n, 4) for i in range(2)]
    bufs = [dev(d) for d in data]
    torch.cuda.synchronize()
    try:
        for i, s in enumerate((a_stream, b_stream)):
            ctx.set_stream(s.cuda_stream)
            ctx.ntt_dev(fid, bufs[i].data_ptr(), log_n, batch=batch)
        torch.cuda.synchronize()
    finally:
        ctx.set_stream(stream.cuda_stream)
    for i in range(2):
        got = host(bufs[i]).reshape(batch, -1, 4)
        for b in range(batch):
            assert np.array_equal(got[b], orc.ntt(fid, data[i][b])), (i, b)


def test_switch_back_to_the_own_stream_with_work_pending(ctx, stream, orc):
    """a forward transform queued on the caller's stream behind the spin, then set_stream(None) and the inverse on the library's
    own stream: the inverse must see the forward's output, so the round trip gives the input back"""
    fid, log_n = zk.FP, 12
    a = mont_rnd(orc, fid, 1 << log_n, 60)
    inp = Inputs()
    d = inp(a)
    torch.cuda.synchronize()
    try:
        with torch.cuda.stream(stream):
            torch.cuda._sleep(SPIN)
            for dst, src in inp.pairs:
                dst.copy_(src)
            ctx.ntt_dev(fid, d, log_n)
        ctx.set_stream(None)
        ctx.ntt_dev(fid, d, log_n, inverse=True)
        got = ctx.dev_download(d, (1 << log_n, 4))               # on the own stream, after the inverse
    finally:
        torch.cuda.synchronize()
        ctx.set_stream(stream.cuda_stream)
    assert np.array_equal(got, a)


# ---------------------------------------------------------------------------------------------------------------- torch's default stream
@pytest.fixture
def on_default_stream(ctx, stream):
    """the context on torch's default stream, whose cuda_stream is 0: the library must run on it, not on its own stream"""
    default = torch.cuda.default_stream()
    assert default.cuda_stream == 0
    ctx.set_stream(default.cuda_stream)
    try:
        yield default
    finally:
        torch.cuda.synchronize()
        ctx.set_stream(stream.cuda_stream)


def test_default_stream_ntt_dev(ctx, orc, on_default_stream):
    fid, log_n = zk.FQ, 12
    a = mont_rnd(orc, fid, 1 << log_n, 70)
    ctx.ntt_dev(fid, dev(a).data_ptr(), log_n)          # warm-up: building the tables and loading the kernels can synchronise the device
    inp = Inputs()
    d = inp(a)
    _, (got,) = on_stream(on_default_stream, inp, lambda: ctx.ntt_dev(fid, d, log_n), [inp.pairs[0][0]])
    assert np.array_equal(got.reshape(-1, 4), orc.ntt(fid, a))


def test_default_stream_msm_dev(ctx, orc, pallas_srs, on_default_stream):
    G, n = pallas_srs, 2048
    sc = orc.random_scalars(G.scalar, n, seed=71)
    with ctx.upload_bases(G.cid, G.g[:n]) as bases:
        warm = dev(sc)
        ctx.msm_dev(bases, warm.data_ptr(), n)           # warm-up, as above
        inp = Inputs()
        d = inp(sc)
        r, _ = on_stream(on_default_stream, inp, lambda: ctx.msm_dev(bases, d, n))
        assert np.array_equal(zk.jacobian_to_affine(G.cid, r), orc.msm(G.cid, G.g[:n], sc))


# ---------------------------------------------------------------------------------------------------------------- profiled runs
@pytest.fixture
def profiled(ctx):
    ctx.set_profile(True)
    try:
        yield ctx
    finally:
        ctx.set_profile(False)


def test_profiled_msm_batch_and_stage_times(ctx, stream, orc, vesta_srs):
    """one MSM per pipeline in profiling mode: msm_batch of five equals the oracle and the unprofiled call; msm_dev reports six
    finite, non-negative stage times"""
    G, n, k = vesta_srs, 2048, 5
    sc = orc.random_scalars(G.scalar, k * n, seed=80).reshape(k, n, 4)
    with ctx.upload_bases(G.cid, G.g[:n]) as bases:
        plain = [zk.jacobian_to_affine(G.cid, r) for r in ctx.msm_batch(bases, sc)]
        ctx.set_profile(True)
        try:
            prof = [zk.jacobian_to_affine(G.cid, r) for r in behind_spin(stream, lambda: ctx.msm_batch(bases, sc))]
            d = dev(sc[2])
            torch.cuda.synchronize()
            one = zk.jacobian_to_affine(G.cid, ctx.msm_dev(bases, d.data_ptr(), n))
            st = ctx.last_stage_ms()
        finally:
            ctx.set_profile(False)
        for j in range(k):
            assert np.array_equal(prof[j], orc.msm(G.cid, G.g[:n], sc[j])), j
            assert np.array_equal(prof[j], plain[j]), j
        assert np.array_equal(one, plain[2])
        times = [st[s] for s in ("recode", "plan", "scatter", "accumulate", "finish", "bitsum")]
        assert all(np.isfinite(t) and t >= 0 for t in times), st
        assert sum(times) > 0, st


def test_profiled_ntt(ctx, stream, orc, profiled):
    """the pinned batch without its pipeline, then a device transform that reports a positive time"""
    check_pinned_ntt_batch(ctx, stream, orc)
    fid, log_n = zk.FP, 14
    a = mont_rnd(orc, fid, 1 << log_n, 81)
    d = dev(a)
    torch.cuda.synchronize()
    ctx.ntt_dev(fid, d.data_ptr(), log_n)
    assert ctx.last_stage_ms()["ntt"] > 0
    stream.synchronize()
    assert np.array_equal(host(d).reshape(-1, 4), orc.ntt(fid, a))


def test_profiled_commit_evaluations_batch(ctx, stream, orc, pallas_srs, profiled):
    G, n = pallas_srs, 2048
    ev15, lag, want = commit_batch_case(orc, G, n)
    with zk.SRS(ctx, G.cid, G.g[:n], G.mont_points(G.h_xy_canon)[0]) as srs:
        srs.add_lagrange_basis(n, lag)
        got = behind_spin(stream, lambda: srs.commit_evaluations_non_hiding_batch(n, ev15))
        for j in range(15):
            assert np.array_equal(got[j].chunks[0], want[j]), j


def test_profiled_srs_open_regression_bytes(ctx, stream, orc, vesta_srs, profiled):
    from test_ser_regression import padded
    want = opening_bytes_want()
    raw = behind_spin(stream, lambda: opening_proof_bytes_product_level(orc, zk, ctx, vesta_srs))
    assert padded(raw, len(want)) == want
