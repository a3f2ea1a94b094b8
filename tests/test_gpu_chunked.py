"""The device stages of a chunked Vesta proof (scalar field Fp): domains of 2^17 to 2^20 rows over the fixture's 2^16 generators, so
max_poly_size = 2^16 and every polynomial is cut into num_chunks = n / 2^16 pieces (kimchi/src/prover.rs:208-212).  t is committed
in 7 num_chunks chunks (prover.rs:923), ft is linearised over them (prover.rs:1184), zk_rows = (16 num_chunks + 5) / 7
(circuits/constraints.rs:965), and the Lagrange bases of commitments (poly-commitment/src/ipa.rs:1145-1171) and of evaluations
(lagrange_basis_evaluations.rs:203-240) are chunked.  kimchi's own test of this is a 2^17-row circuit over a 2^16-point SRS
(kimchi/src/tests/chunked.rs:107-110).

These shapes run kernel paths the per-stage files never reach: more than one (point, chunk) pair group in k_lagrange_evaluate, more
than one point group in k_evaluate_chunks, launch_sum's loop over several k_sum_partials launches, one MSM per basis chunk at an
offset into a windowed table, several fused batches of t's chunk MSMs, and k_linearize_add over 16 chunks in zk_srs_open.  Every
result is compared bit for bit with the CPU oracle or the Python restatements (tests/evals_replay.py, ft_replay.py, perm_replay.py,
verify_replay.py); where a restatement would hold a whole 2^20 x 16 basis in Python integers, the test uses the exact identity
sum_i p[s i] l_{x,k}[i] = chunk k of interpolate(p[::s]) at x.  Each test runs on a context of its own and stays below about
3 GiB of device memory and 6 GiB of host memory."""
import contextlib
import random

import numpy as np
import pytest

import evals_replay as ev
import ft_replay as fr
import perm_replay as pr
import proof_systems_b200 as zk
from test_gpu_ft import check_against_replay, stale
from test_gpu_large_domains import canonical_ints, device_z, draw_scalars
from verify_replay import Entry, HashTranscript, Opening, oracle_verify, to_device

pytestmark = pytest.mark.gpu

M = 1 << 16                     # max_poly_size: the fixture's generators


@pytest.fixture
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.fixture
def srs(ctx, vesta_srs):
    """the 2^16-point Vesta SRS with the default table window (15 bits: 18 x 2^16 table points)"""
    s = zk.SRS(ctx, vesta_srs.cid, vesta_srs.g, vesta_srs.mont_points(vesta_srs.h_xy_canon)[0])
    yield s
    s.close()


def rnd(orc, fid, k, seed):
    return orc.to_mont(fid, orc.random_scalars(fid, k, seed=seed))


def m1(orc, fid, x):
    return ev.mont(orc, fid, [x])[0]


def chunk_evals(orc, fid, p_mont, xs, m=M):
    """[point][chunk] of interpolate(p) split into chunks of m coefficients, each evaluated at x (Horner on Python integers)"""
    P = orc.MODULUS[fid]
    q = ev.ints(orc, fid, orc.ntt(fid, np.ascontiguousarray(p_mont), inverse=True))
    return [[ev.horner(q[k:k + m], x, P) for k in range(0, len(q), m)] for x in xs]


# ---------------------------------------------------------------------------------------------------------------- Lagrange basis of commitments
def test_chunked_lagrange_basis_2_17_over_2_16(ctx, orc, vesta_srs, srs):
    """kimchi's heavy-test shape: SRS::lagrange_basis of D(2^17) over 2^16 generators (group_ntt.cu with chunk > 0, two chunks), then
    commit_evaluations_non_hiding on it (srs.cu: one MSM per chunk at offset c * 2^17 into the basis's windowed table).
    - sampled basis entries of both chunks vs their defining MSM sum_j (w^{-i (c |g| + j)} / n) g[j] on the oracle;
    - ipa_commitment.rs:27-119: commit_evaluations(evals) == commit_non_hiding(iFFT(evals)) chunk by chunk for random evaluations (a
      random combination of every basis entry, so one wrong entry shows), the coefficient chunks vs oracle MSMs, and each evaluation
      chunk vs an oracle MSM over the downloaded basis;
    - the same evaluations handed over on d8 (sub-sampled by 8);
    - commit_evaluations_batch refuses the chunked basis, and 15 single-column calls give each column's interpolated commitment."""
    G = vesta_srs
    fid, n = G.scalar, 1 << 17
    P = orc.MODULUS[fid]
    assert srs.lagrange_basis_chunks(n) == 2
    basis = srs.get_lagrange_basis_from_domain_size(n)
    assert basis.shape == (2, n, 8)
    w = orc.fe_int(fid, orc.root_of_unity(fid, 17))
    winv, ninv = pow(w, -1, P), pow(n, -1, P)
    rng = random.Random(17)
    for i in [0, 1, n // 2, n - 1] + [rng.randrange(n) for _ in range(3)]:
        for c in range(2):
            step, cur, sc = pow(winv, i, P), pow(winv, i * c * M, P) * ninv % P, []
            for _ in range(M):
                sc.append(cur)
                cur = cur * step % P
            assert np.array_equal(basis[c, i], orc.msm(G.cid, G.g, orc.ints_to_limbs(sc))), (c, i)
    evals = rnd(orc, fid, n, 20)
    coeffs = orc.ntt(fid, evals, inverse=True)
    com = srs.commit_evaluations_non_hiding(n, evals)
    via_coeffs = srs.commit_non_hiding(coeffs, 1)
    assert len(com) == len(via_coeffs) == 2
    assert np.array_equal(com.chunks, via_coeffs.chunks)
    for c in range(2):
        assert np.array_equal(via_coeffs.chunks[c], orc.msm_mont(G.cid, G.g, coeffs[c * M:(c + 1) * M])), c
        assert np.array_equal(com.chunks[c], orc.msm_mont(G.cid, basis[c], evals)), c
    del basis
    pad = np.zeros((8 * n, 4), dtype=np.uint64)
    pad[:n] = coeffs
    evals8 = orc.ntt(fid, pad)
    del pad
    assert np.array_equal(srs.commit_evaluations_non_hiding(n, evals8).chunks, com.chunks)
    del evals8
    cols = rnd(orc, fid, 15 * n, 21).reshape(15, n, 4)
    cols[4] = orc.fe(fid, 1)                                     # constant 1: chunk 0 is g[0], chunk 1 the identity
    with pytest.raises(zk.ZkError, match="chunked bases"):
        srs.commit_evaluations_non_hiding_batch(n, cols)
    for j in range(15):
        got = srs.commit_evaluations_non_hiding(n, cols[j]).chunks
        assert np.array_equal(got, srs.commit_non_hiding(orc.ntt(fid, cols[j], inverse=True), 1).chunks), j
        if j == 4:
            assert np.array_equal(got[0], G.g[0]) and not got[1].any()


# ---------------------------------------------------------------------------------------------------------------- t in 7 num_chunks chunks
@pytest.mark.parametrize("nc", [2, 4, 16])
def test_t_commitment_in_7_num_chunks(ctx, orc, vesta_srs, srs, nc):
    """commit_non_hiding of t (prover.rs:923) with 14, 28 and 112 chunks of 2^16: ctx_msm_many_offs fuses up to `msm_batch` chunk
    MSMs per pipeline (api.cu), run here with 16 and with 5 so the last batch is ragged; a t of 7 nc m - m/2 - 3 coefficients also
    sends its short last chunk through zk_msm (srs.cu).  At 14 and 28 chunks every chunk vs the oracle; at 112 the first and last
    chunk of every fused batch of both settings and the ragged tail, the two settings equal everywhere.  At 112, mask_custom with
    112 blinders vs the oracle."""
    G = vesta_srs
    fid, k = G.scalar, 7 * nc
    t = rnd(orc, fid, k * M, 30 + nc)
    short = k * M - M // 2 - 3
    got = {}
    try:
        for batch in (16, 5):
            ctx.set_option("msm_batch", batch)
            got[batch] = (srs.commit_non_hiding(t, k).chunks, srs.commit_non_hiding(t[:short], k).chunks)
    finally:
        ctx.set_option("msm_batch", 16)
    full, ragged = got[16]
    assert full.shape == ragged.shape == (k, 8)
    assert np.array_equal(got[5][0], full) and np.array_equal(got[5][1], ragged)
    assert np.array_equal(ragged[:k - 1], full[:k - 1])
    assert np.array_equal(ragged[k - 1], orc.msm_mont(G.cid, G.g[:M // 2 - 3], t[(k - 1) * M:short]))
    if nc <= 4:
        check = range(k)
    else:
        check = sorted({j for b in (16, 5) for j in range(k) if j % b in (0, b - 1)} | {k - 1})
    for j in check:
        assert np.array_equal(full[j], orc.msm_mont(G.cid, G.g, t[j * M:(j + 1) * M])), j
    if nc == 16:
        bl = orc.random_scalars(fid, k, seed=39)
        masked = srs.mask_custom(zk.PolyComm(full), orc.to_mont(fid, bl))
        h = srs.h
        for j in range(k):
            assert np.array_equal(masked.chunks[j], orc.affine_add(G.cid, full[j], orc.scalar_mul(G.cid, h, orc.limbs_to_int(bl[j])))), j


# ---------------------------------------------------------------------------------------------------------------- Lagrange basis of evaluations
@pytest.mark.parametrize("log_n", [17, 19, 20])
def test_lagrange_evaluate_chunked_at_zeta_and_zeta_omega(ctx, orc, log_n):
    """LagrangeBasisEvaluations::new_with_chunked_segments at zeta and zeta omega with max_poly_size 2^16 (2, 8, 16 chunks: 4, 16, 32
    (point, chunk) pairs, so k_lagrange_evaluate runs 1, 2 and 4 pair groups along blockIdx.z), evaluate of columns at strides 1, 4
    and 8 and evaluate_boolean of a selector, in one zk_lagrange_evaluate_dev call.  At 2^17 the basis values and the evaluations
    vs evals_replay; at 2^19 and 2^20 the evaluations vs the identity sum_i p[s i] l_{x,k}[i] = chunk k of interpolate(p[::s]) at x
    (oracle iNTT, Python Horner), p the 0/1 indicator for the selector."""
    fid = zk.FP
    P, n = orc.MODULUS[fid], 1 << log_n
    nc = n // M
    rng = random.Random(300 + log_n)
    zeta = rng.randrange(P)
    pts = [zeta, zeta * ev.omega(orc, fid, log_n) % P]
    cols = {s: rnd(orc, fid, s * n, 310 + s + log_n) for s in (1, 4, 8)}
    bits = np.random.default_rng(log_n).integers(0, 2, size=(4 * n, 1)) == 1
    sel = np.where(bits, rnd(orc, fid, 4 * n, 320 + log_n), np.uint64(0)).astype(np.uint64)   # nonzero values count as one
    ind = np.where(bits[::4], orc.fe(fid, 1), np.uint64(0)).astype(np.uint64)
    with ctx.buffers() as bufs, contextlib.ExitStack() as stack:
        d = {s: bufs.put(c) for s, c in cols.items()}
        d_sel = bufs.put(sel)
        lbs = [stack.enter_context(zk.LagrangeBasisEvaluations(ctx, fid, M, log_n, m1(orc, fid, x))) for x in pts]
        assert lbs[0].chunks == nc
        got = zk.LagrangeBasisEvaluations.evaluate_all(lbs, [(d[s], s * n, False) for s in (1, 4, 8)] + [(d_sel, 4 * n, True)])
        basis17 = [lb.evals() for lb in lbs] if log_n == 17 else None
    assert got.shape == (4, 2, nc, 4)
    host = [cols[s][::s] for s in (1, 4, 8)] + [ind]
    if log_n == 17:
        for t, x in enumerate(pts):
            basis = ev.lagrange_basis(orc, fid, M, log_n, x)
            assert np.array_equal(basis17[t], np.stack([ev.mont(orc, fid, v) for v in basis])), t
            for j, h in enumerate(host):
                assert np.array_equal(got[j, t], ev.mont(orc, fid, ev.evaluate(basis, ev.ints(orc, fid, h), P))), (j, t)
    else:
        for j, h in enumerate(host):
            want = chunk_evals(orc, fid, h, pts)
            for t in range(2):
                assert np.array_equal(got[j, t], ev.mont(orc, fid, want[t])), (j, t)


@pytest.mark.parametrize("fid", [0, 1])
def test_lagrange_evaluate_partial_second_pair_group(ctx, orc, fid):
    """3 points x 4 chunks = 12 pairs: k_lagrange_evaluate's second group holds 4 of its 8 pairs; strides 1 and 8 and a boolean
    column vs evals_replay, on both fields"""
    P, log_n = orc.MODULUS[fid], 10
    n, m = 1 << log_n, 1 << 8
    rng = random.Random(40 + fid)
    pts = [rng.randrange(P) for _ in range(3)]
    c1, c8 = [rng.randrange(P) for _ in range(n)], [rng.randrange(P) for _ in range(8 * n)]
    bits = [rng.randrange(2) * rng.randrange(1, P) for _ in range(n)]
    with ctx.buffers() as bufs, contextlib.ExitStack() as stack:
        cols = [(bufs.put(ev.mont(orc, fid, c1)), n, False), (bufs.put(ev.mont(orc, fid, c8)), 8 * n, False),
                (bufs.put(ev.mont(orc, fid, bits)), n, True)]
        lbs = [stack.enter_context(zk.LagrangeBasisEvaluations(ctx, fid, m, log_n, m1(orc, fid, x))) for x in pts]
        got = zk.LagrangeBasisEvaluations.evaluate_all(lbs, cols)
    assert got.shape == (3, 3, 4, 4)
    for t, x in enumerate(pts):
        basis = ev.lagrange_basis(orc, fid, m, log_n, x)
        assert np.array_equal(got[0, t], ev.mont(orc, fid, ev.evaluate(basis, c1, P))), t
        assert np.array_equal(got[1, t], ev.mont(orc, fid, ev.evaluate(basis, c8, P))), t
        assert np.array_equal(got[2, t], ev.mont(orc, fid, ev.evaluate_boolean(basis, bits, P))), t


# ---------------------------------------------------------------------------------------------------------------- evaluate_chunks
@pytest.mark.parametrize("nc", [2, 4, 16])
def test_evaluate_chunks_several_point_groups(ctx, orc, nc):
    """to_chunked_polynomial(nc, 2^16).evaluate_chunks at 9 points (k_evaluate_chunks over 3 point groups along blockIdx.z, the
    last one partial) of a full polynomial, a ragged one and a short one, vs evals_replay; the same call at 5 points (2 groups)
    returns the first five points' values"""
    fid = zk.FP
    P = orc.MODULUS[fid]
    rng = random.Random(50 + nc)
    lens = [nc * M, (nc - 1) * M + 777, 1000]
    polys = [canonical_ints(orc.random_scalars(fid, k, seed=51 + k)) for k in lens]
    pts = [0, 1] + [rng.randrange(P) for _ in range(7)]
    with ctx.buffers() as bufs:
        desc = [(bufs.put(ev.mont(orc, fid, p)), len(p)) for p in polys]
        got9 = ctx.poly_evaluate_chunks_dev(fid, desc, nc, M, ev.mont(orc, fid, pts))
        got5 = ctx.poly_evaluate_chunks_dev(fid, desc, nc, M, ev.mont(orc, fid, pts[:5]))
    assert got9.shape == (3, 9, nc, 4) and got5.shape == (3, 5, nc, 4)
    assert np.array_equal(got5, got9[:, :5])
    for j, p in enumerate(polys):
        for t, x in enumerate(pts):
            assert np.array_equal(got9[j, t], ev.mont(orc, fid, ev.evaluate_chunks(p, nc, M, x, P))), (lens[j], t)


# ---------------------------------------------------------------------------------------------------------------- > 65535 reduction outputs
def test_lagrange_evaluate_more_than_65535_outputs(ctx, orc):
    """4097 column descriptors x 16 pairs (2 points x 8 chunks) = 65552 outputs: launch_sum runs k_sum_partials twice, the second
    launch over outputs 65535.. .  The descriptors alternate between two device columns (a plain one at stride 1, a boolean one at
    stride 2); every output vs the two columns' evals_replay values."""
    fid, log_n = zk.FQ, 10
    P, n, m = orc.MODULUS[fid], 1 << log_n, 1 << 7
    rng = random.Random(60)
    pts = [rng.randrange(P) for _ in range(2)]
    a = [rng.randrange(P) for _ in range(n)]
    b = [rng.randrange(2) * rng.randrange(1, P) for _ in range(2 * n)]
    n_cols = 4097
    with ctx.buffers() as bufs, contextlib.ExitStack() as stack:
        d_a, d_b = bufs.put(ev.mont(orc, fid, a)), bufs.put(ev.mont(orc, fid, b))
        lbs = [stack.enter_context(zk.LagrangeBasisEvaluations(ctx, fid, m, log_n, m1(orc, fid, x))) for x in pts]
        got = zk.LagrangeBasisEvaluations.evaluate_all(lbs, [(d_a, n, False) if j % 2 == 0 else (d_b, 2 * n, True) for j in range(n_cols)])
    assert got.shape == (n_cols, 2, 8, 4) and got.shape[0] * 16 > 65535
    bases = [ev.lagrange_basis(orc, fid, m, log_n, x) for x in pts]
    want_a = np.stack([ev.mont(orc, fid, ev.evaluate(bs, a, P)) for bs in bases])
    want_b = np.stack([ev.mont(orc, fid, ev.evaluate_boolean(bs, b, P)) for bs in bases])
    assert np.array_equal(got[0::2], np.broadcast_to(want_a, got[0::2].shape))
    assert np.array_equal(got[1::2], np.broadcast_to(want_b, got[1::2].shape))


def test_evaluate_chunks_more_than_65535_outputs(ctx, orc):
    """821 polynomial descriptors x 5 points x 16 chunks = 65680 outputs (launch_sum's second k_sum_partials launch), alternating
    between a polynomial of 16 full chunks of 64 and one of 1000 coefficients; every output vs evals_replay"""
    fid = zk.FP
    P, nc, cs = orc.MODULUS[fid], 16, 64
    rng = random.Random(61)
    pts = [rng.randrange(P) for _ in range(5)]
    a = [rng.randrange(P) for _ in range(nc * cs)]
    b = [rng.randrange(P) for _ in range(1000)]
    n_polys = 821
    with ctx.buffers() as bufs:
        d_a, d_b = bufs.put(ev.mont(orc, fid, a)), bufs.put(ev.mont(orc, fid, b))
        got = ctx.poly_evaluate_chunks_dev(fid, [(d_a, len(a)) if j % 2 == 0 else (d_b, len(b)) for j in range(n_polys)], nc, cs,
                                           ev.mont(orc, fid, pts))
    assert got.shape == (n_polys, 5, nc, 4) and n_polys * 5 * nc > 65535
    want_a = np.stack([ev.mont(orc, fid, ev.evaluate_chunks(a, nc, cs, x, P)) for x in pts])
    want_b = np.stack([ev.mont(orc, fid, ev.evaluate_chunks(b, nc, cs, x, P)) for x in pts])
    assert np.array_equal(got[0::2], np.broadcast_to(want_a, got[0::2].shape))
    assert np.array_equal(got[1::2], np.broadcast_to(want_b, got[1::2].shape))


# ---------------------------------------------------------------------------------------------------------------- ft
@pytest.mark.parametrize("log_n", [17, 18, 20])
def test_ft_chunked(ctx, orc, log_n):
    """zk_prover_ft_dev with m = 2^16 over D(2^17), D(2^18) and D(2^20): f from sigma_6 over d8 (read at stride 8) in 2, 4 and 16
    chunks linearised at zeta^m, t of 7 nc m coefficients (14, 28, 112 chunks) and a ragged t of 7 nc m - m/2 - 3.  The m
    coefficients, ft_len and ft(zeta omega) vs ft_replay, and Maller's identity ft(zeta) = f(zeta) - (zeta^n - 1) t(zeta) on the
    device's output.  The replay at 2^20 holds 7.3 M Python integers for t and stays within the host budget."""
    fid = zk.FP
    P, n = orc.MODULUS[fid], 1 << log_n
    nc = n // M
    rng = random.Random(70 + log_n)
    perm, zeta = rng.randrange(P), rng.randrange(P)
    s6_8 = rnd(orc, fid, 8 * n, 71 + log_n)
    terms = [(ev.ints(orc, fid, s6_8[::8]), perm)]                 # the entries the device reads: combine_terms at stride 1
    t_full = orc.random_scalars(fid, 7 * nc * M, seed=72 + log_n)
    with ctx.buffers() as bufs:
        d_s8 = bufs.put(s6_8)
        del s6_8
        d_t = bufs.put(orc.to_mont(fid, t_full))
        d_ft = bufs.put(stale(M))
        for t_len in (7 * nc * M, 7 * nc * M - M // 2 - 3):
            ctx.dev_upload(d_ft, stale(M))
            ft_len, e1 = ctx.prover_ft_dev(fid, log_n, M, [(d_s8, 8 * n, m1(orc, fid, perm))], d_t, t_len, m1(orc, fid, zeta), d_ft)
            coeffs = ctx.dev_download(d_ft, (M, 4))
            check_against_replay(orc, fid, log_n, M, terms, canonical_ints(t_full[:t_len]), zeta, (coeffs, ft_len, e1))


# ---------------------------------------------------------------------------------------------------------------- opening and verification
def open_and_check(orc, G, srs, plnms, host, elm, ps, es, draws, seed):
    """zk_srs_open of plnms, then the oracle identities of the proof (as tools/replay_kimchi.py checks them): the combined inner product
    handed to u_base is <a, b> of the combined polynomial a (every chunk at the next power of polyscale) and b; round 0's L and R are
    the reference's two (n/2 + 2)-point MSMs (ipa.rs:938-960); sg = <b_poly_coefficients(chals), g>; z1 = a0 c + d and
    z2 = r_prime c + r_delta; delta = d (sg + b0 U) + r_delta h.  host: per entry (coefficients as ints, blinders as ints).
    Returns the proof as a verify_replay.Entry."""
    fid = G.scalar
    P, N = orc.MODULUS[fid], G.g.shape[0]
    h = srs.h
    u_points = G.g[200:232]
    seen = {"u": []}

    def transcript():
        return HashTranscript(P, u_points, seed)
    tr = transcript()

    def u_base(cip):
        seen["cip"] = orc.fe_int(fid, cip)
        seen["U"] = tr.u_base(seen["cip"])
        return seen["U"]

    def round_challenge(j, l, r):
        u = tr.round(j, l, r)
        seen["u"].append(u)
        return m1(orc, fid, u)

    def final_challenge(d):
        seen["c"] = tr.final(d)
        return m1(orc, fid, seen["c"])

    proof = zk.srs_open(srs, plnms, ev.mont(orc, fid, elm), m1(orc, fid, ps), m1(orc, fid, es), ev.mont(orc, fid, draws), u_base,
                        round_challenge, final_challenge)
    a, blinding, scale = np.zeros(N, dtype=object), 0, 1
    for coeffs, bls in host:
        for k, bl in enumerate(bls):
            chunk = coeffs[k * N:(k + 1) * N]
            a[:len(chunk)] = (a[:len(chunk)] + scale * np.array(chunk, dtype=object)) % P
            blinding = (blinding + scale * bl) % P
            scale = scale * ps % P
    b, sc = np.zeros(N, dtype=object), 1
    for x in elm:
        pw, cur = np.empty(N, dtype=object), 1
        for i in range(N):
            pw[i] = cur
            cur = cur * x % P
        b = (b + sc * pw) % P
        sc = sc * es % P
    cip = int(np.dot(a, b) % P)
    assert seen["cip"] == cip
    U, hh = seen["U"], N // 2
    ip_l, ip_r = int(np.dot(a[hh:], b[:hh]) % P), int(np.dot(a[:hh], b[hh:]) % P)
    l0 = orc.msm(G.cid, np.concatenate([G.g[:hh], h[None], U[None]]), orc.ints_to_limbs([int(x) for x in a[hh:]] + [draws[0], ip_l]))
    r0 = orc.msm(G.cid, np.concatenate([G.g[hh:], h[None], U[None]]), orc.ints_to_limbs([int(x) for x in a[:hh]] + [draws[1], ip_r]))
    assert np.array_equal(proof.lr[0, 0], l0) and np.array_equal(proof.lr[0, 1], r0)
    us = seen["u"]
    assert len(us) == proof.lr.shape[0] == 16
    for u in us:
        ui, half = pow(u, -1, P), len(a) // 2
        a = (a[:half] + ui * a[half:]) % P
        b = (b[:half] + u * b[half:]) % P
    s = [1]
    for u in us:
        s = [v for t in s for v in (t, t * u % P)]
    sg = orc.msm(G.cid, G.g, orc.ints_to_limbs(s))
    assert np.array_equal(proof.sg, sg)
    r_prime = blinding
    for j, u in enumerate(us):
        r_prime = (r_prime + draws[2 * j] * pow(u, -1, P) + draws[2 * j + 1] * u) % P
    a0, b0, c, d, r_delta = int(a[0]), int(b[0]), seen["c"], draws[-2], draws[-1]
    z1, z2 = orc.fe_int(fid, proof.z1), orc.fe_int(fid, proof.z2)
    assert z1 == (a0 * c + d) % P and z2 == (r_prime * c + r_delta) % P
    assert np.array_equal(proof.delta, orc.msm(G.cid, np.stack([sg, U, h]), orc.ints_to_limbs([d, d * b0 % P, r_delta])))
    opening = Opening([(l.copy(), r.copy()) for l, r in proof.lr], proof.delta, z1, z2, proof.sg)
    return Entry(opening, elm, ps, es, None, cip, transcript)


def test_open_and_verify_chunked(ctx, orc, vesta_srs, srs):
    """zk_srs_open on the 2^16 SRS of two coefficient polynomials handed over as device pointers, 2^17 and 2^20 coefficients (2 and 16
    chunks and blinders), and one evaluation-form entry on d8 of D(2^20): combine_polys interpolates it and k_linearize_add folds its
    16 chunks.  Two proofs (their own points, scales, draws and transcripts), each checked by the oracle identities of
    open_and_check; then zk_srs_verify accepts the batch with the 2-, 16- and 16-chunk commitments (the evaluation entry's is the
    commitment of its interpolation, which test_chunked_lagrange_basis_2_17_over_2_16 ties to commit_evaluations), and a batch with
    the last chunk of one 16-chunk commitment replaced fails with oracle_verify's sum."""
    G = vesta_srs
    fid, big = G.scalar, 1 << 20
    P = orc.MODULUS[fid]
    rng = random.Random(80)
    p1, p2 = orc.random_scalars(fid, 1 << 17, seed=81), orc.random_scalars(fid, big, seed=82)
    ev8 = rnd(orc, fid, 8 * big, 83)
    q3 = orc.ntt(fid, np.ascontiguousarray(ev8[::8]), inverse=True)            # the evaluation entry's coefficients (Montgomery)
    bl = [[rng.randrange(P) for _ in range(k)] for k in (2, 16, 16)]
    host = [(canonical_ints(p1), bl[0]), (canonical_ints(p2), bl[1]), (ev.ints(orc, fid, q3), bl[2])]
    comms = [srs.commit_custom(orc.to_mont(fid, p1), 2, ev.mont(orc, fid, bl[0])).chunks,
             srs.commit_custom(orc.to_mont(fid, p2), 16, ev.mont(orc, fid, bl[1])).chunks,
             srs.commit_custom(q3, 16, ev.mont(orc, fid, bl[2])).chunks]
    assert [c.shape[0] for c in comms] == [2, 16, 16]
    del q3
    with ctx.buffers() as bufs:
        entries = []
        d1, d2, d3 = bufs.put(orc.to_mont(fid, p1)), bufs.put(orc.to_mont(fid, p2)), bufs.put(ev8)
        del ev8
        plnms = [((d1, 1 << 17), 0, ev.mont(orc, fid, bl[0])), ((d2, big), 0, ev.mont(orc, fid, bl[1])),
                 ((d3, 8 * big), big, ev.mont(orc, fid, bl[2]))]
        for k in range(2):
            sc = [rng.randrange(P) for _ in range(4 + 2 * 16 + 2)]
            e = open_and_check(orc, G, srs, plnms, host, sc[:2], sc[2], sc[3], sc[4:], 800 + k)
            e.comms = comms
            entries.append(e)
    rb, sgb = rng.randrange(P), rng.randrange(P)
    batch = lambda es: [to_device(zk, orc, fid, e) for e in es]
    ok, pt = zk.srs_verify(srs, batch(entries), m1(orc, fid, rb), m1(orc, fid, sgb), return_sum=True)
    assert ok and not pt.any()
    bad = list(entries)
    e = bad[1]
    bad_comms = [c.copy() for c in comms]
    bad_comms[1][15] = G.g[5]
    bad[1] = Entry(e.opening, e.elm, e.polyscale, e.evalscale, bad_comms, e.cip, e.transcript)
    ok, pt = zk.srs_verify(srs, batch(bad), m1(orc, fid, rb), m1(orc, fid, sgb), return_sum=True)
    assert not ok
    assert np.array_equal(pt, oracle_verify(orc, G.cid, G.g, srs.h, bad, rb, sgb))


# ---------------------------------------------------------------------------------------------------------------- permutation
def test_perm_aggreg_identity_wiring_at_chunked_zk_rows(ctx, orc):
    """kimchi's zk_rows for 16 chunks, (16 * 16 + 5) / 7 = 37, at 2^20: sigma_k = shift_k omega^j wires every cell to itself, so z = 1
    up to row n - 37, then rand0, then rand1 to the end, and the final-value flag is set"""
    fid, log_n, zk_rows = zk.FP, 20, (16 * 16 + 5) // 7
    P, n = orc.MODULUS[fid], 1 << log_n
    assert zk_rows == 37
    last = n - zk_rows
    beta, gamma, shifts, rand = draw_scalars(P, 90)
    sigma = np.empty((7, n, 4), dtype=np.uint64)
    x = np.zeros((n, 4), dtype=np.uint64)
    for k in range(7):
        x[1] = m1(orc, fid, shifts[k])
        sigma[k] = orc.ntt(fid, x)
    del x
    z = np.empty((n, 4), dtype=np.uint64)
    z[:last + 1] = m1(orc, fid, 1)
    z[last + 1], z[last + 2:] = ev.mont(orc, fid, rand)
    want = orc.ntt(fid, z, inverse=True)
    del z
    got, ok = device_z(ctx, orc, fid, log_n, zk_rows, rnd(orc, fid, 7 * n, 91).reshape(7, n, 4), sigma, beta, gamma, shifts, rand)
    assert ok is True
    assert np.array_equal(got, want)


def test_perm_aggreg_random_instance_at_chunked_zk_rows(ctx, orc):
    """zk_rows = 37 at 2^20, random unwired witness and sigma (sigma read at stride 4, over d4): z's coefficients and the final-value
    flag vs perm_replay"""
    fid, log_n, zk_rows, stride = zk.FP, 20, 37, 4
    P, n = orc.MODULUS[fid], 1 << log_n
    beta, gamma, shifts, rand = draw_scalars(P, 92)
    w = orc.random_scalars(fid, 7 * n, seed=93).reshape(7, n, 4)
    sigma = orc.random_scalars(fid, 7 * stride * n, seed=94).reshape(7, stride * n, 4)
    num, den = pr.ratio_factors([canonical_ints(w[k]) for k in range(7)], [canonical_ints(sigma[k, ::stride]) for k in range(7)],
                                shifts, beta, gamma, ev.omega(orc, fid, log_n), P)
    z, want_ok = pr.z_evaluations(num, den, zk_rows, rand, P)
    del num, den
    want = orc.ntt(fid, ev.mont(orc, fid, z), inverse=True)
    del z
    got, ok = device_z(ctx, orc, fid, log_n, zk_rows, orc.to_mont(fid, w), orc.to_mont(fid, sigma), beta, gamma, shifts, rand)
    assert ok == want_ok
    assert np.array_equal(got, want)
