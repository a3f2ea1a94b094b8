"""ft of Maller's optimisation on the device (zk_prover_ft_dev, kimchi/src/prover.rs:1147-1206): every output compared bit for bit
with the Python restatement (tests/ft_replay.py) — the m coefficients (zero past ft_len), ft_len and ft(zeta omega) — over both
fields, unchunked, n < m and chunked shapes, edge lengths of t, special points and cancellations; the verifier's ft_comm against
commit(ft) masked with blinding_ft; one proof's tail from the resident quotient to an opening proof that zk_srs_verify accepts;
errors and two threads on one context."""
import contextlib
import ctypes
import random
import threading

import numpy as np
import pytest

import evals_replay as ev
import ft_replay as fr
import proof_systems_b200 as zk
from verify_replay import HashTranscript

pytestmark = pytest.mark.gpu

SHAPES = [(6, 64), (6, 128), (8, 128), (8, 64)]          # (log_n, m): n = m, n < m, 2 chunks, 4 chunks


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def m1(orc, fid, x):
    return ev.mont(orc, fid, [x])[0]


def stale(m):
    """a recognisable pattern for the ft buffer before a call: nothing of it may survive past ft_len"""
    return np.full((m, 4), 0x0123456789abcdef, dtype=np.uint64)


def device_ft(ctx, orc, fid, log_n, m, terms, t, zeta, bufs):
    """upload terms / t, run the call over a stale ft buffer -> (ft [m, 4] Montgomery, ft_len, ft_eval1 [4], d_ft, d_t)"""
    d_terms = [(bufs.put(ev.mont(orc, fid, e)), len(e), m1(orc, fid, c)) for e, c in terms]
    d_t = bufs.put(ev.mont(orc, fid, t)) if t else 0
    d_ft = bufs.put(stale(m))
    ft_len, e1 = ctx.prover_ft_dev(fid, log_n, m, d_terms, d_t, len(t), m1(orc, fid, zeta), d_ft)
    return ctx.dev_download(d_ft, (m, 4)), ft_len, e1, d_ft, d_t


def check_against_replay(orc, fid, log_n, m, terms, t, zeta, got):
    P = orc.MODULUS[fid]
    coeffs, ft_len, e1 = got[:3]
    f, want, want_e1 = fr.ft(orc, fid, log_n, m, terms, t, zeta)
    assert ft_len == len(want)
    assert np.array_equal(coeffs[:ft_len], ev.mont(orc, fid, want).reshape(-1, 4)[:ft_len])
    assert not coeffs[ft_len:].any()
    assert np.array_equal(e1, m1(orc, fid, want_e1))
    # Maller's identity on the device's output: ft(zeta) = f(zeta) - (zeta^n - 1) t(zeta)
    ft_ints = ev.ints(orc, fid, coeffs[:ft_len]) if ft_len else []
    zh = (pow(zeta, 1 << log_n, P) - 1) % P
    assert fr.evaluate(ft_ints, zeta, P) == (fr.evaluate(f, zeta, P) - zh * fr.evaluate(t, zeta, P)) % P
    return f, want


def make_terms(rng, P, n, kind):
    if kind == "none":
        return []
    if kind == "perm":
        return [([rng.randrange(P) for _ in range(8 * n)], rng.randrange(P))]
    return [([rng.randrange(P) for _ in range(s * n)], rng.randrange(P)) for s in (1, 4, 8)]


# ---------------------------------------------------------------------------------------------------------------- parity
@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,m", SHAPES)
@pytest.mark.parametrize("kind", ["none", "perm", "three"])
def test_ft_matches_the_reference(ctx, orc, fid, log_n, m, kind):
    P, n = orc.MODULUS[fid], 1 << log_n
    nc = fr.num_chunks(n, m)
    rng = random.Random(1000 * fid + 10 * log_n + m + len(kind))
    terms = make_terms(rng, P, n, kind)
    zeta = rng.randrange(P)
    for t_len in (0, 1, m - 1, 7 * nc * m, 7 * nc * m - m // 2 - 3):
        t = [rng.randrange(P) for _ in range(t_len)]
        with ctx.buffers() as bufs:
            got = device_ft(ctx, orc, fid, log_n, m, terms, t, zeta, bufs)
            check_against_replay(orc, fid, log_n, m, terms, t, zeta, got)
            # ft_eval1 is evaluate_chunks of the resident ft at zeta omega
            zo = zeta * ev.omega(orc, fid, log_n) % P
            if got[1]:
                again = ctx.poly_evaluate_chunks_dev(fid, [(got[3], got[1])], 1, m, ev.mont(orc, fid, [zo]))
                assert np.array_equal(again[0, 0, 0], got[2]), t_len
            else:
                assert not got[2].any()


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,m", [(6, 64), (6, 128), (8, 64)])
def test_special_points(ctx, orc, fid, log_n, m):
    """zeta = 0: only the first chunks count and zeta^n - 1 = -1; zeta = 1 and zeta = omega^3: zeta^n - 1 = 0, ft is f linearised"""
    P, n = orc.MODULUS[fid], 1 << log_n
    nc = fr.num_chunks(n, m)
    rng = random.Random(7 + fid + log_n + m)
    terms = make_terms(rng, P, n, "three")
    t = [rng.randrange(P) for _ in range(7 * nc * m - 5)]
    w3 = pow(ev.omega(orc, fid, log_n), 3, P)
    for zeta in (0, 1, w3):
        with ctx.buffers() as bufs:
            got = device_ft(ctx, orc, fid, log_n, m, terms, t, zeta, bufs)
            f, want = check_against_replay(orc, fid, log_n, m, terms, t, zeta, got)
            if zeta == 0:                             # ft = f_0 + t_0
                f0, t0 = (f[:m] + [0] * m)[:m], (t[:m] + [0] * m)[:m]
                assert want == fr.trim([(a + b) % P for a, b in zip(f0, t0)])
            else:
                assert want == fr.linearize(fr.to_chunked_polynomial(f, nc, m), m, pow(zeta, m, P), P)


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,m", [(6, 64), (6, 128), (8, 64)])
def test_cancellation(ctx, orc, fid, log_n, m):
    """t with (zeta^n - 1) t = f linearised: ft = 0, ft_len = 0, ft_eval1 = 0; a perturbed t leaves 0 < ft_len < m"""
    P, n = orc.MODULUS[fid], 1 << log_n
    nc = fr.num_chunks(n, m)
    rng = random.Random(70 + fid + log_n + m)
    terms = make_terms(rng, P, n, "perm")
    zeta = rng.randrange(P)
    f = fr.interpolate(orc, fid, fr.combine_terms(terms, n, P))
    lin_f = fr.linearize(fr.to_chunked_polynomial(f, nc, m), m, pow(zeta, m, P), P)
    inv = pow((pow(zeta, n, P) - 1) % P, P - 2, P)
    t_cancel = [c * inv % P for c in lin_f]
    t_part = list(t_cancel)
    t_part[5] = (t_part[5] + 3) % P
    for t, want_len in ((t_cancel, 0), (t_part, 6), (t_cancel[:len(t_cancel) - 4], len(lin_f))):
        with ctx.buffers() as bufs:
            got = device_ft(ctx, orc, fid, log_n, m, terms, t, zeta, bufs)
            check_against_replay(orc, fid, log_n, m, terms, t, zeta, got)
            assert got[1] == want_len and 0 <= want_len <= m
            if want_len == 0:
                assert not got[0].any() and not got[2].any()


# ---------------------------------------------------------------------------------------------------------------- commitments
def chunk_scalars(orc, fid, zeta, m, k, lead):
    P = orc.MODULUS[fid]
    zm = pow(zeta, m, P)
    return [lead * pow(zm, j, P) % P for j in range(k)]


def verifier_ft_comm(orc, G, f_comm, t_comm, perm, zeta, log_n, m):
    """verifier.rs:957-965: chunk_commitment(f_comm) - (zeta^n - 1) chunk_commitment(t_comm), f_comm = perm_scalar * sigma_comm[6],
    as one MSM over the chunks (identity chunks left out)"""
    fid = G.scalar
    P = orc.MODULUS[fid]
    zh = (pow(zeta, 1 << log_n, P) - 1) % P
    pts = list(f_comm) + list(t_comm)
    sc = chunk_scalars(orc, fid, zeta, m, len(f_comm), perm) + chunk_scalars(orc, fid, zeta, m, len(t_comm), -zh % P)
    keep = [j for j, p in enumerate(pts) if p.any()]
    return orc.msm_mont(G.cid, np.stack([pts[j] for j in keep]), ev.mont(orc, fid, [sc[j] for j in keep]))


def sigma6(orc, fid, rng, n):
    """sigma_6's coefficients and its evaluations over d8 (permutation_coefficients8[6])"""
    P = orc.MODULUS[fid]
    coeffs = [rng.randrange(P) for _ in range(n)]
    evals8 = ev.ints(orc, fid, orc.ntt(fid, ev.mont(orc, fid, coeffs + [0] * (7 * n))))
    return coeffs, evals8


@pytest.mark.parametrize("log_n,m", [(6, 64), (7, 64)])
def test_commitment_equals_the_verifiers_ft_comm(ctx, orc, vesta_srs, log_n, m):
    """commit(ft) masked with blinding_ft == chunk_commitment(f_comm) - (zeta^n - 1) chunk_commitment(t_comm), t_comm hiding"""
    G = vesta_srs
    fid = G.scalar
    P, n = orc.MODULUS[fid], 1 << log_n
    nc = fr.num_chunks(n, m)
    rng = random.Random(log_n + m)
    s6, s6_8 = sigma6(orc, fid, rng, n)
    perm, zeta = rng.randrange(P), rng.randrange(P)
    t = [rng.randrange(P) for _ in range(7 * nc * m - 9)]
    t_bl = [rng.randrange(P) for _ in range(7 * nc)]
    with zk.SRS(ctx, G.cid, G.g[:m], G.mont_points(G.h_xy_canon)[0]) as srs:
        with ctx.buffers() as bufs:
            got = device_ft(ctx, orc, fid, log_n, m, [(s6_8, perm)], t, zeta, bufs)
            check_against_replay(orc, fid, log_n, m, [(s6_8, perm)], t, zeta, got)
            coeffs, ft_len = got[0], got[1]
            t_comm = srs.commit_custom(ev.mont(orc, fid, t), 7 * nc, ev.mont(orc, fid, t_bl)).chunks
            s6_comm = srs.commit_non_hiding(ev.mont(orc, fid, s6), nc).chunks
            assert t_comm.shape[0] == 7 * nc and s6_comm.shape[0] == nc
            bft = fr.blinding_ft(t_bl, zeta, log_n, m, P)
            mine = srs.commit_custom(coeffs[:ft_len], 1, ev.mont(orc, fid, [bft])).chunks
            assert mine.shape[0] == 1
            assert np.array_equal(mine[0], verifier_ft_comm(orc, G, s6_comm, t_comm, perm, zeta, log_n, m))


def test_one_proofs_tail_resident(ctx, orc, vesta_srs):
    """2^10 rows, max_poly_size 2^9 (2 chunks): t from divide_by_vanishing, t_comm by device MSMs, the evaluations at zeta and zeta
    omega from zk_lagrange_* / evaluate_chunks, ft from the new call, then zk_srs_open over the resident ft (length ft_len, blinder
    blinding_ft), t and sigma_6 over d8, verified by zk_srs_verify against the verifier's ft_comm; ft_eval1 + 1 is rejected"""
    G = vesta_srs
    fid, cid = G.scalar, G.cid
    P, log_n, m = orc.MODULUS[fid], 10, 1 << 9
    n, nc = 1 << log_n, 2
    rng = random.Random(2026)
    q = [rng.randrange(P) for _ in range(7 * n)]
    num = [((q[i - n] if i >= n else 0) - (q[i] if i < 7 * n else 0)) % P for i in range(8 * n)]    # q (x^n - 1)
    s6, s6_8 = sigma6(orc, fid, rng, n)
    perm, zeta = rng.randrange(P), rng.randrange(P)
    zo = zeta * ev.omega(orc, fid, log_n) % P
    t_bl = [rng.randrange(P) for _ in range(7 * nc)]
    h = G.mont_points(G.h_xy_canon)[0]
    srs = zk.SRS(ctx, cid, G.g[:m], h)
    bases = ctx.upload_bases(cid, G.g[:m])
    with srs, ctx.buffers() as bufs, contextlib.ExitStack() as stack:
        # 1. t = numerator / Z_H on the device
        d_num = bufs.put(ev.mont(orc, fid, num))
        d_t = bufs.alloc(7 * n * 32)
        assert ctx.poly_divide_by_vanishing_dev(fid, d_num, 8 * n, log_n, d_t) is True
        # 2. t_comm: the 14 chunk MSMs on the resident t, masked with the blinders
        raw = np.stack([zk.jacobian_to_affine(cid, ctx.msm_dev(bases, d_t + c * m * 32, m, mont=True)) for c in range(7 * nc)])
        t_comm = srs.mask_custom(zk.PolyComm(raw), ev.mont(orc, fid, t_bl)).chunks
        assert np.array_equal(t_comm, srs.commit_custom(ev.mont(orc, fid, q), 7 * nc, ev.mont(orc, fid, t_bl)).chunks)
        s6_comm = srs.commit_non_hiding(ev.mont(orc, fid, s6), nc).chunks
        # 3. evaluations at zeta and zeta omega
        d_s8 = bufs.put(ev.mont(orc, fid, s6_8))
        lbs = [stack.enter_context(zk.LagrangeBasisEvaluations(ctx, fid, m, log_n, m1(orc, fid, x))) for x in (zeta, zo)]
        s6_ev = ev.ints(orc, fid, zk.LagrangeBasisEvaluations.evaluate_all(lbs, [(d_s8, 8 * n, False)])[0])    # [point][chunk]
        s6_ev = [s6_ev[:nc], s6_ev[nc:]]
        t_ev = ev.ints(orc, fid, ctx.poly_evaluate_chunks_dev(fid, [(d_t, 7 * n)], 7 * nc, m, ev.mont(orc, fid, [zeta, zo]))[0])
        t_ev = [t_ev[:7 * nc], t_ev[7 * nc:]]
        # 4. ft
        d_ft = bufs.alloc(m * 32)
        ft_len, e1 = ctx.prover_ft_dev(fid, log_n, m, [(d_s8, 8 * n, m1(orc, fid, perm))], d_t, 7 * n, m1(orc, fid, zeta), d_ft)
        _, want, want_e1 = fr.ft(orc, fid, log_n, m, [(s6_8, perm)], q, zeta)
        assert ft_len == len(want) and np.array_equal(e1, m1(orc, fid, want_e1))
        ft_eval1 = ev.ints(orc, fid, e1)[0]
        # ft(zeta) by Maller's identity from the evaluations: perm sigma_6(zeta) - (zeta^n - 1) t(zeta), chunks combined at zeta^m
        zm, zh = pow(zeta, m, P), (pow(zeta, n, P) - 1) % P
        comb = lambda chunks: sum(c * pow(zm, k, P) for k, c in enumerate(chunks)) % P
        ft_eval0 = (perm * comb(s6_ev[0]) - zh * comb(t_ev[0])) % P
        bft = fr.blinding_ft(t_bl, zeta, log_n, m, P)
        ft_comm = verifier_ft_comm(orc, G, s6_comm, t_comm, perm, zeta, log_n, m).reshape(1, 8)
        # 5. the opening proof over the resident polynomials, then the verifier
        sc = [rng.randrange(P) for _ in range(2 + 2 * 9 + 2)]
        ps, es, draws = sc[0], sc[1], sc[2:]
        u_points = G.g[200:232]
        fe_int = lambda limbs: orc.fe_int(fid, np.ascontiguousarray(limbs, dtype=np.uint64).reshape(4))

        def callbacks(seed):
            tr = HashTranscript(P, u_points, seed)
            return (lambda cip: tr.u_base(fe_int(cip)), lambda j, l, r: m1(orc, fid, tr.round(j, l, r)), lambda d: m1(orc, fid, tr.final(d)))

        plnms = [((d_ft, ft_len), 0, ev.mont(orc, fid, [bft])), ((d_t, 7 * n), 0, ev.mont(orc, fid, t_bl)),
                 ((d_s8, 8 * n), n, np.zeros((nc, 4), dtype=np.uint64))]
        elm = ev.mont(orc, fid, [zeta, zo])
        proof = zk.srs_open(srs, plnms, elm, m1(orc, fid, ps), m1(orc, fid, es), ev.mont(orc, fid, draws), *callbacks(5))

        def cip_of(e1_value):
            evals = [[[ft_eval0], [e1_value]], t_ev, s6_ev]            # [polynomial][point][chunk]
            res, scale = 0, 1
            for pe in evals:
                for k in range(len(pe[0])):
                    res = (res + scale * (pe[0][k] + es * pe[1][k])) % P
                    scale = scale * ps % P
            return res

        def verify(e1_value):
            be = zk.BatchEvaluationProof(proof, elm, m1(orc, fid, ps), m1(orc, fid, es), [ft_comm, t_comm, s6_comm],
                                         m1(orc, fid, cip_of(e1_value)), *callbacks(5))
            rb, sgb = rng.randrange(P), rng.randrange(P)
            return zk.srs_verify(srs, [be], m1(orc, fid, rb), m1(orc, fid, sgb))

        assert verify(ft_eval1) is True
        assert verify((ft_eval1 + 1) % P) is False


# ---------------------------------------------------------------------------------------------------------------- errors, threads
def test_errors_leave_ft_untouched(ctx, orc):
    fid, log_n, m = zk.FP, 6, 64
    P, n = orc.MODULUS[fid], 1 << log_n
    L, h = zk.lib(), ctx._h
    rng = random.Random(3)
    z = m1(orc, fid, 5)
    bad = np.array([P & (2**64 - 1), (P >> 64) & (2**64 - 1), (P >> 128) & (2**64 - 1), P >> 192], dtype=np.uint64)
    with ctx.buffers() as bufs:
        d_e = bufs.put(ev.mont(orc, fid, [rng.randrange(P) for _ in range(8 * n)]))
        d_t = bufs.put(ev.mont(orc, fid, [rng.randrange(P) for _ in range(7 * m + 1)]))
        d_ft = bufs.put(stale(m))
        good = [(d_e, 8 * n, z)]
        cases = [
            (-1, dict(field=7)), (-1, dict(log_n=31)), (-1, dict(mps=0)), (-1, dict(log_n=7, mps=48)),
            (-1, dict(terms=[(d_e, 0, z)])), (-1, dict(terms=[(d_e, n + 1, z)])), (-1, dict(terms=[(d_e, 9 * n, z)])),
            (-1, dict(terms=[(0, n, z)])), (-1, dict(zeta=bad)), (-1, dict(terms=[(d_e, n, bad)])),
            (-1, dict(d_t=0, t_len=5)), (-4, dict(t_len=7 * m + 1)), (-4, dict(mps=32, t_len=7 * 2 * 32 + 1)),
        ]
        for code, kw in cases:
            a = dict(field=fid, log_n=log_n, mps=m, terms=good, d_t=d_t, t_len=10, zeta=z)
            a.update(kw)
            with pytest.raises(zk.ZkError) as e:
                ctx.prover_ft_dev(a["field"], a["log_n"], a["mps"], a["terms"], a["d_t"], a["t_len"], a["zeta"], d_ft)
            assert e.value.code == code, (kw, e.value)
            assert np.array_equal(ctx.dev_download(d_ft, (m, 4)), stale(m)), kw
        e1 = np.zeros(4, dtype=np.uint64)
        ln = ctypes.c_size_t()
        zc = np.ascontiguousarray(z)
        assert L.zk_prover_ft_dev(None, fid, log_n, m, None, 0, None, 0, zc.ctypes.data, d_ft, ctypes.byref(ln), e1.ctypes.data) == -1
        assert L.zk_prover_ft_dev(h, fid, log_n, m, None, 0, None, 0, None, d_ft, ctypes.byref(ln), e1.ctypes.data) == -1
        assert L.zk_prover_ft_dev(h, fid, log_n, m, None, 0, None, 0, zc.ctypes.data, None, ctypes.byref(ln), e1.ctypes.data) == -1
        assert L.zk_prover_ft_dev(h, fid, log_n, m, None, 0, None, 0, zc.ctypes.data, d_ft, None, e1.ctypes.data) == -1
        assert L.zk_prover_ft_dev(h, fid, log_n, m, None, 0, None, 0, zc.ctypes.data, d_ft, ctypes.byref(ln), None) == -1
        assert L.zk_prover_ft_dev(h, fid, log_n, m, None, 1, None, 0, zc.ctypes.data, d_ft, ctypes.byref(ln), e1.ctypes.data) == -1
        assert np.array_equal(ctx.dev_download(d_ft, (m, 4)), stale(m))
        # the edges that are valid: f = 0 and t = 0 give ft = 0; t of exactly 7 chunks
        ln0, e0 = ctx.prover_ft_dev(fid, log_n, m, [], 0, 0, z, d_ft)
        assert ln0 == 0 and not e0.any() and not ctx.dev_download(d_ft, (m, 4)).any()
        assert ctx.prover_ft_dev(fid, log_n, m, good, d_t, 7 * m, z, d_ft)[0] > 0


def test_two_threads_share_a_context(ctx, orc):
    fid, log_n, m = zk.FQ, 8, 128
    P, n = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(11)
    cases = []
    for _ in range(2):
        terms = make_terms(rng, P, n, "perm")
        t = [rng.randrange(P) for _ in range(7 * 2 * m - 1)]
        zeta = rng.randrange(P)
        _, want, want_e1 = fr.ft(orc, fid, log_n, m, terms, t, zeta)
        cases.append((terms, t, zeta, want, want_e1))
    errors, dev = [], []

    def work(k):
        try:
            terms, t, zeta, want, want_e1 = cases[k]
            d_terms, d_t, d_ft = dev[k]
            for _ in range(6):
                ln, e1 = ctx.prover_ft_dev(fid, log_n, m, d_terms, d_t, len(t), m1(orc, fid, zeta), d_ft)
                got = ctx.dev_download(d_ft, (m, 4))
                assert ln == len(want) and np.array_equal(e1, m1(orc, fid, want_e1))
                assert np.array_equal(got[:ln], ev.mont(orc, fid, want)) and not got[ln:].any()
        except Exception as e:                    # reported by the main thread
            errors.append(e)

    with ctx.buffers() as bufs:
        for terms, t, zeta, _, _ in cases:
            d_terms = [(bufs.put(ev.mont(orc, fid, e)), len(e), m1(orc, fid, c)) for e, c in terms]
            dev.append((d_terms, bufs.put(ev.mont(orc, fid, t)), bufs.put(stale(m))))
        th = [threading.Thread(target=work, args=(k,)) for k in range(2)]
        for t in th:
            t.start()
        for t in th:
            t.join()
    assert not errors, errors
