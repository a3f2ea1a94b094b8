"""The permutation aggregation polynomial z on the device (zk_perm_aggreg_dev, kimchi's ProverIndex::perm_aggreg): z's coefficients
and the final-value flag compared bit for bit with the Python restatement (tests/perm_replay.py) over both fields, domains of 2^4 to
2^17 rows, zk_rows of 3, 5 and n - 1, sigma read at strides 8 and 1, wired instances, a broken cell, a wired zk row and zero
denominators early, in the middle and inside the tail; on a wired instance, zk_perm_quotient_dev over the device's z vanishes on
d1 and z(1) = z(omega^(n - zk_rows)) = 1; refusals leave d_z untouched; two threads share one context."""
import ctypes
import random
import threading

import numpy as np
import pytest

import evals_replay as ev
import perm_replay as pr
import proof_systems_b200 as zk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def stale(n):
    """a recognisable pattern for d_z before a call"""
    return np.full((n, 4), 0x0123456789abcdef, dtype=np.uint64)


def scalars(orc, fid, inst):
    m = lambda xs: ev.mont(orc, fid, xs)
    return m([inst.beta])[0], m([inst.gamma])[0], m(inst.shifts), m(inst.rand)


def upload(orc, fid, inst, stride, bufs, seed):
    """the 7 witness columns (d1 evaluations) and the 7 sigma columns read at `stride` -> (d_w, d_sigma)"""
    d_w = [bufs.put(ev.mont(orc, fid, inst.w[k])) for k in range(7)]
    d_s = [bufs.put(pr.sigma_strided(orc, fid, inst.sigma[k], stride, seed + k)) for k in range(7)]
    return d_w, d_s


def device_z(ctx, orc, fid, log_n, zk_rows, inst, d_w, d_s, stride, bufs):
    n = 1 << log_n
    d_z = bufs.put(stale(n))
    ok = ctx.perm_aggreg_dev(fid, log_n, zk_rows, d_w, d_s, stride * n, *scalars(orc, fid, inst), d_z)
    return ctx.dev_download(d_z, (n, 4)), ok, d_z


def patch_row(orc, fid, log_n, inst, num, den, j):
    """num / den with row j recomputed from inst"""
    P = orc.MODULUS[fid]
    x = pow(ev.omega(orc, fid, log_n), j, P)
    a = b = 1
    for k in range(7):
        a = a * (inst.w[k][j] + x * inst.beta % P * inst.shifts[k] + inst.gamma) % P
        b = b * (inst.w[k][j] + inst.sigma[k][j] * inst.beta + inst.gamma) % P
    num, den = list(num), list(den)
    num[j], den[j] = a, b
    return num, den


def variants(orc, fid, log_n, zk_rows, inst, rng):
    """(name, instance, sigma stride, changed row or None)"""
    P, n = orc.MODULUS[fid], 1 << log_n
    last = n - zk_rows
    out = [("valid", inst, 8, None)]
    bad = inst.copy()
    k, j = rng.choice(inst.wired)
    bad.w[k][j] = (bad.w[k][j] + rng.randrange(1, P)) % P
    out.append(("broken", bad, 1, j))
    for name, j, stride in (("zero early", 0, 1), ("zero middle", last // 2, 8),
                            ("zero in the tail", last + 2 + (zk_rows - 3) // 2 if zk_rows > 3 else last + 1, 8)):
        zi = inst.copy()
        pr.zero_denominator(zi, P, rng.randrange(7), j)
        out.append((name, zi, stride, j))
    if zk_rows > 3:
        tw = inst.copy()
        j = last + 2 + rng.randrange(zk_rows - 3)
        tw.sigma[rng.randrange(7)][j] = rng.randrange(P)
        out.append(("wired zk row", tw, 1, j))
    return out


# 2^12 rows: last = n - zk_rows just past, on and just before the 2048-row block boundary (2049, 2048, 2047), on a 16-row
# thread boundary (16), and a tail warp scan over 31 or 32 rows (zk_rows 35, 36)
CASES = [(log_n, zk) for log_n in (4, 10, 16, 17) for zk in (3, 5, (1 << log_n) - 1)] + [(12, zk) for zk in (35, 36, 2047, 2048, 2049, 4080)]


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,zk_rows", CASES)
def test_z_matches_the_reference(ctx, orc, fid, log_n, zk_rows):
    P, n = orc.MODULUS[fid], 1 << log_n
    inst = pr.wired_instance(orc, fid, log_n, zk_rows, seed=1000 * fid + 10 * log_n + zk_rows)
    rng = random.Random(fid + log_n + zk_rows)
    num0, den0 = pr.ratio_factors(inst.w, inst.sigma, inst.shifts, inst.beta, inst.gamma, ev.omega(orc, fid, log_n), P)
    for name, vi, stride, j in variants(orc, fid, log_n, zk_rows, inst, rng):
        num, den = (num0, den0) if j is None or j >= n - 1 else patch_row(orc, fid, log_n, vi, num0, den0, j)
        z, want_ok = pr.z_evaluations(num, den, zk_rows, vi.rand, P)
        want = ev.mont(orc, fid, pr.interpolate(orc, fid, z))
        with ctx.buffers() as bufs:
            d_w, d_s = upload(orc, fid, vi, stride, bufs, seed=log_n + zk_rows)
            got, ok, _ = device_z(ctx, orc, fid, log_n, zk_rows, vi, d_w, d_s, stride, bufs)
        assert ok == want_ok, name
        assert want_ok == (name in ("valid", "zero in the tail", "wired zk row")), name
        assert np.array_equal(got, want), name


# ---------------------------------------------------------------------------------------------------------------- the property
def vanishing_coeffs(orc, fid, log_n, zk_rows):
    """permutation_vanishing_polynomial(d1, zk_rows) = (x - w^(n - zk_rows)) (x - w^(n - zk_rows + 1)) (x - w^(n - 1)): 4 coefficients"""
    P, n = orc.MODULUS[fid], 1 << log_n
    w = ev.omega(orc, fid, log_n)
    c = [1]
    for r in (pow(w, n - zk_rows, P), pow(w, n - zk_rows + 1, P), pow(w, n - 1, P)):
        c = [((c[i - 1] if i else 0) - r * (c[i] if i < len(c) else 0)) % P for i in range(len(c) + 1)]
    return c


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,zk_rows", [(10, 3), (10, 5), (12, 17)])
def test_perm_quotient_over_the_device_z_vanishes_on_d1(ctx, orc, fid, log_n, zk_rows):
    """z from the device; witness and z to d8 with zk_ntt_dev_oop; zkpm over d8 from its four coefficients; zk_perm_quotient_dev is
    then zero at every point of d1 (positions 8 j) and not everywhere; z(1) = z(omega^(n - zk_rows)) = 1"""
    P, n = orc.MODULUS[fid], 1 << log_n
    m8 = 8 * n
    inst = pr.wired_instance(orc, fid, log_n, zk_rows, seed=77 + fid + log_n + zk_rows)
    beta, gamma, shifts, rand = scalars(orc, fid, inst)
    alpha0 = ev.mont(orc, fid, [random.Random(fid).randrange(1, P)])[0]
    with ctx.buffers() as bufs:
        d_wev = bufs.put(np.concatenate([ev.mont(orc, fid, inst.w[k]) for k in range(7)]))
        d_s8 = bufs.put(np.concatenate([pr.sigma_d8(orc, fid, inst.sigma[k]) for k in range(7)]))
        d_w = [d_wev + k * n * 32 for k in range(7)]
        d_s = [d_s8 + k * m8 * 32 for k in range(7)]
        d_z = bufs.put(stale(n))
        assert ctx.perm_aggreg_dev(fid, log_n, zk_rows, d_w, d_s, m8, beta, gamma, shifts, rand, d_z) is True
        d_wc, d_w8, d_z8, d_zk8, d_out = (bufs.put(np.zeros((k, 4), dtype=np.uint64)) for k in (7 * n, 7 * m8, m8, m8, m8))
        ctx.ntt_dev_oop(fid, d_wev, n, n, d_wc, log_n, batch=7, inverse=True)             # the witness polynomials
        ctx.ntt_dev_oop(fid, d_wc, n, n, d_w8, log_n + 3, batch=7)                        # ... over d8
        ctx.ntt_dev_oop(fid, d_z, n, n, d_z8, log_n + 3)                                  # z over d8
        d_zk = bufs.put(ev.mont(orc, fid, vanishing_coeffs(orc, fid, log_n, zk_rows)))
        ctx.ntt_dev_oop(fid, d_zk, 4, 4, d_zk8, log_n + 3)                                # zkpm over d8
        ctx.perm_quotient_dev(fid, log_n + 3, [d_w8 + k * m8 * 32 for k in range(7)], d_z8, d_s, d_zk8, beta, gamma, alpha0, shifts, d_out)
        out = ctx.dev_download(d_out, (m8, 4))
        assert not out[::8].any()
        assert out.any()
        w = ev.omega(orc, fid, log_n)
        at = ctx.poly_evaluate_chunks_dev(fid, [(d_z, n)], 1, n, ev.mont(orc, fid, [1, pow(w, n - zk_rows, P)]))
        one = ev.mont(orc, fid, [1])[0]
        assert np.array_equal(at[0, 0, 0], one) and np.array_equal(at[0, 1, 0], one)


# ---------------------------------------------------------------------------------------------------------------- errors, threads
def test_refusals_leave_z_untouched(ctx, orc):
    fid, log_n, zk_rows = zk.FQ, 6, 4
    P, n = orc.MODULUS[fid], 1 << log_n
    inst = pr.wired_instance(orc, fid, log_n, zk_rows, seed=3)
    beta, gamma, shifts, rand = scalars(orc, fid, inst)
    bad = np.array([P & (2**64 - 1), (P >> 64) & (2**64 - 1), (P >> 128) & (2**64 - 1), P >> 192], dtype=np.uint64)
    with ctx.buffers() as bufs:
        d_w, d_s = upload(orc, fid, inst, 8, bufs, seed=3)
        d_z = bufs.put(stale(n))
        sh_bad, rn_bad = shifts.copy(), rand.copy()
        sh_bad[6], rn_bad[1] = bad, bad
        cases = [dict(field=7), dict(log_n=31), dict(zk_rows=2), dict(zk_rows=0), dict(zk_rows=n), dict(zk_rows=n + 1),
                 dict(sigma_len=0), dict(sigma_len=n // 2), dict(sigma_len=n + 1), dict(sigma_len=9 * n), dict(sigma_len=3 * n + 5),
                 dict(beta=bad), dict(gamma=bad), dict(shifts=sh_bad), dict(rand=rn_bad),
                 dict(d_z=d_w[3]), dict(d_z=d_s[6] + 32 * (8 * n - 1)), dict(d_z=d_w[0] - 32 * (n - 1))]
        for kw in cases:
            a = dict(field=fid, log_n=log_n, zk_rows=zk_rows, sigma_len=8 * n, beta=beta, gamma=gamma, shifts=shifts, rand=rand, d_z=d_z)
            a.update(kw)
            with pytest.raises(zk.ZkError) as e:
                ctx.perm_aggreg_dev(a["field"], a["log_n"], a["zk_rows"], d_w, d_s, a["sigma_len"], a["beta"], a["gamma"], a["shifts"],
                                    a["rand"], a["d_z"])
            assert e.value.code == -1, (kw, e.value)
            assert np.array_equal(ctx.dev_download(d_z, (n, 4)), stale(n)), kw
        with pytest.raises(zk.ZkError) as e:
            ctx.perm_aggreg_dev(fid, log_n, zk_rows, d_w[:6] + [0], d_s, 8 * n, beta, gamma, shifts, rand, d_z)
        assert e.value.code == -1
        with pytest.raises(zk.ZkError) as e:
            ctx.perm_aggreg_dev(fid, log_n, zk_rows, d_w, [0] + d_s[1:], 8 * n, beta, gamma, shifts, rand, d_z)
        assert e.value.code == -1
        # null pointers through the C ABI itself
        L, h = zk.lib(), ctx._h
        pw = (ctypes.c_void_p * 7)(*d_w)
        ps = (ctypes.c_void_p * 7)(*d_s)
        arrs = [np.ascontiguousarray(x, dtype=np.uint64).reshape(-1) for x in (beta, gamma, shifts, rand)]
        ptrs = [a.ctypes.data for a in arrs]
        ok = ctypes.c_int(7)
        full = [h, fid, log_n, zk_rows, pw, ps, 8 * n, *ptrs, d_z, ctypes.byref(ok)]
        for pos in (0, 4, 5, 7, 8, 9, 10, 11, 12):
            args = list(full)
            args[pos] = None
            assert L.zk_perm_aggreg_dev(*args) == -1, pos
        assert ok.value == 7
        assert np.array_equal(ctx.dev_download(d_z, (n, 4)), stale(n))
        # the edges that are valid: zk_rows = n - 1, sigma read at strides 1 .. 8
        assert ctx.perm_aggreg_dev(fid, log_n, n - 1, d_w, d_s, 8 * n, beta, gamma, shifts, rand, d_z) in (True, False)
        for s in range(1, 9):
            ctx.perm_aggreg_dev(fid, log_n, zk_rows, d_w, d_s, s * n, beta, gamma, shifts, rand, d_z)
        assert ctx.perm_aggreg_dev(fid, log_n, zk_rows, d_w, d_s, 8 * n, beta, gamma, shifts, rand, d_z) is True


def test_two_threads_share_a_context(ctx, orc):
    fid, log_n, zk_rows = zk.FP, 12, 6
    P, n = orc.MODULUS[fid], 1 << log_n
    cases, errors = [], []

    def work(t):
        try:
            inst, d_w, d_s, d_z, want, want_ok = cases[t]
            for _ in range(6):
                ok = ctx.perm_aggreg_dev(fid, log_n, zk_rows, d_w, d_s, 8 * n, *scalars(orc, fid, inst), d_z)
                assert ok == want_ok and np.array_equal(ctx.dev_download(d_z, (n, 4)), want)
        except Exception as e:                    # reported by the main thread
            errors.append(e)

    with ctx.buffers() as bufs:
        for t in range(2):
            inst = pr.wired_instance(orc, fid, log_n, zk_rows, seed=500 + t)
            if t:
                k, j = inst.wired[0]
                inst.w[k][j] = (inst.w[k][j] + 1) % P                     # one thread's instance fails the final-value check
            _, coeffs, ok = pr.perm_aggreg(orc, fid, log_n, zk_rows, inst.w, inst.sigma, inst.shifts, inst.beta, inst.gamma, inst.rand)
            d_w, d_s = upload(orc, fid, inst, 8, bufs, seed=t)
            cases.append((inst, d_w, d_s, bufs.put(stale(n)), ev.mont(orc, fid, coeffs), ok))
        th = [threading.Thread(target=work, args=(t,)) for t in range(2)]
        for t in th:
            t.start()
        for t in th:
            t.join()
    assert not errors, errors
    assert cases[0][5] is True and cases[1][5] is False
