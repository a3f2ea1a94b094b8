"""Device-resident folding rounds of the IPA opening (proof_systems_b200.IpaRounds over ipa.cu) against the oracle, following
  poly-commitment/src/ipa.rs:929-1007        the round structure of SRS::open (L, R, the folds of a, b and g)
  poly-commitment/src/commitment.rs:528-581  b_poly_coefficients: the folded base g0 equals <s, g> with s_i = prod u_{k-j}^{bit_j(i)}
"""
import numpy as np
import pytest

import proof_systems_b200 as zk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def b_poly_coefficients(chals, m):
    """commitment.rs:565-581: s[i] = prod over set bits j of i of chals[k-1-j]"""
    k = len(chals)
    s = [1] * (1 << k)
    for i in range(1, 1 << k):
        kk = i.bit_length() - 1
        s[i] = s[i - (1 << kk)] * chals[k - 1 - kk] % m
    return s


@pytest.mark.parametrize("name", ["pallas_srs", "vesta_srs"])
@pytest.mark.parametrize("window_bits", [-1, 0])
def test_every_round_matches_the_oracle(ctx, orc, request, name, window_bits):
    """L, R, the inner products and the folded a, b of every round against an explicit restatement of ipa.rs:929-1007 that
    folds the bases point by point (g <- g_lo + [u] g_hi) on the CPU."""
    G = request.getfixturevalue(name)
    m = orc.FQ_MODULUS if G.scalar == orc.FQ else orc.FP_MODULUS
    n = 16
    g = G.g[:n].copy()
    a = orc.limbs_to_ints(orc.random_scalars(G.scalar, n, seed=11))
    b = orc.limbs_to_ints(orc.random_scalars(G.scalar, n, seed=12))
    mont = lambda xs: orc.to_mont(G.scalar, orc.ints_to_limbs(xs))
    bases = ctx.upload_bases(G.cid, g, window_bits=window_bits)
    rounds = zk.IpaRounds(ctx, bases, mont(a), mont(b))
    chals = orc.limbs_to_ints(orc.random_scalars(G.scalar, 4, seed=13))
    for u in chals:
        h = len(a) // 2
        assert len(rounds) == 2 * h
        l, r, ipl, ipr = rounds.lr()
        assert np.array_equal(zk.jacobian_to_affine(G.cid, l), orc.msm(G.cid, g[:h], orc.ints_to_limbs(a[h:])))
        assert np.array_equal(zk.jacobian_to_affine(G.cid, r), orc.msm(G.cid, g[h:], orc.ints_to_limbs(a[:h])))
        assert orc.fe_int(G.scalar, ipl) == sum(x * y for x, y in zip(a[h:], b[:h])) % m
        assert orc.fe_int(G.scalar, ipr) == sum(x * y for x, y in zip(a[:h], b[h:])) % m
        ui = pow(u, -1, m)
        rounds.fold(mont([u])[0], mont([ui])[0])
        a = [(a[i] + ui * a[i + h]) % m for i in range(h)]
        b = [(b[i] + u * b[i + h]) % m for i in range(h)]
        g = np.stack([orc.affine_add(G.cid, g[i], orc.scalar_mul(G.cid, g[i + h], u)) for i in range(h)])
        da, db = rounds.state()
        assert orc.limbs_to_ints(orc.from_mont(G.scalar, da)) == a
        assert orc.limbs_to_ints(orc.from_mont(G.scalar, db)) == b
    assert len(rounds) == 1
    assert np.array_equal(zk.jacobian_to_affine(G.cid, rounds.sg()), g[0])
    with pytest.raises(zk.ZkError):
        rounds.lr()
    rounds.close()
    bases.free()


def test_folded_base_is_the_b_poly_commitment(ctx, orc, pallas_srs):
    """After all rounds g0 = <b_poly_coefficients(chals), g> — the `sg` the verifier recomputes (ipa.rs:248-262)."""
    G = pallas_srs
    m = orc.FQ_MODULUS
    k = 12
    n = 1 << k
    g = G.g[:n]
    a = orc.limbs_to_ints(orc.random_scalars(G.scalar, n, seed=21))
    b = orc.limbs_to_ints(orc.random_scalars(G.scalar, n, seed=22))
    a[5] = 0
    mont = lambda xs: orc.to_mont(G.scalar, orc.ints_to_limbs(xs))
    bases = ctx.upload_bases(G.cid, g)
    rounds = zk.IpaRounds(ctx, bases, mont(a), mont(b))
    chals = orc.limbs_to_ints(orc.random_scalars(G.scalar, k, seed=23))
    ca = list(a)
    for j, u in enumerate(chals):
        l, r, _, _ = rounds.lr()
        if j in (0, 3, k - 1):
            # explicit scalars over the original bases: L = sum_t sum_{i<h} a_j[h+i] s_j[t] g[t m_j + i]
            sj = b_poly_coefficients(chals[:j], m)
            mj = n >> j
            h = mj // 2
            scl, scr = [0] * n, [0] * n
            for t in range(1 << j):
                for i in range(h):
                    scl[t * mj + i] = ca[h + i] * sj[t] % m
                    scr[t * mj + h + i] = ca[i] * sj[t] % m
            assert np.array_equal(zk.jacobian_to_affine(G.cid, l), orc.msm(G.cid, g, orc.ints_to_limbs(scl)))
            assert np.array_equal(zk.jacobian_to_affine(G.cid, r), orc.msm(G.cid, g, orc.ints_to_limbs(scr)))
        ui = pow(u, -1, m)
        rounds.fold(mont([u])[0], mont([ui])[0])
        h = len(ca) // 2
        ca = [(ca[i] + ui * ca[i + h]) % m for i in range(h)]
    a0, b0 = rounds.state()
    s = b_poly_coefficients(chals, m)
    s_inv = b_poly_coefficients([pow(u, -1, m) for u in chals], m)
    assert np.array_equal(zk.jacobian_to_affine(G.cid, rounds.sg()), orc.msm(G.cid, g, orc.ints_to_limbs(s)))
    assert orc.fe_int(G.scalar, a0[0]) == sum(x * y for x, y in zip(a, s_inv)) % m == ca[0]
    assert orc.fe_int(G.scalar, b0[0]) == sum(x * y for x, y in zip(b, s)) % m
    rounds.close()
    bases.free()


def test_identity_padding_and_argument_checks(ctx, orc, pallas_srs):
    """SRS::open pads g with the identity and a with zeros up to a power of two (ipa.rs:848-862)."""
    import ctypes
    G = pallas_srs
    m = orc.FQ_MODULUS
    g = G.g[:6]
    a = orc.limbs_to_ints(orc.random_scalars(G.scalar, 6, seed=31))
    b = orc.limbs_to_ints(orc.random_scalars(G.scalar, 8, seed=32))
    mont = lambda xs: orc.to_mont(G.scalar, orc.ints_to_limbs(xs))
    bases = ctx.upload_bases(G.cid, g)
    rounds = zk.IpaRounds(ctx, bases, mont(a), mont(b))
    assert len(rounds) == 8
    chals = [3, 5, m - 1]
    gp = np.concatenate([g, np.zeros((2, 8), dtype=np.uint64)])
    l, r, _, _ = rounds.lr()
    assert np.array_equal(zk.jacobian_to_affine(G.cid, l), orc.msm(G.cid, gp[:4], orc.ints_to_limbs(a[4:] + [0, 0])))
    assert np.array_equal(zk.jacobian_to_affine(G.cid, r), orc.msm(G.cid, gp[4:], orc.ints_to_limbs(a[:4])))
    for j, u in enumerate(chals):
        if j:
            rounds.lr()
        rounds.fold(mont([u])[0], mont([pow(u, -1, m)])[0])
    assert np.array_equal(zk.jacobian_to_affine(G.cid, rounds.sg()), orc.msm(G.cid, gp, orc.ints_to_limbs(b_poly_coefficients(chals, m))))
    rounds.close()
    with pytest.raises(ValueError):
        zk.IpaRounds(ctx, bases, mont(a + a + a), mont(b))
    out = ctypes.c_void_p()
    z = np.zeros((16, 4), dtype=np.uint64)
    zp = ctypes.c_void_p(z.ctypes.data)
    assert zk.lib().zk_ipa_begin(ctx._h, bases._h, None, None, 8, ctypes.byref(out)) == -1    # ZK_ERR_INVALID: null argument
    assert zk.lib().zk_ipa_begin(ctx._h, bases._h, zp, zp, 16, ctypes.byref(out)) == -1        # n is not the padded SRS size
    assert zk.lib().zk_ipa_begin(ctx._h, bases._h, zp, zp, 6, ctypes.byref(out)) == -1         # not a power of two
    bases.free()


@pytest.mark.parametrize("name", ["pallas_srs", "vesta_srs"])
def test_direct_base_fold_building_block(ctx, orc, request, name):
    """zk_points_fold_dev (the reference's own per-round fold g'[i] = g[i] + [u] g[h + i], ipa.rs:1002-1006) against the oracle's
    scalar multiplication and addition — full-width and 128-bit (endo-form length) challenges, identity padding on either side."""
    G = request.getfixturevalue(name)
    h = 37
    g = G.g[: 2 * h].copy()
    g[3] = 0                      # identity in the low half
    g[h + 5] = 0                  # identity in the high half (the reference's zero padding, ipa.rs:848-850)
    with ctx.buffers() as bufs:
        d_g, d_out = bufs.put(g), bufs.alloc(g.nbytes // 2)
        for bits in (255, 128, 1):
            u = orc.limbs_to_ints(orc.random_scalars(G.scalar, 1, seed=bits))[0] % (1 << bits) or 1
            ctx.points_fold_dev(G.cid, d_g, h, orc.to_mont(G.scalar, orc.ints_to_limbs([u]))[0], d_out)
            got = ctx.dev_download(d_out, (h, 8))
            for i in (0, 3, 5, 11, h - 1):
                hi = orc.scalar_mul(G.cid, g[h + i], u) if g[h + i].any() else np.zeros(8, dtype=np.uint64)
                want = g[i] if not hi.any() else (hi if not g[i].any() else orc.affine_add(G.cid, g[i], hi))
                assert np.array_equal(got[i], want), (bits, i)
