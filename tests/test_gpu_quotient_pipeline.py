"""SURVEY.md §8f row 3 end to end: one quotient polynomial computed without leaving the device — the prover's sequence
kimchi/src/prover.rs:370-381 (iFFT(n) of the columns) -> circuits/constraints.rs:488-507 (FFT(8n)) -> prover.rs:794-892 (gate constraints
through the expression evaluator into t4 / t8, the permutation part through its kernel) -> prover.rs:905-918 (iFFT(4n) + iFFT(8n),
+ public, division by the vanishing polynomial, + bnd) -> prover.rs:921 (the 7 chunk commitments of t).  ONE upload of the d1
evaluations, ONE download of 7 points; every intermediate the test reads back is compared bit for bit with the oracle's chain
(ntt, expr_eval, perm_quot, divide_by_vanishing, msm)."""
import numpy as np
import pytest

import gate_programs as gp
import proof_systems_b200 as zk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("length,log_n", [(8 * 7 + 3, 3), (64, 3), (8, 3), (5, 3), (4096 * 8, 12), (4096 * 7 + 1, 12), (9, 0)])
def test_divide_by_vanishing_vs_oracle(ctx, orc, length, log_n):
    fid, n = zk.FQ, 1 << log_n
    f = orc.to_mont(fid, orc.random_scalars(fid, length, seed=length))
    want_q, want_r = orc.divide_by_vanishing(fid, f, log_n)
    with ctx.buffers() as bufs:
        d_f, d_q = bufs.put(f), bufs.alloc(max(length - n, 1) * 32)
        zero_rem = ctx.poly_divide_by_vanishing_dev(fid, d_f, length, log_n, d_q)
        assert zero_rem == (not want_r.any())
        if length > n:
            assert np.array_equal(ctx.dev_download(d_q, (length - n, 4)), want_q)


def test_exact_multiple_of_the_vanishing_polynomial_has_zero_remainder(ctx, orc):
    """f = q (x^n - 1) built on the host: the call returns q and reports a zero remainder — the prover's check at prover.rs:910-914"""
    fid, log_n = zk.FP, 10
    n, P = 1 << log_n, orc.FP_MODULUS
    q = orc.limbs_to_ints(orc.random_scalars(fid, 7 * n, seed=5))
    f = [0] * (8 * n)
    for j, c in enumerate(q):
        f[j + n] = (f[j + n] + c) % P
        f[j] = (f[j] - c) % P
    fm, qm = orc.to_mont(fid, orc.ints_to_limbs(f)), orc.to_mont(fid, orc.ints_to_limbs(q))
    with ctx.buffers() as bufs:
        d_f, d_q = bufs.put(fm), bufs.alloc(qm.nbytes)
        assert ctx.poly_divide_by_vanishing_dev(fid, d_f, 8 * n, log_n, d_q) is True
        assert np.array_equal(ctx.dev_download(d_q, (7 * n, 4)), qm)
        fm[3] = orc.to_mont(fid, orc.ints_to_limbs([(f[3] + 1) % P]))[0]                # one coefficient off: remainder != 0
        ctx.dev_upload(d_f, fm)
        assert ctx.poly_divide_by_vanishing_dev(fid, d_f, 8 * n, log_n, d_q) is False


class QuotientCase:
    """The inputs of one quotient polynomial over d1 = 2^log_n (Vesta's scalar field) and the oracle's chain over them: t4, t8, the
    quotient and its 7 chunk commitments on the generators of G."""

    def __init__(self, orc, G, log_n=9):
        fid = self.fid = zk.FP
        self.log_n, self.G = log_n, G
        n, m4, m8 = 1 << log_n, 4 << log_n, 8 << log_n
        rnd = lambda k, seed: orc.to_mont(fid, orc.random_scalars(fid, k, seed=seed))
        self.cols = rnd(16 * n, 11).reshape(16, n, 4)                # w_0..w_14 and z as evaluations over d1
        self.coeff8 = rnd(15 * m8, 12).reshape(15, m8, 4)            # per-index arrays, resident in a real prover (zk_index_cache_section)
        self.sigma8, self.zkpm = rnd(7 * m8, 13).reshape(7, m8, 4), rnd(m8, 14)
        self.gen_sel4, self.pos_sel8 = rnd(m4, 15), rnd(m8, 16)
        self.beta, self.gamma, self.alpha0, self.shifts = rnd(1, 17)[0], rnd(1, 18)[0], rnd(1, 19)[0], rnd(7, 20)
        self.alphas, self.mds = rnd(17, 21), rnd(9, 22).reshape(3, 3, 4)
        self.public, self.bnd = rnd(n, 23), rnd(7 * n, 24)
        # ---------------------------------------------------------------- oracle
        coeffs = np.stack([orc.ntt(fid, self.cols[j], inverse=True) for j in range(16)])
        ev8 = []
        for j in range(16):
            pad = np.zeros((m8, 4), dtype=np.uint64); pad[:n] = coeffs[j]
            ev8.append(orc.ntt(fid, pad))
        gen = gp.generic_gate(gp.Recorder(), self.alphas[:2])
        pos = gp.poseidon_gate(gp.Recorder(), self.alphas[2:], self.mds)
        cols_gen = [(ev8[k], 8) for k in range(15)] + [(self.coeff8[k], 8) for k in range(15)] + [(self.gen_sel4, 4)]
        cols_pos = cols_gen[:30] + [(self.pos_sel8, 8)]
        self.t4 = orc.expr_eval(fid, gen.ops, gen.args, gen.literals, cols_gen, m4)
        t8 = orc.perm_quot(fid, np.stack(ev8[:7]), ev8[15], self.sigma8, self.zkpm, self.beta, self.gamma, self.alpha0, self.shifts)
        self.t8 = orc.expr_eval(fid, pos.ops, pos.args, pos.literals, cols_pos, m8, acc=t8)
        t4c, f = orc.ntt(fid, self.t4, inverse=True), orc.ntt(fid, self.t8, inverse=True)
        add = lambda a, b: orc.to_mont(fid, orc.ints_to_limbs([(x + y) % orc.FP_MODULUS for x, y in zip(orc.limbs_to_ints(orc.from_mont(fid, a)), orc.limbs_to_ints(orc.from_mont(fid, b)))]))
        f[:m4] = add(f[:m4], t4c)
        f[:n] = add(f[:n], self.public)
        quot, rem = orc.divide_by_vanishing(fid, f, log_n)
        assert rem.any()                                        # random columns satisfy no circuit: the prover would stop here
        self.quot = add(quot, self.bnd)
        self.want_comm = [orc.msm(G.cid, G.g[:n], orc.from_mont(fid, self.quot[c * n:(c + 1) * n])) for c in range(7)]

    INPUTS = ("cols", "coeff8", "sigma8", "zkpm", "gen_sel4", "pos_sel8", "public", "bnd")

    def scratch_bytes(self):
        """sizes of the device chain's intermediates: d_ev8, d_t4, d_t8, d_q"""
        n = 1 << self.log_n
        return {"ev8": 16 * 8 * n * 32, "t4": 4 * n * 32, "t8": 8 * n * 32, "q": 7 * n * 32}

    def run_on_device(self, ctx, d, bases, check=None):
        """The prover's sequence on the context's stream over the resident inputs d[name] (INPUTS) and the scratch d["ev8"], d["t4"],
        d["t8"], d["q"]; check(stage) is called after the expression evaluations ("t") and after the division ("q").  Returns the 7
        chunk commitments (affine)."""
        fid, log_n = self.fid, self.log_n
        n, m4, m8 = 1 << log_n, 4 << log_n, 8 << log_n
        ctx.ntt_dev(fid, d["cols"], log_n, batch=16, inverse=True)                           # prover.rs:370-381
        ctx.ntt_dev_oop(fid, d["cols"], n, n, d["ev8"], log_n + 3, batch=16)                  # constraints.rs:488-507
        w8 = [(d["ev8"] + k * m8 * 32, m8, 8) for k in range(15)]
        c8 = [(d["coeff8"] + k * m8 * 32, m8, 8) for k in range(15)]
        gp.generic_gate(zk.ExprProgram(), self.alphas[:2]).evaluations(ctx, fid, w8 + c8 + [(d["gen_sel4"], m4, 4)], m4, 4, d["t4"])   # prover.rs:794-812
        ctx.perm_quotient_dev(fid, log_n + 3, [w[0] for w in w8[:7]], d["ev8"] + 15 * m8 * 32, [d["sigma8"] + k * m8 * 32 for k in range(7)],
                              d["zkpm"], self.beta, self.gamma, self.alpha0, self.shifts, d["t8"])                                 # prover.rs:815-824
        gp.poseidon_gate(zk.ExprProgram(), self.alphas[2:], self.mds).evaluations(ctx, fid, w8 + c8 + [(d["pos_sel8"], m8, 8)], m8, 8, d["t8"],
                                                                                  accumulate=True)                                 # :826-882
        if check:
            check("t")
        ctx.ntt_dev(fid, d["t4"], log_n + 2, inverse=True)                                  # prover.rs:906: t4.interpolate() + t8.interpolate()
        ctx.ntt_dev(fid, d["t8"], log_n + 3, inverse=True)
        ctx.poly_add_dev(fid, d["t8"], d["t4"], m4)
        ctx.poly_add_dev(fid, d["t8"], d["public"], n)                                      # f += &public_poly
        assert ctx.poly_divide_by_vanishing_dev(fid, d["t8"], m8, log_n, d["q"]) is False   # prover.rs:909-914
        ctx.poly_add_dev(fid, d["q"], d["bnd"], 7 * n)                                      # quotient += &bnd
        if check:
            check("q")
        return [zk.jacobian_to_affine(self.G.cid, ctx.msm_dev(bases, d["q"] + c * n * 32, n, mont=True)) for c in range(7)]   # prover.rs:921


def test_one_quotient_polynomial_without_leaving_the_device(ctx, orc, vesta_srs):
    case = QuotientCase(orc, vesta_srs)
    n, m4, m8 = 1 << case.log_n, 4 << case.log_n, 8 << case.log_n
    with ctx.upload_bases(vesta_srs.cid, vesta_srs.g[:n]) as bases, ctx.buffers() as bufs:
        d = {}
        for name in QuotientCase.INPUTS:                        # the ONE upload of per-proof data (cols); the rest is per-index, resident
            d[name] = bufs.put(getattr(case, name))
        for name, nb in case.scratch_bytes().items():
            d[name] = bufs.alloc(nb)

        def check(stage):
            if stage == "t":
                assert np.array_equal(ctx.dev_download(d["t4"], (m4, 4)), case.t4) and np.array_equal(ctx.dev_download(d["t8"], (m8, 4)), case.t8)
            else:
                assert np.array_equal(ctx.dev_download(d["q"], (7 * n, 4)), case.quot)
        got = case.run_on_device(ctx, d, bases, check)
        for c in range(7):
            assert np.array_equal(got[c], case.want_comm[c]), c
