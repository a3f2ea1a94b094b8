"""SURVEY.md §8f row 3, the evaluator: kimchi's expression framework on the device.  zk_expr_eval_dev runs the reference's RPN form
of a constraint (PolishToken, kimchi/src/circuits/expr.rs:819-836) at every point of d4 / d8 with the semantics of
PolishToken::evaluate (:856-940) and the cell indexing of Expr::evaluations (:1938-1990).  Checked bit for bit against the oracle's
own restatement (pinned to the gates' closed forms in tests/test_oracle_expr.py) on the programs of five real gates
(generic: kimchi/src/circuits/polynomials/generic.rs:83-120; poseidon: poseidon.rs:351-436; complete add: complete_add.rs:103-222;
endomul: endosclmul.rs:475-549; endomul scalar: endomul_scalar.rs:174-220), on random programs that use every
opcode, on the permutation quotient written as a program (against the dedicated kernel), and on the reference's failure modes."""
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


def _columns(orc, fid, log_n, seed):
    n, m = 1 << log_n, 8 << log_n
    rnd = lambda k, s: orc.to_mont(fid, orc.random_scalars(fid, k, seed=s))
    return n, m, rnd, [rnd(m, seed + k) for k in range(15)], [rnd(m, seed + 100 + k) for k in range(15)]


@pytest.mark.parametrize("fid,log_n", [(0, 6), (1, 10)])
def test_generic_gate_over_d4(ctx, orc, fid, log_n):
    n, m, rnd, w, co = _columns(orc, fid, log_n, 1)
    sel4, alphas = rnd(4 * n, 900), rnd(2, 901)
    rec = gp.generic_gate(gp.Recorder(), alphas)
    want = orc.expr_eval(fid, rec.ops, rec.args, rec.literals, [(a, 8) for a in w + co] + [(sel4, 4)], 4 * n)
    with ctx.buffers() as r:
        cols = [(r.put(a), m, 8) for a in w + co] + [(r.put(sel4), 4 * n, 4)]
        d_out = r.alloc(4 * n * 32)
        prog = gp.generic_gate(zk.ExprProgram(), alphas)
        prog.evaluations(ctx, fid, cols, 4 * n, 4, d_out)
        assert np.array_equal(ctx.dev_download(d_out, (4 * n, 4)), want)


@pytest.mark.parametrize("fid,log_n", [(1, 6), (0, 11)])
def test_complete_add_gate_over_d4(ctx, orc, fid, log_n):
    """complete_add.rs:103-222: three cached sub-expressions reused across constraints, the literal 1, doublings (Dup + Add)"""
    n, m, rnd, w, co = _columns(orc, fid, log_n, 21)
    sel4, alphas = rnd(4 * n, 960), rnd(7, 961)
    one = orc.to_mont(fid, orc.ints_to_limbs([1]))[0]
    rec = gp.complete_add_gate(gp.Recorder(), alphas, one)
    want = orc.expr_eval(fid, rec.ops, rec.args, rec.literals, [(a, 8) for a in w + co] + [(sel4, 4)], 4 * n)
    with ctx.buffers() as r:
        cols = [(r.put(a), m, 8) for a in w + co] + [(r.put(sel4), 4 * n, 4)]
        d_out = r.alloc(4 * n * 32)
        gp.complete_add_gate(zk.ExprProgram(), alphas, one).evaluations(ctx, fid, cols, 4 * n, 4, d_out)
        assert np.array_equal(ctx.dev_download(d_out, (4 * n, 4)), want)


class _Lit:
    def __init__(self, orc, fid):
        self.orc, self.fid, self.modulus = orc, fid, (orc.FP_MODULUS if fid == orc.FP else orc.FQ_MODULUS)
    def __call__(self, v):
        return self.orc.to_mont(self.fid, self.orc.ints_to_limbs([v % self.modulus]))[0]


@pytest.mark.parametrize("fid,log_n", [(0, 7), (1, 10)])
def test_endomul_scalar_gate_over_d8(ctx, orc, fid, log_n):
    """endomul_scalar.rs:174-220: 11 constraints with rational literals (11/6, -5/2, 2/3), Horner folds from zero, eight cached values"""
    n, m, rnd, w, co = _columns(orc, fid, log_n, 33)
    sel8, alphas = rnd(m, 970), rnd(11, 971)
    rec = gp.endomul_scalar_gate(gp.Recorder(), alphas, _Lit(orc, fid))
    want = orc.expr_eval(fid, rec.ops, rec.args, rec.literals, [(a, 8) for a in w + co] + [(sel8, 8)], m)
    with ctx.buffers() as r:
        cols = [(r.put(a), m, 8) for a in w + co] + [(r.put(sel8), m, 8)]
        d_out = r.alloc(m * 32)
        gp.endomul_scalar_gate(zk.ExprProgram(), alphas, _Lit(orc, fid)).evaluations(ctx, fid, cols, m, 8, d_out)
        assert np.array_equal(ctx.dev_download(d_out, (m, 4)), want)


@pytest.mark.parametrize("fid,log_n", [(1, 5), (0, 11)])
def test_endomul_gate_over_d8(ctx, orc, fid, log_n):
    """endosclmul.rs:475-549: 12 constraints with the endo coefficient as a literal, squares (Pow 2), eight cached sub-expressions and
    three next-row cells (the last 8 rows of d8 wrap to row 0)"""
    n, m, rnd, w, co = _columns(orc, fid, log_n, 44)
    sel8, alphas, endo = rnd(m, 980), rnd(12, 981), rnd(1, 982)[0]
    one = orc.to_mont(fid, orc.ints_to_limbs([1]))[0]
    rec = gp.endomul_gate(gp.Recorder(), alphas, one, endo)
    want = orc.expr_eval(fid, rec.ops, rec.args, rec.literals, [(a, 8) for a in w + co] + [(sel8, 8)], m)
    with ctx.buffers() as r:
        cols = [(r.put(a), m, 8) for a in w + co] + [(r.put(sel8), m, 8)]
        d_out = r.alloc(m * 32)
        gp.endomul_gate(zk.ExprProgram(), alphas, one, endo).evaluations(ctx, fid, cols, m, 8, d_out)
        assert np.array_equal(ctx.dev_download(d_out, (m, 4)), want)


@pytest.mark.parametrize("fid,log_n", [(0, 5), (1, 13)])
def test_poseidon_gate_over_d8_and_accumulation_into_t8(ctx, orc, fid, log_n):
    """2^13 gates -> d8 of 2^16 points: the size of a 2^13-row circuit; the last 8 rows read their `next` cells from row 0"""
    n, m, rnd, w, co = _columns(orc, fid, log_n, 7)
    sel8, alphas, mds, t8 = rnd(m, 950), rnd(15, 951), rnd(9, 952).reshape(3, 3, 4), rnd(m, 953)
    rec = gp.poseidon_gate(gp.Recorder(), alphas, mds)
    cols_h = [(a, 8) for a in w + co] + [(sel8, 8)]
    want = orc.expr_eval(fid, rec.ops, rec.args, rec.literals, cols_h, m)
    want_acc = orc.expr_eval(fid, rec.ops, rec.args, rec.literals, cols_h, m, acc=t8)
    with ctx.buffers() as r:
        cols = [(r.put(a), m, 8) for a in w + co] + [(r.put(sel8), m, 8)]
        d_out, d_t8 = r.alloc(m * 32), r.put(t8)
        prog = gp.poseidon_gate(zk.ExprProgram(), alphas, mds)
        prog.evaluations(ctx, fid, cols, m, 8, d_out)
        assert np.array_equal(ctx.dev_download(d_out, (m, 4)), want)
        prog.evaluations(ctx, fid, cols, m, 8, d_t8, accumulate=True)          # t8 += eval (prover.rs:876-882)
        assert np.array_equal(ctx.dev_download(d_t8, (m, 4)), want_acc)


def _random_program(rng, n_cols, n_lit, length):
    """a valid program that uses every opcode: keeps the stack between 1 and 8 and ends with one value"""
    rec, depth = gp.Recorder(), 0
    lits = []
    while len(rec.ops) < length or depth != 1:
        choices = []
        if depth < 8 and len(rec.ops) < length: choices += ["lit", "cell", "cell", "load"] + (["dup"] if depth else [])
        if depth >= 2: choices += ["add", "mul", "sub"] * (3 if len(rec.ops) >= length else 1)
        if depth >= 1 and len(rec.ops) < length: choices += ["pow", "store"]
        c = choices[rng.integers(len(choices))]
        if c == "lit": rec._t(0, int(rng.integers(n_lit))); depth += 1
        elif c == "cell": rec.cell(int(rng.integers(n_cols)), bool(rng.integers(2))); depth += 1
        elif c == "load":
            if rec.n_cached == 0: continue
            rec.load(int(rng.integers(rec.n_cached))); depth += 1
        elif c == "dup": rec.dup(); depth += 1
        elif c == "pow": rec.pow(int(rng.choice([0, 1, 2, 3, 5, 7, 8, 255])))
        elif c == "store":
            if rec.n_cached >= 90: continue
            rec.store()
        else: getattr(rec, c)(); depth -= 1
    return rec


@pytest.mark.parametrize("seed", range(6))
def test_random_programs_use_every_opcode_and_mixed_domains(ctx, orc, seed):
    """columns over d8, d4, d2 and d1 read from an output domain of d1, d2, d4 or d8 (every legal scale), current and next rows"""
    rng = np.random.default_rng(seed)
    fid, log_n = seed & 1, 5
    n = 1 << log_n
    out_mult = [1, 2, 4, 8][seed % 4]
    mults = [mlt for mlt in (1, 2, 4, 8) if mlt >= out_mult]
    rnd = lambda k, s: orc.to_mont(fid, orc.random_scalars(fid, k, seed=s))
    col_mults = [mults[int(rng.integers(len(mults)))] for _ in range(9)]
    cols_h = [(rnd(cm * n, 40 + k), cm) for k, cm in enumerate(col_mults)]
    lits = rnd(5, 77)
    rec = _random_program(rng, len(cols_h), 5, 120)
    assert set(rec.ops) == set(range(9))
    want = orc.expr_eval(fid, rec.ops, rec.args, lits, cols_h, out_mult * n)
    with ctx.buffers() as r:
        cols = [(r.put(a), a.shape[0], cm) for a, cm in cols_h]
        d_out = r.alloc(out_mult * n * 32)
        ctx.expr_eval_dev(fid, list(zip(rec.ops, rec.args)), lits, cols, out_mult * n, out_mult, d_out)
        assert np.array_equal(ctx.dev_download(d_out, (out_mult * n, 4)), want)


def test_permutation_quotient_as_a_program_equals_the_dedicated_kernel(ctx, orc):
    """perm (permutation.rs:223-357) written as an RPN program over the same resident columns — x_i supplied as a column, the way
    the reference supplies poly_x_d1 evaluated over d8 — equals zk_perm_quotient_dev and the oracle's orc_perm_quot"""
    fid, log_m = zk.FP, 11
    m = 1 << log_m
    rnd = lambda k, s: orc.to_mont(fid, orc.random_scalars(fid, k, seed=s))
    w, sigma = rnd(7 * m, 1).reshape(7, m, 4), rnd(7 * m, 2).reshape(7, m, 4)
    z, zkpm = rnd(m, 3), rnd(m, 4)
    beta, gamma, alpha0, shifts = rnd(1, 5)[0], rnd(1, 6)[0], rnd(1, 7)[0], rnd(7, 8)
    want = orc.perm_quot(fid, w, z, sigma, zkpm, beta, gamma, alpha0, shifts)
    omega = orc.fe_int(fid, orc.root_of_unity(fid, log_m))
    P = orc.FP_MODULUS
    xs, cur = [], 1
    for _ in range(m):
        xs.append(cur); cur = cur * omega % P
    x_col = orc.to_mont(fid, orc.ints_to_limbs(xs))
    Wc, S, Z, ZK, X = 0, 7, 14, 15, 16
    p = zk.ExprProgram()
    p.cell(Z)
    for k in range(7):
        p.cell(Wc + k).literal(gamma).add().literal(beta).literal(shifts[k]).mul().cell(X).mul().add().mul()
    p.cell(Z, next_row=True)
    for k in range(7):
        p.cell(Wc + k).literal(gamma).add().literal(beta).cell(S + k).mul().add().mul()
    p.sub().literal(alpha0).mul().cell(ZK).mul()
    with ctx.buffers() as r:
        cols = [(r.put(w[k]), m, 8) for k in range(7)] + [(r.put(sigma[k]), m, 8) for k in range(7)] + [(r.put(z), m, 8), (r.put(zkpm), m, 8), (r.put(x_col), m, 8)]
        d_out, d_out2 = r.alloc(m * 32), r.alloc(m * 32)
        p.evaluations(ctx, fid, cols, m, 8, d_out)
        got = ctx.dev_download(d_out, (m, 4))
        assert np.array_equal(got, want)
        ctx.perm_quotient_dev(fid, log_m, [c[0] for c in cols[:7]], cols[14][0], [c[0] for c in cols[7:14]], cols[15][0], beta, gamma, alpha0, shifts, d_out2)
        assert np.array_equal(ctx.dev_download(d_out2, (m, 4)), got)


def test_malformed_programs_are_refused_before_anything_runs(ctx, orc):
    one = orc.to_mont(zk.FP, orc.ints_to_limbs([1]))
    with ctx.buffers() as r:
        col = [(r.put(orc.to_mont(zk.FP, orc.random_scalars(zk.FP, 16, seed=3))), 16, 8)]
        d_out = r.alloc(16 * 32)
        E = zk.ExprProgram
        ctx.expr_eval_dev(zk.FP, [(E.CONST, 0), (E.CELL, 0), (E.ADD, 0)], one, col, 16, 8, d_out)
        bad = [([(E.ADD, 0)], "empty stack"),                                   # ExprError::EmptyStack
               ([(E.CONST, 0), (E.CONST, 0)], "leaves 2 values"),               # assert_eq!(stack.len(), 1)
               ([(E.LOAD, 0)], "before it is stored"),
               ([(E.CELL, 5)], "column 5"),
               ([(E.CONST, 3)], "constant 3"),
               ([(99, 0)], "unknown opcode"),
               ([(E.CONST, 0)] * 30 + [(E.ADD, 0)] * 29, "deeper")]
        for toks, msg in bad:
            with pytest.raises(zk.ZkError, match=msg):
                ctx.expr_eval_dev(zk.FP, toks, one, col, 16, 8, d_out)
        with pytest.raises(zk.ZkError, match="not a power-of-two multiple"):   # a column coarser than the output domain
            ctx.expr_eval_dev(zk.FP, [(E.CELL, 0)], one, [(col[0][0], 8, 4)], 16, 8, d_out)
        with pytest.raises(zk.ZkError, match="domain multiple"):
            ctx.expr_eval_dev(zk.FP, [(E.CELL, 0)], one, [(col[0][0], 16, 4)], 16, 8, d_out)
