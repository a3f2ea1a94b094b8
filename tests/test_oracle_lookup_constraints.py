"""kimchi's lookup constraints (tests/lookup_constraints.py) against the lookup argument's Python restatement (tests/lookup_replay.py),
on the CPU: the RPN programs equal their closed forms at every row; the VanishesOnZK and Lagrange columns equal their definitions;
every honest instance's constraints divide exactly by Z_H and `verify` accepts its sorted columns; each perturbation fails exactly
the constraints it must; and a consistent misreading of the argument that the replay's own invariants cannot see is caught."""
import importlib.util
import random

import numpy as np
import pytest

import evals_replay as ev
import gate_programs as gp
import lookup_constraints as lc
import lookup_replay as lr
import proof_systems_b200 as zk
import test_oracle_lookup


def lit_of(orc, fid):
    return lambda v: ev.mont(orc, fid, [v])[0]


def entries_over_d8(orc, fid, inst, cols1, cfg):
    """every entry's d8 evaluations for the instance's d1 columns, and whether each divides by Z_H"""
    log_n = inst.n.bit_length() - 1
    cols8 = [lc.to_d8(orc, fid, c) for c in cols1] + lc.env_d8(orc, fid, log_n, inst.zk_rows)
    evals = lc.oracle_evals(orc, fid, lc.constraints(gp.Recorder, cfg), cols8)
    return evals, [lc.divides(orc, fid, e, log_n) for e in evals]


# ---------------------------------------------------------------------------------------------------------------- programs
@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("m", [1, 2, 3, 4])
def test_programs_equal_the_closed_forms_at_every_row(orc, fid, m):
    """random columns over d1 (selectors and environment columns too), the instance's patterns with the synthetic next-row lookup"""
    P, log_n = orc.MODULUS[fid], 5
    n = 1 << log_n
    inst = lr.instance(P, log_n, 3, m, seed=10 * fid + m, tic="kimchi")
    cfg = lc.of_instance(inst, lit_of(orc, fid))
    assert any(nxt for pat in cfg.patterns for _, entries in pat for e in entries for _, _, nxt in e)
    rng = random.Random(fid * 10 + m)
    cols = [[rng.randrange(P) for _ in range(n)] for _ in range(cfg.n_columns)]
    progs = lc.constraints(gp.Recorder, cfg)
    assert len(progs) == len(lc.ENTRIES)
    got = [ev.ints(orc, fid, orc.expr_eval(fid, p.ops, p.args, p.literals, [(ev.mont(orc, fid, c), 1) for c in cols], n)) for p in progs]
    for i in range(n):
        assert [g[i] for g in got] == lc.closed_form(cfg, cols, i), i
    assert all(got[3 + k] == [0] * n for k in range(m, 4))
    # the library's builder records the same program
    for rec, prog in zip(progs, lc.constraints(zk.ExprProgram, cfg)):
        assert [(o, a) for o, a in zip(rec.ops, rec.args)] == prog.tokens
        assert np.array_equal(np.array(rec.literals), np.array(prog.constants))


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,zk_rows", [(3, 3), (4, 5), (5, 3), (4, 14)])
def test_environment_columns_equal_their_definitions(orc, fid, log_n, zk_rows):
    """the coefficient forms through the oracle's FFT(8n) against the pointwise definitions, including the points x = w^i of d1"""
    P, n = orc.MODULUS[fid], 1 << log_n
    w, w8 = ev.omega(orc, fid, log_n), ev.omega(orc, fid, log_n + 3)
    got = [ev.ints(orc, fid, c) for c in lc.env_d8(orc, fid, log_n, zk_rows)]
    assert got == lc.env_d8_pointwise(P, n, zk_rows, w, w8)
    L = n - zk_rows - 1
    zkv, l0, lL = got
    assert [r for r in range(n) if zkv[8 * r] == 0] == list(range(L, n))
    assert l0[0] == n and lL[8 * L] == n * pow(w, n - L, P) % P
    assert all(l0[8 * r] == 0 for r in range(1, n)) and all(lL[8 * r] == 0 for r in range(n) if r != L)


# ---------------------------------------------------------------------------------------------------------------- honest instances
# the shapes of test_gpu_lookup.CASES with m <= 4, kept small
CASES = [(4, 3, 1, "first"), (4, 5, 3, "middle"), (4, 14, 4, "last"), (6, 62, 3, "end"), (7, 5, 4, "end"), (8, 3, 2, "middle"),
         (8, 5, 4, "first")]


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,zk_rows,m,where", CASES)
def test_honest_instances_divide_by_the_vanishing_polynomial(orc, fid, log_n, zk_rows, m, where):
    P = orc.MODULUS[fid]
    inst = lr.instance(P, log_n, zk_rows, m, seed=300 + 10 * fid + log_n + m, dummy_at=where, tic="kimchi")
    s = lr.sorted_patched(inst)
    agg, ok = lr.aggregation(inst, s)
    assert ok and lc.verify(inst, s) is None
    cfg = lc.of_instance(inst, lit_of(orc, fid))
    evals, div = entries_over_d8(orc, fid, inst, lc.instance_columns(inst, s, agg), cfg)
    assert all(div), [e for e, d in zip(lc.ENTRIES, div) if not d]
    assert all(e.any() for e in evals[:3 + m])            # zero on d1, not everywhere


def test_a_random_table_id_combiner_breaks_the_constraints(orc):
    """the constraints compute table_id_combiner = jc^max_joint_size themselves: a table and lookups combined with another
    combiner sort and aggregate consistently, and still fail the aggregation"""
    fid, log_n, zk_rows, m = 0, 5, 3, 3
    P = orc.MODULUS[fid]
    inst = lr.instance(P, log_n, zk_rows, m, seed=5)
    assert inst.tic != lc.of_instance(inst, None).table_id_combiner
    s = lr.sorted_patched(inst)
    agg, ok = lr.aggregation(inst, s)
    assert ok and lc.verify(inst, s) is None
    _, div = entries_over_d8(orc, fid, inst, lc.instance_columns(inst, s, agg), lc.of_instance(inst, lit_of(orc, fid)))
    assert not div[0] and all(div[1:])


# ---------------------------------------------------------------------------------------------------------------- negative cases
@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("kind", list(lc.NEGATIVE))
def test_each_perturbation_fails_exactly_its_constraints(orc, fid, kind):
    P, log_n, zk_rows, m = orc.MODULUS[fid], 6, 3, 4
    inst = lr.instance(P, log_n, zk_rows, m, seed=400 + fid, tic="kimchi")
    s0 = lr.sorted_patched(inst)
    s, row = lc.perturb(inst, s0, kind)
    agg, _ = lr.aggregation(inst, s)
    if kind == "agg scaled":
        agg = [lc.SCALE * a % P for a in agg]
    must_fail, verdict = lc.NEGATIVE[kind]
    assert agg[inst.L] != 1 and lc.verify(inst, s) == verdict
    cfg = lc.of_instance(inst, lit_of(orc, fid))
    cols = lc.instance_columns(inst, s, agg)
    _, div = entries_over_d8(orc, fid, inst, cols, cfg)
    assert {e for e, d in zip(lc.ENTRIES, div) if not d} == must_fail
    # over d1 the recurrence is nonzero at the zero denominator's row alone (the environment columns as 0 / 1 indicators)
    n, L = inst.n, inst.L
    cols = cols + [[int(r < L) for r in range(n)], [int(r == 0) for r in range(n)], [int(r == L) for r in range(n)]]
    bad = [r for r in range(n) if lc.closed_form(cfg, cols, r)[0]]
    assert bad == ([] if row is None else [row])


# ---------------------------------------------------------------------------------------------------------------- a mutation
def misread_next_row_cells():
    """lookup_replay with one consistent misreading: a lookup's next-row cell read at the current row, in the generator and in
    joint_value, so the sorted columns and the aggregation both follow it"""
    src = open(lr.__file__).read()
    for old in ("w[col][i + int(nxt)]", "w[col][i + int(nx)]"):
        assert src.count(old) == 1, old
        src = src.replace(old, "w[col][i]")
    spec = importlib.util.spec_from_loader("lookup_replay_misread", loader=None)
    mod = importlib.util.module_from_spec(spec)
    exec(compile(src, lr.__file__, "exec"), mod.__dict__)
    return mod


def test_a_consistent_misreading_passes_the_replay_invariants_and_fails_the_constraints(orc, monkeypatch):
    mutant = misread_next_row_cells()
    monkeypatch.setattr(test_oracle_lookup, "lr", mutant)
    test_oracle_lookup.test_hand_worked_instance()
    for case in test_oracle_lookup.CASES[::5]:
        test_oracle_lookup.test_invariants_of_random_instances(*case)
    test_oracle_lookup.test_gates_by_row_and_a_hot_value()
    monkeypatch.undo()

    fid, log_n, zk_rows, m = 1, 6, 3, 3
    P = orc.MODULUS[fid]
    inst = mutant.instance(P, log_n, zk_rows, m, seed=500, tic="kimchi")
    s = mutant.sorted_patched(inst)
    agg, ok = mutant.aggregation(inst, s)
    assert ok
    cfg = lc.of_instance(inst, lit_of(orc, fid))
    cols = lc.instance_columns(inst, s, agg)
    _, div = entries_over_d8(orc, fid, inst, cols, cfg)
    assert not div[0] and all(div[1:])
    assert lc.verify(inst, s) == "multiset"
    # the recurrence fails on the rows of the pattern with a next-row cell, and only there
    n, L = inst.n, inst.L
    syn = inst.names.index("synthetic") + 1
    cols = cols + [[int(r < L) for r in range(n)], [0] * n, [0] * n]
    assert [r for r in range(n) if lc.closed_form(cfg, cols, r)[0]] == [r for r in range(L) if inst.row_pattern[r] == syn]
