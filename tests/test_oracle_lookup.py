"""The Python restatement of kimchi's lookup argument (tests/lookup_replay.py) pinned on its own, since the reference holds no vectors
for it: one instance worked out by hand with its sorted columns written out, and random instances checked against the argument's
invariants — the sorted columns are the multiset of the lookups, the padding and the table; neighbouring columns meet in the snake;
agg[0] = 1 and agg[L] = 1 exactly when the columns are a sorting; the smallest row with a missing value is reported."""
import random
from collections import Counter

import pytest

import lookup_replay as lr

P = 0x40000000000000000000000000000000224698FC094CF91B992D30ED00000001      # Fp (Pallas base, Vesta scalar)


def hand_instance():
    """n = 16, zk_rows = 3 (L = 12), m = 1, jc = tic = 0: T1[0 .. 12) = 0 5 7 5 9 0 0 0 0 0 0 0 (a duplicate 5 and zero padding,
    the dummy 0 first), T1[12] = 0; rows 0 .. 3 look up w_0 = 7 5 5 9, rows 4 .. 11 have no lookup (8 padded slots)"""
    n = 16
    w = [[0] * n for _ in range(lr.COLUMNS)]
    w[0][:4] = [7, 5, 5, 9]
    T1 = [0, 5, 7, 5, 9, 0, 0, 0, 0, 0, 0, 0, 0, 11, 12, 13]
    return lr.Instance(P=P, n=n, zk_rows=3, m=1, jc=0, tic=0, dummy=0, T1=T1, w=w, patterns=[[(0, [[(None, 0, False)]])]],
                       row_pattern=[1, 1, 1, 1] + [0] * 8, beta=3, gamma=1000, rand_sorted=[101, 102, 103, 201, 202, 203],
                       rand_agg=[301, 302, 303])


def test_hand_worked_instance():
    """counts: 0 -> 1 + 8 padding, 5 -> 1 + 2, 7 -> 1 + 1, 9 -> 1 + 1; the duplicates 5 and 0 once each.  seq = 0 x9, 5 5 5, 7 7,
    5, 9 9, 0 x7 (24 = (m + 1) L); column 0 = seq[0 .. 12) then seq[12] = 7; column 1 = seq[12 .. 24) then its last value again,
    reversed"""
    inst = hand_instance()
    cols = lr.sorted_columns(inst)
    assert cols[0] == [0] * 9 + [5, 5, 5, 7]
    assert cols[1] == [0] * 8 + [9, 9, 5, 7, 7]
    s = lr.sorted_patched(inst)
    assert s[0] == cols[0] + [101, 102, 103] and s[1] == cols[1] + [201, 202, 203]
    agg, ok = lr.aggregation(inst, s)
    assert ok and agg[0] == 1 and agg[13:] == [301, 302, 303]


def seq_of(cols, L):
    """the pre-snake sequence: each column's first L entries in table order (the m joins and the final duplicate dropped)"""
    return [x for k, c in enumerate(cols) for x in (c[:L] if k % 2 == 0 else c[1:][::-1][:L])]


CASES = [(log_n, zk, m, where) for log_n, zk in ((4, 3), (5, 5), (7, 3), (8, 6)) for m in (1, 3, 4) for where in ("first", "middle", "end", "last")]


@pytest.mark.parametrize("log_n,zk_rows,m,where", CASES)
def test_invariants_of_random_instances(log_n, zk_rows, m, where):
    inst = lr.instance(P, log_n, zk_rows, m, seed=log_n * 100 + zk_rows * 10 + m, dummy_at=where)
    L = inst.L
    cols = lr.sorted_columns(inst)
    assert all(len(c) == L + 1 for c in cols)
    fs = [lr.joint_value(lk, inst.w, i, inst.jc, inst.tic, P) for i in range(L) for lk in lr.row_lookups(inst, i)]
    pad = sum(m - len(lr.row_lookups(inst, i)) for i in range(L))
    assert Counter(seq_of(cols, L)) == Counter(fs + [inst.dummy] * pad + inst.T1[:L])
    for k in range(m):
        if k % 2 == 0:
            assert cols[k][L] == cols[k + 1][L]
        else:
            assert cols[k][0] == cols[k + 1][0]
    s = lr.sorted_patched(inst)
    agg, ok = lr.aggregation(inst, s)
    assert agg[0] == 1 and ok and len(agg) == inst.n and agg[L + 1:] == inst.rand_agg
    # two unequal sorted entries swapped: the product no longer telescopes
    rng = random.Random(log_n + m)
    k = rng.randrange(m + 1)
    pos = [(a, b) for a in range(L + 1) for b in range(a + 1, L + 1) if s[k][a] != s[k][b]]
    if pos:
        a, b = rng.choice(pos)
        bad = [list(c) for c in s]
        bad[k][a], bad[k][b] = bad[k][b], bad[k][a]
        assert not lr.aggregation(inst, bad)[1]


@pytest.mark.parametrize("seed", range(6))
def test_the_smallest_missing_row_is_reported(seed):
    rng = random.Random(seed)
    inst = lr.instance(P, 6, 3, 4, seed=seed)
    rows = [i for i in range(inst.L) if inst.row_pattern[i]]
    a, b = sorted(rng.sample(rows, 2))
    assert lr.break_row(inst, b, rng) and lr.break_row(inst, a, rng)
    with pytest.raises(lr.ValueNotInTable) as e:
        lr.sorted_columns(inst)
    assert e.value.row == a


def test_gates_by_row_and_a_hot_value():
    """by_row: ForeignFieldMul and RangeCheck1 also mark the next row, a later gate's own pattern overrides that; every lookup on
    one table value still sorts"""
    assert lr.by_row(["ForeignFieldMul", "Zero", "RangeCheck1", "Xor16", "Zero"]) == [
        "foreign_field_mul", "foreign_field_mul", "range_check", "xor", None, None]
    inst = lr.instance(P, 7, 3, 4, seed=9, gates=["RangeCheck0"] * 124, hot=True)
    fs = {lr.joint_value(lk, inst.w, i, inst.jc, inst.tic, P) for i in range(inst.L) for lk in lr.row_lookups(inst, i)}
    assert len(fs) == 1
    assert lr.aggregation(inst, lr.sorted_patched(inst))[1]


def test_dummy_missing_while_padding_is_malformed():
    inst = hand_instance()
    inst.T1 = [5, 7, 9, 5, 7, 9, 5, 7, 9, 5, 7, 9, 9, 1, 2, 3]
    with pytest.raises(lr.Malformed):
        lr.sorted_columns(inst)
    inst.row_pattern = [1] * 12                      # every slot used: nothing is padded, the columns form without the dummy
    inst.w[0][:12] = [7, 5, 5, 9, 9, 9, 7, 7, 5, 5, 9, 7]
    cols = lr.sorted_columns(inst)
    assert lr.aggregation(inst, lr.sorted_patched(inst))[1] and len(cols[0]) == 13
