"""kimchi's lookup argument restated with Python integers: the joint table (prover.rs:500-568, combine_table_entry), `sorted`
(lookup/constraints.rs:90-201), `zk_patch` (:35-48) and `aggregation` (:233-338), plus generators of instances for them.  Field
elements are canonical ints; `evals_replay.mont` / `ints` convert from / to the library's Montgomery limbs.

A joint lookup is (table_id, entries) as proof_systems_b200.LookupSpec takes it: table_id an int (LookupTableID::Constant) or
("witness", column); entries a list of linear combinations, each a list of (coeff or None for one, column, next_row)."""
import random

import evals_replay as ev

COLUMNS = 15
XOR_TABLE_ID, RANGE_CHECK_TABLE_ID = 0, 1


class ValueNotInTable(Exception):
    """ProverError::ValueNotInTable(row)"""

    def __init__(self, row):
        super().__init__(row)
        self.row = row


class Malformed(Exception):
    """the reference's sorted columns come out with the wrong lengths (or it panics): the dummy is missing from the table"""


def combine(entries, jc, tic, tid, P):
    """combine_table_entry: Horner over the reversed entries, plus tic * table id"""
    acc = 0
    for x in reversed(entries):
        acc = (acc * jc + x) % P
    return (acc + tic * tid) % P


def joint_table(cols8, jc, tic, P, tid8=None, runtime8=None):
    """the joint lookup table over d8: combine_table_entry at every point, column 1 plus the runtime table if there is one"""
    out = []
    for i in range(len(cols8[0])):
        row = [(c[i] + runtime8[i]) % P if k == 1 and runtime8 is not None else c[i] for k, c in enumerate(cols8)]
        out.append(combine(row, jc, tic, 0 if tid8 is None else tid8[i], P))
    return out


def kimchi_lookups(pattern):
    """LookupPattern::lookups() (lookups.rs:448-528)"""
    one = lambda col: [(None, col, False)]
    if pattern == "xor":
        return [(XOR_TABLE_ID, [one(3 + i), one(7 + i), one(11 + i)]) for i in range(4)]
    if pattern == "lookup":
        return [(("witness", 0), [one(2 * i + 1), one(2 * i + 2)]) for i in range(3)]
    if pattern == "range_check":
        return [(RANGE_CHECK_TABLE_ID, [one(c)]) for c in range(3, 7)]
    if pattern == "foreign_field_mul":
        return [(RANGE_CHECK_TABLE_ID, [one(c)]) for c in range(7, 11)]
    raise ValueError(pattern)


def from_gate(gate, nxt):
    """LookupPattern::from_gate (lookups.rs:541-553)"""
    if gate == "Lookup" and not nxt:
        return "lookup"
    if (gate == "RangeCheck0" and not nxt) or gate == "RangeCheck1" or (gate == "Rot64" and not nxt):
        return "range_check"
    if gate == "ForeignFieldMul":
        return "foreign_field_mul"
    if gate == "Xor16" and not nxt:
        return "xor"
    return None


def by_row(gates):
    """LookupInfo::by_row (lookups.rs:286-299) as pattern names per row (None: no lookups); gates.len() + 1 entries"""
    kinds = [None] * (len(gates) + 1)
    for i, g in enumerate(gates):
        if from_gate(g, False):
            kinds[i] = from_gate(g, False)
        if from_gate(g, True):
            kinds[i + 1] = from_gate(g, True)
    return kinds


def joint_value(lookup, w, i, jc, tic, P):
    """JointLookupSpec::evaluate at row i"""
    table_id, entries = lookup
    vals = [sum((1 if c is None else c) * w[col][i + int(nxt)] for c, col, nxt in entry) % P for entry in entries]
    tid = w[table_id[1]][i] if isinstance(table_id, tuple) else table_id % P      # i32_to_field: -F(|id|) for a negative id
    return combine(vals, jc, tic, tid, P)


def row_lookups(inst, i):
    p = inst.row_pattern[i]
    return inst.patterns[p - 1] if p else []


def sorted_columns(inst):
    """lookup::constraints::sorted: the m + 1 columns of L + 1 entries each (snake-shaped).  Raises ValueNotInTable(row) or
    Malformed like the reference's Err / malformed result."""
    P, m, L, T1 = inst.P, inst.m, inst.L, inst.T1
    counts = {}
    for t in T1[:L]:
        counts.setdefault(t, 1)
    for i in range(L):
        spec = row_lookups(inst, i)
        for lk in spec:
            f = joint_value(lk, inst.w, i, inst.jc, inst.tic, P)
            if f not in counts:
                raise ValueNotInTable(i)
            counts[f] += 1
        counts[inst.dummy] = counts.get(inst.dummy, 0) + m - len(spec)
    cols = [[] for _ in range(m + 1)]
    i = 0
    for t in T1[:L]:
        c = counts[t]
        counts[t] = 1
        for j in range(c):
            if (i + j) // L > m:
                raise Malformed()
            cols[(i + j) // L].append(t)
        i += c
    if i != (m + 1) * L:
        raise Malformed()
    for k in range(m):
        cols[k].append(cols[k + 1][0])
    cols[m].append(cols[m][-1])
    for k in range(1, m + 1, 2):
        cols[k].reverse()
    return cols


def zk_patch(e, n, zk_rows, rand):
    """lookup::constraints::zk_patch: zeros up to n - zk_rows, then the zk_rows random values"""
    assert len(e) <= n - zk_rows and len(rand) == zk_rows
    return list(e) + [0] * (n - zk_rows - len(e)) + list(rand)


def sorted_patched(inst):
    """the prover's sorted columns: `sorted`, then zk_patch per column with the column's zk_rows draws"""
    cols = sorted_columns(inst)
    z = inst.zk_rows
    return [zk_patch(c, inst.n, z, inst.rand_sorted[k * z:(k + 1) * z]) for k, c in enumerate(cols)]


def aggregation(inst, s):
    """lookup::constraints::aggregation over the patched sorted columns s -> (agg over d1, agg[L] == 1)"""
    P, m, L = inst.P, inst.m, inst.L
    beta, gamma = inst.beta, inst.gamma
    beta1 = (1 + beta) % P
    gb1 = gamma * beta1 % P
    den = []
    for row in range(L):
        acc = 1
        for k, col in enumerate(s):
            a, b = (row, row + 1) if k % 2 == 0 else (row + 1, row)
            acc = acc * (gb1 + col[a] + beta * col[b]) % P
        den.append(acc)
    agg = [1] + ev.batch_inversion_and_mul(den, 1, P)
    base = pow(beta1, m, P)
    for i in range(L):
        spec = row_lookups(inst, i)
        f = base * pow(gamma + inst.dummy, m - len(spec), P) % P
        for lk in spec:
            f = f * (gamma + joint_value(lk, inst.w, i, inst.jc, inst.tic, P)) % P
        t = (gb1 + inst.T1[i] + beta * inst.T1[i + 1]) % P
        agg[i + 1] = agg[i + 1] * f % P * t % P * agg[i] % P
    res = zk_patch(agg, inst.n, inst.zk_rows, inst.rand_agg)
    return res, res[L] == 1


# ------------------------------------------------------------------------------------------------------------ instances
class Instance:
    """one call's inputs: the joint table T1 over d1 (n values), the 15 witness columns, the patterns and each lookup row's pattern
    (0: none, p + 1: patterns[p]), m, the scalars and the random values"""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    @property
    def L(self):
        return self.n - self.zk_rows - 1

    def copy(self):
        c = Instance(**self.__dict__)
        c.w = [list(col) for col in self.w]
        c.T1 = list(self.T1)
        c.row_pattern = list(self.row_pattern)
        return c


SYNTHETIC_ID = -5


def synthetic_lookups(coeff):
    """a pattern kimchi does not have: one lookup of table -5 whose first entry is coeff * w_13[next row] + w_14 and second w_12"""
    return [(SYNTHETIC_ID, [[(coeff, 13, True), (None, 14, False)], [(None, 12, False)]])]


def make_tables(rng, P, n_rows):
    """table rows (table id, [c0, c1, c2]) without the all-zero row of id 0 (the dummy), duplicates included"""
    rows = []
    while len(rows) < n_rows:
        kind = rng.randrange(5)
        if kind == 0:
            a, b = rng.randrange(16), rng.randrange(1, 16)
            rows.append((XOR_TABLE_ID, [a, b, a ^ b]))
        elif kind == 1:
            rows.append((RANGE_CHECK_TABLE_ID, [rng.randrange(1 << 12), 0, 0]))
        elif kind in (2, 3):
            rows.append((kind, [rng.randrange(P), rng.randrange(P), 0]))
        else:
            rows.append((SYNTHETIC_ID, [rng.randrange(P), rng.randrange(P), 0]))
        if rng.random() < 0.1:
            rows.append(rows[-1])                   # a duplicate table row
    return rows[:n_rows]


def instance(P, log_n, zk_rows, m, seed, dummy_at="end", jc=None, empty_frac=0.3, gates=None, hot=False, table=None):
    """A valid instance: every lookup of rows < L hits the table.  The table has L rows: random rows of the XOR, range-check, two
    width-2 (Lookup-pattern) and synthetic tables, duplicates, and the dummy row (0, 0, 0) of id 0 placed at the start, the middle
    or the end (dummy_at: "first", "middle", "end" = zero padding at the end, "last" = exactly one dummy row, at L - 1).
    T1[L] = T1[L - 1] (kimchi pads past L with the dummy too) and random beyond.  gates: a gate list for by_row, else random gates
    drawn from those whose patterns fit m.  hot: every lookup hits one table row.  table: the L table rows to use instead."""
    rng = random.Random(seed)
    n = 1 << log_n
    L = n - zk_rows - 1
    assert L >= 1
    jc = rng.randrange(P) if jc is None else jc
    tic = rng.randrange(P)
    coeff = rng.randrange(2, P)
    names = [p for p, k in (("xor", 4), ("lookup", 3), ("range_check", 4), ("foreign_field_mul", 4)) if k <= m] + ["synthetic"]
    patterns = [kimchi_lookups(p) if p != "synthetic" else synthetic_lookups(coeff) for p in names]
    pidx = {p: k + 1 for k, p in enumerate(names)}
    n_real = L - 1 if dummy_at == "last" else L - max(1, L // 4)
    real = make_tables(rng, P, n_real)
    dummy_row = (XOR_TABLE_ID, [0, 0, 0])
    n_dummy = L - len(real)
    if table is not None:
        assert len(table) == L
        rows = list(table)
    elif dummy_at == "first":
        rows = [dummy_row] * n_dummy + real
    elif dummy_at == "middle":
        h = len(real) // 2
        rows = real[:h] + [dummy_row] * n_dummy + real[h:]
    else:
        rows = real + [dummy_row] * n_dummy
    T1 = [combine(c, jc, tic, tid % P, P) for tid, c in rows]
    T1 += [T1[L - 1]] + [rng.randrange(P) for _ in range(n - L - 1)]
    dummy = combine([0, 0, 0], jc, tic, 0, P)
    # row patterns: by_row over the gates, or a random choice per row
    if gates is not None:
        kinds = by_row(gates)
        row_pattern = [pidx[kinds[i]] if i < len(kinds) and kinds[i] else 0 for i in range(L)]
    else:
        row_pattern = [0 if rng.random() < empty_frac else rng.randrange(1, len(names) + 1) for _ in range(L)]
    # witness: random, then for rows L - 1 down to 0 the cells that make each lookup hit a table row (a next-row cell is final by then)
    w = [[rng.randrange(P) for _ in range(n)] for _ in range(COLUMNS)]
    by_id = {}
    for r, (tid, c) in enumerate(rows):
        by_id.setdefault(tid, []).append(r)
    hot_row = {}
    for i in reversed(range(L)):
        p = row_pattern[i]
        if not p:
            continue
        spec = patterns[p - 1]
        wid = None
        if isinstance(spec[0][0], tuple):
            cands = [t for t in (2, 3) if t in by_id]
            wid = rng.choice(cands) if cands else None
            w[spec[0][0][1]][i] = wid or 0
        if any((wid if isinstance(t, tuple) else t) not in by_id for t, _ in spec):
            row_pattern[i] = 0                                      # no table row this pattern could hit
            continue
        for table_id, entries in spec:
            tid = wid if isinstance(table_id, tuple) else table_id
            r = hot_row.setdefault(tid, rng.choice(by_id[tid])) if hot else rng.choice(by_id[tid])
            target = rows[r][1]
            for e, entry in enumerate(entries):
                *others, (c_last, col_last, nxt_last) = entry
                assert not nxt_last
                acc = sum((1 if c is None else c) * w[col][i + int(nx)] for c, col, nx in others) % P
                cl = 1 if c_last is None else c_last
                w[col_last][i] = (target[e] - acc) * pow(cl, P - 2, P) % P
    return Instance(P=P, n=n, zk_rows=zk_rows, m=m, jc=jc, tic=tic, dummy=dummy, T1=T1, w=w, patterns=patterns, names=names,
                    row_pattern=row_pattern, beta=rng.randrange(P), gamma=rng.randrange(P),
                    rand_sorted=[rng.randrange(P) for _ in range((m + 1) * zk_rows)], rand_agg=[rng.randrange(P) for _ in range(zk_rows)])


def break_row(inst, i, rng):
    """row i gets a lookup whose value is not in the table (a fresh random cell under its first lookup); returns False if the row
    has no lookup"""
    spec = row_lookups(inst, i)
    if not spec:
        return False
    col = spec[0][1][0][-1][1]
    while True:
        inst.w[col][i] = rng.randrange(inst.P)
        if joint_value(spec[0], inst.w, i, inst.jc, inst.tic, inst.P) not in set(inst.T1[:inst.L]):
            return True


def zero_denominator(inst, s, row, rng):
    """sorted column 0 made to vanish one factor of den_row: s_0[row] = -(gamma (1 + beta) + beta s_0[row + 1])"""
    P = inst.P
    gb1 = inst.gamma * (1 + inst.beta) % P
    s[0][row] = (-(gb1 + inst.beta * s[0][row + 1])) % P
