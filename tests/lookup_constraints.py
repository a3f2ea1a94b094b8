"""kimchi's lookup constraints restated for the evaluator: the RPN program of every entry of `lookup::constraints::constraints(
configuration, false)` (kimchi/src/circuits/lookup/constraints.rs:378-682; "false" is the generate_feature_flags value the prover
uses, prover.rs:877), their closed forms with Python integers, the two kinds of environment column they read over d8, and the
reference's own post-condition on the sorted columns, `verify` (:690-796).

The prover scales entry k by its own alpha power and adds it into t8 (prover.rs:874-902); for honest inputs every entry vanishes
on d1, so each divides exactly by Z_H.  The entries, in order (ENTRIES):

  aggregation   VanishesOnZK * (agg(xw) * den - agg(x) * f * t)
  initial       l_0 * (agg - 1)
  final         l_L * (agg - 1),  L = n - zk_rows - 1 (RowOffset { zk_rows: true, offset: -1 })
  compat i      l_L (i even) or l_0 (i odd) times (sorted_i - sorted_(i+1)), for i < m; the literal zero for m <= i < 4, which
                keeps the alpha positions of the runtime-table entries fixed

with f = (1 - sum_p sel_p) * pad(0) + sum_p sel_p * pad(|p|) * prod_(j in p) (gamma + joint_j), pad(k) = (gamma + dummy)^(m - k) *
(1 + beta)^m, t = gamma (1 + beta) + T(x) + beta T(xw), den = prod_(i <= m) (gamma (1 + beta) + s_i(x) + beta s_i(xw)) with x and xw
swapped on odd i.  joint_j is JointLookupSpec::evaluate: Horner in the joint combiner jc over the reversed entries, plus
table_id_combiner * table id, where table_id_combiner = jc^max_joint_size is computed inside the expression, as the reference does.
The dummy lookup has no entries and table id 0.

Column order (what cell() indices refer to): 15 witness | one selector per pattern (LookupKindIndex) | LookupTable | m + 1
LookupSorted | LookupAggreg | VanishesOnZeroKnowledgeAndPreviousRows | UnnormalizedLagrangeBasis(0) | UnnormalizedLagrangeBasis(L).

Degree bound: the largest term is VanishesOnZK * agg * sel * prod_(j <= m) (gamma + joint_j) * T, of degree zk_rows + 1 + (m + 3)(n - 1)
for m <= 4 (kimchi's max_per_row); that is below 8n for every zk_rows < n, so evaluations over d8 hold each entry exactly."""
import numpy as np

import evals_replay as ev
import lookup_replay as lr

COLUMNS = 15
ENTRIES = ["aggregation", "initial", "final", "compat 0", "compat 1", "compat 2", "compat 3"]


class Config:
    """one configuration of the constraints: the field modulus, m = max_per_row (1 .. 4), the patterns (lookup_replay's joint-lookup
    lists, one selector column each), the challenges as canonical ints, and lit(v): the Montgomery limbs of the canonical int v"""

    def __init__(self, P, m, patterns, beta, gamma, jc, lit):
        assert 1 <= m <= 4 and all(len(p) <= m for p in patterns)
        self.P, self.m, self.patterns, self.beta, self.gamma, self.jc, self.lit = P, m, patterns, beta, gamma, jc, lit
        self.max_joint_size = lr.max_joint_size(patterns)
        self.SEL = COLUMNS
        self.TABLE = self.SEL + len(patterns)
        self.SORTED = self.TABLE + 1
        self.AGG = self.SORTED + m + 1
        self.ZKV = self.AGG + 1
        self.L0 = self.ZKV + 1
        self.LL = self.L0 + 1
        self.n_columns = self.LL + 1

    @property
    def table_id_combiner(self):
        return pow(self.jc, self.max_joint_size, self.P)


def of_instance(inst, lit, patterns=None):
    """the configuration of a lookup_replay instance (its patterns unless others are given)"""
    return Config(inst.P, inst.m, inst.patterns if patterns is None else patterns, inst.beta, inst.gamma, inst.jc, lit)


# ------------------------------------------------------------------------------------------------------------ the programs
def constraints(new_program, cfg):
    """the RPN program of every entry of ENTRIES, each built by new_program() (tests/gate_programs.Recorder or
    proof_systems_b200.ExprProgram: any object with ExprProgram's methods)"""
    P, m = cfg.P, cfg.m
    lit = lambda p, v: p.literal(cfg.lit(v % P))

    def gammabeta1(p):                                  # gamma * (beta + 1)
        lit(p, cfg.gamma); lit(p, cfg.beta); lit(p, 1); p.add().mul()

    def table_id_combiner(p):                           # (1 .. max_joint_size).fold(jc, |acc, _| acc * jc)
        lit(p, cfg.jc)
        for _ in range(1, cfg.max_joint_size):
            lit(p, cfg.jc); p.mul()

    def joint(p, table_id, entries):                    # JointLookupSpec::evaluate (lookups.rs:372-408, tables/mod.rs:167-182)
        lit(p, 0)
        for entry in reversed(entries):
            lit(p, cfg.jc); p.mul()                     # joint_combiner * acc + x
            lit(p, 0)                                   # SingleLookup::evaluate: fold(zero, acc + eval(pos) * coeff)
            for c, col, nxt in entry:
                p.cell(col, nxt); lit(p, 1 if c is None else c); p.mul().add()
            p.add()
        table_id_combiner(p)
        if isinstance(table_id, tuple):                 # LookupTableID::WitnessColumn, read at the current row
            p.cell(table_id[1])
        else:
            lit(p, table_id)                            # i32_to_field
        p.mul().add()

    def dummy_padding(p, spec_len):                     # (gamma + dummy)^(m - spec_len) * (1 + beta)^m
        lit(p, 1)
        for _ in range(spec_len, m):
            lit(p, cfg.gamma)
            joint(p, 0, [])                             # the dummy lookup: no entries, table id 0
            p.add().mul()
        lit(p, 1); lit(p, cfg.beta); p.add()            # beta1_per_row: beta1 times beta1, m - 1 times
        for _ in range(1, m):
            lit(p, 1); lit(p, cfg.beta); p.add().mul()
        p.mul()

    def f_term(p, spec):
        dummy_padding(p, len(spec))
        for table_id, entries in spec:
            lit(p, cfg.gamma); joint(p, table_id, entries); p.add().mul()

    def numerator(p):
        lit(p, 1)                                       # non_lookup_indicator = 1 - sum of the selectors
        lit(p, 0)
        for k in range(len(cfg.patterns)):
            p.cell(cfg.SEL + k).add()
        p.sub()
        f_term(p, [])
        p.mul()
        for k, spec in enumerate(cfg.patterns):
            p.cell(cfg.SEL + k); f_term(p, spec); p.mul().add()
        gammabeta1(p)                                   # t
        p.cell(cfg.TABLE).add()
        lit(p, cfg.beta); p.cell(cfg.TABLE, True).mul().add()
        p.mul()

    def denominator(p):
        lit(p, 1)
        for i in range(m + 1):
            s1, s2 = (False, True) if i % 2 == 0 else (True, False)
            gammabeta1(p)
            p.cell(cfg.SORTED + i, s1).add()
            lit(p, cfg.beta); p.cell(cfg.SORTED + i, s2).mul().add()
            p.mul()

    def aggregation(p):
        p.cell(cfg.ZKV)
        p.cell(cfg.AGG, True); denominator(p); p.mul()
        p.cell(cfg.AGG); numerator(p); p.mul()
        p.sub().mul()

    def boundary(p, lagrange, build):
        p.cell(lagrange); build(); p.mul()

    progs = []
    p = new_program(); aggregation(p); progs.append(p)
    for lag in (cfg.L0, cfg.LL):
        p = new_program(); boundary(p, lag, lambda: (p.cell(cfg.AGG), lit(p, 1), p.sub())); progs.append(p)
    for i in range(4):
        p = new_program()
        if i < m:
            boundary(p, cfg.LL if i % 2 == 0 else cfg.L0, lambda: (p.cell(cfg.SORTED + i), p.cell(cfg.SORTED + i + 1), p.sub()))
        else:
            lit(p, 0)
        progs.append(p)
    return progs


# ------------------------------------------------------------------------------------------------------------ closed forms
def joint_value(lookup, w, row, nxt_row, jc, tic, P):
    """JointLookupSpec::evaluate at one row, next-row cells read at nxt_row"""
    table_id, entries = lookup
    acc = 0
    for entry in reversed(entries):
        acc = acc * jc + sum((1 if c is None else c) * w[col][nxt_row if nxt else row] for c, col, nxt in entry)
    tid = w[table_id[1]][row] if isinstance(table_id, tuple) else table_id
    return (acc + tic * tid) % P


def closed_form(cfg, cols, i):
    """the value of every entry of ENTRIES at row i of columns cols given over d1 (lists of canonical ints, the program's order)"""
    P, m, beta, gamma = cfg.P, cfg.m, cfg.beta, cfg.gamma
    n = len(cols[0])
    j = (i + 1) % n
    tic = cfg.table_id_combiner
    w = cols[:COLUMNS]
    gb1 = gamma * (1 + beta)
    dummy = 0                                           # JointLookup { entry: [], table_id: 0 }

    def f_term(spec):
        v = pow(gamma + dummy, m - len(spec), P) * pow(1 + beta, m, P)
        for lk in spec:
            v = v * (gamma + joint_value(lk, w, i, j, cfg.jc, tic, P)) % P
        return v

    sel = [cols[cfg.SEL + k][i] for k in range(len(cfg.patterns))]
    f = (1 - sum(sel)) * f_term([]) + sum(s * f_term(spec) for s, spec in zip(sel, cfg.patterns))
    T = cols[cfg.TABLE]
    t = gb1 + T[i] + beta * T[j]
    den = 1
    for k in range(m + 1):
        s = cols[cfg.SORTED + k]
        a, b = (i, j) if k % 2 == 0 else (j, i)
        den = den * (gb1 + s[a] + beta * s[b]) % P
    agg, l0, lL = cols[cfg.AGG], cols[cfg.L0][i], cols[cfg.LL][i]
    out = [cols[cfg.ZKV][i] * (agg[j] * den - agg[i] * f * t), l0 * (agg[i] - 1), lL * (agg[i] - 1)]
    for k in range(4):
        s = lambda q: cols[cfg.SORTED + q][i]
        out.append((lL if k % 2 == 0 else l0) * (s(k) - s(k + 1)) if k < m else 0)
    return [v % P for v in out]


# ------------------------------------------------------------------------------------------------------------ environment columns
def vanishing_zk_coeffs(P, w, n, zk_rows):
    """vanishes_on_last_n_rows(d1, zk_rows + 1) (permutation.rs:93-106): prod_(n - zk_rows - 1 <= k < n) (x - w^k), coefficients"""
    c = [1]
    for k in range(n - zk_rows - 1, n):
        r = pow(w, k, P)
        c = [((c[e - 1] if e else 0) - r * (c[e] if e < len(c) else 0)) % P for e in range(len(c) + 1)]
    return c


def lagrange_coeffs(P, w, n, i):
    """the unnormalized Lagrange basis l_i(x) = (x^n - 1) / (x - w^i): the coefficient of x^k is w^(i (n - 1 - k))"""
    wi = pow(w, i % n, P)
    out, cur = [0] * n, 1
    for k in reversed(range(n)):
        out[k] = cur
        cur = cur * wi % P
    return out


def env_d8(orc, fid, log_n, zk_rows):
    """[VanishesOnZK, l_0, l_L] over d8 (Montgomery [8n, 4] each): the coefficient forms above through the oracle's FFT(8n), as
    domain_constant_evaluation.rs:48-49 evaluates the first"""
    P, n = orc.MODULUS[fid], 1 << log_n
    w = ev.omega(orc, fid, log_n)
    out = []
    for c in (vanishing_zk_coeffs(P, w, n, zk_rows), lagrange_coeffs(P, w, n, 0), lagrange_coeffs(P, w, n, -(zk_rows + 1))):
        pad = np.zeros((8 * n, 4), dtype=np.uint64)
        pad[:len(c)] = ev.mont(orc, fid, c)
        out.append(orc.ntt(fid, pad))
    return out


def env_d8_pointwise(P, n, zk_rows, w, w8):
    """the same three columns from their definitions at every x = w8^k of d8, Python integers: the product for VanishesOnZK, and
    unnormalized_lagrange_evals (expr.rs:1055-1127) for l_i: (x^n - 1) / (x - w^i), which is 0 at the other points of d1 and
    n * w^(-i) at x = w^i"""
    xs = [pow(w8, k, P) for k in range(8 * n)]
    zkv = []
    for x in xs:
        v = 1
        for k in range(n - zk_rows - 1, n):
            v = v * (x - pow(w, k, P)) % P
        zkv.append(v)
    out = [zkv]
    for i in (0, n - zk_rows - 1):
        wi = pow(w, i, P)
        col = []
        for k, x in enumerate(xs):
            if k % 8:
                col.append((pow(x, n, P) - 1) * pow(x - wi, P - 2, P) % P)
            else:
                col.append(n * pow(wi, P - 2, P) % P if k == 8 * i else 0)
        out.append(col)
    return out


# ------------------------------------------------------------------------------------------------------------ instances over d8
def instance_columns(inst, s, agg, n_patterns=None):
    """an instance's d1 columns in the program's order, the three environment columns left out: witness, one selector per pattern
    (1 on the rows < L that use it), T1, the sorted columns s and agg (canonical ints)"""
    L = inst.L
    n_patterns = len(inst.patterns) if n_patterns is None else n_patterns
    sel = [[1 if r < L and inst.row_pattern[r] == k + 1 else 0 for r in range(inst.n)] for k in range(n_patterns)]
    return list(inst.w) + sel + [list(inst.T1)] + [list(c) for c in s] + [list(agg)]


def to_d8(orc, fid, col):
    """d1 evaluations (canonical ints) -> d8 evaluations (Montgomery), through the oracle's iFFT(n) and FFT(8n)"""
    n = len(col)
    pad = np.zeros((8 * n, 4), dtype=np.uint64)
    pad[:n] = orc.ntt(fid, ev.mont(orc, fid, col), inverse=True)
    return orc.ntt(fid, pad)


def oracle_evals(orc, fid, progs, cols8):
    """oracle.expr_eval of each program over d8; cols8: the program's columns over d8 (Montgomery)"""
    m8 = len(cols8[0])
    return [orc.expr_eval(fid, p.ops, p.args, p.literals, [(c, 8) for c in cols8], m8) for p in progs]


def divides(orc, fid, evals8, log_n):
    """whether the polynomial of these d8 evaluations divides exactly by Z_H = x^n - 1"""
    _, rem = orc.divide_by_vanishing(fid, orc.ntt(fid, evals8, inverse=True), log_n)
    return not rem.any()


# ------------------------------------------------------------------------------------------------------------ negative cases
# each perturbation of honest sorted columns or agg: the entries that must fail (every other entry must still vanish) and
# verify's verdict.  agg is recomputed by `aggregation` from the perturbed columns, except for "agg scaled".
NEGATIVE = {
    "agg scaled": ({"initial", "final"}, None),            # the recurrence is homogeneous in agg
    "swapped": ({"final"}, "sorting"),                     # the recurrence holds for any columns; the product no longer telescopes
    "zero den": ({"aggregation", "final"}, "sorting"),     # batch_inversion leaves the zero: agg is 0 from the next row on
    "turning even": ({"compat 0", "final"}, "overlap"),
    "turning odd": ({"compat 1", "final"}, "overlap"),
}
SCALE = 5


def perturb(inst, s, kind):
    """the sorted columns of a NEGATIVE case (a copy), and the row the recurrence must fail at (None: it must vanish)"""
    P, L = inst.P, inst.L
    s = [list(c) for c in s]
    if kind == "swapped":
        # two entries of one column whose values occur once each in the table, away from the turning rows: after the swap the
        # snake meets the later table value first and can never come back to the earlier one
        once = {t for t, c in _counts(inst.T1[:L]).items() if c == 1}
        k = 1
        rows = [r for r in range(1, L) if s[k][r] in once]
        a, b = next((a, b) for a in rows for b in rows if s[k][a] != s[k][b])
        s[k][a], s[k][b] = s[k][b], s[k][a]
    elif kind == "zero den":
        row = L // 2
        lr.zero_denominator(inst, s, row, None)
        return s, row
    elif kind.startswith("turning"):
        k = 0 if kind.endswith("even") else 1
        pos = L if k % 2 == 0 else 0
        s[k][pos] = (s[k][pos] + 1) % P
    return s, None


def _counts(xs):
    c = {}
    for x in xs:
        c[x] = c.get(x, 0) + 1
    return c


# ------------------------------------------------------------------------------------------------------------ verify
def verify(inst, sorted_cols, tic=None, table_entries=None):
    """lookup::constraints::verify (constraints.rs:690-796) on canonical-int sorted columns: None when every check passes, else the
    first that fails: "overlap" (neighbouring columns disagree where the snake turns), "sorting" (the joined snake does not follow
    the table order), "count" (it holds the wrong number of values) or "multiset" (not lookups + dummies + table).  tic: the
    table id combiner (the instance's by default); table_entries: lookup_table_entries (L by default)."""
    P, m, n = inst.P, inst.m, inst.n
    L = n - inst.zk_rows - 1
    tic = inst.tic if tic is None else tic
    for i in range(len(sorted_cols) - 1):
        pos = L if i % 2 == 0 else 0
        if sorted_cols[i][pos] != sorted_cols[i + 1][pos]:
            return "overlap"
    joined = []
    for i, s in enumerate(sorted_cols):
        es = list(s[:L + 1])
        joined += es if i % 2 == 0 else es[::-1]
    k = 0
    for t in inst.T1[:L if table_entries is None else table_entries]:
        while k < len(joined) and joined[k] == t:
            k += 1
    if k != len(joined):
        return "sorting"
    sorted_counts = {}
    for i, s in enumerate(sorted_cols):
        for x in (s[:L] if i % 2 == 0 else s[1:L + 1]):
            sorted_counts[x] = sorted_counts.get(x, 0) + 1
    all_lookups = {}
    for t in inst.T1[:L]:
        all_lookups[t] = all_lookups.get(t, 0) + 1
    for r in range(L):
        spec = lr.row_lookups(inst, r)
        for lk in spec:
            v = joint_value(lk, inst.w, r, r + 1, inst.jc, tic, P)
            all_lookups[v] = all_lookups.get(v, 0) + 1
        all_lookups[inst.dummy] = all_lookups.get(inst.dummy, 0) + m - len(spec)
    if sum(all_lookups.values()) != sum(sorted_counts.values()):
        return "count"
    if all_lookups != sorted_counts:
        return "multiset"
    return None
