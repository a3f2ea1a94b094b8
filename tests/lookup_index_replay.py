"""The lookup index and the lookup commitments of its verifier index, restated from the reference:
  LookupConstraintSystem::create                  kimchi/src/circuits/lookup/index.rs:202-482 (check_id_duplicates :487-502)
  LookupInfo::selector_polynomials_and_tables     kimchi/src/circuits/lookup/lookups.rs:235-283 (from_gate :541-553)
  the gate tables                                 lookup/tables/mod.rs:15-46 (RangeCheck before Xor), xor.rs:22-44, range_check.rs
  LookupVerifierIndex's commitments               kimchi/src/verifier_index.rs:196-215 (mask_fixed :179-185)
  Builder::build's domain for lookups             kimchi/src/circuits/constraints.rs:897-1006
and the cache file's encoding of the sections (cached_prover_index.rs:258-268, :1560-1620).

Gates are their tags (gate_type_to_tag); tables are (id, columns) with canonical ints; runtime is None or a list of
(id, first_column).  Interpolation and evaluation take their FFTs from the CPU oracle, the commitments their MSMs from orc.msm_mont."""
import numpy as np

import evals_replay as ev
import index_replay as ir
import lookup_replay as lr

GATE_NAMES = {7: "Lookup", 8: "RangeCheck0", 9: "RangeCheck1", 10: "ForeignFieldAdd", 11: "ForeignFieldMul", 12: "Xor16", 13: "Rot64"}
TAGS = {name: tag for tag, name in GATE_NAMES.items()}
PATTERNS = ["xor", "lookup", "range_check", "foreign_field_mul"]      # sections 0x52 .. 0x55, LookupSelectorBits 1 .. 4
MAX_JOINT_SIZE = {"xor": 3, "lookup": 2, "range_check": 1, "foreign_field_mul": 1}
ID_COLLISION, TABLE_ID_ZERO, TOO_LONG = 1, 2, 3
XOR_TABLE_ID, RANGE_CHECK_TABLE_ID = lr.XOR_TABLE_ID, lr.RANGE_CHECK_TABLE_ID


class LookupError_(Exception):
    """LookupError: kind (ID_COLLISION, TABLE_ID_ZERO, TOO_LONG) and the reference's Display message"""

    def __init__(self, kind, message):
        super().__init__(message)
        self.kind, self.message = kind, message


class Panics(Exception):
    """the reference panics (an index past the domain, a usize underflow)"""


def xor_table():
    """xor_table: (i, j, i ^ j) for i, j < 16, every column reversed, so (0, 0, 0) is the last row"""
    rows = [(i, j, i ^ j) for i in range(16) for j in range(16)][::-1]
    return (XOR_TABLE_ID, [[r[c] for r in rows] for c in range(3)])


def range_check_table():
    return (RANGE_CHECK_TABLE_ID, [list(range(1 << 12))])


def id_duplicates(ids, msg):
    """check_id_duplicates: None, or the collision_type "msg: [a, b]" listing every id already seen, in order"""
    seen, dups = set(), []
    for i in ids:
        if i in seen:
            dups.append(i)
        seen.add(i)
    return f"{msg}: [{', '.join(map(str, dups))}]" if dups else None


def patterns_of(tags):
    """LookupPatterns::from_gates: the patterns the gates use, in section order"""
    used = set()
    for t in tags:
        for nxt in (False, True):
            p = lr.from_gate(GATE_NAMES.get(t), nxt)
            if p:
                used.add(p)
    return [p for p in PATTERNS if p in used]


def selectors(n, tags):
    """selector_polynomials_and_tables: pattern -> 0/1 column over d1; a Next pattern sets row i + 1"""
    pats = patterns_of(tags)
    out = {p: [0] * n for p in pats}
    for i, t in enumerate(tags[:n]):
        for nxt in (False, True):
            p = lr.from_gate(GATE_NAMES.get(t), nxt)
            if p:
                if i + nxt >= n:
                    raise Panics(f"selector row {i + nxt} of {n}")
                out[p][i + nxt] = 1
    return out


def gate_tables(pats):
    """the gate tables of the patterns in GateLookupTable's order: RangeCheck (RangeCheck, ForeignFieldMul), then Xor"""
    out = []
    if "range_check" in pats or "foreign_field_mul" in pats:
        out.append(range_check_table())
    if "xor" in pats:
        out.append(xor_table())
    return out


def concatenated(tables, width, rows, P=None):
    """the concatenated table: each table's columns, narrower ones filled with 0, rows padded with 0 to `rows`; and the table ids
    (i32_to_field: a negative id is -|id|), padded with 0"""
    cols = [[] for _ in range(width)]
    ids = []
    for tid, data in tables:
        ln = len(data[0])
        ids += [tid % P if P else tid] * ln
        for c in range(width):
            cols[c] += list(data[c]) if c < len(data) else [0] * ln
    return [c + [0] * (rows - len(c)) for c in cols], ids + [0] * (rows - len(ids))


def create(P, n, zk_rows, tags, tables, runtime=None):
    """LookupConstraintSystem::create over d1: None without a pattern, else a dict with the d1 columns (Python ints) cols (w table
    columns), ids (None without a nonzero id), selectors (pattern -> column, present ones), runtime_selector (None without runtime
    tables) and runtime_table_offset.  Raises LookupError_ or Panics like the reference."""
    pats = patterns_of(tags)
    if not pats:
        return None
    max_num_entries = n - zk_rows - 1
    sel = selectors(n, tags)
    gt = gate_tables(pats)
    dup = id_duplicates([t[0] for t in tables] + [t[0] for t in gt], "duplicates between fixed given and fixed from-gate tables")
    if dup is None and runtime is not None:
        dup = id_duplicates([r[0] for r in runtime], "runtime table duplicates")
    if dup is not None:
        raise LookupError_(ID_COLLISION, "Cannot create a combined table since ids for sub-tables are colliding. The collision type is: " + dup)
    all_tables = list(tables) + gt
    offset = rsel = None
    if runtime is not None:
        offset = sum(len(d[0]) for _, d in all_tables)
        rlen = sum(len(c) for _, c in runtime)
        if offset + rlen > n:
            raise Panics("d1_size - runtime_table_offset - runtime_len underflows")
        rsel = [1] * offset + [0] * rlen + [1] * (n - offset - rlen)
        for i in range(n - zk_rows, n):
            rsel[i] = 0
        all_tables += [(tid, [list(c), [0] * len(c)]) for tid, c in runtime]
    width = max([len(d) for _, d in all_tables] + [MAX_JOINT_SIZE[p] for p in pats])
    has0 = any(tid == 0 for tid, _ in all_tables)
    zero_entry = any(tid == 0 and any(all(col[r] == 0 for col in d) for r in range(len(d[0]))) for tid, d in all_tables)
    if has0 and not zero_entry:
        raise LookupError_(TABLE_ID_ZERO, "The table with id 0 must have an entry of all zeros")
    total = sum(len(d[0]) for _, d in all_tables)
    if total >= max_num_entries:
        raise LookupError_(TOO_LONG, "The combined lookup table is larger than allowed by the domain size. "
                                     f"Observed: {total}, expected: {max_num_entries - 1}")
    cols, ids = concatenated(all_tables, width, n, P)
    return {"cols": cols, "ids": ids if any(tid != 0 for tid, _ in all_tables) else None, "selectors": sel, "runtime_selector": rsel,
            "runtime_table_offset": offset}


def header_bits(res) -> int:
    """lookup_selectors_present, bits 0 .. 5: table ids, the selectors xor, lookup, range_check, ffmul, the runtime selector"""
    bits = 1 if res["ids"] is not None else 0
    for k, p in enumerate(PATTERNS):
        if p in res["selectors"]:
            bits |= 2 << k
    return bits | (0x20 if res["runtime_selector"] is not None else 0)


def columns(res):
    """(section tag, d1 column) in the order of the sections and of the commitments; 0x50 once per table column"""
    out = [(0x50, c) for c in res["cols"]]
    if res["ids"] is not None:
        out.append((0x51, res["ids"]))
    out += [(0x52 + k, res["selectors"][p]) for k, p in enumerate(PATTERNS) if p in res["selectors"]]
    if res["runtime_selector"] is not None:
        out.append((0x56, res["runtime_selector"]))
    return out


def sections(orc, fid, res) -> dict:
    """section tag -> (Montgomery payload, elem_domain_size) as the reference's writer records them: 0x50 the w columns over d8
    back to back with elem_domain_size w, the others over d8 with 8n"""
    out = {}
    cols = columns(res)
    n = len(cols[0][1])
    for tag, c in cols:
        e = ir.evaluate(orc, fid, ev.mont(orc, fid, c), 8)
        if tag == 0x50:
            prev = out.get(0x50, (np.zeros((0, 4), dtype=np.uint64), 0))[0]
            out[0x50] = (np.concatenate([prev, e]), len(res["cols"]))
        else:
            out[tag] = (e, 8 * n)
    return out


def commitments(orc, cid, g, h, res) -> np.ndarray:
    """[count, chunks, 8]: commit_evaluations_non_hiding of each column in columns() order, plus h on every chunk of the table
    columns and the table ids (mask_fixed)"""
    fid = orc.SCALAR_FIELD[cid]
    out = []
    for tag, c in columns(res):
        coeffs = orc.ntt(fid, ev.mont(orc, fid, c), inverse=True)
        n, m = coeffs.shape[0], g.shape[0]
        chunks = []
        for k in range(max(1, n // m)):
            part = coeffs[k * m:(k + 1) * m]
            p = orc.msm_mont(cid, g[:part.shape[0]], part)
            chunks.append(orc.affine_add(cid, p, h) if tag in (0x50, 0x51) else p)
        out.append(np.stack(chunks))
    return np.stack(out)


def builder_domain(n_gates, tags, tables, runtime=None):
    """Builder::build without max_poly_size (constraints.rs:897-1006): zk_rows = 3 and the smallest power of two holding
    max(gates, lookup_domain_size + 1) + 3 rows, where lookup_domain_size counts the fixed, runtime and gate tables and a dummy row
    when no fixed table has id 0"""
    size = sum(len(d[0]) if d else 0 for _, d in tables) + sum(len(c) for _, c in (runtime or []))
    size += sum(len(d[0]) for _, d in gate_tables(patterns_of(tags)))
    size += 0 if any(tid == 0 for tid, _ in tables) else 1
    lower = max(n_gates, size + 1) + 3
    return 1 << (lower - 1).bit_length(), 3


def mont_table(orc, fid, data) -> np.ndarray:
    """a table's columns as IndexCache.build_lookup takes them: Montgomery uint64 [width, len, 4]"""
    return np.stack([ev.mont(orc, fid, c) if len(c) else np.zeros((0, 4), dtype=np.uint64) for c in data])
