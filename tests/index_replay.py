"""The prover index's column evaluations and the commitments of its verifier index, restated from the reference:
  ConstraintSystem::evaluated_column_coefficients   kimchi/src/circuits/constraints.rs:510-587 (sigma, coefficients, generic, poseidon)
  ConstraintSystem::column_evaluations              constraints.rs:590-760 (over d8 / d4), selector_polynomial at :334-362
  padding of the gate list                          constraints.rs:1010-1020 (CircuitGate::zero wired to itself)
  Shifts::map / cell_to_field                       kimchi/src/circuits/polynomials/permutation.rs:150-170, :201-203
  ProverIndex::verifier_index                       kimchi/src/verifier_index.rs:171-300 (mask_fixed at :179-185)
and the circuit encodings of the cache file (kimchi/src/cached_prover_index.rs): PrunedGate records (:270-300, write_pruned_gate at
:1007-1015, gate_type_to_tag at :965-982) and the GateCoeffs section (:1472-1479).

A gate is (tag, wires, coeffs): wires 7 (row, col) pairs, coeffs canonical ints.  Columns are Montgomery arrays [n, 4]; interpolation
and evaluation take their FFTs from the CPU oracle (orc.ntt), the commitments their MSMs from orc.msm_mont."""
import struct

import numpy as np

import evals_replay as ev

PERMUTS, COLUMNS, GATE_BYTES = 7, 15, 60
ZERO, GENERIC, POSEIDON, COMPLETE_ADD, VAR_BASE_MUL, ENDO_MUL, ENDO_MUL_SCALAR, LOOKUP = range(8)
RANGE_CHECK0 = 8                                          # optional selector bit b <-> tag 8 + b (OptionalSelectorBits, :246-255)
OPTIONAL_TAGS = 0x40


# ------------------------------------------------------------------------------------------------------------ encodings
def pruned_gates(gates) -> bytes:
    """write_pruned_gate: typ_tag u16 | pad[2] | 7 x (row u32, col u32)"""
    out = bytearray()
    for tag, wires, _ in gates:
        out += struct.pack("<H2x", tag)
        for row, col in wires:
            out += struct.pack("<II", row, col)
    return bytes(out)


def gate_coeffs(orc, fid, gates) -> bytes:
    """the GateCoeffs section: per gate a u32 count, then that many Montgomery field elements"""
    out = bytearray()
    for _, _, coeffs in gates:
        out += struct.pack("<I", len(coeffs))
        if coeffs:
            out += ev.mont(orc, fid, coeffs).astype("<u8").tobytes()
    return bytes(out)


def padded(gates, n):
    """constraints.rs:1010-1020: rows len(gates) .. n - 1 are zero gates wired to themselves, without coefficients"""
    return list(gates) + [(ZERO, [(r, k) for k in range(PERMUTS)], []) for r in range(len(gates), n)]


def header(zk, n, zk_rows, shifts_mont, optional=0, **kw):
    """a zk_index_header with the fields zk_index_build reads; the others from kw"""
    h = zk.IndexHeader()
    h.domain_d1_size, h.zk_rows, h.optional_selectors_present = n, zk_rows, optional
    for k in range(PERMUTS):
        for j in range(4):
            h.shift[k][j] = int(shifts_mont[k][j])
    for name, v in kw.items():
        if name in ("endo", "verifier_index_digest"):
            for j in range(4):
                getattr(h, name)[j] = int(v[j])
        else:
            setattr(h, name, v)
    return h


# ------------------------------------------------------------------------------------------------------------ d1 columns
def sid(orc, fid, n) -> np.ndarray:
    """sid[j] = omega^j: the forward FFT of the vector with 1 at position 1"""
    e1 = np.zeros((n, 4), dtype=np.uint64)
    e1[1 % n] = ev.mont(orc, fid, [1])[0]
    return orc.ntt(fid, e1)


def selector_tags(optional: int) -> dict:
    """section tag -> gate tag of the selectors built with selector_polynomial (zeroed by zero_selectors)"""
    tags = {0x22: COMPLETE_ADD, 0x23: VAR_BASE_MUL, 0x24: ENDO_MUL, 0x25: ENDO_MUL_SCALAR}
    for b in range(6):
        if optional >> b & 1:
            tags[OPTIONAL_TAGS + b] = RANGE_CHECK0 + b
    return tags


def columns_d1(orc, fid, n, zk_rows, gates, shifts, optional=0, zero_selectors=False) -> dict:
    """section tag -> the column over d1 (Montgomery [n, 4]) before interpolation; shifts canonical ints.  0x01 is sid itself."""
    P = orc.MODULUS[fid]
    gates = padded(gates, n)
    pw = sid(orc, fid, n)
    cols = {0x01: pw}
    real = [r for r, g in enumerate(gates) if g[0] != ZERO or any(w != (r, k) for k, w in enumerate(g[1]))]
    rows = sorted({row for r in real for row, _ in gates[r][1]})
    pw_int = dict(zip(rows, ev.ints(orc, fid, pw[rows]))) if rows else {}
    for k in range(PERMUTS):
        # self-wired rows: shift_k omega^r (the FFT of shift_k at position 1); the others shift[col] omega^row (cell_to_field)
        e = np.zeros((n, 4), dtype=np.uint64)
        e[1 % n] = ev.mont(orc, fid, [shifts[k]])[0]
        s = orc.ntt(fid, e)
        if real:
            s[real] = ev.mont(orc, fid, [shifts[gates[r][1][k][1]] * pw_int[gates[r][1][k][0]] % P for r in real])
        s[n + 2 - zk_rows:n - 1] = 0                       # constraints.rs:516-530
        cols[0x30 + k] = s
    for i in range(COLUMNS):                               # gate.coeffs.get(i) or zero
        c = np.zeros((n, 4), dtype=np.uint64)
        has = [r for r, g in enumerate(gates) if len(g[2]) > i]
        if has:
            c[has] = ev.mont(orc, fid, [gates[r][2][i] for r in has])
        cols[0x10 + i] = c
    one = ev.mont(orc, fid, [1])[0]

    def selector(tag):
        c = np.zeros((n, 4), dtype=np.uint64)
        c[[r for r, g in enumerate(gates) if g[0] == tag]] = one
        return c
    cols[0x20] = selector(GENERIC)
    cols[0x21] = selector(POSEIDON)                        # gate.ps()
    for sec, tag in selector_tags(optional).items():       # selector_polynomial: zero when cfg!(debug_assertions) && disable_gates_checks
        cols[sec] = np.zeros((n, 4), dtype=np.uint64) if zero_selectors else selector(tag)
    return cols


def domain_mult(tag) -> int:
    """the evaluation domain of a section, as a multiple of d1"""
    return 1 if tag == 0x01 else 4 if tag in (0x20, 0x22) else 8


def evaluate(orc, fid, col, mult) -> np.ndarray:
    """Evaluations::interpolate over d1, then evaluate_over_domain_by_ref over the domain mult times larger"""
    n = col.shape[0]
    pad = np.zeros((mult * n, 4), dtype=np.uint64)
    pad[:n] = orc.ntt(fid, col, inverse=True)
    return orc.ntt(fid, pad)


def sections(orc, fid, n, zk_rows, gates, shifts, optional=0, zero_selectors=False, tags=None) -> dict:
    """section tag -> (Montgomery payload, elem_domain_size) as the reference's writer records them (cached_prover_index.rs:1434-1560)"""
    cols = columns_d1(orc, fid, n, zk_rows, gates, shifts, optional, zero_selectors)
    out = {}
    for tag, c in cols.items():
        if tags is None or tag in tags:
            m = domain_mult(tag)
            out[tag] = (c if m == 1 else evaluate(orc, fid, c, m), m * n)
    return out


# ------------------------------------------------------------------------------------------------------------ commitments
def commitment_tags(optional: int) -> list:
    """verifier_index.rs:221-300: sigma_comm, coefficients_comm, generic, psm, complete_add, mul, emul, endomul_scalar, optional"""
    return ([0x30 + k for k in range(PERMUTS)] + [0x10 + i for i in range(COLUMNS)] + list(range(0x20, 0x26))
            + [OPTIONAL_TAGS + b for b in range(6) if optional >> b & 1])


MASKED = set(range(0x20, 0x26))                            # mask_fixed: blinder one


def commitments(orc, cid, g, h, cols, optional: int) -> np.ndarray:
    """[count, chunks, 8]: commit_evaluations_non_hiding(d1, e) == commit_non_hiding(interpolate(e)) (poly-commitment/tests/
    ipa_commitment.rs) -- chunk c is the MSM of coefficients c |g| .. (c + 1) |g| over g -- plus h on every chunk of the masked ones.
    cols: section tag -> d1 column."""
    fid = orc.SCALAR_FIELD[cid]
    out = []
    for tag in commitment_tags(optional):
        coeffs = orc.ntt(fid, cols[tag], inverse=True)
        n, m = coeffs.shape[0], g.shape[0]
        chunks = []
        for c in range(max(1, n // m)):
            part = coeffs[c * m:(c + 1) * m]
            p = orc.msm_mont(cid, g[:part.shape[0]], part)
            chunks.append(orc.affine_add(cid, p, h) if tag in MASKED else p)
        out.append(np.stack(chunks))
    return np.stack(out)
