"""CPU checks of tests/index_replay.py, the restatement of kimchi's prover-index columns (constraints.rs:510-760) that the device's
zk_index_build is compared with: a worked 2^3-row circuit by hand, the padding, the zeroed sigma rows, and the d8 / d4 sections
agreeing with their d1 columns."""
import random
import struct

import numpy as np
import pytest

import evals_replay as ev
import index_replay as ir


def random_circuit(orc, fid, n, n_gates, seed, tags=range(14)):
    """gates of random tags and random wires into the first n_gates rows, with 0 .. 20 coefficients each"""
    rng = random.Random(seed)
    P = orc.MODULUS[fid]
    tags = list(tags)
    gates = []
    for r in range(n_gates):
        wires = [(rng.randrange(max(1, n_gates)), rng.randrange(7)) for _ in range(7)]
        gates.append((tags[r % len(tags)], wires, [rng.randrange(P) for _ in range(rng.choice([0, 1, 5, 15, 20]))]))
    shifts = [1] + [rng.randrange(2, P) for _ in range(6)]
    return gates, shifts


def test_a_worked_eight_row_circuit(orc):
    """n = 8, zk_rows = 3, two gates: a Generic gate at row 0 with coefficients (2, 3) whose wire 0 points at (1, 2), and a Poseidon
    gate at row 1; rows 2 .. 7 are padding.  With zk_rows = 3 no sigma row is zeroed (the range n - 1 .. n - 2 is empty)."""
    fid, n = 0, 8
    P = orc.MODULUS[fid]
    w = ev.omega(orc, fid, 3)
    shifts = [1, 5, 7, 11, 13, 17, 19]
    gates = [(ir.GENERIC, [(1, 2)] + [(0, k) for k in range(1, 7)], [2, 3]),
             (ir.POSEIDON, [(1, k) for k in range(7)], [])]
    cols = {t: ev.ints(orc, fid, c) for t, c in ir.columns_d1(orc, fid, n, 3, gates, shifts).items()}
    assert cols[0x01] == [pow(w, j, P) for j in range(n)]
    assert cols[0x30] == [7 * w % P] + [shifts[0] * pow(w, j, P) % P for j in range(1, n)]
    for k in range(1, 7):
        assert cols[0x30 + k] == [shifts[k] * pow(w, j, P) % P for j in range(n)]
    assert cols[0x10] == [2] + [0] * 7 and cols[0x11] == [3] + [0] * 7
    assert all(cols[0x10 + i] == [0] * n for i in range(2, 15))
    assert cols[0x20] == [1] + [0] * 7 and cols[0x21] == [0, 1] + [0] * 6
    for t in (0x22, 0x23, 0x24, 0x25):
        assert cols[t] == [0] * n
    # the encodings: 60-byte records, and a u32 count before each gate's coefficients
    g = ir.pruned_gates(gates)
    assert len(g) == 120 and struct.unpack_from("<HxxII", g, 0) == (ir.GENERIC, 1, 2) and struct.unpack_from("<H", g, 60) == (ir.POSEIDON,)
    c = ir.gate_coeffs(orc, fid, gates)
    assert len(c) == 4 + 64 + 4 and struct.unpack_from("<I", c, 0) == (2,) and struct.unpack_from("<I", c, 68) == (0,)
    assert ev.ints(orc, fid, np.frombuffer(c[4:68], dtype="<u8").reshape(2, 4)) == [2, 3]


def test_padding_rows_are_self_wired_zero_gates():
    gates = [(ir.GENERIC, [(0, 3)] * 7, [1])]
    p = ir.padded(gates, 4)
    assert p[0] == gates[0]
    for r in range(1, 4):
        assert p[r] == (ir.ZERO, [(r, k) for k in range(7)], [])


@pytest.mark.parametrize("zk_rows", [3, 5, 15])
def test_sigma_is_zero_on_exactly_the_zk_rows_past_the_first_two(orc, zk_rows):
    fid, n = 1, 16
    gates, shifts = random_circuit(orc, fid, n, n, seed=zk_rows)
    cols = ir.columns_d1(orc, fid, n, zk_rows, gates, shifts)
    zero = set(range(n + 2 - zk_rows, n - 1))
    for k in range(7):
        s = ev.ints(orc, fid, cols[0x30 + k])
        assert {j for j in range(n) if s[j] == 0} == zero      # shifts and omega^j are nonzero, so no other row is zero


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("optional", [0, 0b111111])
def test_each_section_sub_sampled_is_its_d1_column(orc, fid, optional):
    n, zk_rows = 32, 5
    gates, shifts = random_circuit(orc, fid, n, 20, seed=fid + optional)
    cols = ir.columns_d1(orc, fid, n, zk_rows, gates, shifts, optional)
    secs = ir.sections(orc, fid, n, zk_rows, gates, shifts, optional)
    assert set(secs) == set(cols) and len(secs) == 1 + 7 + 15 + 6 + bin(optional).count("1")
    for tag, (payload, dom) in secs.items():
        m = ir.domain_mult(tag)
        assert dom == m * n and payload.shape == (m * n, 4)
        assert np.array_equal(payload[::m], cols[tag]), hex(tag)
    for tag in (0x20, 0x22):
        assert ir.domain_mult(tag) == 4
    # every tag selects its rows
    for sec, tag in ir.selector_tags(optional).items():
        assert ev.ints(orc, fid, cols[sec]) == [int(r < 20 and gates[r][0] == tag) for r in range(n)]


def test_zero_selectors_zeroes_only_selector_polynomials_sections(orc):
    fid, n = 0, 16
    gates, shifts = random_circuit(orc, fid, n, 14, seed=3)
    a = ir.columns_d1(orc, fid, n, 3, gates, shifts, 0b101, zero_selectors=False)
    b = ir.columns_d1(orc, fid, n, 3, gates, shifts, 0b101, zero_selectors=True)
    zeroed = {0x22, 0x23, 0x24, 0x25, 0x40, 0x42}
    for tag in a:
        if tag in zeroed:
            assert a[tag].any() and not b[tag].any(), hex(tag)
        else:
            assert np.array_equal(a[tag], b[tag]), hex(tag)


def test_commitment_order():
    assert ir.commitment_tags(0b100001) == ([0x30 + k for k in range(7)] + [0x10 + i for i in range(15)]
                                            + [0x20, 0x21, 0x22, 0x23, 0x24, 0x25, 0x40, 0x45])
