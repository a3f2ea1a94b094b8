"""BASELINE config 5 proxy under pytest: the MSM / NTT schedule of one kimchi proof at 2^16 gates (tools/replay_kimchi.py,
SURVEY.md §3.1) on the REAL srs/vesta.srs generators, with the 2^16 Lagrange basis computed on the device and required to equal the
one stored in srs/test_vesta.srs (digest of all 65 536 entries), and EVERY stage output compared bit for bit with the CPU oracle:
15 witness commitments, 15 iFFT(n), z, 16 FFT(8n), the quotient's iFFT(4n) + iFFT(8n), the 7 chunks of t, and the opening proof
through zk_srs_open (round 0's L and R, sg, delta, the z1 / z2 identity)."""
import os
import sys

import pytest

import proof_systems_b200 as zk

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))


def test_replay_of_a_2_16_proof_every_stage_bit_exact(orc):
    from replay_kimchi import replay
    with zk.Context(0) as ctx:
        rep = replay(zk, orc, ctx, log_n=16, check=True)
    assert rep["checks"]["lagrange_basis_equals_srs_test_vesta"]
    assert all(rep["checks"].values())
    assert set(rep["stages_s"]) <= set(rep["checks"]) | {"lagrange_basis_equals_srs_test_vesta"}
