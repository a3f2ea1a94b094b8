"""SRS::verify (poly-commitment/src/ipa.rs:301-502) restated on the CPU oracle (tests/verify_replay.py), on the reference's own
randomised batch-verification test (poly-commitment/tests/commitment.rs:119-257): 7 aggregated proofs over SRS::create(128), made by
the oracle restatement of SRS::open, verified with rand_base and sg_rand_base drawn from the same StdRng([0; 32]) stream."""
import json
import os

import numpy as np
import pytest

from verify_replay import TAMPERINGS, oracle_open, oracle_verify, opening_bytes, reference_batch, tamper

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ser_regression.json")


@pytest.fixture(scope="module")
def batch(orc, vesta_srs):
    h = vesta_srs.mont_points(vesta_srs.h_xy_canon)[0]
    g = vesta_srs.g[:128]
    return reference_batch(orc, vesta_srs, lambda polys, elm, ps, es, draws, tr: oracle_open(orc, g, h, polys, elm, ps, es, draws, tr))


def test_first_proof_is_the_reference_opening_proof(orc, batch):
    """the restated stream reproduces the reference's bytes of its first proof (ser_regression_canonical_opening_proof)"""
    entries = batch[0]
    want = json.load(open(GOLDEN))["opening_proof_vesta_srs128"]
    raw = opening_bytes(orc, entries[0].opening)
    assert list(raw) + [0] * (len(want) - len(raw)) == want


def test_the_reference_batch_verifies(orc, batch):
    entries, rand_base, sg_rand_base, g, h = batch
    assert not np.any(oracle_verify(orc, orc.VESTA, g, h, entries, rand_base, sg_rand_base))


@pytest.mark.parametrize("kind", TAMPERINGS)
def test_a_tampered_batch_fails(orc, batch, kind):
    entries, rand_base, sg_rand_base, g, h = batch
    bad = tamper(entries, kind, orc.FP_MODULUS, g[5])
    assert np.any(oracle_verify(orc, orc.VESTA, g, h, bad, rand_base, sg_rand_base))
