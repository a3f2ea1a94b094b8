"""Device-side ingestion of kimchi's mmap prover-index cache (kimchi/src/cached_prover_index.rs:26-56): a cache image written in the
reference's layout (tests/index_cache_writer.py restates its serializer) is parsed by zk_index_cache_load, its field-element sections
arrive on the device bit for bit, the header fields come back, malformed files are rejected with the reference's error classes, and
permutation_coefficients8 taken straight from the cache feeds the permutation quotient kernel."""
import numpy as np
import pytest

import proof_systems_b200 as zk
from index_cache_writer import write_cache

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def make_image(orc, fid, log_n, ident="vk-digest-abc", **kw):
    n, m8, m4 = 1 << log_n, 8 << log_n, 4 << log_n
    rnd = lambda k, seed: orc.to_mont(fid, orc.random_scalars(fid, k, seed=seed))
    arrays = {0x01: (rnd(n, 1), 0)}
    for i in range(15):
        arrays[0x10 + i] = (rnd(m8, 10 + i), m8)
    arrays[0x20] = (rnd(m4, 40), m4)                      # generic selector over d4
    arrays[0x21] = (rnd(m8, 41), m8)
    for i in range(7):
        arrays[0x30 + i] = (rnd(m8, 50 + i), m8)
    arrays[0x40] = (rnd(m8, 60), m8)                      # one optional selector
    header = {"public": 3, "prev_challenges": 2, "zk_rows": 3, "max_poly_size": n, "domain_d1_size": n, "feature_flags": 1,
              "optional_selectors_present": 1, "endo_limbs": [int(x) for x in rnd(1, 70)[0]], "shift_limbs": [[int(x) for x in r] for r in rnd(7, 71)]}
    gates = bytes(60 * 5)                                  # a non-field section (PrunedGate records): skipped by the device copy
    sections = [(0x02, gates, 0)] + [(tag, a.astype("<u8").tobytes(), dom) for tag, (a, dom) in arrays.items()]
    return write_cache(ident, header, sections, **kw), arrays, header


@pytest.mark.parametrize("fid", [0, 1])
def test_sections_arrive_on_the_device_bit_for_bit(ctx, orc, fid):
    image, arrays, header = make_image(orc, fid, 8)
    with zk.IndexCache(ctx, image, expect_identifier="vk-digest-abc") as cache:
        h = cache.header
        assert (h.public_inputs, h.prev_challenges, h.zk_rows, h.max_poly_size, h.domain_d1_size) == (3, 2, 3, 256, 256)
        assert h.identifier == b"vk-digest-abc" and h.feature_flags == 1 and h.num_sections == len(arrays) + 1
        assert list(h.endo) == header["endo_limbs"] and [list(r) for r in h.shift] == header["shift_limbs"]
        for tag, (a, dom) in arrays.items():
            ptr, n_el, d = cache.section(tag)
            assert n_el == a.shape[0] and d == dom
            assert np.array_equal(ctx.dev_download(ptr, a.shape), a), hex(tag)
        with pytest.raises(zk.ZkError):
            cache.section(0x02)                            # gates are not field elements
        with pytest.raises(zk.ZkError):
            cache.section(0x41)                            # optional selector not in this file


def test_malformed_files_are_rejected(ctx, orc):
    image, _, _ = make_image(orc, 0, 6)
    for bad in (image[:100], b"MINAPK00" + image[8:], image[:8] + (2).to_bytes(4, "little") + image[12:], image[:-500]):
        with pytest.raises(zk.ZkError):
            zk.IndexCache(ctx, bad)
    with pytest.raises(zk.ZkError):
        zk.IndexCache(ctx, image, expect_identifier="another-key")      # CacheError::IdentifierMismatch
    # a section table entry pointing past the end, and a missing permutation column
    trunc, _, _ = make_image(orc, 0, 6)
    with pytest.raises(zk.ZkError):
        zk.IndexCache(ctx, trunc[: len(trunc) // 2])


def test_cached_sigma_feeds_the_permutation_quotient(ctx, orc):
    """permutation_coefficients8 read from the cache image (no host re-encoding) as the sigma operand of zk_perm_quotient_dev"""
    fid, log_n = zk.FQ, 7
    image, arrays, header = make_image(orc, fid, log_n)
    m = 8 << log_n
    rnd = lambda k, seed: orc.to_mont(fid, orc.random_scalars(fid, k, seed=seed))
    w, z, zkpm = rnd(7 * m, 81).reshape(7, m, 4), rnd(m, 82), rnd(m, 83)
    beta, gamma, alpha0 = rnd(1, 84)[0], rnd(1, 85)[0], rnd(1, 86)[0]
    shifts = np.array(header["shift_limbs"], dtype=np.uint64)
    sigma = np.stack([arrays[0x30 + i][0] for i in range(7)])
    want = orc.perm_quot(fid, w, z, sigma, zkpm, beta, gamma, alpha0, shifts)
    with zk.IndexCache(ctx, image) as cache, ctx.buffers() as bufs:
        d_w, d_z, d_zkpm, d_out = bufs.put(w), bufs.put(z), bufs.put(zkpm), bufs.alloc(z.nbytes)
        d_sigma = [cache.section(0x30 + i)[0] for i in range(7)]
        ctx.perm_quotient_dev(fid, log_n + 3, [d_w + k * m * 32 for k in range(7)], d_z, d_sigma, d_zkpm, beta, gamma, alpha0, shifts, d_out)
        assert np.array_equal(ctx.dev_download(d_out, (m, 4)), want)
