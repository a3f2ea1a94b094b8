"""tests/msm_plan.py against the facts the library states about its own planner, and against itself (no GPU): the signed digits add up
to the scalar, scalars built for a bucket layout land where they were aimed, and the regime table used by
tests/test_gpu_msm_regimes.py names regimes the planner really selects."""
import random

import numpy as np
import pytest

import msm_plan as mp

FP_MODULUS = 28948022309329048855892746252171976963363056481941560715954676764349967630337
FQ_MODULUS = 28948022309329048855892746252171976963363056481941647379679742748393362948097
H100_SMS = 132


@pytest.mark.parametrize("c", range(2, 17))
def test_signed_digits_reassemble_the_scalar(c):
    half, nwin = 1 << (c - 1), mp.num_windows(c)
    rng = random.Random(c)
    vals = [0, 1, half, half + 1, sum((half + 1) << (c * w) for w in range(nwin - 1)) % (1 << 254)]
    vals += [1 << k for k in range(0, 254, 7)] + [(1 << k) - 1 for k in (c - 1, c, c + 1, 128, 254)]
    for m in (FP_MODULUS, FQ_MODULUS):
        vals += [m - 1, m - 2, m >> 1] + [rng.randrange(m) for _ in range(200)]
    for s in vals:
        d = mp.digits(s, c)                    # asserts that no carry leaves the top window
        assert len(d) == nwin and all(-half < x <= half for x in d)
        assert sum(x << (c * w) for w, x in enumerate(d)) == s
    assert mp.digits(half, c)[0] == half                                    # 2^(c-1) stays positive
    assert mp.digits(half + 1, c)[:2] == [half + 1 - (1 << c), 1]           # one more goes negative and carries
    assert all(x < 0 for x in mp.digits(vals[4], c)[:1])


@pytest.mark.parametrize("c", range(2, 17))
@pytest.mark.parametrize("table", [True, False])
def test_scalars_for_lands_in_the_aimed_buckets(c, table):
    half = 1 << (c - 1)
    p = mp.plan(1, 1, c if table else 0, c, H100_SMS)
    top = p.nwin - 3
    pops = [(0, 1, 3), (0, half, 2), (top, 1, 4), (1, half, 1)]
    if half > 1:
        pops += [(0, -(half - 1), 5), (2, -1, 2), (top, half - 1, 7)]
    sc = mp.scalars_for(pops, c)
    p = p._replace(n=len(sc))
    want = np.zeros(p.NB, dtype=np.int64)
    for w, d, cnt in pops:
        want[mp.bucket_of(p, 0, w, d)] += cnt
        if d < 0:
            want[mp.bucket_of(p, 0, w + 1, 1)] += cnt       # the carry of a negative digit
    assert np.array_equal(mp.buckets([sc], p), want)
    assert len(sc) == sum(cnt for _, _, cnt in pops) and all(0 <= s < mp.SCALAR_LIMIT for s in sc)
    # a batch puts MSM j's entries into its own groups
    p2 = p._replace(k=2, G=2 * p.gpm, NB=2 * p.NB)
    got = mp.buckets([sc, [0] * len(sc)], p2)
    assert np.array_equal(got[:p.NB], want) and not got[p.NB:].any()


def test_plan_reproduces_the_documented_choices():
    """msm_default_window's comment: with a table 2^16 points -> c = 15 and 2^11 -> c = 10; test_config4 asserts 16 at 2^20"""
    assert mp.default_window(1 << 16, True) == 15 and mp.default_window(1 << 11, True) == 10 and mp.default_window(1 << 20, True) == 16
    assert mp.default_window(1 << 16, False) == 12 and mp.default_window(1, False) == 4 and mp.default_window(100, True) == 5
    assert [mp.num_windows(c) for c in (2, 7, 8, 15, 16)] == [128, 37, 32, 18, 16]
    # window 16 table, one MSM of 2^16: 2^15 buckets > 64 quads x 132 SMs -> thread-per-bucket finish, one launch more
    p = mp.plan(1 << 16, 1, 16, 0, H100_SMS)
    assert (p.c, p.nwin, p.gpm, p.G, p.B, p.NB, p.Mmax) == (16, 16, 1, 1, 32768, 32768, 1 << 20)
    assert p.many_buckets and p.launches == 9 and p.ntiles == 8 and p.capacity == 132 * 512 and p.K == 6 and p.log_g == 0 and p.smax == 32
    q = mp.plan(1 << 11, 1, 10, 0, H100_SMS)
    assert not q.many_buckets and q.launches == 8 and q.ntiles == 1 and q.NB == 512 and q.nwin == 26
    # without a table every window has a bucket set of its own
    t = mp.plan(4096, 1, 0, 0, H100_SMS)
    assert (t.c, t.gpm, t.NB) == (8, 32, 32 * 128)
    # a batch of 16 at window 16: 128 scan tiles
    assert mp.plan(2048, 16, 16, 0, H100_SMS).ntiles == 128
    # the options
    assert mp.plan(1 << 15, 1, 16, 0, H100_SMS, chunk=1).K == 1 and mp.plan(1 << 15, 1, 16, 0, H100_SMS, wave_threads=32).capacity == 132 * 32
    assert [mp.plan(1000, 1, 10, 0, H100_SMS, chunk=k).log_g for k in (64, 6, 2, 1)] == [0, 1, 2, 3]


def test_regime_counts_tasks_and_giants():
    p = mp.plan(5000, 1, 10, 0, H100_SMS, chunk=3)
    counts = np.zeros(p.NB, dtype=np.int64)
    counts[[0, 5, 6, 511]] = [1, 3 * p.smax, 3 * p.smax + 1, 7]
    r = mp.regime(counts, p)
    assert list(r.s_b[[0, 5, 6, 511]]) == [1, p.smax, p.smax + 1, 3] and list(r.giants) == [6] and not r.overflow
    assert (r.empty, r.single, r.multi, r.tasks) == (p.NB - 4, 1, 2, 1 + 2 * p.smax + 1 + 3)
    assert r.task_off[6] == 1 + p.smax and r.task_off[-1] == r.tasks
    counts[100:165] = 3 * p.smax + 1
    assert mp.regime(counts, p).overflow and len(mp.regime(counts, p).giants) == 66
