"""Every regime of the MSM accumulation and bucket-finish pipeline (csrc/msm.cu), steered through the public options `msm_chunk` and
`msm_wave_threads` and through the scalars alone, each result bit-exact against the oracle.

Every case first asserts, with the planner mirror tests/msm_plan.py, that the call is in the regime the case is named after: the
finish variant (thread per bucket behind k_run_sum, or quads per bucket), K entries per task, log_g / smax, how many buckets are
giant and whether their list overflows, the scan tiles of k_plan.  Two facts of the mirror are checked on the device with every call:
the kernel launches of the call (one more with the thread-per-bucket finish) and, for zk_msm_partial, the (c, groups) it reports.
The giant list and log_g cannot be observed from outside the library; for those the mirror alone is the witness."""
from contextlib import contextmanager

import numpy as np
import pytest

import msm_plan as mp
import proof_systems_b200 as zk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@contextmanager
def options(ctx, chunk=0, wave_threads=0):
    ctx.set_option("msm_chunk", chunk)
    ctx.set_option("msm_wave_threads", wave_threads)
    try:
        yield
    finally:
        ctx.set_option("msm_chunk", 0)
        ctx.set_option("msm_wave_threads", 0)


def negated(orc, srs, pts):
    out = np.array(pts, dtype=np.uint64, copy=True).reshape(-1, 8)
    zero = np.zeros(4, dtype=np.uint64)
    for row in out:
        if row.any():
            row[4:] = orc.fe_sub(srs.base, zero, row[4:])
    return out.reshape(np.shape(pts))


def run(ctx, orc, srs, bases, g, sc_ints, p, window_bits=0, off=0):
    """one MSM (sc_ints: n ints) or one fused batch (a list of k such lists) over g[off : off + n]; checks the launches the mirror
    predicts and the oracle's result"""
    batch = isinstance(sc_ints[0], (list, tuple))
    sets = sc_ints if batch else [sc_ints]
    assert (len(sets), len(sets[0])) == (p.k, p.n)
    limbs = np.stack([orc.ints_to_limbs(s) for s in sets])
    before = ctx.launch_count
    if batch:
        got = [zk.jacobian_to_affine(srs.cid, r) for r in ctx.msm_batch(bases, limbs, off=off, window_bits=window_bits)]
    else:
        got = [ctx.msm_affine(bases, limbs[0], off=off, window_bits=window_bits)]
    assert ctx.launch_count - before == p.launches
    for j in range(p.k):
        assert np.array_equal(got[j], orc.msm(srs.cid, g[off:off + p.n], limbs[j])), j


# ------------------------------------------------------------------------------------------ a. finish variant x K x log_g
# (bases, call window, n): NB = 32768 and 45056 are far above 64 quads x SMs, 512 and 832 far below, on any H100
VARIANTS = {"serial-table16": (16, 0, 1 << 15), "serial-table15": (15, 0, 30000), "serial-plain12": (0, 12, 3000), "quad-table10": (10, 0, 1000),
            "quad-plain5": (0, 5, 700)}
# log_g = f(Mmax / (K NB)) for the explicit chunks; with chunk 0 the heuristic's K depends on the SM count: the mirror's value is used
LOG_G = {"serial-table16": {1: 2, 2: 1, 3: 0, 6: 0, 64: 0, 4096: 0}, "serial-table15": {1: 3, 2: 2, 3: 1, 6: 0, 64: 0, 4096: 0},
         "serial-plain12": {1: 0, 2: 0, 3: 0, 6: 0, 64: 0, 4096: 0},
         "quad-table10": {1: 3, 2: 2, 3: 2, 6: 1, 64: 0, 4096: 0}, "quad-plain5": {1: 3, 2: 2, 3: 1, 6: 0, 64: 0, 4096: 0}}
TUNINGS = [(0, 0), (1, 0), (2, 0), (3, 0), (6, 0), (64, 0), (4096, 0), (0, 32), (0, 2048)]


@pytest.mark.parametrize("chunk,wave", TUNINGS, ids=[f"chunk{c}-wave{w}" for c, w in TUNINGS])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_finish_variant_x_chunk_x_log_g(ctx, orc, pallas_srs, sms, variant, chunk, wave):
    srs = pallas_srs
    wb, window, n = VARIANTS[variant]
    g = srs.g[:n].copy()
    g[n // 3] = 0
    sc = orc.limbs_to_ints(orc.random_scalars(srs.scalar, n, seed=n + chunk))
    sc[1:40] = [1] * 39                       # one heavier bucket: more than one task at the small chunks
    with ctx.upload_bases(srs.cid, g, window_bits=wb) as bases:
        p = mp.plan(n, 1, bases.window_bits, window, sms, chunk, wave)
        assert p.many_buckets == variant.startswith("serial") and p.capacity == sms * (wave or 512)
        if chunk:
            assert p.K == chunk and p.log_g == LOG_G[variant][chunk] and p.smax == 32 << p.log_g
        r = mp.regime(mp.buckets([sc], p), p)
        if chunk == 4096:
            assert r.multi == 0 and len(r.giants) == 0          # nothing goes through the partials
        if chunk == 1:
            assert r.tasks == int(mp.buckets([sc], p).sum()) and r.multi > 0   # every entry a task
        with options(ctx, chunk, wave):
            run(ctx, orc, srs, bases, g, sc, p, window_bits=window)


def test_log_g_takes_every_value_in_both_finish_variants():
    for prefix in ("serial", "quad"):
        assert {v for name, d in LOG_G.items() if name.startswith(prefix) for v in d.values()} == {0, 1, 2, 3}


def test_launch_count_tells_the_finish_variant(ctx, orc, pallas_srs, sms):
    """the same bases and scalars at windows 8 and 10: k_run_sum is the one kernel more of the thread-per-bucket finish"""
    srs = pallas_srs
    n = 500
    sc = orc.random_scalars(srs.scalar, n, seed=8)
    with ctx.upload_bases(srs.cid, srs.g[:n], window_bits=0) as bases:
        delta = {}
        for window in (8, 10):
            before = ctx.launch_count
            ctx.msm(bases, sc, window_bits=window)
            delta[window] = ctx.launch_count - before
        quad, serial = mp.plan(n, 1, 0, 8, sms), mp.plan(n, 1, 0, 10, sms)
        assert not quad.many_buckets and serial.many_buckets
        assert delta[10] - delta[8] == 1 and (delta[8], delta[10]) == (quad.launches, serial.launches)


# ------------------------------------------------------------------------------------------ b. bucket populations at the boundaries
def boundary_layout(B, K, smax, giant_at):
    """(bucket, entries) pairs in bucket order for a table (one group, window 0: digit v fills bucket v - 1).  `s` tasks are asked for
    as s K - 1 entries when K > 1, so that the tasks of a bucket are unequal (base / rem of k_accumulate)."""
    ent = lambda s: s * K - (1 if K > 1 and s > 0 else 0)
    GIANT = 2000
    lay, b, t = [], 0, 0

    def put(s, gap=0):
        nonlocal b, t
        b += gap
        lay.append((b, ent(s)))
        b += 1
        t += s

    def align(m):                                   # single-task buckets until the next bucket starts at task offset m mod 4
        while t % 4 != m:
            put(1)

    put(GIANT if giant_at == "first" else 1)        # bucket 0: digit 1
    align(0)
    for _ in range(4):                              # a run of four one-task buckets
        put(1)
    for m in range(4):                              # multi-task buckets that start at task offset 0, 1, 2, 3 mod 4
        align(m)
        put(2 + m)
    align(3)
    put(6); put(1); put(1); put(6)                  # the run [tail of a bucket, two whole buckets, head of a fourth]
    for s in (7, 8, 9):
        put(s)
    put(smax - 1, gap=1)                            # one empty bucket in front
    put(smax)
    put(smax + 1)                                   # the smallest giant
    put(3, gap=5)
    for j in range(1, GIANT_SLICES + 1):            # k_giant_finish cuts a giant into 16 slices of ceil(s / 16)
        put(16 * j - 1)
        put(16 * j + 1)
    if B >= 16384:
        put(2, gap=5000)                            # more than a whole k_plan tile of empty buckets
        put(5, gap=4096)
    if giant_at == "middle":
        put(GIANT)
        put(2)
    assert b < B - 1
    lay.append((B - 1, ent(GIANT if giant_at == "last" else 2)))      # digit 2^(c-1): the lone bucket of k_gridsum's extra row
    return lay


GIANT_SLICES = mp.GIANT_SLICES


def layout_scalars(lay):
    return [b + 1 for b, cnt in lay for _ in range(cnt)]


def check_boundary_facts(lay, p, r, giant_at):
    s_b = dict((b, int(r.s_b[b])) for b, _ in lay)
    assert {0, 1, 2, 3, 4, 5, 7, 8, 9, p.smax - 1, p.smax, p.smax + 1} <= set(r.s_b.tolist())
    assert {16 * j + d for j in range(1, 17) for d in (-1, 1)} <= set(s_b.values())
    multi = [b for b, _ in lay if s_b[b] >= 2]
    assert {int(r.task_off[b]) % 4 for b in multi} == {0, 1, 2, 3}
    off = r.task_off
    owner = np.searchsorted(off, np.arange(r.tasks), side="right") - 1       # bucket of every task
    runs = [(i, owner[i:i + 4]) for i in range(0, r.tasks - 3, 4)]                 # what one thread of k_run_sum sums
    assert any(len(set(q)) == 4 and all(r.s_b[x] == 1 for x in q) for _, q in runs)
    assert any(len(set(q)) == 4 and off[q[0]] < i and off[q[3] + 1] > i + 4 for i, q in runs)
    gaps = np.diff([b for b, _ in lay]) - 1
    assert 1 in gaps and 5 in gaps and (p.B < 16384 or gaps.max() > mp.PLAN_TILE)
    assert r.s_b[0] > 0 and r.s_b[p.B - 1] > 0
    assert 1 <= len(r.giants) <= mp.MAX_GIANTS and not r.overflow
    where = {"first": 0, "last": p.B - 1}.get(giant_at)
    if where is not None:
        assert where in r.giants
    elif giant_at == "middle":
        assert any(0 < x < p.B - 1 and r.s_b[x] >= 2000 for x in r.giants)


@pytest.mark.parametrize("giant_at", ["first", "middle", "last", "none"])
@pytest.mark.parametrize("chunk", [1, 3])
@pytest.mark.parametrize("wb", [16, 13], ids=["serial-table16", "quad-table13"])
def test_bucket_populations_at_the_boundaries(ctx, orc, pallas_srs, sms, wb, chunk, giant_at):
    srs = pallas_srs
    for smax in (32, 64, 128, 256):                 # smax depends on n, which depends on the layout: take the consistent one
        lay = boundary_layout(1 << (wb - 1), chunk, smax, giant_at)
        sc = layout_scalars(lay)
        p = mp.plan(len(sc), 1, wb, 0, sms, chunk)
        if p.smax == smax:
            break
    else:
        pytest.fail("no consistent smax")
    assert len(sc) <= len(srs.g) and p.many_buckets == (wb == 16) and p.K == chunk
    counts = mp.buckets([sc], p)
    assert [(b, int(counts[b])) for b in np.flatnonzero(counts)] == lay
    check_boundary_facts(lay, p, mp.regime(counts, p), giant_at)
    g = srs.g[:len(sc)]
    with ctx.upload_bases(srs.cid, g, window_bits=wb) as bases:
        with options(ctx, chunk):
            run(ctx, orc, srs, bases, g, sc, p)


@pytest.mark.parametrize("entries", [1, 5, 3000])
@pytest.mark.parametrize("wb", [16, 13], ids=["serial-table16", "quad-table13"])
def test_a_single_populated_bucket(ctx, orc, vesta_srs, sms, wb, entries):
    srs = vesta_srs
    g = srs.g[:entries]
    with ctx.upload_bases(srs.cid, g, window_bits=wb) as bases:
        for digit in (1, 1234, 1 << (wb - 1)):
            sc = [digit] * entries
            p = mp.plan(entries, 1, wb, 0, sms, 1)
            r = mp.regime(mp.buckets([sc], p), p)
            assert r.empty == p.NB - 1 and r.s_b[digit - 1] == entries and len(r.giants) == (entries > p.smax)
            with options(ctx, 1):
                run(ctx, orc, srs, bases, g, sc, p)


# ------------------------------------------------------------------------------------------ c. how many giants
def giants_scalars(p, count, extra=()):
    """`count` giant buckets (digits 2, 4, 6, ... of window 0, of sizes just above smax K) and a few ordinary ones"""
    pops = [(0, 2 * (i + 1), (p.smax + 1 + i % 7) * p.K) for i in range(count)] + [(0, 1, 1), (0, 3, 2 * p.K), (1, 5, 3)] + list(extra)
    return mp.scalars_for(pops, p.c)


def consistent(build, make_plan):
    """scalars and plan that agree on smax (it depends on n, and n on smax)"""
    p = make_plan(1)
    for _ in range(5):
        sc = build(p)
        n = len(sc[0]) if isinstance(sc[0], list) else len(sc)
        q = make_plan(n)
        if q.smax == p.smax:
            return sc, q
        p = q
    pytest.fail("no consistent smax")


@pytest.mark.parametrize("count", [0, 1, 2, 63, 64, 65, 100])
@pytest.mark.parametrize("wb", [16, 10], ids=["serial-table16", "quad-table10"])
def test_number_of_giant_buckets(ctx, orc, vesta_srs, sms, wb, count):
    srs = vesta_srs
    sc, p = consistent(lambda p: giants_scalars(p, count), lambda n: mp.plan(n, 1, wb, 0, sms, 1))
    r = mp.regime(mp.buckets([sc], p), p)
    assert len(r.giants) == count and r.overflow == (count > 64) and p.many_buckets == (wb == 16) and r.multi >= 1 and r.single >= 1
    g = srs.g[:p.n]
    with ctx.upload_bases(srs.cid, g, window_bits=wb) as bases:
        with options(ctx, 1):
            run(ctx, orc, srs, bases, g, sc, p)


@pytest.mark.parametrize("per_msm", [(0, 1, 20, 30), (0, 1, 30, 40)], ids=["51-giants", "71-giants-overflow"])
@pytest.mark.parametrize("wb", [16, 10], ids=["serial-table16", "quad-table10"])
def test_giants_spread_over_the_groups_of_a_fused_batch(ctx, orc, vesta_srs, sms, wb, per_msm):
    srs = vesta_srs

    def build(p):
        n = max(len(giants_scalars(p, c)) for c in per_msm)
        return [(giants_scalars(p, c) + [0] * n)[:n] for c in per_msm]

    sc, p = consistent(build, lambda n: mp.plan(n, len(per_msm), wb, 0, sms, 1))
    r = mp.regime(mp.buckets(sc, p), p)
    assert [int(np.sum(r.giants // p.B == j)) for j in range(p.k)] == list(per_msm) and r.overflow == (sum(per_msm) > 64)
    assert p.many_buckets == (wb == 16) and p.ntiles == (32 if wb == 16 else 1)
    g = srs.g[:p.n]
    with ctx.upload_bases(srs.cid, g, window_bits=wb) as bases:
        with options(ctx, 1):
            run(ctx, orc, srs, bases, g, sc, p)


@pytest.mark.parametrize("count", [3, 70])
@pytest.mark.parametrize("window", [10, 8], ids=["serial-plain10", "quad-plain8"])
def test_giants_spread_over_the_windows_of_a_plain_run(ctx, orc, pallas_srs, sms, window, count):
    srs = pallas_srs

    def build(p):        # giant i in window 3 i mod (nwin - 2), alternating signs
        pops = [((3 * i) % (p.nwin - 2), (7 + i) * (-1 if i % 2 else 1), p.smax + 1 + i % 5) for i in range(count)]
        return mp.scalars_for(pops + [(0, 1, 2), (p.nwin - 2, 3, 5)], p.c)

    sc, p = consistent(build, lambda n: mp.plan(n, 1, 0, window, sms, 1))
    r = mp.regime(mp.buckets([sc], p), p)
    assert len(r.giants) >= count and r.overflow == (count > 64) and len(set(r.giants // p.B)) > 2 and p.many_buckets == (window == 10)
    g = srs.g[:p.n]
    with ctx.upload_bases(srs.cid, g, window_bits=0) as bases:
        with options(ctx, 1):
            run(ctx, orc, srs, bases, g, sc, p, window_bits=window)


@pytest.mark.parametrize("wb", [16, 10], ids=["serial-table16", "quad-table10"])
def test_giant_list_starts_clean_after_an_overflow(ctx, orc, vesta_srs, sms, wb):
    """overflow -> one giant -> none -> one giant -> overflow on one context: the giant counter and the arrival tickets of one call
    leave nothing behind for the next"""
    srs = vesta_srs
    cases = {}
    for count in (65, 1, 0):
        cases[count] = consistent(lambda p: giants_scalars(p, count), lambda n: mp.plan(n, 1, wb, 0, sms, 1))
    with ctx.upload_bases(srs.cid, srs.g[:max(p.n for _, p in cases.values())], window_bits=wb) as bases:
        with options(ctx, 1):
            for count in (65, 1, 0, 1, 65):
                sc, p = cases[count]
                r = mp.regime(mp.buckets([sc], p), p)
                assert len(r.giants) == count and r.overflow == (count == 65)
                run(ctx, orc, srs, bases, srs.g, sc, p)


# ------------------------------------------------------------------------------------------ d. coinciding partials and buckets
def coinciding_case(orc, srs, c, K):
    """bases (copies of P = g[0], of -P, of the identity, and ordinary points) and scalars such that partial sums coincide in every
    addition of the finish and of the bucket reduction.  Returns (points, scalars, facts) for a table of window c (window 0 only)."""
    P, Q = srs.g[0], srs.g[1]
    nP, nQ = negated(orc, srs, P), negated(orc, srs, Q)
    zero = np.zeros(8, dtype=np.uint64)
    W = 1 << ((c - 1) // 2)
    pts, sc = [], []

    def fill(digit, points):
        for x in points:
            pts.append(x)
            sc.append(digit)

    fill(1, [P] * K + [P] * K)                            # two equal partials: the finish doubles
    fill(2, [P] * K + [nP] * K)                           # P, -P (any task split sums to the identity)
    fill(3, srs.g[2:4])                                   # spacer: shifts the next bucket's task offset
    fill(4, [P] * (2 * K) + [nP] * (2 * K))               # P, P, -P, -P
    fill(5, [srs.g[5]])
    fill(6, [P] * (2 * K) + [nP] * (2 * K))               # the same one task later: across a boundary of k_run_sum's runs of 4
    fill(7, [zero] * (3 * K))                             # only identity bases, several tasks
    fill(8, [zero])                                       # only the identity, one task
    fill(9, [P] * (1024 * K))                             # a giant of 2^10 equal partials: every level of the tree doubles
    fill(10, [P] * (600 * K) + [nP] * (600 * K))          # a giant that sums to the identity
    # k_gridsum: digit v sits in row v / W, column v % W
    r0 = 4 * W
    fill(r0 + 1, [Q]); fill(r0 + 2, [Q])                  # one row, equal sums
    fill(5 * W + 1, [Q])                                  # one column (with r0 + 1), equal sums
    fill(6 * W + 3, [Q, P]); fill(6 * W + 4, [nQ, nP])    # one row, opposite sums
    fill(7 * W + 5, [srs.g[6]]); fill(9 * W + 5, [negated(orc, srs, srs.g[6])])   # one column, opposite sums
    # k_gridsum_final: rows 10 and 11 (both have bit 1), columns W - 1 and W - 2 likewise: equal row / column sums
    fill(10 * W + W - 1, [srs.g[7]]); fill(11 * W + W - 2, [srs.g[7]])
    return np.stack(pts), sc


@pytest.mark.parametrize("chunk", [1, 2])
@pytest.mark.parametrize("wb", [16, 10], ids=["serial-table16", "quad-table10"])
def test_coinciding_partials_and_buckets(ctx, orc, pallas_srs, sms, wb, chunk):
    srs = pallas_srs
    g, sc = coinciding_case(orc, srs, wb, chunk)
    p = mp.plan(len(sc), 1, wb, 0, sms, chunk)
    r = mp.regime(mp.buckets([sc], p), p)
    assert p.many_buckets == (wb == 16) and p.K == chunk
    assert list(r.s_b[:10]) == [2, 2, 2 // chunk, 4, 1, 4, 3, 1, 1024, 1200] and list(r.giants) == [8, 9] and 1024 > p.smax
    # the two P, P, -P, -P buckets cross a boundary of k_run_sum's runs of 4 at different places
    assert r.task_off[3] % 4 != 0 and r.task_off[5] % 4 != 0 and r.task_off[3] % 4 != r.task_off[5] % 4
    with ctx.upload_bases(srs.cid, g, window_bits=wb) as bases:
        with options(ctx, chunk):
            run(ctx, orc, srs, bases, g, sc, p)


@pytest.mark.parametrize("wb,window", [(16, 0), (10, 0), (0, 9)], ids=["serial-table16", "quad-table10", "plain9"])
def test_groups_that_sum_to_the_identity(ctx, orc, vesta_srs, sms, wb, window):
    """every bucket holds P and -P: the whole MSM is the identity; without a table, also one window alone"""
    srs = vesta_srs
    m = 300
    g = np.concatenate([srs.g[:m], negated(orc, srs, srs.g[:m])])
    c = wb or window
    half = orc.limbs_to_ints(orc.random_scalars(srs.scalar, m, seed=5))
    with ctx.upload_bases(srs.cid, g, window_bits=wb) as bases:
        for chunk in (1, 2):
            p = mp.plan(2 * m, 1, wb, window, sms, chunk)
            with options(ctx, chunk):
                run(ctx, orc, srs, bases, g, half + half, p, window_bits=window)
                assert not ctx.msm_affine(bases, orc.ints_to_limbs(half + half), window_bits=window).any()
                if not wb:       # window 2 cancels, the others do not
                    low = [s % (1 << c) for s in half]
                    mixed = [a + (d << (2 * c)) for a, d in zip(low, low)] + [a + (1 << (3 * c)) + (d << (2 * c)) for a, d in zip(low, low)]
                    counts = mp.buckets([mixed], p)
                    assert counts[2 * p.B:3 * p.B].sum() > 0
                    run(ctx, orc, srs, bases, g, mixed, p, window_bits=window)


# ------------------------------------------------------------------------------------------ e. tables and windows
@pytest.mark.parametrize("table", [True, False], ids=["table", "plain"])
@pytest.mark.parametrize("c", range(2, 17))
def test_every_window_with_and_without_a_table(ctx, orc, pallas_srs, sms, c, table):
    """windows 2..7 take k_build_table (more than 33 rows), 8..16 k_build_table_batched; identity points among the bases; a slice at
    an offset (the table's row stride is the resident n, not the slice's); canonical and Montgomery scalars"""
    srs = pallas_srs
    assert (mp.num_windows(c) > 33) == (c < 8)
    N = 1000
    g = srs.g[:N].copy()
    g[[0, 30, 128, 999]] = 0
    sc = orc.random_scalars(srs.scalar, N, seed=c)
    sc[3] = orc.int_to_limbs(orc.MODULUS[srs.scalar] - 1)
    sc[4] = orc.int_to_limbs((1 << (c - 1)) + 1)
    with ctx.upload_bases(srs.cid, g, window_bits=c if table else 0) as bases:
        assert bases.window_bits == (c if table else 0)
        for n in (1, 31, 33, 127, 129, 1000):
            p = mp.plan(n, 1, bases.window_bits, c, sms)
            run(ctx, orc, srs, bases, g, orc.limbs_to_ints(sc[:n]), p, window_bits=0 if table else c)
        off, n = 127, 129
        p = mp.plan(n, 1, bases.window_bits, c, sms)
        run(ctx, orc, srs, bases, g, orc.limbs_to_ints(sc[:n]), p, window_bits=0 if table else c, off=off)
        mont = orc.to_mont(srs.scalar, sc[:n])
        assert np.array_equal(ctx.msm_affine(bases, mont, off=off, mont=True, window_bits=0 if table else c), orc.msm(srs.cid, g[off:off + n], sc[:n]))


# ------------------------------------------------------------------------------------------ f. gathered partials
def gathered(ctx, orc, srs, bases, d_sc, slices, window, p):
    """zk_msm_partial per (offset, scalar offset, n) slice, written side by side like an all-gather, then zk_msm_finish_gathered"""
    import torch
    cnt = p.c * p.gpm
    d_all = torch.zeros((len(slices), cnt, 16), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()           # torch fills on its stream, the context runs on its own
    for r, (off, s_off, n) in enumerate(slices):
        before = ctx.launch_count
        assert ctx.msm_partial(bases, d_sc.data_ptr() + 32 * s_off, n, d_all[r].data_ptr(), cnt, off=off, window_bits=window) == (p.c, p.gpm)
        assert ctx.launch_count - before == p.launches
    return zk.jacobian_to_affine(srs.cid, ctx.msm_finish_gathered(srs.cid, d_all.data_ptr(), len(slices), p.c, p.gpm))


@pytest.mark.parametrize("world", [1, 3, 8, 9, 17])
@pytest.mark.parametrize("wb,window", [(9, 0), (0, 7)], ids=["table9", "plain7"])
def test_gathered_partials_of_equal_slices(ctx, orc, vesta_srs, sms, wb, window, world):
    """k_sum_partials strides the ranks by its 8 quads: 1, 3, 8, 9 and 17 ranks"""
    import torch
    srs = vesta_srs
    m = 120
    n = world * m
    sc = orc.random_scalars(srs.scalar, n, seed=world)
    d_sc = torch.from_numpy(sc.view(np.int64)).cuda()
    with ctx.upload_bases(srs.cid, srs.g[:n], window_bits=wb) as bases:
        p = mp.plan(m, 1, bases.window_bits, window, sms)
        got = gathered(ctx, orc, srs, bases, d_sc, [(r * m, r * m, m) for r in range(world)], window, p)
        assert np.array_equal(got, orc.msm(srs.cid, srs.g[:n], sc))


@pytest.mark.parametrize("wb,window", [(9, 0), (0, 7)], ids=["table9", "plain7"])
def test_gathered_partials_that_coincide(ctx, orc, vesta_srs, sms, wb, window):
    """ranks whose slice sums are equal (the same slice twice), opposite (the negated points) and the identity (zero scalars)"""
    import torch
    srs = vesta_srs
    m = 120
    g = np.concatenate([srs.g[:m], negated(orc, srs, srs.g[:m])])
    sc = np.concatenate([orc.random_scalars(srs.scalar, m, seed=9), np.zeros((m, 4), dtype=np.uint64)])
    d_sc = torch.from_numpy(sc.view(np.int64)).cuda()
    A, NEG, ZERO = (0, 0, m), (m, 0, m), (0, m, m)
    want = {1: orc.msm(srs.cid, g[:m], sc[:m]), 2: orc.msm(srs.cid, np.concatenate([g[:m], g[:m]]), np.concatenate([sc[:m], sc[:m]])),
            0: np.zeros(8, dtype=np.uint64)}
    with ctx.upload_bases(srs.cid, g, window_bits=wb) as bases:
        p = mp.plan(m, 1, bases.window_bits, window, sms)
        for slices, mult in (([A, A], 2), ([A, NEG], 0), ([A, ZERO], 1), ([ZERO, A, A, NEG], 1), ([ZERO, ZERO, ZERO], 0),
                             ([A, A, NEG, NEG, A, ZERO, NEG, A, A, NEG], 1)):
            assert np.array_equal(gathered(ctx, orc, srs, bases, d_sc, slices, window, p), want[mult]), (slices, mult)


# ------------------------------------------------------------------------------------------ g. workspace reuse
def test_workspace_reuse_across_shapes(orc, pallas_srs, sms):
    """one context of its own, one pass: the scan tiles go 1 -> 8 -> 128 -> 1 -> 8 -> 11 -> 1 with plain and table bases interleaved and
    msm_chunk changed in between (chain flags re-allocated only when they grow, epoch stamps, scratch of a larger call under a
    smaller one)"""
    srs = pallas_srs
    n = 2048
    g = srs.g[:n]
    with zk.Context(0) as ctx:
        plain = ctx.upload_bases(srs.cid, g, window_bits=0)
        t16 = ctx.upload_bases(srs.cid, g, window_bits=16)
        t10 = ctx.upload_bases(srs.cid, g, window_bits=10)
        ones = [1] * (n - 3) + [0, 5, 7]          # one giant bucket
        rnd = lambda seed, m=n: orc.limbs_to_ints(orc.random_scalars(srs.scalar, m, seed=seed))
        steps = [(plain, 8, 1, 0, rnd(1), 1), (t16, 0, 1, 0, rnd(2), 8), (t16, 0, 16, 0, [rnd(10 + j) for j in range(16)], 128),
                 (t10, 0, 1, 1, ones, 1), (t16, 0, 1, 3, ones, 8), (plain, 12, 1, 2, rnd(3), 11), (t10, 0, 1, 0, rnd(4, 100), 1),
                 (t16, 0, 16, 1, [ones] + [rnd(30 + j) for j in range(15)], 128), (plain, 8, 1, 0, ones, 1)]
        for bases, window, k, chunk, sc, ntiles in steps:
            m = len(sc[0]) if k > 1 else len(sc)
            p = mp.plan(m, k, bases.window_bits, window, sms, chunk)
            assert p.ntiles == ntiles
            with options(ctx, chunk):
                run(ctx, orc, srs, bases, g, sc, p, window_bits=window)
