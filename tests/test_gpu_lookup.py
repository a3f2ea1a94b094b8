"""kimchi's lookup argument on the device (zk_lookup_joint_table_dev, zk_lookup_sorted_dev, zk_lookup_aggreg_dev) compared bit for bit
with the Python restatement (tests/lookup_replay.py) over both fields: the joint table with 1 and 3 columns, table ids and a runtime
column; sorted columns and the aggregation for m = 1, 3, 4, zk_rows of 3, 5 and n - 2, domains of 2^4 to 2^17 rows, the dummy first,
in the middle and last, kimchi's gates through by_row, one value hit by every lookup, missing values, a missing dummy, zero
denominators and a perturbed column; a chain from an index-cache image to the commitments; refusals; a caller's stream; two
threads on one context."""
import ctypes
import random
import threading

import numpy as np
import pytest
import torch

import evals_replay as ev
import lookup_replay as lr
import proof_systems_b200 as zk
from index_cache_writer import write_cache
from test_gpu_streams import Inputs, on_stream

pytestmark = pytest.mark.gpu

STALE = 0x0123456789ABCDEF


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


class Bufs:
    """device buffers of one test, freed at the end"""

    def __init__(self, ctx):
        self.ctx, self.ptrs = ctx, []

    def put(self, a):
        a = np.ascontiguousarray(a, dtype=np.uint64)
        p = self.ctx.dev_alloc(max(a.nbytes, 32))
        self.ptrs.append(p)
        if a.nbytes:
            self.ctx.dev_upload(p, a)
        return p

    def stale(self, n):
        return self.put(np.full((n, 4), STALE, dtype=np.uint64))

    def free(self):
        for p in self.ptrs:
            self.ctx.dev_free(p)


def mont(orc, fid, xs):
    return ev.mont(orc, fid, [int(x) for x in xs])


def spec_of(orc, fid, inst):
    """the instance's patterns as a LookupSpec (coefficients to Montgomery)"""
    s = zk.LookupSpec(fid, inst.m)
    for pat in inst.patterns:
        s.add_pattern([(tid, [[(None if c is None else mont(orc, fid, [c])[0], col, nxt) for c, col, nxt in e] for e in entries])
                       for tid, entries in pat])
    return s


def info_of(orc, fid, inst, row_pattern=None):
    sc = mont(orc, fid, [inst.jc, inst.tic, inst.dummy])
    return spec_of(orc, fid, inst).info(np.array(inst.row_pattern if row_pattern is None else row_pattern, dtype=np.uint8), *sc)


def table_strided(orc, fid, T1, stride, seed):
    """T1 as the device reads it: T1[i] at stride i, random elements elsewhere"""
    n = len(T1)
    out = orc.to_mont(fid, orc.random_scalars(fid, stride * n, seed=seed))
    out[::stride] = mont(orc, fid, T1)
    return np.ascontiguousarray(out)


def upload(orc, fid, inst, bufs, stride=1):
    d_w = [bufs.put(mont(orc, fid, c)) for c in inst.w]
    return d_w, bufs.put(table_strided(orc, fid, inst.T1, stride, 5))


def run_sorted(ctx, orc, fid, inst, d_w, d_t, stride, bufs, info=None):
    n = inst.n
    d_s = [bufs.stale(n) for _ in range(inst.m + 1)]
    row = ctx.lookup_sorted_dev(fid, n.bit_length() - 1, inst.zk_rows, d_w, d_t, stride, info or info_of(orc, fid, inst),
                                mont(orc, fid, inst.rand_sorted), d_s)
    return row, d_s, [ctx.dev_download(p, (n, 4)) for p in d_s]


def run_aggreg(ctx, orc, fid, inst, d_w, d_t, stride, d_s, bufs):
    n = inst.n
    d_a = bufs.stale(n)
    b, g = mont(orc, fid, [inst.beta, inst.gamma])
    ok = ctx.lookup_aggreg_dev(fid, n.bit_length() - 1, inst.zk_rows, d_w, d_t, stride, info_of(orc, fid, inst), d_s, b, g,
                               mont(orc, fid, inst.rand_agg), d_a)
    return ok, ctx.dev_download(d_a, (n, 4))


def stale_cols(k, n):
    return [np.full((n, 4), STALE, dtype=np.uint64)] * k


# ---------------------------------------------------------------------------------------------------------------- joint table
@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n", [4, 10, 16])
@pytest.mark.parametrize("n_cols,ids,runtime", [(1, False, False), (1, True, False), (3, False, False), (3, True, True), (3, False, True)])
def test_joint_table(ctx, orc, fid, log_n, n_cols, ids, runtime):
    P, m8 = orc.MODULUS[fid], 8 << log_n
    rng = random.Random(fid * 100 + log_n * 10 + n_cols)
    rnd = lambda seed: orc.to_mont(fid, orc.random_scalars(fid, m8, seed=seed))
    cols = [rnd(10 + c) for c in range(n_cols)]
    tid8 = rnd(20) if ids else None
    rt8 = rnd(21) if runtime else None
    jc, tic = rng.randrange(P), rng.randrange(P)
    ints = lambda a: ev.ints(orc, fid, a)
    want = mont(orc, fid, lr.joint_table([ints(c) for c in cols], jc, tic, P, ints(tid8) if ids else None, ints(rt8) if runtime else None))
    bufs = Bufs(ctx)
    try:
        d_c = [bufs.put(c) for c in cols]
        d8, d1 = bufs.stale(m8), bufs.stale(m8 // 8)
        ctx.lookup_joint_table_dev(fid, log_n, d_c, *mont(orc, fid, [jc, tic]), d8, bufs.put(tid8) if ids else None,
                                   bufs.put(rt8) if runtime else None, d1)
        assert np.array_equal(ctx.dev_download(d8, (m8, 4)), want)
        assert np.array_equal(ctx.dev_download(d1, (m8 // 8, 4)), want[::8])
    finally:
        bufs.free()


# ---------------------------------------------------------------------------------------------------------------- sorted + aggregation
CASES = [(4, 3, 1, "first", 1), (4, 5, 3, "middle", 8), (4, 14, 4, "last", 8), (6, 62, 3, "end", 1), (10, 3, 4, "end", 8),
         (10, 5, 1, "middle", 1), (12, 5, 4, "first", 8), (12, 3, 3, "last", 1), (16, 3, 4, "middle", 8), (17, 5, 4, "end", 8),
         # L + 1 = n - zk_rows just past, on and just before the 2048-row block boundary of the aggregation
         (12, 2047, 2, "first", 8), (12, 2048, 4, "end", 1), (12, 2049, 3, "middle", 8)]


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,zk_rows,m,where,stride", CASES)
def test_sorted_and_aggregation_match_the_reference(ctx, orc, fid, log_n, zk_rows, m, where, stride):
    P = orc.MODULUS[fid]
    inst = lr.instance(P, log_n, zk_rows, m, seed=1000 * fid + 10 * log_n + m, dummy_at=where)
    s = lr.sorted_patched(inst)
    agg, ok = lr.aggregation(inst, s)
    assert ok
    bufs = Bufs(ctx)
    try:
        d_w, d_t = upload(orc, fid, inst, bufs, stride)
        row, d_s, got = run_sorted(ctx, orc, fid, inst, d_w, d_t, stride, bufs)
        assert row == -1
        for k in range(m + 1):
            assert np.array_equal(got[k], mont(orc, fid, s[k])), k
        dok, got_a = run_aggreg(ctx, orc, fid, inst, d_w, d_t, stride, d_s, bufs)
        assert dok is True and np.array_equal(got_a, mont(orc, fid, agg))
    finally:
        bufs.free()


GATES = ["Xor16", "Lookup", "RangeCheck0", "RangeCheck1", "ForeignFieldMul", "Rot64", "Zero", "Generic"]


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("hot", [False, True])
def test_kimchi_gates_and_one_hot_value(ctx, orc, fid, hot):
    """rows from by_row over kimchi gates (ForeignFieldMul and RangeCheck1 on the next row too), or every lookup on one range-check
    value (all count increments on one address)"""
    P, log_n, zk_rows = orc.MODULUS[fid], 12, 3
    L = (1 << log_n) - zk_rows - 1
    rng = random.Random(fid)
    gates = ["RangeCheck0"] * L if hot else [rng.choice(GATES) for _ in range(L)]
    inst = lr.instance(P, log_n, zk_rows, 4, seed=7 + fid, gates=gates, hot=hot)
    s = lr.sorted_patched(inst)
    agg, ok = lr.aggregation(inst, s)
    bufs = Bufs(ctx)
    try:
        d_w, d_t = upload(orc, fid, inst, bufs, 8)
        row, d_s, got = run_sorted(ctx, orc, fid, inst, d_w, d_t, 8, bufs)
        assert row == -1 and all(np.array_equal(got[k], mont(orc, fid, s[k])) for k in range(5))
        dok, got_a = run_aggreg(ctx, orc, fid, inst, d_w, d_t, 8, d_s, bufs)
        assert ok and dok and np.array_equal(got_a, mont(orc, fid, agg))
    finally:
        bufs.free()


@pytest.mark.parametrize("fid", [0, 1])
def test_missing_values_report_the_smallest_row_and_write_nothing(ctx, orc, fid):
    P, log_n, zk_rows, m = orc.MODULUS[fid], 10, 5, 4
    for case in ("early", "last row", "two rows"):
        inst = lr.instance(P, log_n, zk_rows, m, seed=50 + fid)
        rng = random.Random(fid)
        L = inst.L
        syn = inst.names.index("synthetic") + 1
        rows = {"early": [2], "last row": [L - 1], "two rows": [L // 2, 7]}[case]
        for i in rows:
            inst.row_pattern[i] = syn
            assert lr.break_row(inst, i, rng)
        with pytest.raises(lr.ValueNotInTable) as e:
            lr.sorted_columns(inst)
        assert e.value.row == min(rows)
        bufs = Bufs(ctx)
        try:
            d_w, d_t = upload(orc, fid, inst, bufs, 1)
            row, _, got = run_sorted(ctx, orc, fid, inst, d_w, d_t, 1, bufs)
            assert row == min(rows), case
            assert all(np.array_equal(g, s) for g, s in zip(got, stale_cols(m + 1, inst.n))), case
        finally:
            bufs.free()


@pytest.mark.parametrize("fid", [0, 1])
def test_dummy_missing_while_padding_is_refused(ctx, orc, fid):
    P, log_n, zk_rows, m = orc.MODULUS[fid], 8, 3, 3
    inst = lr.instance(P, log_n, zk_rows, m, seed=60 + fid, dummy_at="last")
    L = inst.L
    inst.T1[L - 1] = inst.T1[0]                     # the only dummy row replaced by a duplicate: no lookup referred to it
    inst.row_pattern = [p if i != 3 else 0 for i, p in enumerate(inst.row_pattern)]
    with pytest.raises(lr.Malformed):
        lr.sorted_columns(inst)
    bufs = Bufs(ctx)
    try:
        d_w, d_t = upload(orc, fid, inst, bufs, 1)
        with pytest.raises(zk.ZkError) as e:
            run_sorted(ctx, orc, fid, inst, d_w, d_t, 1, bufs)
        assert e.value.code == -1 and "dummy" in str(e.value)
        got = [ctx.dev_download(p, (inst.n, 4)) for p in bufs.ptrs[-(m + 1):]]
        assert all(np.array_equal(g, s) for g, s in zip(got, stale_cols(m + 1, inst.n)))
    finally:
        bufs.free()


@pytest.mark.parametrize("fid", [0, 1])
def test_zero_denominators_and_a_perturbed_column(ctx, orc, fid):
    """the aggregation over sorted columns the caller changed: a zero den in the first row, the middle and row L - 1 (inverted to
    zero), and two unequal entries swapped (final value not one)"""
    P, log_n, zk_rows, m = orc.MODULUS[fid], 11, 5, 3
    inst = lr.instance(P, log_n, zk_rows, m, seed=70 + fid)
    L = inst.L
    rng = random.Random(fid)
    s0 = lr.sorted_patched(inst)
    variants = []
    for row in (0, L // 2, L - 1):
        s = [list(c) for c in s0]
        lr.zero_denominator(inst, s, row, rng)
        variants.append((f"zero den at {row}", s))
    s = [list(c) for c in s0]
    a, b = next((a, b) for a in range(L) for b in range(a + 1, L) if s[2][a] != s[2][b])
    s[2][a], s[2][b] = s[2][b], s[2][a]
    variants.append(("swapped", s))
    bufs = Bufs(ctx)
    try:
        d_w, d_t = upload(orc, fid, inst, bufs, 1)
        for name, s in variants:
            want, ok = lr.aggregation(inst, s)
            d_s = [bufs.put(mont(orc, fid, c)) for c in s]
            dok, got = run_aggreg(ctx, orc, fid, inst, d_w, d_t, 1, d_s, bufs)
            assert dok == ok and not ok, name
            assert np.array_equal(got, mont(orc, fid, want)), name
    finally:
        bufs.free()


# ---------------------------------------------------------------------------------------------------------------- the chain
def test_chain_from_an_index_cache_to_the_commitments(ctx, orc, pallas_srs):
    """sections 0x50 (the table's 3 columns over d8, packed) and 0x51 (table ids) of a cache image -> joint table -> sorted ->
    aggregation -> zk_msm_dev of the m + 2 resident columns over the Lagrange basis, against the oracle's MSM"""
    G = pallas_srs
    fid, log_n, zk_rows, m = G.scalar, 8, 3, 4
    P, n = orc.MODULUS[fid], 1 << log_n
    L = n - zk_rows - 1
    table = lr.make_tables(random.Random(4), P, L - 5) + [(lr.XOR_TABLE_ID, [0, 0, 0])] * 5      # kimchi: zero padding at the end
    inst = lr.instance(P, log_n, zk_rows, m, seed=81, table=table)
    cols1 = [[c[k] for _, c in table] + [0] * (n - L) for k in range(3)]
    ids1 = [tid % P for tid, _ in table] + [0] * (n - L)
    T1 = [lr.combine([cols1[k][i] for k in range(3)], inst.jc, inst.tic, ids1[i], P) for i in range(n)]
    assert inst.T1[:L + 1] == T1[:L + 1]
    inst.T1 = T1
    s = lr.sorted_patched(inst)
    agg, ok = lr.aggregation(inst, s)
    assert ok

    def d8(vals):
        c = orc.ntt(fid, mont(orc, fid, vals), inverse=True)
        pad = np.zeros((8 * n, 4), dtype=np.uint64)
        pad[:n] = c
        return orc.ntt(fid, pad)

    zeros8 = bytes(8 * n * 32)                 # coefficients8 and permutation_coefficients8: sections every cache must carry
    sections = ([(0x10 + i, zeros8, 8 * n) for i in range(15)] + [(0x30 + i, zeros8, 8 * n) for i in range(7)] +
                [(0x50, np.concatenate([d8(c) for c in cols1]).astype("<u8").tobytes(), 8 * n), (0x51, d8(ids1).astype("<u8").tobytes(), 8 * n)])
    header = {"public": 0, "prev_challenges": 0, "zk_rows": zk_rows, "max_poly_size": n, "domain_d1_size": n, "lookup_selectors_present": 1,
              "endo_limbs": [0] * 4, "shift_limbs": [[0] * 4] * 7}
    cache = zk.IndexCache(ctx, write_cache("lookup-chain", header, sections))
    bufs = Bufs(ctx)
    lag = G.lagrange_small(n)
    bases = ctx.upload_bases(G.cid, lag)
    try:
        p50, n50, dom50 = cache.section(0x50)
        p51, _, _ = cache.section(0x51)
        assert n50 == 3 * 8 * n and dom50 == 8 * n
        d_t8, d_t1 = bufs.stale(8 * n), bufs.stale(n)
        ctx.lookup_joint_table_dev(fid, log_n, [p50 + k * 8 * n * 32 for k in range(3)], *mont(orc, fid, [inst.jc, inst.tic]), d_t8, p51, None, d_t1)
        assert np.array_equal(ctx.dev_download(d_t1, (n, 4)), mont(orc, fid, T1))
        d_w = [bufs.put(mont(orc, fid, c)) for c in inst.w]
        row, d_s, got = run_sorted(ctx, orc, fid, inst, d_w, d_t8, 8, bufs)
        assert row == -1 and all(np.array_equal(got[k], mont(orc, fid, s[k])) for k in range(m + 1))
        d_a = bufs.stale(n)
        b, g = mont(orc, fid, [inst.beta, inst.gamma])
        assert ctx.lookup_aggreg_dev(fid, log_n, zk_rows, d_w, d_t8, 8, info_of(orc, fid, inst), d_s, b, g, mont(orc, fid, inst.rand_agg), d_a)
        assert np.array_equal(ctx.dev_download(d_a, (n, 4)), mont(orc, fid, agg))
        for k, (d, col) in enumerate(zip(d_s + [d_a], s + [agg])):
            com = zk.jacobian_to_affine(G.cid, ctx.msm_dev(bases, d, n, mont=True))
            assert np.array_equal(com, orc.msm_mont(G.cid, lag, mont(orc, fid, col))), k
    finally:
        bases.free()
        bufs.free()
        cache.close()


# ---------------------------------------------------------------------------------------------------------------- refusals
def test_refusals_leave_the_outputs_untouched(ctx, orc):
    fid, log_n, zk_rows, m = zk.FQ, 6, 4, 3
    P, n = orc.MODULUS[fid], 1 << log_n
    inst = lr.instance(P, log_n, zk_rows, m, seed=90)
    L = inst.L
    bad = np.array([P & (2**64 - 1), (P >> 64) & (2**64 - 1), (P >> 128) & (2**64 - 1), P >> 192], dtype=np.uint64)
    bufs = Bufs(ctx)
    try:
        d_w, d_t = upload(orc, fid, inst, bufs, 1)
        d_s = [bufs.stale(n) for _ in range(m + 1)]
        d_a = bufs.stale(n)
        rs, ra = mont(orc, fid, inst.rand_sorted), mont(orc, fid, inst.rand_agg)
        b, g = mont(orc, fid, [inst.beta, inst.gamma])
        spec = spec_of(orc, fid, inst)
        sc = list(mont(orc, fid, [inst.jc, inst.tic, inst.dummy]))

        def info(rows=None, mm=None, jc=None, dummy=None):
            i = spec.info(np.array(inst.row_pattern if rows is None else rows, dtype=np.uint8), jc if jc is not None else sc[0], sc[1],
                          dummy if dummy is not None else sc[2])
            if mm is not None:
                i.max_per_row = mm
            return i

        def untouched():
            return all(np.array_equal(ctx.dev_download(p, (n, 4)), stale_cols(1, n)[0]) for p in d_s + [d_a])

        rs_bad = rs.copy()
        rs_bad[-1] = bad
        bad_rows = list(inst.row_pattern)
        bad_rows[5] = len(inst.patterns) + 1
        cases = [dict(field=7), dict(log_n=31), dict(zk_rows=0), dict(zk_rows=n - 1), dict(zk_rows=n), dict(stride=0), dict(stride=9),
                 dict(info=info(mm=0)), dict(info=info(mm=9)), dict(info=info(mm=2)), dict(info=info(rows=bad_rows)), dict(info=info(jc=bad)),
                 dict(info=info(dummy=bad)), dict(rs=rs_bad), dict(d_s=[d_w[3]] + d_s[1:]), dict(d_s=d_s[:2] + [d_t] + d_s[3:]),
                 dict(d_s=[d_s[0], d_s[0] + 32 * (n - 1)] + d_s[2:]), dict(d_s=d_s[:3] + [0])]
        for kw in cases:
            a = dict(field=fid, log_n=log_n, zk_rows=zk_rows, stride=1, info=info(), rs=rs, d_s=d_s)
            a.update(kw)
            with pytest.raises(zk.ZkError) as e:
                ctx.lookup_sorted_dev(a["field"], a["log_n"], a["zk_rows"], d_w, d_t, a["stride"], a["info"], a["rs"], a["d_s"])
            assert e.value.code == -1, kw
        ra_bad = ra.copy()
        ra_bad[0] = bad
        for kw in [dict(field=7), dict(zk_rows=n - 1), dict(beta=bad), dict(gamma=bad), dict(ra=ra_bad), dict(d_a=d_w[0]), dict(d_a=d_s[2]),
                   dict(d_a=d_t + 32), dict(info=info(mm=9)), dict(stride=0)]:
            a = dict(field=fid, zk_rows=zk_rows, beta=b, gamma=g, ra=ra, d_a=d_a, info=info(), stride=1)
            a.update(kw)
            with pytest.raises(zk.ZkError) as e:
                ctx.lookup_aggreg_dev(a["field"], log_n, a["zk_rows"], d_w, d_t, a["stride"], a["info"], d_s, a["beta"], a["gamma"], a["ra"], a["d_a"])
            assert e.value.code == -1, kw
        assert untouched()
        # the lookup info's own checks: a term column, next, entries, a table id column, a pattern larger than m or out of range
        L_ = zk.lib()
        for field, val in (("column", 15), ("next", 2)):
            i = info()
            setattr(i.terms[0], field, val)
            with pytest.raises(zk.ZkError):
                ctx.lookup_sorted_dev(fid, log_n, zk_rows, d_w, d_t, 1, i, rs, d_s)
        for field, val in (("n_entries", 5), ("table_id_column", 15), ("table_id_column", -2), ("first_term", 10**6)):
            i = info()
            setattr(i.lookups[0], field, val)
            with pytest.raises(zk.ZkError):
                ctx.lookup_sorted_dev(fid, log_n, zk_rows, d_w, d_t, 1, i, rs, d_s)
        i = info()
        i.pattern_first[0] = 10**6
        with pytest.raises(zk.ZkError):
            ctx.lookup_sorted_dev(fid, log_n, zk_rows, d_w, d_t, 1, i, rs, d_s)
        i = info()
        i.terms[0].coeff[:] = [int(x) for x in bad]
        with pytest.raises(zk.ZkError):
            ctx.lookup_sorted_dev(fid, log_n, zk_rows, d_w, d_t, 1, i, rs, d_s)
        # null pointers through the C ABI
        i = info()
        pw = (ctypes.c_void_p * 15)(*d_w)
        ps = (ctypes.c_void_p * (m + 1))(*d_s)
        row = ctypes.c_int64(7)
        full = [ctx._h, fid, log_n, zk_rows, pw, ctypes.c_void_p(d_t), 1, ctypes.byref(i), rs.ctypes.data, ps, ctypes.byref(row)]
        for pos in (0, 4, 5, 7, 8, 9, 10):
            args = list(full)
            args[pos] = None
            assert L_.zk_lookup_sorted_dev(*args) == -1, pos
        assert row.value == 7 and untouched()
        # the joint table's refusals
        m8 = 8 * n
        cols = [bufs.put(orc.to_mont(fid, orc.random_scalars(fid, m8, seed=k))) for k in range(3)]
        d8 = bufs.stale(m8)
        jc, tic = sc[0], sc[1]
        for kw in [dict(field=7), dict(log_n=31), dict(cols=[]), dict(cols=cols[:1], rt=cols[1]), dict(jc=bad), dict(tic=bad), dict(out8=cols[2]),
                   dict(out8=cols[0] + 32 * 5), dict(out1=d8 + 32), dict(out1=cols[1]), dict(ids=d8)]:
            a = dict(field=fid, log_n=log_n, cols=cols, jc=jc, tic=tic, out8=d8, ids=None, rt=None, out1=None)
            a.update(kw)
            with pytest.raises(zk.ZkError) as e:
                ctx.lookup_joint_table_dev(a["field"], a["log_n"], a["cols"], a["jc"], a["tic"], a["out8"], a["ids"], a["rt"], a["out1"])
            assert e.value.code == -1, kw
        assert np.array_equal(ctx.dev_download(d8, (m8, 4)), stale_cols(1, m8)[0])
        # the valid edges: zk_rows = n - 2 (one lookup row), strides 1 .. 8
        edge = lr.instance(P, log_n, n - 2, m, seed=91)
        row0, _, _ = run_sorted(ctx, orc, fid, edge, *upload(orc, fid, edge, bufs, 1), 1, bufs)
        assert row0 == -1
    finally:
        bufs.free()


# ---------------------------------------------------------------------------------------------------------------- streams, threads
def test_all_three_calls_on_a_callers_stream(orc):
    """inputs copied in behind a spin kernel on the caller's stream: any of the three calls running elsewhere reads zeros"""
    stream = torch.cuda.Stream()
    c = zk.Context(0)
    c.set_stream(stream.cuda_stream)
    try:
        fid, log_n, zk_rows, m = zk.FP, 10, 3, 4
        P, n = orc.MODULUS[fid], 1 << log_n
        inst = lr.instance(P, log_n, zk_rows, m, seed=100)
        s = lr.sorted_patched(inst)
        agg, _ = lr.aggregation(inst, s)
        cols = [orc.to_mont(fid, orc.random_scalars(fid, 8 * n, seed=k)) for k in range(2)]
        jt = lr.joint_table([ev.ints(orc, fid, x) for x in cols], inst.jc, inst.tic, P)
        inp = Inputs()
        d_c = [inp(x) for x in cols]
        d_w = [inp(mont(orc, fid, col)) for col in inst.w]
        d_t = inp(mont(orc, fid, inst.T1))
        out8 = torch.full((8 * n, 4), STALE, dtype=torch.int64, device="cuda")
        d_s = [torch.full((n, 4), STALE, dtype=torch.int64, device="cuda") for _ in range(m + 1)]
        d_a = torch.full((n, 4), STALE, dtype=torch.int64, device="cuda")
        info = info_of(orc, fid, inst)
        b, g = mont(orc, fid, [inst.beta, inst.gamma])

        def calls():
            c.lookup_joint_table_dev(fid, log_n, d_c, *mont(orc, fid, [inst.jc, inst.tic]), out8.data_ptr())
            row = c.lookup_sorted_dev(fid, log_n, zk_rows, d_w, d_t, 1, info, mont(orc, fid, inst.rand_sorted), [t.data_ptr() for t in d_s])
            ok = c.lookup_aggreg_dev(fid, log_n, zk_rows, d_w, d_t, 1, info, [t.data_ptr() for t in d_s], b, g, mont(orc, fid, inst.rand_agg),
                                     d_a.data_ptr())
            return row, ok

        (row, ok), got = on_stream(stream, inp, calls, [out8] + d_s + [d_a])
        assert row == -1 and ok
        assert np.array_equal(got[0], mont(orc, fid, jt))
        for k in range(m + 1):
            assert np.array_equal(got[1 + k], mont(orc, fid, s[k])), k
        assert np.array_equal(got[-1], mont(orc, fid, agg))
    finally:
        c.close()


def test_two_threads_share_a_context(ctx, orc):
    fid, log_n, zk_rows, m = zk.FQ, 11, 5, 4
    P, n = orc.MODULUS[fid], 1 << log_n
    bufs, cases, errors = Bufs(ctx), [], []
    for t in range(2):
        inst = lr.instance(P, log_n, zk_rows, m - t, seed=200 + t)
        s = lr.sorted_patched(inst)
        agg, _ = lr.aggregation(inst, s)
        d_w, d_t = upload(orc, fid, inst, bufs, 1)
        cases.append((inst, d_w, d_t, s, agg))

    def work(t):
        try:
            inst, d_w, d_t, s, agg = cases[t]
            mine = Bufs(ctx)
            try:
                for _ in range(4):
                    row, d_s, got = run_sorted(ctx, orc, fid, inst, d_w, d_t, 1, mine)
                    assert row == -1 and all(np.array_equal(got[k], mont(orc, fid, s[k])) for k in range(inst.m + 1))
                    ok, got_a = run_aggreg(ctx, orc, fid, inst, d_w, d_t, 1, d_s, mine)
                    assert ok and np.array_equal(got_a, mont(orc, fid, agg))
            finally:
                mine.free()
        except Exception as e:                    # reported by the main thread
            errors.append(e)

    try:
        th = [threading.Thread(target=work, args=(t,)) for t in range(2)]
        for t in th:
            t.start()
        for t in th:
            t.join()
    finally:
        bufs.free()
    assert not errors, errors
