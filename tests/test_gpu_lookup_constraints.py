"""The device's lookup argument against kimchi's own lookup constraints (tests/lookup_constraints.py): zk_lookup_sorted_dev and
zk_lookup_aggreg_dev give the sorted columns and agg over d1; zk_ntt_dev_oop takes every column to d8; zk_expr_eval_dev evaluates each
entry of lookup::constraints::constraints into its own buffer and, scaled by its alpha power, into one t8 (prover.rs:874-902); each
result is compared bit for bit with oracle.expr_eval and, after iFFT(8n), must divide exactly by Z_H (zk_poly_divide_by_vanishing_dev).
`verify` (constraints.rs:690-796) checks the downloaded sorted columns, and the device's final-value flag must agree with the final-value
entry.  Degree bound: with m <= 4 the largest term has degree zk_rows + 1 + (m + 3)(n - 1) < 8n, so d8 holds every entry exactly.

Cases: both fields; the sorted-and-aggregation shapes of test_gpu_lookup (L + 1 around the 2048-row aggregation block, zk_rows = n - 2,
2^4 to 2^17 rows); kimchi's gates through by_row at 2^12 and 2^16, and one value hit by every lookup; the chain from an index-cache image
with the table, its ids and the four pattern selectors read from the cache's sections; no table ids; and the perturbations of
lookup_constraints.NEGATIVE, agg recomputed on the device, each failing exactly its entries."""
import random

import numpy as np
import pytest

import evals_replay as ev
import gate_programs as gp
import lookup_constraints as lc
import lookup_replay as lr
import proof_systems_b200 as zk
from index_cache_writer import write_cache
from test_gpu_lookup import CASES, GATES, Bufs, info_of, mont

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def lit_of(orc, fid):
    return lambda v: ev.mont(orc, fid, [v])[0]


def to_d8(ctx, fid, log_n, d1, k, bufs):
    """k contiguous d1 columns -> k contiguous d8 columns: iFFT(n), then FFT(8n) with in_len = n"""
    n = 1 << log_n
    coef, out = bufs.stale(k * n), bufs.stale(k * 8 * n)
    ctx.ntt_dev_oop(fid, d1, n, n, coef, log_n, batch=k, inverse=True)
    ctx.ntt_dev_oop(fid, coef, n, n, out, log_n + 3, batch=k)
    return out


def run(ctx, orc, fid, inst, bufs, patterns=None, table8=None, selectors8=None, device_tic=None, kind=None):
    """the device chain for one instance; table8 / selectors8: device pointers of d8 columns taken as given (else built from the
    instance over d1); device_tic: the table id combiner handed to the lookup calls (the instance's by default); kind: a
    lookup_constraints.NEGATIVE perturbation.  Returns (per-entry divisibility, t8 divisibility, final_is_one, verify's verdict,
    the aggregation entry's nonzero rows of d1)."""
    P, n, m = inst.P, inst.n, inst.m
    log_n, m8, B = n.bit_length() - 1, 8 * n, 32
    cfg = lc.of_instance(inst, lit_of(orc, fid), patterns)
    n_pat = len(cfg.patterns)
    w1 = bufs.put(np.concatenate([mont(orc, fid, c) for c in inst.w]))
    d_w = [w1 + k * n * B for k in range(15)]
    if table8 is None:
        table8 = to_d8(ctx, fid, log_n, bufs.put(mont(orc, fid, inst.T1)), 1, bufs)
    tic = inst.tic if device_tic is None else device_tic
    info = info_of(orc, fid, inst)
    info.table_id_combiner[:] = [int(x) for x in mont(orc, fid, [tic])[0]]
    sa1 = bufs.stale((m + 2) * n)
    d_s = [sa1 + k * n * B for k in range(m + 1)]
    d_a = sa1 + (m + 1) * n * B
    assert ctx.lookup_sorted_dev(fid, log_n, inst.zk_rows, d_w, table8, 8, info, mont(orc, fid, inst.rand_sorted), d_s) == -1
    row = None
    if kind is not None and kind != "agg scaled":
        s, row = lc.perturb(inst, [ev.ints(orc, fid, ctx.dev_download(p, (n, 4))) for p in d_s], kind)
        ctx.dev_upload(sa1, np.concatenate([mont(orc, fid, c) for c in s]))
    b, g = mont(orc, fid, [inst.beta, inst.gamma])
    final_is_one = ctx.lookup_aggreg_dev(fid, log_n, inst.zk_rows, d_w, table8, 8, info, d_s, b, g, mont(orc, fid, inst.rand_agg), d_a)
    if kind == "agg scaled":
        agg = ev.ints(orc, fid, ctx.dev_download(d_a, (n, 4)))
        ctx.dev_upload(d_a, mont(orc, fid, [lc.SCALE * a % P for a in agg]))
    # every column over d8, in the program's order
    w8 = to_d8(ctx, fid, log_n, w1, 15, bufs)
    if selectors8 is None:
        sel1 = [[1 if r < inst.L and inst.row_pattern[r] == k + 1 else 0 for r in range(n)] for k in range(n_pat)]
        sel = to_d8(ctx, fid, log_n, bufs.put(np.concatenate([mont(orc, fid, c) for c in sel1])), n_pat, bufs)
        selectors8 = [sel + k * m8 * B for k in range(n_pat)]
    sa8 = to_d8(ctx, fid, log_n, sa1, m + 2, bufs)
    env = lc.env_d8(orc, fid, log_n, inst.zk_rows)
    ptrs = ([w8 + k * m8 * B for k in range(15)] + list(selectors8) + [table8] + [sa8 + k * m8 * B for k in range(m + 2)] +
            [bufs.put(e) for e in env])
    assert len(ptrs) == cfg.n_columns
    cols = [(p, m8, 8) for p in ptrs]
    # each entry into its own buffer, and alpha-scaled into t8
    alphas = [random.Random(n + fid).randrange(1, P) for _ in lc.ENTRIES]
    scaled = lc.constraints(zk.ExprProgram, cfg)
    d_e, d_t8 = [bufs.stale(m8) for _ in lc.ENTRIES], bufs.put(np.zeros((m8, 4), dtype=np.uint64))
    for prog, sp, a, d in zip(lc.constraints(zk.ExprProgram, cfg), scaled, alphas, d_e):
        prog.evaluations(ctx, fid, cols, m8, 8, d)
        sp.literal(mont(orc, fid, [a])[0]).mul().evaluations(ctx, fid, cols, m8, 8, d_t8, accumulate=True)
    got = [ctx.dev_download(d, (m8, 4)) for d in d_e]
    got_t8 = ctx.dev_download(d_t8, (m8, 4))
    host8 = [ctx.dev_download(p, (m8, 4)) for p in ptrs]
    want = lc.oracle_evals(orc, fid, lc.constraints(gp.Recorder, cfg), host8)
    del host8
    for name, gt, wt in zip(lc.ENTRIES, got, want):
        assert np.array_equal(gt, wt), name
    comb = gp.Recorder()
    for k, a in enumerate(alphas):
        comb.cell(k).literal(mont(orc, fid, [a])[0]).mul()
        if k:
            comb.add()
    assert np.array_equal(got_t8, orc.expr_eval(fid, comb.ops, comb.args, comb.literals, [(e, 1) for e in want], m8))
    bad_rows = [r for r in range(n) if got[0][8 * r].any()]
    # iFFT(8n), then the division by Z_H on the device
    d_q = bufs.stale(m8)
    div = []
    for d in d_e + [d_t8]:
        ctx.ntt_dev(fid, d, log_n + 3, inverse=True)
        div.append(ctx.poly_divide_by_vanishing_dev(fid, d, m8, log_n, d_q))
    s_now = [ev.ints(orc, fid, ctx.dev_download(p, (n, 4))) for p in d_s]
    return div[:-1], div[-1], final_is_one, lc.verify(inst, s_now), bad_rows, row


def check_honest(res, kind="honest"):
    div, div_t8, final_is_one, verdict, bad_rows, _ = res
    assert all(div), (kind, [e for e, d in zip(lc.ENTRIES, div) if not d])
    assert div_t8 and final_is_one is True and verdict is None and bad_rows == []


# ---------------------------------------------------------------------------------------------------------------- honest instances
@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,zk_rows,m,where,stride", CASES)
def test_the_device_lookup_argument_satisfies_the_constraints(ctx, orc, fid, log_n, zk_rows, m, where, stride):
    """stride 8: the lookup calls read the table from its d8 evaluations, as the prover's lookup_table8; stride 1 cases do too
    here, since the constraints need the table over d8 anyway"""
    inst = lr.instance(orc.MODULUS[fid], log_n, zk_rows, m, seed=1000 * fid + 10 * log_n + m, dummy_at=where, tic="kimchi")
    bufs = Bufs(ctx)
    try:
        check_honest(run(ctx, orc, fid, inst, bufs))
    finally:
        bufs.free()


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,hot", [(12, False), (12, True), (16, False)])
def test_kimchi_gates_and_one_hot_value(ctx, orc, fid, log_n, hot):
    """rows from by_row over kimchi's gates (2^16: the prover's size), or every lookup on one range-check value"""
    P, zk_rows = orc.MODULUS[fid], 3
    L = (1 << log_n) - zk_rows - 1
    rng = random.Random(fid + log_n)
    gates = ["RangeCheck0"] * L if hot else [rng.choice(GATES) for _ in range(L)]
    inst = lr.instance(P, log_n, zk_rows, 4, seed=7 + fid + log_n, gates=gates, hot=hot, tic="kimchi")
    bufs = Bufs(ctx)
    try:
        check_honest(run(ctx, orc, fid, inst, bufs))
    finally:
        bufs.free()


def test_no_table_ids(ctx, orc):
    """kimchi's prover hands the lookup calls table_id_combiner = 0 when the index has no table ids (prover.rs:480-486), while the
    constraints still use jc^max_joint_size: the two agree only because every table id and every lookup's id is then 0, as here
    (XOR rows and the dummy, Xor16 gates only)"""
    fid, log_n, zk_rows, m = zk.FQ, 10, 5, 4
    P, n = orc.MODULUS[fid], 1 << log_n
    L = n - zk_rows - 1
    rng = random.Random(3)
    table = [(lr.XOR_TABLE_ID, [a, b, a ^ b]) for a, b in ((rng.randrange(16), rng.randrange(16)) for _ in range(L - 9))]
    table += [(lr.XOR_TABLE_ID, [0, 0, 0])] * 9
    inst = lr.instance(P, log_n, zk_rows, m, seed=31, gates=["Xor16"] * L, table=table, tic=0)
    assert inst.tic == 0 and any(inst.row_pattern)
    bufs = Bufs(ctx)
    try:
        check_honest(run(ctx, orc, fid, inst, bufs, device_tic=0))
    finally:
        bufs.free()


def test_chain_from_an_index_cache(ctx, orc, pallas_srs):
    """sections 0x50 (the table's 3 columns over d8) and 0x51 (table ids) -> zk_lookup_joint_table_dev -> the lookup calls and the
    table column; the four pattern selectors (xor, lookup, range_check, ffmul) read from sections 0x52 - 0x55
    (cached_prover_index.rs:122-134)"""
    fid, log_n, zk_rows, m = pallas_srs.scalar, 8, 3, 4
    P, n = orc.MODULUS[fid], 1 << log_n
    L = n - zk_rows - 1
    table = lr.make_tables(random.Random(4), P, L - 5) + [(lr.XOR_TABLE_ID, [0, 0, 0])] * 5
    rng = random.Random(5)
    inst = lr.instance(P, log_n, zk_rows, m, seed=82, table=table, gates=[rng.choice(GATES) for _ in range(L)], tic="kimchi")
    kimchi = [inst.patterns[inst.names.index(p)] for p in zk.LookupSpec.KIMCHI_PATTERNS]
    assert inst.names[:4] == list(zk.LookupSpec.KIMCHI_PATTERNS) and lr.max_joint_size(kimchi) == lr.max_joint_size(inst.patterns)
    cols1 = [[c[k] for _, c in table] + [0] * (n - L) for k in range(3)]
    ids1 = [tid % P for tid, _ in table] + [0] * (n - L)
    sel1 = [[1 if r < L and inst.row_pattern[r] == k + 1 else 0 for r in range(n)] for k in range(4)]
    d8 = lambda vals: lc.to_d8(orc, fid, vals).astype("<u8").tobytes()
    zeros8 = bytes(8 * n * 32)
    sections = ([(0x10 + i, zeros8, 8 * n) for i in range(15)] + [(0x30 + i, zeros8, 8 * n) for i in range(7)] +
                [(0x50, b"".join(d8(c) for c in cols1), 8 * n), (0x51, d8(ids1), 8 * n)] +
                [(0x52 + k, d8(sel1[k]), 8 * n) for k in range(4)])
    header = {"public": 0, "prev_challenges": 0, "zk_rows": zk_rows, "max_poly_size": n, "domain_d1_size": n,
              "lookup_selectors_present": 0x1F, "endo_limbs": [0] * 4, "shift_limbs": [[0] * 4] * 7}
    cache = zk.IndexCache(ctx, write_cache("lookup-constraints", header, sections))
    bufs = Bufs(ctx)
    try:
        p50, _, _ = cache.section(0x50)
        p51, _, _ = cache.section(0x51)
        sel8 = []
        for k in range(4):
            p, cnt, dom = cache.section(0x52 + k)
            assert cnt == 8 * n and dom == 8 * n
            sel8.append(p)
        d_t8, d_t1 = bufs.stale(8 * n), bufs.stale(n)
        ctx.lookup_joint_table_dev(fid, log_n, [p50 + k * 8 * n * 32 for k in range(3)], *mont(orc, fid, [inst.jc, inst.tic]), d_t8, p51,
                                   None, d_t1)
        inst.T1 = ev.ints(orc, fid, ctx.dev_download(d_t1, (n, 4)))
        check_honest(run(ctx, orc, fid, inst, bufs, patterns=kimchi, table8=d_t8, selectors8=sel8))
    finally:
        bufs.free()
        cache.close()


# ---------------------------------------------------------------------------------------------------------------- negative cases
@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("kind", list(lc.NEGATIVE))
def test_each_perturbation_fails_exactly_its_constraints(ctx, orc, fid, kind):
    inst = lr.instance(orc.MODULUS[fid], 10, 5, 4, seed=600 + fid, tic="kimchi")
    must_fail, verdict = lc.NEGATIVE[kind]
    bufs = Bufs(ctx)
    try:
        div, div_t8, final_is_one, got_verdict, bad_rows, row = run(ctx, orc, fid, inst, bufs, kind=kind)
    finally:
        bufs.free()
    assert {e for e, d in zip(lc.ENTRIES, div) if not d} == must_fail
    assert not div_t8 and got_verdict == verdict
    assert bad_rows == ([] if row is None else [row])
    # the device's flag is about the agg it computed: for "agg scaled" that agg was honest, and the scaling came after
    assert final_is_one is (kind == "agg scaled")
