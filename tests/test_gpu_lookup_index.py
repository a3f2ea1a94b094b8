"""The lookup index built on the device (zk_lookup_index_build) and the lookup commitments of its verifier index
(zk_lookup_index_commitments), bit for bit against tests/lookup_index_replay.py, the restatement of kimchi's
LookupConstraintSystem::create (lookup/index.rs:202-482) and of LookupVerifierIndex's commitments (verifier_index.rs:196-215).  The built
index also equals a loaded cache image of the same sections, its refusals leave no handle, and the resident lookup chain (joint table,
sorted, aggregation, kimchi's lookup constraints, division by Z_H) runs on its sections."""
import ctypes
import random
import threading

import numpy as np
import pytest
import torch

import evals_replay as ev
import index_replay as ir
import lookup_index_replay as li
import lookup_replay as lr
import proof_systems_b200 as zk
from index_cache_writer import write_cache
from test_gpu_index_build import srs_of, view
from test_gpu_lookup_constraints import check_honest, run
from test_gpu_lookup import stale

pytestmark = pytest.mark.gpu

T = li.TAGS
MIXES = {"xor": [T["Xor16"]], "lookup": [T["Lookup"]], "range_check": [T["RangeCheck0"], T["RangeCheck1"], T["Rot64"]],
         "ffmul": [T["ForeignFieldMul"]], "all": list(T.values()), "none": [0, 1, 2, 10]}


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def circuit(n, mix, seed, n_gates=None):
    """gate tags: the mix's gates and Zero / Generic gates at random, none using the next row on the last row"""
    rng = random.Random(seed)
    n_gates = min(n - 1, 3000) if n_gates is None else n_gates
    return [rng.choice(MIXES[mix] + [0, 1]) for _ in range(n_gates)]


def gates_of(tags) -> bytes:
    return ir.pruned_gates([(t, [(r, k) for k in range(7)], []) for r, t in enumerate(tags)])


def table(rng, P, tid, width, rows, zero_row=False):
    cols = [[rng.randrange(P) for _ in range(rows)] for _ in range(width)]
    if zero_row:                                                    # one all-zero row, as a table of id 0 needs
        r = rng.randrange(rows)
        for c in cols:
            c[r] = 0
    return (tid, cols)


def tables_of(kind, P, seed):
    """(fixed tables, runtime): ids 0, positive and negative, a table wider than any max_joint_size, runtime None / [] / two / id 0"""
    rng = random.Random(seed)
    if kind == "plain":
        return [table(rng, P, 2, 2, 5)], None
    if kind == "ids":
        return [table(rng, P, 0, 1, 4, zero_row=True), table(rng, P, 5, 2, 3), table(rng, P, -7, 4, 6)], []
    if kind == "neg":                                               # no id 0: the XOR table may join
        return [table(rng, P, 5, 2, 3), table(rng, P, -7, 4, 6)], []
    if kind == "runtime2":
        return [table(rng, P, 3, 1, 7)], [(9, [rng.randrange(P) for _ in range(6)]), (10, [rng.randrange(P) for _ in range(2)])]
    if kind == "runtime0":
        return [table(rng, P, 4, 3, 9)], [(0, [rng.randrange(P), 0, rng.randrange(P)])]
    raise ValueError(kind)


def build(ctx, orc, fid, n, zk_rows, tags, tables, runtime):
    mont_rt = None if runtime is None else [(tid, ev.mont(orc, fid, c)) for tid, c in runtime]
    return zk.IndexCache.build_lookup(ctx, fid, n, zk_rows, gates_of(tags), [(tid, li.mont_table(orc, fid, d)) for tid, d in tables], mont_rt)


def section(ctx, idx, tag):
    p, n_el, dom = idx.section(tag)
    return ctx.dev_download(p, (n_el, 4)), dom


# ---------------------------------------------------------------------------------------------------------------- sections
CASES = [(4, 3, "lookup", "plain"), (6, 5, "lookup", "ids"), (8, 3, "lookup", "runtime2"), (10, 4, "xor", "runtime2"),
         (10, 3, "xor", "runtime0"), (13, 3, "range_check", "ids"), (13, 6, "ffmul", "plain"), (14, 3, "all", "runtime2"),
         (14, 3, "all", "runtime0"), (16, 3, "all", "neg")]


@pytest.mark.parametrize("fid", [0, 1])
@pytest.mark.parametrize("log_n,zk_rows,mix,kind", CASES)
def test_sections_match_the_restatement(ctx, orc, fid, log_n, zk_rows, mix, kind):
    P, n = orc.MODULUS[fid], 1 << log_n
    tags = circuit(n, mix, seed=log_n + fid)
    tables, runtime = tables_of(kind, P, seed=log_n * 10 + fid)
    res = li.create(P, n, zk_rows, tags, tables, runtime)
    want = li.sections(orc, fid, res)
    idx, offset = build(ctx, orc, fid, n, zk_rows, tags, tables, runtime)
    with idx:
        h = idx.header
        assert (h.domain_d1_size, h.zk_rows, h.lookup_selectors_present, h.num_sections) == (n, zk_rows, li.header_bits(res), len(want))
        assert offset == res["runtime_table_offset"]
        for tag, (payload, dom) in want.items():
            got, d = section(ctx, idx, tag)
            assert d == dom and np.array_equal(got, payload), hex(tag)
        for tag in set(range(0x50, 0x57)) - set(want) | {0x01, 0x30}:
            with pytest.raises(zk.ZkError):
                idx.section(tag)


@pytest.mark.parametrize("fid", [0, 1])
def test_no_pattern_gives_no_index(ctx, orc, fid):
    tables, runtime = tables_of("ids", orc.MODULUS[fid], seed=1)
    assert build(ctx, orc, fid, 64, 3, circuit(64, "none", seed=2), tables, runtime) == (None, None)
    assert build(ctx, orc, fid, 64, 3, [], [], None) == (None, None)


def test_two_to_the_20_rows(ctx, orc):
    """every section sub-sampled at stride 8 against its d1 column, and two sections in full"""
    fid, log_n, zk_rows = 0, 20, 3
    P, n = orc.MODULUS[fid], 1 << log_n
    rng = random.Random(20)
    tags = circuit(n, "all", seed=20, n_gates=n - 1)
    tables = [table(rng, P, 2, 2, 1 << 10)]
    runtime = [(6, [rng.randrange(P) for _ in range(64)])]
    res = li.create(P, n, zk_rows, tags, tables, runtime)
    idx, offset = build(ctx, orc, fid, n, zk_rows, tags, tables, runtime)
    try:
        assert offset == (1 << 10) + 4096 + 256 and idx.header.lookup_selectors_present == 0x3F
        cols = li.columns(res)
        p50, n50, w = idx.section(0x50)
        assert w == len(res["cols"]) == 3 and n50 == 3 * 8 * n
        for k, (tag, c) in enumerate(cols):
            p = p50 + k * 8 * n * 32 if tag == 0x50 else idx.section(tag)[0]
            got = view(p, 8 * n)[::8].cpu().numpy().view(np.uint64)
            assert np.array_equal(got, ev.mont(orc, fid, c)), (hex(tag), k)
        for tag in (0x51, 0x55):
            c = dict(cols)[tag]
            p, n_el, _ = idx.section(tag)
            assert np.array_equal(view(p, n_el).cpu().numpy().view(np.uint64), ir.evaluate(orc, fid, ev.mont(orc, fid, c), 8)), hex(tag)
    finally:
        idx.close()
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------- refusals
def raw_build(ctx, fid, n, zk_rows, g, n_gates, tables, runtime, has_runtime, out_null=False, err_null=False, off_null=False):
    fixed = (zk._lib.LookupTable * max(1, len(tables)))(*tables)
    rt = (zk._lib.RuntimeTableCfg * max(1, len(runtime)))(*runtime)
    err, off, out = ctypes.c_int(-5), ctypes.c_uint64(12345), ctypes.c_void_p(0xdead)
    rc = zk.lib().zk_lookup_index_build(ctx._h if ctx else None, fid, n, zk_rows, g, n_gates, fixed if tables else None, len(tables),
                                        rt if runtime else None, len(runtime), has_runtime, None if err_null else ctypes.byref(err),
                                        None if off_null else ctypes.byref(off), None if out_null else ctypes.byref(out))
    return rc, out.value, err.value, off.value


def test_refusals_leave_no_handle(ctx, orc):
    fid, n, zk_rows = 0, 64, 3
    P = orc.MODULUS[fid]
    keep = []

    def tab(tid, width, rows, fill=1):
        a = np.ascontiguousarray(np.broadcast_to(ev.mont(orc, fid, [fill]), (width * max(rows, 1), 4))[:width * rows])
        keep.append(a)
        return zk._lib.LookupTable(tid, width, rows, a.ctypes.data if a.size else None)

    def rtab(tid, rows, fill=1):
        a = np.ascontiguousarray(np.broadcast_to(ev.mont(orc, fid, [fill]), (max(rows, 1), 4))[:rows])
        keep.append(a)
        return zk._lib.RuntimeTableCfg(tid, rows, a.ctypes.data if a.size else None)
    g = gates_of([T["Lookup"], 0, T["RangeCheck1"]] + [0] * 10)
    ng = len(g) // 60
    bad = np.ascontiguousarray(np.array([[P & (2 ** 64 - 1), (P >> 64) & (2 ** 64 - 1), (P >> 128) & (2 ** 64 - 1), P >> 192]], dtype=np.uint64))
    non_canonical = zk._lib.LookupTable(3, 1, 1, bad.ctypes.data)
    big = 1 << 13                                                    # room for the range-check table
    ok = raw_build(ctx, fid, big, zk_rows, g, ng, [tab(2, 2, 5)], [rtab(7, 3)], 1)
    assert ok[0] == 0 and ok[1] and ok[2] == 0 and ok[3] == 4096 + 5
    zk.lib().zk_index_cache_free(ctypes.c_void_p(ok[1]))
    errors = {                                                       # LookupError: kind and the start of the reference's message
        "fixed id collides with the range-check table": ((big, [tab(1, 1, 4)], [], 0), 1, "Cannot create a combined table since ids for "
                                                                                            "sub-tables are colliding. The collision type is: duplicates between fixed given and fixed from-gate tables: [1]"),
        "two fixed tables of id 5": ((big, [tab(5, 1, 4), tab(5, 2, 3), tab(5, 1, 1)], [], 0), 1, "Cannot create a combined table since ids "
                                                                                                    "for sub-tables are colliding. The collision type is: duplicates between fixed given and fixed from-gate tables: [5, 5]"),
        "runtime duplicates": ((big, [tab(5, 1, 4)], [rtab(5, 2), rtab(5, 3)], 1), 1, "Cannot create a combined table since ids for "
                                                                                        "sub-tables are colliding. The collision type is: runtime table duplicates: [5]"),
        "id 0 without a zero row": ((big, [tab(0, 2, 4)], [], 0), 2, "The table with id 0 must have an entry of all zeros"),
        "id-0 runtime table without a zero": ((big, [], [rtab(0, 4)], 1), 2, "The table with id 0 must have an entry of all zeros"),
        "too long": ((big, [tab(2, 1, big - zk_rows - 1 - 4096)], [], 0), 3, "The combined lookup table is larger than allowed by the "
                                                                               f"domain size. Observed: {big - zk_rows - 1}, expected: {big - zk_rows - 2}"),
    }
    for name, ((nn, tabs, rts, has), kind, msg) in errors.items():
        rc, out, err, off = raw_build(ctx, fid, nn, zk_rows, g, ng, tabs, rts, has)
        assert (rc, out, err, off) == (-1, None, kind, 12345), name
        assert zk.lib().zk_last_error().decode() == msg, name
    last_next = gates_of([0] * (n - 1) + [T["ForeignFieldMul"]])
    invalid = {
        "null context": dict(ctx=None),
        "null out": dict(out_null=True),
        "null lookup_error": dict(err_null=True),
        "null runtime_table_offset with runtime": dict(off_null=True, runtime=[rtab(7, 3)], has_runtime=1),
        "runtime without has_runtime": dict(runtime=[rtab(7, 3)]),
        "unknown field": dict(fid=2),
        "n not a power of two": dict(n=48),
        "n beyond 2^27": dict(n=1 << 28),
        "zk_rows 0": dict(zk_rows=0),
        "zk_rows n - 1": dict(zk_rows=n - 1),
        "more gates than rows": dict(n=8),
        "tag 14": dict(g=gates_of([14])),
        "width 0": dict(tables=[tab(2, 0, 0)]),
        "width 17": dict(tables=[tab(2, 17, 2)]),
        "a non-canonical entry": dict(tables=[non_canonical]),
        "a non-canonical runtime entry": dict(runtime=[zk._lib.RuntimeTableCfg(3, 1, bad.ctypes.data)], has_runtime=1),
        "next row on the last row": dict(g=last_next),
        "gates null with a count": dict(g=None, n_gates=3),
        "more rows than the domain with runtime tables": dict(n=64, g=gates_of([T["RangeCheck0"]]), runtime=[rtab(7, 3)], has_runtime=1),
    }
    for name, kw in invalid.items():
        a = dict(ctx=ctx, fid=fid, n=n, zk_rows=zk_rows, g=g, tables=[], runtime=[], has_runtime=0)
        a.update(kw)
        a.setdefault("n_gates", len(a["g"]) // 60 if a["g"] else 0)
        rc, out, err, off = raw_build(**a)
        assert rc == -1 and off == 12345, name
        if not kw.get("out_null"):                                   # else nothing can be written there
            assert out is None, name
        if not kw.get("err_null"):
            assert err == 0, name


# ---------------------------------------------------------------------------------------------------------------- commitments
@pytest.mark.parametrize("curve,log_n,m,mix,kind", [("pallas", 10, 1 << 16, "xor", "neg"), ("vesta", 13, 1 << 16, "all", "runtime2"),
                                                    ("pallas", 14, 1 << 16, "range_check", "ids"), ("vesta", 17, 1 << 16, "lookup", "runtime2")])
def test_commitments(ctx, orc, pallas_srs, vesta_srs, curve, log_n, m, mix, kind):
    golden = pallas_srs if curve == "pallas" else vesta_srs
    fid = orc.SCALAR_FIELD[golden.cid]
    P, n, zk_rows = orc.MODULUS[fid], 1 << log_n, 3
    tags = circuit(n, mix, seed=log_n)
    tables, runtime = tables_of(kind, P, seed=log_n)
    res = li.create(P, n, zk_rows, tags, tables, runtime)
    with srs_of(ctx, golden, m) as srs:
        idx, _ = build(ctx, orc, fid, n, zk_rows, tags, tables, runtime)
        with idx:
            got = srs.lookup_index_commitments(idx)
            chunks = max(1, n // m)
            assert got.shape == (len(li.columns(res)), chunks, 8)
            assert np.array_equal(got, li.commitments(orc, golden.cid, golden.g[:m], srs.h, res))
            # the table columns and the table ids are h away from commit_evaluations_non_hiding, the selectors equal it
            for k, (tag, c) in enumerate(li.columns(res)):
                plain = srs.commit_evaluations_non_hiding(n, ev.mont(orc, fid, c)).chunks
                want = np.stack([orc.affine_add(golden.cid, p, srs.h) for p in plain]) if tag in (0x50, 0x51) else plain
                assert np.array_equal(got[k], want), hex(tag)


def test_commitment_refusals(ctx, orc, vesta_srs):
    fid, n = 0, 1 << 10                                             # Vesta's scalars: Fp
    P = orc.MODULUS[fid]
    tags = circuit(n, "xor", seed=3)
    with srs_of(ctx, vesta_srs, 1 << 10) as srs:
        other, _ = build(ctx, orc, 1, n, 3, tags, [], None)          # over Fq
        good, _ = build(ctx, orc, fid, n, 3, tags, *tables_of("neg", P, seed=3))
        prover = zk.IndexCache.build(ctx, fid, ir.header(zk, n, 3, ev.mont(orc, fid, [1] * 7)), ir.pruned_gates([]), b"")
        with other, good, prover:
            out = np.zeros((64, 8), dtype=np.uint64)
            k = ctypes.c_size_t()
            call = lambda idx, cap=64: zk.lib().zk_lookup_index_commitments(srs._h, idx._h if idx else None,
                                                                            out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)), cap, ctypes.byref(k))
            for name, idx in {"null index": None, "other field": other, "no section 0x50": prover}.items():
                assert call(idx) == -1, name
            count = good.section(0x50)[2] + bin(good.header.lookup_selectors_present).count("1")
            assert call(good, cap=count - 1) == -1 and k.value == count
            assert call(good) == 0 and k.value == count


# ---------------------------------------------------------------------------------------------------------------- built == loaded
@pytest.mark.parametrize("fid", [0, 1])
def test_built_index_equals_the_loaded_file(ctx, orc, vesta_srs, pallas_srs, fid):
    P, n, zk_rows = orc.MODULUS[fid], 1 << 10, 4
    tags = circuit(n, "all", seed=50 + fid, n_gates=200)
    tags = [t for t in tags if t not in (T["RangeCheck0"], T["RangeCheck1"], T["Rot64"], T["ForeignFieldMul"])]   # no 4096-row table
    tables, runtime = tables_of("runtime2", P, seed=fid)
    res = li.create(P, n, zk_rows, tags, tables, runtime)
    want = li.sections(orc, fid, res)
    zeros8 = bytes(8 * n * 32)
    sections = [(0x30 + i, zeros8, 8 * n) for i in range(7)] + [(t, a.astype("<u8").tobytes(), d) for t, (a, d) in want.items()]
    header = {"public": 0, "prev_challenges": 0, "zk_rows": zk_rows, "max_poly_size": n, "domain_d1_size": n,
              "lookup_selectors_present": li.header_bits(res), "endo_limbs": [0] * 4, "shift_limbs": [[0] * 4] * 7}
    golden = vesta_srs if fid == 0 else pallas_srs
    built, _ = build(ctx, orc, fid, n, zk_rows, tags, tables, runtime)
    with built, zk.IndexCache(ctx, write_cache("lookup", header, sections)) as loaded, srs_of(ctx, golden, 1 << 10) as srs:
        assert loaded.header.lookup_selectors_present == built.header.lookup_selectors_present
        for tag in want:
            a, da = section(ctx, built, tag)
            b, db = section(ctx, loaded, tag)
            assert da == db and np.array_equal(a, b), hex(tag)
        assert np.array_equal(srs.lookup_index_commitments(built), srs.lookup_index_commitments(loaded))


# ---------------------------------------------------------------------------------------------------------------- the resident chain
def test_chain_on_a_built_index(ctx, orc, pallas_srs):
    """a circuit of Lookup, Xor16, RangeCheck0/1 and ForeignFieldMul gates whose witness is drawn from the built table: sections
    0x50 / 0x51 -> zk_lookup_joint_table_dev -> sorted, aggregation, kimchi's lookup constraints with the selectors 0x52 - 0x55 of the
    built index -> division by Z_H with a zero remainder"""
    fid, log_n, zk_rows, m = pallas_srs.scalar, 13, 3, 4
    P, n = orc.MODULUS[fid], 1 << log_n
    L = n - zk_rows - 1
    rng = random.Random(13)
    names = ["Lookup", "Xor16", "RangeCheck0", "RangeCheck1", "ForeignFieldMul", "Zero"]
    gates = []
    while len(gates) < L - 2:                   # as in kimchi's gadgets, the row a Next pattern looks up holds a Zero gate
        gates.append(rng.choice(names))
        if gates[-1] in ("RangeCheck1", "ForeignFieldMul"):
            gates.append("Zero")
    gates = gates[:L - 2] + ["Zero"] * 2
    tags = [T.get(g, 0) for g in gates]
    user = (2, [[rng.randrange(P) for _ in range(300)], [rng.randrange(P) for _ in range(300)]])
    res = li.create(P, n, zk_rows, tags, [user])
    assert len(res["cols"]) == 3 and set(res["selectors"]) == set(li.PATTERNS)
    ids = [0] * n if res["ids"] is None else res["ids"]
    table_rows = [(ids[r], [res["cols"][c][r] for c in range(3)]) for r in range(L)]
    inst = lr.instance(P, log_n, zk_rows, m, seed=84, table=table_rows, gates=gates, tic="kimchi")
    kimchi = [inst.patterns[inst.names.index(p)] for p in zk.LookupSpec.KIMCHI_PATTERNS]
    assert inst.names[:4] == list(zk.LookupSpec.KIMCHI_PATTERNS) and any(inst.row_pattern)
    idx, _ = build(ctx, orc, fid, n, zk_rows, tags, [user], None)
    with idx, ctx.buffers() as bufs:
        p50, _, w = idx.section(0x50)
        p51, _, _ = idx.section(0x51)
        sel8 = [idx.section(0x52 + k)[0] for k in range(4)]
        d_t8, d_t1 = stale(bufs, 8 * n), stale(bufs, n)
        ctx.lookup_joint_table_dev(fid, log_n, [p50 + k * 8 * n * 32 for k in range(w)], *ev.mont(orc, fid, [inst.jc, inst.tic]), d_t8, p51,
                                   None, d_t1)
        inst.T1 = ev.ints(orc, fid, ctx.dev_download(d_t1, (n, 4)))
        check_honest(run(ctx, orc, fid, inst, bufs, patterns=kimchi, table8=d_t8, selectors8=sel8))


# ---------------------------------------------------------------------------------------------------------------- streams, threads
def test_on_a_callers_stream(orc, vesta_srs):
    """both calls on a caller's stream, queued behind a spin kernel"""
    fid, n, zk_rows = 0, 1 << 12, 4
    P = orc.MODULUS[fid]
    tags = circuit(n, "xor", seed=7)
    tables, runtime = tables_of("runtime0", P, seed=7)
    res = li.create(P, n, zk_rows, tags, tables, runtime)
    want = li.sections(orc, fid, res)
    stream = torch.cuda.Stream()
    with zk.Context(0) as c:
        c.set_stream(stream.cuda_stream)
        with srs_of(c, vesta_srs, 1 << 16) as srs:
            srs.get_lagrange_basis_from_domain_size(n)
            torch.cuda.synchronize()
            with torch.cuda.stream(stream):
                torch.cuda._sleep(20_000_000)
                idx, _ = build(c, orc, fid, n, zk_rows, tags, tables, runtime)
                torch.cuda._sleep(20_000_000)
                got = srs.lookup_index_commitments(idx)
            with idx:
                for tag, (payload, _) in want.items():
                    assert np.array_equal(section(c, idx, tag)[0], payload), hex(tag)
            assert np.array_equal(got, li.commitments(orc, vesta_srs.cid, vesta_srs.g[:1 << 16], srs.h, res))


def test_two_threads_share_a_context(ctx, orc):
    fid, n = 1, 1 << 10
    P = orc.MODULUS[fid]
    work = [(circuit(n, "xor" if t else "lookup", seed=30 + t), *tables_of("runtime2" if t else "ids", P, seed=t)) for t in range(2)]
    want = [li.sections(orc, fid, li.create(P, n, 5, *w)) for w in work]
    errors = []

    def go(t):
        try:
            for _ in range(3):
                idx, _ = build(ctx, orc, fid, n, 5, *work[t])
                with idx:
                    for tag, (payload, _) in want[t].items():
                        assert np.array_equal(section(ctx, idx, tag)[0], payload), hex(tag)
        except Exception as e:             # noqa: BLE001 - reported below
            errors.append(e)
    th = [threading.Thread(target=go, args=(t,)) for t in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
