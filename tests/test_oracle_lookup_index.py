"""tests/lookup_index_replay.py, the restatement of LookupConstraintSystem::create (kimchi/src/circuits/lookup/index.rs:202-482),
pinned to the reference's own examples and tests: the worked concatenation of :334-366, test_check_id_duplicates and
test_colliding_table_ids (:517-627) on create_multi_range_check(0)'s gates with the domain Builder::build picks, the XOR table's
rows (tables/xor.rs:22-44), the Next-row selectors (lookups.rs:235-283), the runtime selector (:269-289) and the length limit."""
import pytest

import lookup_index_replay as li

P = 0x40000000000000000000000000000000224698FC094CF91B992D30ED00000001        # Fp
MULTI_RANGE_CHECK = [li.TAGS["RangeCheck0"], li.TAGS["RangeCheck0"], li.TAGS["RangeCheck1"], 0]   # create_multi_range_check(0)


def test_the_worked_example():
    """index.rs:334-366: a 3-column table of id 0 and a 2-column table of id 1 in a domain of 5 rows"""
    cols, ids = li.concatenated([(0, [[1, 5, 0], [2, 6, 0], [3, 7, 0]]), (1, [[8], [9]])], 3, 5)
    assert [[c[r] for c in cols] for r in range(5)] == [[1, 2, 3], [5, 6, 7], [0, 0, 0], [8, 9, 0], [0, 0, 0]]
    assert ids == [0, 0, 0, 1, 0]


def test_check_id_duplicates():
    assert li.id_duplicates([1, 2, 3], "test no duplicates") is None
    assert li.id_duplicates([1, 2, 3, 2, 4, 1], "test-with-dups") == "test-with-dups: [2, 1]"


def fixed(tid, value, rows=16):
    return (tid, [[value] * rows])


COLLIDING = {                                           # test_colliding_table_ids: tables, runtime, collision_type or None (Ok)
    "range table passed twice": ([li.range_check_table()], None, "duplicates between fixed given and fixed from-gate tables: [1]"),
    "xor table, no duplicates": ([li.xor_table()], None, None),
    "collision in fixed ids": ([fixed(5, 0), fixed(5, 1)], None, "duplicates between fixed given and fixed from-gate tables: [5]"),
    "collision in runtime ids": ([], [(5, [0] * 16), (5, [1] * 16)], "runtime table duplicates: [5]"),
    "runtime and fixed ids may collide": ([fixed(5, 0)], [(5, [1] * 16)], None),
}


@pytest.mark.parametrize("case", list(COLLIDING))
def test_colliding_table_ids(case):
    tables, runtime, collision = COLLIDING[case]
    n, zk_rows = li.builder_domain(4, MULTI_RANGE_CHECK, tables, runtime)
    assert (n, zk_rows) == ((1 << 14, 3) if case == "range table passed twice" else (1 << 13, 3))
    if collision is None:
        res = li.create(P, n, zk_rows, MULTI_RANGE_CHECK, tables, runtime)
        assert res is not None and list(res["selectors"]) == ["range_check"]
    else:
        with pytest.raises(li.LookupError_) as e:
            li.create(P, n, zk_rows, MULTI_RANGE_CHECK, tables, runtime)
        assert e.value.kind == li.ID_COLLISION
        assert e.value.message == "Cannot create a combined table since ids for sub-tables are colliding. The collision type is: " + collision


def test_xor_table_rows():
    tid, cols = li.xor_table()
    rows = [tuple(c[r] for c in cols) for r in range(256)]
    assert tid == 0 and rows[0] == (15, 15, 0) and rows[1] == (15, 14, 1) and rows[16] == (14, 15, 1) and rows[-1] == (0, 0, 0)
    assert len(set(rows)) == 256


def test_gate_tables_come_range_check_first():
    """Xor16 and RangeCheck0: the range-check table (id 1, 4096 rows) before the XOR table (id 0)"""
    res = li.create(P, 1 << 13, 3, [li.TAGS["Xor16"], li.TAGS["RangeCheck0"]], [])
    assert len(res["cols"]) == 3 and res["cols"][0][:3] == [0, 1, 2] and res["cols"][1][4095] == 0
    assert [res["cols"][c][4096] for c in range(3)] == [15, 15, 0] and res["ids"][:4097] == [1] * 4096 + [0]
    assert list(res["selectors"]) == ["xor", "range_check"]


@pytest.mark.parametrize("gate,pattern", [("RangeCheck1", "range_check"), ("ForeignFieldMul", "foreign_field_mul")])
def test_next_row_patterns_mark_two_rows(gate, pattern):
    n = 1 << 13
    tags = [0] * 10 + [li.TAGS[gate]]
    res = li.create(P, n, 3, tags, [])
    sel = res["selectors"][pattern]
    assert [r for r in range(n) if sel[r]] == [10, 11]
    with pytest.raises(li.Panics):                                  # the next row of the last row is past the domain
        li.create(P, 16, 3, [0] * 15 + [li.TAGS[gate]], [])


def test_no_pattern_is_none():
    assert li.create(P, 64, 3, [0, 1, 2, 10], [fixed(3, 0)], runtime=[]) is None


@pytest.mark.parametrize("runtime", [[], [(7, [1, 2, 3]), (8, [4, 5])]])
def test_runtime_selector(runtime):
    n, zk_rows = 1 << 13, 4
    res = li.create(P, n, zk_rows, [li.TAGS["Lookup"]], [fixed(2, 9, 10)], runtime)
    rlen = sum(len(c) for _, c in runtime)
    assert res["runtime_table_offset"] == 10
    want = [1] * 10 + [0] * rlen + [1] * (n - 10 - rlen - zk_rows) + [0] * zk_rows
    assert res["runtime_selector"] == want
    assert len(res["cols"]) == 2                                    # max_joint_size of Lookup, and a runtime table's width
    if runtime:
        assert res["cols"][0][10:15] == [1, 2, 3, 4, 5] and res["cols"][1][10:15] == [0] * 5 and res["ids"][10:16] == [7, 7, 7, 8, 8, 0]


def test_table_ids_and_the_zero_entry():
    n = 1 << 6
    tags = [li.TAGS["Lookup"]]
    assert li.create(P, n, 3, tags, [fixed(0, 0)])["ids"] is None                  # only id 0: no table_ids
    assert li.create(P, n, 3, tags, [fixed(-3, 1)])["ids"][:17] == [P - 3] * 16 + [0]
    with pytest.raises(li.LookupError_) as e:
        li.create(P, n, 3, tags, [fixed(0, 1)])
    assert e.value.kind == li.TABLE_ID_ZERO and e.value.message == "The table with id 0 must have an entry of all zeros"
    with pytest.raises(li.LookupError_) as e:                                       # an id-0 runtime table counts, with its placeholder
        li.create(P, n, 3, tags, [], runtime=[(0, [1, 2])])
    assert e.value.kind == li.TABLE_ID_ZERO
    assert li.create(P, n, 3, tags, [], runtime=[(0, [1, 0])]) is not None


def test_too_long_at_exactly_max_num_entries():
    n, zk_rows = 64, 5
    max_num_entries = n - zk_rows - 1
    tags = [li.TAGS["Lookup"]]
    assert li.create(P, n, zk_rows, tags, [fixed(2, 1, max_num_entries - 1)]) is not None
    with pytest.raises(li.LookupError_) as e:
        li.create(P, n, zk_rows, tags, [fixed(2, 1, max_num_entries)])
    assert e.value.kind == li.TOO_LONG
    assert e.value.message == ("The combined lookup table is larger than allowed by the domain size. "
                               f"Observed: {max_num_entries}, expected: {max_num_entries - 1}")
