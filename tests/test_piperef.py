"""The specialised-pipeline reference of tests/_piperef.py against values worked out by hand, and its generators' determinism (no GPU)."""
import pytest

import _piperef as P

S = P.schema_of()


def test_mul_1minus_1plus_with_a_negative_multiplier():
    # a * (1 - b) * (1 + c) with one + c = -2^40: 2^40 * 2^40 * -2^40
    assert P.agg_term("mul_1minus_1plus", 1 << 40, 100 - (1 << 40), -100 - (1 << 40)) == -(1 << 120)
    # 2^59 * 2^59 * 2^9 = 2^127 wraps to INT128_MIN
    assert P.finish_sum("mul_1minus_1plus", P.agg_term("mul_1minus_1plus", 1 << 59, 100 - (1 << 59), (1 << 9) - 100)) == -(1 << 127)
    assert P.agg_term("mul_1minus_minus_paymul", 3, 10, pay=-7, d=2) == 3 * 90 + 14


def test_64_bit_sums_wrap_and_read_back_sign_extended():
    big = 10**18 - 1
    cols = {"a": [big] * 10, "k": [0] * 10}
    out = P.scan_groupby(cols, S, [], [], [("col", ["a"]), ("one", [])])
    assert out == {(): [10**19 - 10 - (1 << 64), 10]}  # 9 999 999 999 999 999 990 wraps past 2^63
    assert P.scan_groupby({"a": [-5], "k": [3]}, S, [], ["k"], [("col", ["a"]), ("one", [])]) == {(3, 0): [-5, 1]}
    # an i128 sum does not wrap at 64 bits
    assert P.scan_groupby({"a": [big] * 10, "b": [0] * 10}, S, [], [], [("mul_1minus", ["a", "b"])]) == {(): [10 * big * 100]}


def test_fsb4_and_date_constants():
    assert P.constant(S, "fs", "A") == 65
    assert P.constant(S, "fs", "AB") == 0x4241
    assert P.constant(S, "fs", "") == 0
    assert P.constant(S, "dt", "1970-01-02") == 1
    assert P.constant(S, "dt", "1969-12-31") == -1
    with pytest.raises(P.PipeError) as e:
        P.constant(S, "fs", "ABCDE")
    assert e.value.code == P.LDB_ERR_INVALID


def test_decimal_constants():
    assert P.constant(S, "a", "0.05") == 5
    assert P.constant(S, "a", "-1.5") == -150
    assert P.constant(S, "a", "12") == 1200
    assert P.constant(S, "a", 7) == 700
    assert P.constant(S, "a", -((1 << 63) // 100)) == -9223372036854775800
    for bad in ((1 << 62), -(1 << 62), "92233720368547758.08"):
        with pytest.raises(P.PipeError) as e:
            P.constant(S, "a", bad)
        assert e.value.code == P.LDB_ERR_UNSUPPORTED
    with pytest.raises(P.PipeError) as e:
        P.constant(S, "a", "1.234")
    assert e.value.code == P.LDB_ERR_INVALID


def test_string_filters():
    cols = {"s": [b"", b"x", b"green", b"\xc3\xa9t\xc3\xa9"]}
    assert P.filter_rows(cols, S, [("s", "contains", "")]) == [True] * 4
    assert P.filter_rows(cols, S, [("s", "contains", "re")]) == [False, False, True, False]
    assert P.filter_rows(cols, S, [("s", "contains", "é")]) == [False, False, False, True]
    assert P.filter_rows(cols, S, [("s", "=", "")]) == [True, False, False, False]
    assert P.filter_rows(cols, S, [("s", "!=", "")]) == [False, True, True, True]


def test_filter_entries_ranges_and_in():
    cols = {"i": [-5, 0, 5, 10], "a": [-100, 0, 100, 250], "dt": [0, 1, 2, 3], "fs": [65, 66, 67, 68]}
    assert P.filter_rows(cols, S, [("i", ">", -5), ("i", "<=", 5)]) == [False, True, True, False]
    assert P.filter_rows(cols, S, [("a", ">=", "-1"), ("a", "<", 2)]) == [True, True, True, False]
    assert P.filter_rows(cols, S, [("i", "in", [10])]) == [False, False, False, True]
    assert P.filter_rows(cols, S, [("fs", "in", ["B", "D"]), ("i", "notnull", 0)]) == [False, True, False, True]
    # a second compare on a column joins the first: four columns with ranges are four entries, a fifth column is one too many
    four = [("i", ">", -9), ("i", "<", 9), ("a", "!=", 0), ("dt", ">=", "1970-01-01"), ("dt", "<", "1970-01-04"), ("fs", "=", "A")]
    assert P.filter_rows(cols, S, four) == [True, False, False, False]
    with pytest.raises(P.PipeError) as e:
        P.filter_rows(cols, S, four + [("i", "=", 1)])
    assert e.value.code == P.LDB_ERR_UNSUPPORTED
    with pytest.raises(P.PipeError) as e:
        P.filter_rows(cols, S, [("i", "in", list(range(9)))])
    assert e.value.code == P.LDB_ERR_UNSUPPORTED


def test_topk_tie_breaking_and_64_bit_lanes():
    t = P.JoinTable(n_side=2, n_aggs=1, unique=False)
    for key, side0 in ((5, 2), (3, 2), (9, 1), (1, 0), (7, 0), (4, 4)):
        t.insert(key, 0, side0, 0)
    cols = {"k": [5, 3, 9, 1, 1, 4], "a": [10, 10, 10, 15, 5, -5]}
    P.probe_agg(cols, S, [], t, "k", ("col", ["a"]))
    assert [r[0] for r in P.topk(t, 64)] == [1, 9, 3, 5, 4]  # 20; then 10 by side0, then key; -5 last; 7 never probed
    assert P.topk(t, 64)[-1][3] == -5
    assert [r[0] for r in P.topk(t, 2)] == [1, 9]
    with pytest.raises(P.PipeError) as e:  # the lane is 64-bit now: a 128-bit sum may not join it
        P.probe_agg(cols, S, [], t, "k", ("mul", ["a", "a"]))
    assert e.value.code == P.LDB_ERR_UNSUPPORTED


def test_join_table_errors():
    with pytest.raises(ValueError):  # overflow of a larger directory depends on the insert order
        P.JoinTable(expected_rows=16384)
    t = P.JoinTable(expected_rows=8)
    for k in range(17):
        t.insert(k, k)
    with pytest.raises(P.PipeError) as e:
        t.count()
    assert e.value.code == P.LDB_ERR_CAPACITY  # 16 slots
    cases = [(P.JoinTable(), [(1, 0), (1, 1)], P.LDB_ERR_INVALID), (P.JoinTable(unique=False), [(-1, -1)], P.LDB_ERR_UNSUPPORTED),
             (P.JoinTable(n_side=1), [(1, -3)], P.LDB_ERR_UNSUPPORTED), (P.JoinTable("direct", key_min=0, key_max=9), [(10, 1)], P.LDB_ERR_INVALID),
             (P.JoinTable("direct", key_min=0, key_max=9), [(3, 1), (3, 2)], P.LDB_ERR_INVALID), (P.JoinTable("pair"), [((-1, -1), 5)], P.LDB_ERR_UNSUPPORTED)]
    for tab, rows, code in cases:
        for k, p in rows:
            tab.insert(k, p)
        with pytest.raises(P.PipeError) as e:
            tab.count()
        assert e.value.code == code
    ok = P.JoinTable(unique=False)
    ok.insert(-1, 0)
    ok.insert(-1, 0)
    ok.insert(0, -1)
    assert ok.count() == 3 and ok.multimap() == {-1: [0, 0], 0: [-1]}


def test_pipelines_on_hand_worked_rows():
    cols = {"k": [1, 2, 2, 3], "i": [10, 20, 20, 30], "a": [100, 200, 300, 400], "b": [0, 10, 20, 30], "c": [5, 5, 5, 5], "dt": [0, 365, -1, 10957]}
    build = P.JoinTable(unique=False)
    P.scan_build(cols, S, [("a", ">", "1.00")], build, "k", payload="i")
    assert build.multimap() == {2: [20, 20], 3: [30]}
    assert sorted(P.materialize(cols, S, [], ["k", "$payload"], probe=(build, "k"))) == [(2, 20), (2, 20), (2, 20), (2, 20), (3, 30)]
    years = P.JoinTable()
    P.scan_build({"k": [1, 2, 3, 4], "dt": [0, 365, -1, 10957]}, S, [], years, "k", payload="dt", payload_expr="year")
    assert years.multimap() == {1: [1970], 2: [1971], 3: [1969], 4: [2000]}
    a, b = P.JoinTable(), P.JoinTable(n_side=1)
    for k, p in ((1, 7), (2, 8), (3, 9)):
        a.insert(k, p)
        b.insert(k, p if k != 3 else 4, 0)
    got = P.probe2_groupby(cols, S, [], a, "k", b, "k", ("mul_1minus", ["a", "b"]))
    assert got == {(7, 0): [100 * 100], (8, 0): [200 * 90 + 300 * 80]}
    p = P.JoinTable("pair")
    p.insert((1, 10), -3)
    s, o = P.JoinTable("direct", key_min=0, key_max=3), P.JoinTable()
    s.insert(1, -1)
    o.insert(10, -1)
    star = P.star_probe_groupby(cols, S, [], p, ("k", "i"), s, "k", o, "i", ("a", "b", "c"))
    assert star == {(-1, -1): [100 * 100 + 3 * 5]}


def test_generators_are_deterministic():
    assert P.gen_table(7, 300) == P.gen_table(7, 300)
    assert P.gen_table(7, 300) != P.gen_table(8, 300)
    vals = P.gen_table(3, 500)
    assert all(-(10**18) < v < 10**18 for c in ("a", "b", "c") for v in vals[c])
    ks = P.colliding_keys(16, 4093, 50)
    assert ks == P.colliding_keys(16, 4093, 50) and len(set(ks)) == 50
    assert all(int(h) & 0xFFFF == 4093 for h in P.h64(ks))
    h = P.h64([0, 1, -1, 12345])
    assert int(h[0]) == 0 and all(int(x) == int(x.byteswap()) for x in h)  # h64 is bswap-symmetric
