"""Builder side of general joins in program pipelines (lingodb_b200/program.py): row ids, PROBE_EACH and side columns ("fetch"),
without a GPU."""
import ctypes as C

import pytest

from lingodb_b200 import program as P

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))


def _reads(op, a, b, arg):
    """registers an instruction reads"""
    if op in (P.OPS["load"], P.OPS["const"], P.OPS["rowid"], P.OPS["strcmp"], P.OPS["strlike"], P.OPS["strkey8"]):
        return []
    if op in (P.OPS["neg"], P.OPS["not"], P.OPS["isnull"], P.OPS["i2f"], P.OPS["year"], P.OPS["probe"], P.OPS["probe_each"]):
        return [a]
    if op == P.OPS["select"]:
        return [a, b, arg]
    return [a, b]


def test_probe_each_is_emitted_once_and_a_second_one_is_refused():
    b = P.Builder()
    lines = C.c_void_p(7)
    m = ("probe_each", lines, col("ps_partkey"))
    b.expr(("cmp", ">", m, const(3)))
    b.expr(("add", m, const(1)))
    b.expr(m)
    each = [i for i in b.instr if i[0] == P.OPS["probe_each"]]
    assert len(each) == 1 and each[0][3] == 0 and b.tables == [lines]
    outer = P.Builder()
    outer.expr(("probe_each", lines, col("c_custkey"), "outer"))
    assert outer.instr[-1][0] == P.OPS["probe_each"] and outer.instr[-1][3] == 1
    with pytest.raises(ValueError, match="at most one probe_each"):
        b.expr(("probe_each", C.c_void_p(8), col("ps_suppkey")))


def test_fetched_columns_are_bound_to_their_row_registers_after_the_source_columns():
    b = P.Builder()
    part, supp = C.c_void_p(11), C.c_void_p(12)
    prow = ("probe", C.c_void_p(3), col("l_partkey"))
    srow = ("probe", C.c_void_p(4), col("l_suppkey"))
    size = b.expr(("fetch", part, prow, "p_size"))
    b.expr(("add", ("fetch", supp, srow, "s_acctbal"), ("fetch", part, prow, "p_size")))
    b.expr(col("l_quantity"))
    assert b.side_tables == [11, 12]
    assert [(t, c) for t, c, _ in b.side_columns] == [(0, "p_size"), (1, "s_acctbal")]
    ins = b.instructions()
    loads = [i for i in ins if i[0] == P.OPS["load"]]
    n_src = len(b.columns)
    assert b.columns == ["l_partkey", "l_suppkey", "l_quantity"]
    side_loads = [i for i in loads if i[4] >= n_src]
    assert [i[4] - n_src for i in side_loads] == [0, 1]  # the p_size load is emitted once
    for t, c, r in b.side_columns:  # each side column's row register holds the probe payload, written before the load
        probe_at = next(k for k, i in enumerate(ins) if i[1] == r)
        load_at = next(k for k, i in enumerate(ins) if i[0] == P.OPS["load"] and i[4] == n_src + b.side_columns.index((t, c, r)))
        assert ins[probe_at][0] == P.OPS["probe"] and probe_at < load_at
    assert size == side_loads[0][1]


def test_string_ops_accept_fetched_columns_and_rowid_is_a_payload():
    b = P.Builder()
    part = C.c_void_p(21)
    row = ("probe", C.c_void_p(5), col("l_partkey"))
    b.expr(("like", "prefix", ("fetch", part, row, "p_type"), "PROMO"))
    b.expr(("strcmp", "=", ("fetch", part, row, "p_brand"), "Brand#23"))
    b.expr(("strkey8", ("fetch", part, row, "p_container")))
    b.expr(("strcmp", "=", "l_shipinstruct", "DELIVER IN PERSON"))
    ins = b.instructions()
    n_src = len(b.columns)
    assert b.columns == ["l_partkey", "l_shipinstruct"]
    strs = [i for i in ins if i[0] in (P.OPS["strlike"], P.OPS["strcmp"], P.OPS["strkey8"])]
    assert [i[2] for i in strs] == [n_src + 0, n_src + 1, n_src + 2, 1]
    assert [c for _, c, _ in b.side_columns] == ["p_type", "p_brand", "p_container"]
    assert len({r for _, _, r in b.side_columns}) == 1  # one probe: the three columns share one row register
    r = P.Builder()
    rid = r.expr(("rowid",))
    assert r.instr == [(P.OPS["rowid"], rid, 0, 0, 0)]
    with pytest.raises(ValueError, match="not a column"):
        P.Builder().expr(("strcmp", "=", ("col", "x"), "a"))


def test_every_register_read_is_written_earlier():
    b = P.Builder()
    part, groups = C.c_void_p(31), C.c_void_p(32)
    each = ("probe_each", C.c_void_p(6), col("ps_partkey"))
    grow = ("probe", C.c_void_p(7), ("add", ("mul", col("ps_partkey"), const(1 << 14)), col("ps_suppkey")))
    b.expr(("and", ("like", "prefix", ("fetch", part, ("probe", C.c_void_p(8), col("ps_partkey")), "p_name"), "forest"),
            ("cmp", ">", ("mul", col("ps_availqty"), const(200)), ("fetch", groups, grow, "a0"))))
    b.expr(("case", ("isnull", each), const(0), ("fetch", groups, each, "k0")))
    written = set()
    side_row = {len(b.columns) + k: r for k, (_, _, r) in enumerate(b.side_columns)}
    for op, dst, a, bb, arg in b.instructions():
        for r in _reads(op, a, bb, arg):
            assert r in written, (op, r)
        if op == P.OPS["load"] and arg in side_row:
            assert side_row[arg] in written
        if op in (P.OPS["strcmp"], P.OPS["strlike"], P.OPS["strkey8"]) and a in side_row:
            assert side_row[a] in written
        assert dst not in written  # single assignment: nothing after PROBE_EACH overwrites what it reads on the next match
        written.add(dst)
