"""Builder side of join-table markers (lingodb_b200/program.py): the encoding of ("mark", probe, cond), where the builder puts the
probe relative to the condition, the LDB_SINK_NONE runner's descriptor, and the builder's refusals — without a GPU."""
import ctypes as C

import pytest

from lingodb_b200 import capi, program as P

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))


def test_mark_after_probe_encodes_condition_and_table():
    b = P.Builder()
    t = C.c_void_p(71)
    cond = ("cmp", "!=", col("x"), const(3))
    r = b.expr(("mark", ("probe", t, col("k")), cond))
    ins = b.instructions()
    assert [i[0] for i in ins] == [P.OPS["load"], P.OPS["const"], P.OPS["cmp"], P.OPS["load"], P.OPS["probe"], P.OPS["mark"]]
    c, probe, mark = ins[2], ins[4], ins[5]
    # (op, dst, a = condition register, b = 0, arg = table index); the probe comes after the condition, right before the mark
    assert mark == (P.OPS["mark"], r, c[1], 0, 0)
    assert probe[4] == 0 and b.tables == [t]
    assert P.OPS["mark"] == 28 and P.SINK_NONE == 4


def test_mark_of_probe_each_reuses_the_probe_each():
    b = P.Builder()
    t, side = C.c_void_p(72), C.c_void_p(73)
    each = ("probe_each", t, col("k"), "outer")
    cond = ("cmp", "!=", ("fetch", side, each, "s"), col("s"))
    r = b.expr(("mark", each, cond))
    ops = [i[0] for i in b.instr]
    assert ops.count(P.OPS["probe_each"]) == 1
    pe = next(i for i in b.instr if i[0] == P.OPS["probe_each"])
    assert pe[3] == 1  # outer
    assert b.instr[-1][0] == P.OPS["mark"] and b.instr[-1][1] == r and b.instr[-1][4] == b.tables.index(t)
    assert b.side_columns == [(0, "s", pe[1])]
    # the same mark twice is one instruction
    assert b.expr(("mark", each, cond)) == r and [i[0] for i in b.instr].count(P.OPS["mark"]) == 1


def test_mark_on_a_second_table_and_key_tuples():
    b = P.Builder()
    t0, t1 = C.c_void_p(74), C.c_void_p(75)
    b.expr(("probe", t0, col("a")))
    r = b.expr(("mark", ("probe", t1, col("a"), col("b")), const(1)))
    mark = b.instr[-1]
    assert mark[0] == P.OPS["mark"] and mark[1] == r and mark[4] == 1
    probe = b.instr[-2]
    assert probe[0] == P.OPS["probe"] and probe[4] == 1


def test_mark_needs_a_probe_expression():
    t = C.c_void_p(76)
    for bad in [("mark", col("k"), const(1)), ("mark", ("strcode", t, "s"), const(1)), ("mark", ("probe", t, col("k"))), ("mark",)]:
        with pytest.raises(ValueError, match="mark takes a probe or probe_each expression and a condition"):
            P.Builder().expr(bad)


def test_mark_refuses_a_probe_on_a_dictionary():
    b = P.Builder()
    d = C.c_void_p(77)
    b.expr(("strcode", d, "s"))
    with pytest.raises(ValueError, match="the probed table is a string dictionary"):
        b.expr(("mark", ("probe", d, col("k")), const(1)))


def test_mark_refuses_a_later_probe_of_the_same_table():
    b = P.Builder()
    t = C.c_void_p(78)
    each = ("probe_each", t, col("k"))
    b.expr(each)
    with pytest.raises(ValueError, match="another probe of the same table runs between the probe and the mark"):
        b.expr(("mark", each, ("isnull", ("probe", t, col("j")))))


def test_effects_only_descriptor():
    b = P.Builder()
    t = C.c_void_p(79)
    b.expr(("mark", ("probe", t, col("k")), const(1)))
    d, keep = P._desc(None, type("T", (), {"h": None})(), b, -1)
    d.sink_kind = P.SINK_NONE
    assert d.sink_kind == 4 and not d.sink and d.n_tables == 1 and d.n_instr == 4 and d.filter_reg == -1
    assert d.instr[3].op == P.OPS["mark"]


def test_marks_entry_points_are_bound():
    assert capi.SIGNATURES["ldb_gpu_join_table_marks"] == (C.c_int, [C.c_void_p, C.c_int32, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(capi.Error)])
    assert capi.SIGNATURES["ldb_gpu_join_table_clear_marks"] == (C.c_int, [C.c_void_p, C.POINTER(capi.Error)])
    assert (P.MARKED, P.UNMARKED, P.ALL) == (1, 0, -1)
