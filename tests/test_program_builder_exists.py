"""Builder side of probe-side EXISTS joins (lingodb_b200/program.py): the encoding of ("exists", table, key, …, cond) and of the outer
probe_each with a residual, the scoping of the expression cache around residual blocks, and the builder's refusals — without a GPU."""
import ctypes as C

import pytest

from lingodb_b200 import program as P

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))
O = P.OPS


def _block(b, at):
    """the EXISTS instruction at `at` and its block"""
    ex = b.instr[at]
    assert ex[0] == O["exists"]
    return ex, b.instr[at + 1:at + 1 + ex[3]]


def test_exists_block_length_and_match():
    b = P.Builder()
    t, side = C.c_void_p(81), C.c_void_p(82)
    cond = ("cmp", "!=", ("fetch", side, ("match", t), "v"), col("pv"))
    r = b.expr(("exists", t, col("k"), cond))
    ins = b.instructions()
    assert [i[0] for i in ins] == [O["load"], O["exists"], O["load"], O["load"], O["cmp"]]
    ex, block = _block(b, 1)
    # (op, dst, a = key register, b = block length, arg = table index); the block's last write is the residual
    assert ex == (O["exists"], r, ins[0][1], 3, 0) and b.tables == [t]
    assert b.side_columns == [(0, "v", r)]  # ("match", t) is the EXISTS's own register
    assert ins[2] == (O["load"], ins[2][1], 0, 0, 2)  # the side column, numbered after the two source columns
    assert O["exists"] == 29


def test_exists_without_residual_and_key_tuples():
    b = P.Builder()
    t = C.c_void_p(83)
    r = b.expr(("exists", t, col("a"), col("b"), None))
    ex = b.instr[-1]
    assert ex == (O["exists"], r, b.instr[0][1], 0, 0) and b.instr[1][1] == b.instr[0][1] + 1
    # keys that are not consecutive are moved first; the EXISTS reads the moved pair
    b2 = P.Builder()
    b2.expr(col("b"))
    b2.expr(col("x"))
    r2 = b2.expr(("exists", t, col("a"), col("b"), None))
    ex2 = b2.instr[-1]
    moves = b2.instr[-3:-1]
    assert all(m[0] == O["select"] for m in moves) and ex2[2] == moves[0][1] and moves[1][1] == moves[0][1] + 1 and ex2[1] == r2


def test_cache_is_scoped_to_the_block():
    b = P.Builder()
    t, side = C.c_void_p(84), C.c_void_p(85)
    pv = b.expr(col("pv"))  # cached before the block: reused inside it
    cond = ("and", ("cmp", "!=", ("fetch", side, ("match", t), "v"), col("pv")), ("cmp", ">", col("q"), const(1)))
    b.expr(("exists", t, col("k"), cond))
    ex, block = _block(b, 2)
    assert ex[3] == len(block) == len(b.instr) - 3
    assert not any(i[0] == O["load"] and i[1] == pv for i in block)
    q_in_block = next(i[1] for i in block if i[0] == O["load"] and i[4] == b.columns.index("q"))
    # after the block: "q" and the fetched column are evaluated again, pv is not
    n = len(b.instr)
    assert b.expr(col("q")) != q_in_block and len(b.instr) == n + 1
    assert b.expr(col("pv")) == pv and len(b.instr) == n + 1
    written = {i[1] for i in block}
    assert not written & set(b._cache.values()) and not written & set(b._rows.values()) and b._match is None


def test_forced_move_for_a_cached_condition():
    b = P.Builder()
    t = C.c_void_p(86)
    c = b.expr(("cmp", ">", col("x"), const(0)))
    r = b.expr(("exists", t, col("k"), ("cmp", ">", col("x"), const(0))))
    ex, block = _block(b, len(b.instr) - 2)
    assert block == [(O["select"], block[0][1], c, c, c)] and ex[3] == 1 and ex[1] == r
    # the match itself as the condition: a move too, never an empty block (b = 0 means no residual)
    b2 = P.Builder()
    r2 = b2.expr(("exists", t, col("k"), ("match", t)))
    assert b2.instr[-1] == (O["select"], b2.instr[-1][1], r2, r2, r2) and b2.instr[-2][3] == 1


def test_two_exists_and_placement_around_probe_each():
    b = P.Builder()
    t0, t1, t2 = C.c_void_p(87), C.c_void_p(88), C.c_void_p(89)
    e0 = b.expr(("exists", t0, col("k"), ("cmp", "=", col("x"), const(1))))
    m = ("probe_each", t1, col("k"))
    b.expr(m)
    e1 = b.expr(("exists", t2, col("j"), ("cmp", "!=", ("fetch", t2, ("match", t2), "s"), ("fetch", t1, m, "s"))))
    ops = [i[0] for i in b.instr]
    assert ops.count(O["exists"]) == 2 and ops.index(O["exists"]) < ops.index(O["probe_each"]) < len(ops) - 1 - ops[::-1].index(O["exists"])
    assert [i[4] for i in b.instr if i[0] == O["exists"]] == [0, 2] and b.tables == [t0, t1, t2]
    assert e0 != e1 and b.expr(("exists", t0, col("k"), ("cmp", "=", col("x"), const(1)))) == e0  # cached after its block


def test_outer_probe_each_with_residual_composition():
    b = P.Builder()
    t, side = C.c_void_p(90), C.c_void_p(91)
    cond = ("cmp", "<", ("fetch", side, ("match", t), "d"), ("col", "bound"))
    m = b.expr(("probe_each", t, col("k"), "outer", ("on", cond)))
    f = b.where(b.expr(("cmp", ">", col("z"), const(0))))
    ops = [i[0] for i in b.instr]
    ex_at = ops.index(O["exists"])
    ex, block = _block(b, ex_at)
    key = ex[2]
    after = b.instr[ex_at + 1 + ex[3]:]
    # NULL = 0 / 0, k' = SELECT(v, k, NULL), PROBE_EACH(k', outer), the residual against m, OR ISNULL(m), then the user's WHERE AND it
    div = next(i for i in after if i[0] == O["div"])
    sel = next(i for i in after if i[0] == O["select"])
    pe = next(i for i in after if i[0] == O["probe_each"])
    assert sel[2:] == (key, div[1], ex[1]) and pe == (O["probe_each"], m, sel[1], 1, 0)
    isnull = next(i for i in after if i[0] == O["isnull"])
    orr = next(i for i in after if i[0] == O["or"])
    assert isnull[2] == m and orr[3] == isnull[1]
    res = next(i for i in after if i[1] == orr[2])
    assert res[0] == O["cmp"] and after.index(res) > after.index(pe)
    assert b.instr[-1] == (O["and"], f, b.instr[-1][2], orr[1], 0)
    assert b.side_columns == [(0, "d", ex[1]), (0, "d", m)]
    # without a user WHERE the residual condition is the WHERE; where() adds it once
    b2 = P.Builder()
    b2.expr(("probe_each", t, col("k"), "outer", ("on", cond)))
    f2 = b2.where(-1)
    assert b2.instr[-1][0] == O["or"] and f2 == b2.instr[-1][1] and b2.where(-1) == -1
    b3 = P.Builder()
    b3.expr(("probe_each", t, col("k"), "outer", ("on", cond)))
    d, keep = P._desc(None, type("T", (), {"h": None})(), b3, -1)  # the descriptor takes the residual as its filter
    assert d.filter_reg == f2 and d.n_instr == len(b3.instr)


@pytest.mark.parametrize("bad,msg", [
    (lambda t, u: ("exists", t, col("k"), ("exists", u, col("j"), None)), "exists inside the condition"),
    (lambda t, u: ("exists", t, col("k"), ("mark", ("probe", u, col("j")), const(1))), "mark inside the condition"),
    (lambda t, u: ("exists", t, col("k"), ("isnull", ("probe_each", u, col("j")))), "probe_each inside the condition"),
    (lambda t, u: ("exists", t, col("k"), ("isnull", ("strcode", u, "s"))), "strcode inside the condition"),
    (lambda t, u: ("probe_each", t, col("k"), "outer", ("on", ("exists", u, col("j"), None))), "exists inside the condition"),
    (lambda t, u: ("isnull", ("match", t)), "match: only inside"),
    (lambda t, u: ("exists", t, col("k"), ("isnull", ("match", u))), "match: only inside"),
    (lambda t, u: ("probe_each", t, col("k"), ("on", const(1))), "takes the outer form"),
    (lambda t, u: ("exists", t, col("k")), "exists takes a join table"),
])
def test_builder_rejections(bad, msg):
    t, u = C.c_void_p(92), C.c_void_p(93)
    with pytest.raises(ValueError, match=msg):
        P.Builder().expr(bad(t, u))


def test_lookup_strcode_is_allowed_in_a_block_and_match_after_the_block_is_not():
    b = P.Builder()
    t, d = C.c_void_p(94), C.c_void_p(95)
    b.expr(("exists", t, col("k"), ("isnull", ("strcode", d, "s", "lookup"))))
    assert b.instr[2][0] == O["strcode"] and b.instr[2][3] == 0
    with pytest.raises(ValueError, match="match: only inside"):
        b.expr(("match", t))
