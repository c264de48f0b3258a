"""The nested-loop join model (tests/_nljoinref.py) pinned to the reference's answers and to hand-worked cases of every rule in
include/ldb_gpu.h.

1. The reference's answers (tests/golden/nljoins.json, made by make_nljoins.py): every select1-3.test query whose only subquery is
   (SELECT count(*) FROM t1 AS x WHERE x.b<t1.b).  The model's COUNT join of t1 with itself on  b > b  gives the subquery's column; a
   small host evaluator (`run_query`) gives the query's other terms, its WHERE, ORDER BY and the sqllogictest answer form.
2. Hand-worked cases: NULL and NaN operands, signed zeros, integers of mixed widths, decimals beyond 64 bits, single-side conditions
   inside ON, cross products and the fixed output order of every kind."""
import hashlib
import json
import os
import re

import _nljoinref as N

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nljoins.json")
SUB = "(SELECT count(*) FROM t1 AS x WHERE x.b<t1.b)"


def golden() -> dict:
    return json.load(open(GOLDEN))


# ---------------------------------------------------------------------------------------------------- the host evaluator
_TOKEN = re.compile(r"\s*(?:(__CNT__)|([A-Za-z_][A-Za-z_0-9]*)|(\d+)|(<=|>=|<>|!=|[-+*(),<>=]))")


def _tokens(sql: str) -> list:
    rest, pos, out = sql.replace(SUB, " __CNT__ "), 0, []
    while rest[pos:].strip():
        m = _TOKEN.match(rest, pos)
        assert m, rest[pos:]
        out.append(m.group(1) or m.group(2) or m.group(3) or m.group(4))
        pos = m.end()
    return out


class _Parser:
    """SELECT exprs FROM t1 [WHERE expr] [ORDER BY n, ...] over the tokens make_nljoins.py admits; expressions as closures of
    (row, count) with SQLite's values: NULL is None, a comparison 1 / 0 / None, AND / OR / NOT three-valued"""

    def __init__(self, toks):
        self.t, self.i = toks, 0

    def peek(self, k=0):
        return self.t[self.i + k] if self.i + k < len(self.t) else None

    def take(self, want=None):
        tok = self.t[self.i]
        assert want is None or tok == want, (tok, want)
        self.i += 1
        return tok

    def query(self):
        self.take("SELECT")
        cols = [self.expr()]
        while self.peek() == ",":
            self.take()
            cols.append(self.expr())
        self.take("FROM"), self.take("t1")
        where = None
        if self.peek() == "WHERE":
            self.take()
            where = self.expr()
        order = []
        if self.peek() == "ORDER":
            self.take(), self.take("BY")
            order.append(int(self.take()))
            while self.peek() == ",":
                self.take()
                order.append(int(self.take()))
        assert self.peek() is None
        return cols, where, order

    def expr(self):
        a = self.conj()
        while self.peek() == "OR":
            self.take()
            a = (lambda x, y: lambda r: _or(x(r), y(r)))(a, self.conj())
        return a

    def conj(self):
        a = self.neg()
        while self.peek() == "AND":
            self.take()
            a = (lambda x, y: lambda r: _and(x(r), y(r)))(a, self.neg())
        return a

    def neg(self):
        if self.peek() == "NOT":
            self.take()
            x = self.neg()
            return lambda r: None if x(r) is None else int(not x(r))
        return self.pred()

    def pred(self):
        a = self.add()
        op = self.peek()
        if op in ("<", "<=", ">", ">=", "=", "<>", "!="):
            self.take()
            b = self.add()
            f = N.OPS["!=" if op == "<>" else op]
            return lambda r: None if a(r) is None or b(r) is None else int(f(a(r), b(r)))
        negate = op == "NOT" and self.peek(1) == "BETWEEN"
        if negate or op == "BETWEEN":
            if negate:
                self.take()
            self.take("BETWEEN")
            lo = self.add()
            self.take("AND")
            hi = self.add()
            inside = lambda r: _and(None if a(r) is None or lo(r) is None else int(a(r) >= lo(r)),
                                    None if a(r) is None or hi(r) is None else int(a(r) <= hi(r)))
            return (lambda r: None if inside(r) is None else int(not inside(r))) if negate else inside
        if op == "IS":
            self.take()
            want_null = True
            if self.peek() == "NOT":
                self.take()
                want_null = False
            self.take("NULL")
            return lambda r: int((a(r) is None) == want_null)
        return a

    def add(self):
        a = self.mul()
        while self.peek() in ("+", "-"):
            op = self.take()
            b = self.mul()
            a = (lambda x, y, o: lambda r: None if x(r) is None or y(r) is None else (x(r) + y(r) if o == "+" else x(r) - y(r)))(a, b, op)
        return a

    def mul(self):
        a = self.unary()
        while self.peek() == "*":
            self.take()
            a = (lambda x, y: lambda r: None if x(r) is None or y(r) is None else x(r) * y(r))(a, self.unary())
        return a

    def unary(self):
        if self.peek() in ("-", "+"):
            op = self.take()
            x = self.unary()
            return (lambda r: None if x(r) is None else -x(r)) if op == "-" else x
        tok = self.take()
        if tok == "(":
            x = self.expr()
            self.take(")")
            return x
        if tok == "__CNT__":
            return lambda r: r[1]
        if tok.isdigit():
            v = int(tok)
            return lambda r: v
        k = "abcde".index(tok)
        return lambda r: r[0][k]


def _and(x, y):
    if x == 0 or y == 0:
        return 0
    return None if x is None or y is None else 1


def _or(x, y):
    if x not in (None, 0) or y not in (None, 0):
        return 1
    return None if x is None or y is None else 0


def run_query(sql: str, rows: list, counts: list) -> list:
    """the result rows of one query over t1's rows, `counts[i]` the subquery's value for row i"""
    cols, where, order = _Parser(_tokens(sql)).query()
    out = []
    for r, c in zip(rows, counts):
        if where is None or where((r, c)) not in (None, 0):
            out.append(tuple(f((r, c)) for f in cols))
    # ORDER BY: SQLite puts NULL first; a stable sort from the last key
    for k in reversed(order):
        out.sort(key=lambda row: (row[k - 1] is not None, row[k - 1] if row[k - 1] is not None else 0))
    return out


def answer_matches(q: dict, rows: list) -> bool:
    """the answer as sqllogictest states it: nosort in result order, rowsort with rows sorted as text; listed, or counted and hashed
    (md5 of every value + newline, NULL as "NULL")"""
    text = [["NULL" if v is None else str(v) for v in r] for r in rows]
    if q["sort"] == "rowsort":
        text.sort()
    vals = [v for r in text for v in r]
    if "md5" in q:
        return len(vals) == q["n_values"] and hashlib.md5("".join(v + "\n" for v in vals).encode()).hexdigest() == q["md5"]
    return vals == q["values"]


def counts_of(t1: list) -> list:
    """the subquery's column: the model's COUNT join of t1 with itself, left.b > right.b"""
    rows = [{"b": r[1]} for r in t1]
    return [c for _, c in N.nl_join("count", rows, rows, [("b", ">", "b")])]


# ---------------------------------------------------------------------------------------------------- 1. the reference's answers
def test_reference_answers():
    g = golden()
    total = 0
    for f, v in g["files"].items():
        cnt = counts_of(v["t1"])
        for q in v["queries"]:
            assert answer_matches(q, run_query(q["sql"], v["t1"], cnt)), (f, q["line"])
            total += 1
    assert total == 154


def test_the_evaluator_is_not_vacuous():
    """a wrong count column (the subquery with <= instead of <) fails most answers, so the answers pin the count"""
    g = golden()
    wrong = right = 0
    for v in g["files"].values():
        rows = [{"b": r[1]} for r in v["t1"]]
        bad = [c for _, c in N.nl_join("count", rows, rows, [("b", ">=", "b")])]
        for q in v["queries"]:
            right += 1
            wrong += not answer_matches(q, run_query(q["sql"], v["t1"], bad))
    assert wrong > right * 0.8, (wrong, right)


# the unnesting.test / join.test queries as joins: (left values, right values, kind, conditions on the column "v"); i2.i > i1.i reads
# right.v > left.v, i.e. left.v < right.v.  x = ALL(SELECT y … WHERE y <= x) is TRUE when no y <= x differs from x: a mark join on
# (x >= y AND x != y) whose marker is FALSE.  COUNT(i) counts like COUNT(*) there: the condition already excludes a NULL i2.i.
def small_joins(ints: list) -> dict:
    lt = [("v", "<", "v")]
    return {("unnesting", 195): (ints, ints, "count", lt), ("unnesting", 281): (ints, ints, "left", lt), ("unnesting", 572): (ints, ints, "mark", lt),
            ("unnesting", 662): (ints, ints, "semi", [("v", ">", "v"), ("v", "!=", "v")]), ("unnesting", 814): (ints, ints, "count", lt),
            ("unnesting", 830): (ints, ints, "count", lt), ("join", 133): ([1, 2, 3], [2, 3, 4, 5], "mark", [("v", ">=", "v"), ("v", "!=", "v")])}


def small_answer(key, left: list, per_left: list) -> list:
    """a query's answer rows (tsv text) from its join's outcome per left row: the count (COUNT), the marker (MARK), the matched right
    values (LEFT, for MIN) or whether the row is kept (SEMI); ORDER BY i puts NULL last, as the reference does"""
    txt = lambda v: "NULL" if v is None else str(v)
    by_i = lambda rows: sorted(rows, key=lambda r: (r[0] is None, r[0] if r[0] is not None else 0))
    line = key[1]
    if line in (195, 814, 830):
        return ["\t".join(map(txt, r)) for r in by_i(list(zip(left, per_left)))]
    if line == 281:
        return ["\t".join(map(txt, r)) for r in by_i([(i, min(ms) if ms else None) for i, ms in zip(left, per_left)])]
    if line == 572:
        return ["t" if m else "f" for m in per_left]
    if line == 662:
        return [txt(r[0]) for r in by_i([(i,) for i, k in zip(left, per_left) if k])]
    return sorted(f"{x}\t{'f' if m else 't'}" for x, m in zip(left, per_left))  # join.test, rowsort


def test_unnesting_and_join_answers():
    g = golden()["small"]
    joins = small_joins(g["integers"])
    assert len(g["queries"]) == len(joins) == 7
    for q in g["queries"]:
        key = (q["file"], q["line"])
        lv, rv, kind, conds = joins[key]
        left, right = [{"v": v} for v in lv], [{"v": v} for v in rv]
        m = N.matches(left, right, conds)
        per = {"count": [len(js) for js in m], "mark": [bool(js) for js in m], "semi": [bool(js) for js in m],
               "left": [[rv[j] for j in js] for js in m]}[kind]
        assert small_answer(key, lv, per) == q["rows"], key


# ---------------------------------------------------------------------------------------------------- 2. hand-worked cases

NAN = float("nan")


def test_row_order_of_every_kind():
    left = [{"a": 1}, {"a": None}, {"a": 3}, {"a": 0}]
    right = [{"b": 0}, {"b": 2}, {"b": 5}, {"b": None}]
    c = [("a", "<", "b")]
    assert N.nl_join("inner", left, right, c) == [(0, 1), (0, 2), (2, 2), (3, 1), (3, 2)]
    assert N.nl_join("left", left, right, c) == [(0, 1), (0, 2), (1, None), (2, 2), (3, 1), (3, 2)]
    assert N.nl_join("right", left, right, c) == [(0, 1), (0, 2), (2, 2), (3, 1), (3, 2), (None, 0), (None, 3)]
    assert N.nl_join("full", left, right, c) == [(0, 1), (0, 2), (1, None), (2, 2), (3, 1), (3, 2), (None, 0), (None, 3)]
    assert N.nl_join("semi", left, right, c) == [0, 2, 3]
    assert N.nl_join("anti", left, right, c) == [1]
    assert N.nl_join("mark", left, right, c) == [(0, 1), (1, 0), (2, 1), (3, 1)]
    assert N.nl_join("count", left, right, c) == [(0, 2), (1, 0), (2, 1), (3, 2)]


def test_nan_is_never_true_and_zeros_are_equal():
    left = [{"f": NAN}, {"f": -0.0}, {"f": 1.5}]
    right = [{"g": 0.0}, {"g": NAN}, {"g": 1.5}]
    assert N.nl_join("inner", left, right, [("f", "=", "g")]) == [(1, 0), (2, 2)]
    # <> is ONE: a NaN on either side is not TRUE
    assert N.nl_join("inner", left, right, [("f", "!=", "g")]) == [(1, 2), (2, 0)]
    assert N.nl_join("count", left, right, [("f", "<=", "g")]) == [(0, 0), (1, 2), (2, 1)]
    assert N.cond_true(-0.0, ">=", 0.0) and not N.cond_true(-0.0, "<", 0.0)


def test_mixed_widths_and_decimal_cells():
    # int8 against int64 by value; decimals past 2^64 compare by their 128-bit value (the model sees values, not cells: which cell width
    # holds them is the device test's part, test_gpu_nljoin.py's "decimals" sets)
    left = [{"i8": -128, "d": 10 ** 17}, {"i8": 127, "d": -(10 ** 17)}]
    right = [{"i64": -(1 << 40), "w": (1 << 70) + 1}, {"i64": 127, "w": -(1 << 70)}, {"i64": 1 << 40, "w": 10 ** 17}]
    assert N.nl_join("inner", left, right, [("i8", "<", "i64")]) == [(0, 1), (0, 2), (1, 2)]
    assert N.nl_join("inner", left, right, [("d", "<", "w")]) == [(0, 0), (1, 0), (1, 2)]
    assert N.nl_join("inner", left, right, [("d", "=", "w")]) == [(0, 2)]


def test_single_side_conditions_are_part_of_on():
    left = [{"a": 1, "k": 5}, {"a": 2, "k": -1}, {"a": 3, "k": None}]
    right = [{"b": 9, "z": 0}, {"b": 9, "z": 7}]
    c = [("k", ">", None, 0), (None, "<=", "z", 3), ("a", "<", "b")]  # k > 0  AND  3 <= z  AND  a < b
    assert N.nl_join("inner", left, right, c) == [(0, 1)]
    # a left row failing its own condition is unmatched, not dropped
    assert N.nl_join("left", left, right, c) == [(0, 1), (1, None), (2, None)]
    assert N.nl_join("anti", left, right, c) == [1, 2]
    assert N.nl_join("count", left, right, c) == [(0, 1), (1, 0), (2, 0)]
    assert N.nl_join("full", left, right, c) == [(0, 1), (1, None), (2, None), (None, 0)]


def test_cross_product_and_empty_sides():
    left, right = [{"a": None}, {"a": 1}], [{"b": None}, {"b": 2}, {"b": 3}]
    assert N.nl_join("inner", left, right, []) == [(i, j) for i in range(2) for j in range(3)]
    assert N.nl_join("count", left, right, []) == [(0, 3), (1, 3)]
    assert N.nl_join("left", left, [], []) == [(0, None), (1, None)]
    assert N.nl_join("right", [], right, []) == [(None, 0), (None, 1), (None, 2)]
    assert N.nl_join("anti", left, [], [("a", "<", "b")]) == [0, 1]
    assert N.nl_join("mark", [], right, []) == []


def test_band_join():
    events = [{"ts": t} for t in (5, 10, 15, 20)]
    windows = [{"start": 0, "stop": 10}, {"start": 10, "stop": 19}, {"start": 30, "stop": 40}]
    c = [("ts", ">=", "start"), ("ts", "<=", "stop")]  # ts BETWEEN start AND stop
    assert N.nl_join("inner", events, windows, c) == [(0, 0), (1, 0), (1, 1), (2, 1)]
    assert N.nl_join("right", events, windows, c) == [(0, 0), (1, 0), (1, 1), (2, 1), (None, 2)]
