"""The set-operation model (tests/_setopref.py) against the reference's own answers: the six queries of test/sqlite-small/setops.test and
every 8th compound query of test/sqlite/select4.test whose reading does not depend on operator precedence (tests/golden/setops.json, made by
tests/golden/make_setops.py), and hand-worked cases of the rules the reference's tests do not reach: NULL rows, float zeros and NaN,
narrowed against wide decimals, '' against NULL, t EXCEPT ALL t and ALL counts of 0, 1 and many."""
import hashlib
import json
import os
import re

import pytest

import _setopref as S

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "setops.json")
OP_KIND = {"UNION ALL": "union_all", "UNION": "union", "EXCEPT": "except", "INTERSECT": "intersect", "EXCEPT ALL": "except_all",
           "INTERSECT ALL": "intersect_all"}
OP_LINE = re.compile(r"^\s*(UNION ALL|UNION|EXCEPT ALL|EXCEPT|INTERSECT ALL|INTERSECT)\s*$")


def golden():
    with open(GOLDEN) as fh:
        return json.load(fh)


def split_compound(sql: str):
    """operands and the operators between them, from a compound query written one operator per line"""
    operands, ops, cur = [], [], []
    for ln in sql.split("\n"):
        m = OP_LINE.match(ln)
        if m:
            operands.append(" ".join(cur))
            ops.append(OP_KIND[m.group(1)])
            cur = []
        else:
            cur.append(ln.strip())
    operands.append(" ".join(cur))
    return operands, ops


def chain(operands: list, ops: list) -> list:
    """the operators applied left to right, each result the next left side"""
    acc = operands[0]
    for op, rows in zip(ops, operands[1:]):
        acc = S.setop(op, acc, rows)
    return acc


# ---------------------------------------------------------------------------------------------------- a small WHERE evaluator
TOKEN = re.compile(r"\s*(?:(\d+)|([A-Za-z_]\w*)|(<>|<=|>=|!=|[=<>(),]))")


def tokens(s: str) -> list:
    out, pos = [], 0
    s = s.strip()
    while pos < len(s):
        m = TOKEN.match(s, pos)
        assert m and m.end() > pos, f"cannot read {s[pos:]!r}"
        pos = m.end()
        out.append(int(m.group(1)) if m.group(1) else m.group(2).upper() if m.group(2) and m.group(2).upper() in ("AND", "OR", "NOT", "IN") else
                   ("col", m.group(2)) if m.group(2) else m.group(3))
    return out


class Where:
    """=, <>, <, <=, >, >=, IN (…), AND, OR, NOT and parentheses over integer columns and integer literals"""

    def __init__(self, text: str):
        self.t, self.i = tokens(text), 0
        self.tree = self.disj()
        assert self.i == len(self.t), f"trailing tokens in {text!r}"

    def peek(self):
        return self.t[self.i] if self.i < len(self.t) else None

    def take(self, want=None):
        x = self.t[self.i]
        assert want is None or x == want, (x, want)
        self.i += 1
        return x

    def disj(self):
        x = self.conj()
        while self.peek() == "OR":
            self.take()
            x = ("or", x, self.conj())
        return x

    def conj(self):
        x = self.neg()
        while self.peek() == "AND":
            self.take()
            x = ("and", x, self.neg())
        return x

    def neg(self):
        if self.peek() == "NOT":
            self.take()
            return ("not", self.neg())
        return self.pred()

    def pred(self):
        if self.peek() == "(":
            self.take()
            x = self.disj()
            self.take(")")
            return x
        a = self.take()
        if self.peek() == "NOT" and self.t[self.i + 1] == "IN":
            self.take()
            return ("not", self.in_list(a))
        if self.peek() == "IN":
            return self.in_list(a)
        op = self.take()
        return ("cmp", op, a, self.take())

    def in_list(self, a):
        self.take("IN")
        self.take("(")
        vals = [self.take()]
        while self.peek() == ",":
            self.take()
            vals.append(self.take())
        self.take(")")
        return ("in", a, vals)

    def eval(self, row: dict, x=None):
        x = self.tree if x is None else x
        val = lambda v: row[v[1]] if isinstance(v, tuple) else v
        if x[0] == "or":
            return self.eval(row, x[1]) or self.eval(row, x[2])
        if x[0] == "and":
            return self.eval(row, x[1]) and self.eval(row, x[2])
        if x[0] == "not":
            return not self.eval(row, x[1])
        if x[0] == "in":
            return val(x[1]) in [val(v) for v in x[2]]
        a, b = val(x[2]), val(x[3])
        return {"=": a == b, "<>": a != b, "!=": a != b, "<": a < b, "<=": a <= b, ">": a > b, ">=": a >= b}[x[1]]


SELECT = re.compile(r"^SELECT (.+?) FROM (t\d)(?: WHERE (.*))?$")


def operand_rows(text: str, tables: dict) -> list:
    """the rows of one `SELECT cols FROM tN [WHERE …]` operand, in table order"""
    m = SELECT.match(text.strip())
    assert m, text
    cols = [c.strip() for c in m.group(1).split(",")]
    tab = m.group(2)
    names = [f"{c}{tab[1:]}" for c in "abcde"]
    where = Where(m.group(3)) if m.group(3) else None
    out = []
    for r in tables[tab]:
        row = dict(zip(names, r))
        if where is None or where.eval(row):
            out.append(tuple(row[c] for c in cols))
    return out


def valuesort_answer(rows: list):
    """the answer as select4.test states it: every value as text, sorted; listed, or counted and hashed (md5 of value + newline each)"""
    vals = sorted(str(v) for r in rows for v in r)
    return vals, len(vals), hashlib.md5("".join(v + "\n" for v in vals).encode()).hexdigest()


def values_rows(text: str) -> list:
    """`(values (1),(2),…)` as single-column rows"""
    return [(int(v),) for v in re.findall(r"\((-?\d+)\)", text)]


# ---------------------------------------------------------------------------------------------------- the reference's answers
def test_setops_test_answers():
    g = golden()["setops_test"]
    assert len(g) == 6
    for q in g:
        operands, ops = split_compound(q["sql"])
        got = chain([values_rows(o) for o in operands], ops)
        assert sorted(str(r[0]) for r in got) == sorted(q["rows"]), q["sql"]


def test_select4_answers():
    g = golden()["select4"]
    tables = {k: [tuple(r) for r in v] for k, v in g["tables"].items()}
    assert sum(len(v) for v in tables.values()) == 1000
    assert len(g["queries"]) == (g["qualifying_queries_in_file"] + 7) // 8  # every 8th query whose reading has no precedence question
    for q in g["queries"]:
        operands, ops = split_compound(q["sql"])
        assert "intersect" not in ops[1:]
        got = chain([operand_rows(o, tables) for o in operands], ops)
        vals, n, md5 = valuesort_answer(got)
        if "md5" in q:
            assert (n, md5) == (q["n_values"], q["md5"]), f"select4.test:{q['line']}"
        else:
            assert vals == sorted(q["values"]), f"select4.test:{q['line']}"


# ---------------------------------------------------------------------------------------------------- hand-worked cases
def test_null_rows():
    L = [(1, None), (None, None), (1, None), (None, 2), (None, None)]
    R = [(None, None), (1, 2)]
    assert S.setop("distinct", L) == [(1, None), (None, None), (None, 2)]
    assert S.setop("union", L, R) == [(1, None), (None, None), (None, 2), (1, 2)]
    assert S.setop("intersect", L, R) == [(None, None)]
    assert S.setop("except", L, R) == [(1, None), (None, 2)]
    assert S.setop("intersect_all", L, R) == [(None, None)]
    assert S.setop("except_all", L, R) == [(1, None), (1, None), (None, None), (None, 2)]
    assert S.setop("union_all", L, R) == L + R


def test_float_zero_and_nan():
    nan = float("nan")
    L = [(-0.0,), (0.0,), (nan,), (float("-nan"),), (1.5,)]
    got = S.setop("distinct", L)
    assert len(got) == 3
    assert S.same_cells(got[0], (-0.0,)) and not S.same_cells(got[0], (0.0,))  # the first occurrence's cells: the sign of its zero
    assert S.same_cells(got[1], (nan,)) and S.same_cells(got[2], (1.5,))
    got = S.setop("intersect", [(0.0,), (nan,)], [(-0.0,), (float("nan"),)])
    assert len(got) == 2 and S.same_cells(got[0], (0.0,)) and S.same_cells(got[1], (nan,))
    assert S.setop("except", [(0.0,), (nan,), (2.0,)], [(-0.0,), (float("nan"),)]) == [(2.0,)]
    got = S.setop("intersect_all", [(-0.0,)] * 3, [(0.0,)] * 2)
    assert len(got) == 2 and all(S.same_cells(r, (-0.0,)) for r in got)

def test_narrow_and_wide_decimals():
    # a decimal is its raw value whatever cell width held it: 8-byte 12345 and 16-byte 12345 are one row; values past 64 bits differ
    L = [(12345,), (-1,), ((1 << 64) + 5,)]
    R = [(12345,), (5,), (-1,)]
    assert S.setop("intersect", L, R) == [(12345,), (-1,)]
    assert S.setop("except", L, R) == [((1 << 64) + 5,)]


def test_empty_string_is_not_null():
    L = [(b"",), (None,), (b"",), (b"a",)]
    R = [(None,)]
    assert S.setop("distinct", L) == [(b"",), (None,), (b"a",)]
    assert S.setop("except", L, R) == [(b"",), (b"a",)]
    assert S.setop("intersect", L, R) == [(None,)]


def test_same_table_both_sides():
    t = [(1,), (2,), (2,), (None,)]
    assert S.setop("except_all", t, t) == []
    assert S.setop("except", t, t) == []
    assert S.setop("intersect_all", t, t) == t
    assert S.setop("intersect", t, t) == [(1,), (2,), (None,)]
    assert S.setop("union", t, t) == [(1,), (2,), (None,)]
    assert S.setop("union_all", t, t) == t + t


@pytest.mark.parametrize("cl,cr", [(0, 3), (1, 0), (1, 1), (3, 1), (1, 3), (1000, 999), (999, 1000), (5000, 0)])
def test_all_counts(cl, cr):
    L = [(7,)] * cl + [(8,)]
    R = [(9,)] + [(7,)] * cr
    ia = S.setop("intersect_all", L, R)
    ea = S.setop("except_all", L, R)
    assert ia == [(7,)] * min(cl, cr)
    assert ea == [(7,)] * max(cl - cr, 0) + [(8,)]
    assert S.setop("intersect", L, R) == ([(7,)] if cl and cr else [])
    assert S.setop("except", L, R) == ([(7,)] if cl and not cr else []) + [(8,)]
