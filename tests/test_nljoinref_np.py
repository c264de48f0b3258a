"""The vectorised twin (tests/_nljoinref_np.py) against the exact nested-loop join model (tests/_nljoinref.py): seeded tables with
NULLs, NaN, signed zeros and 16-byte decimals, every kind, and the condition shapes of the sorted-ranges path (a range, a band, a
band of two probe columns, equality plus range, equality only, residuals, constants in ON, a cross product)."""
import pytest

import _nljoinref as N
import _nljoinref_np as V
from test_gpu_setop import gen_rows, group_fn

SHAPES = [
    ("range", [("i32", "<", "i32")]),
    ("band", [("i32", ">=", "i32"), ("i32", "<", "j32")]),
    ("band_two_probe", [("i32", "<=", "i32"), ("j32", ">", "i32")]),
    ("eq_range", [("i8", "=", "i8"), ("dt", "<", "dt")]),
    ("eq_only", [("fs", "=", "fs")]),
    ("residual_ne", [("i64", "<=", "i64"), ("i16", "!=", "k16")]),
    ("residual_range", [("i32", "<", "i32"), ("f8", ">=", "f4")]),
    ("decimals", [("dn", "<", "dw"), ("dw", ">=", "dn")]),
    ("floats", [("f4", "<", "f8"), ("e8", ">", "f8")]),
    ("constants", [("i8", ">", None, -20), (None, "<=", "i16", 0), ("i32", ">", "i32")]),
    ("cross", []),
]


@pytest.mark.parametrize("name,conds", SHAPES)
@pytest.mark.parametrize("n,m", [(0, 5), (5, 0), (40, 57), (131, 64)])
def test_twin_equals_the_model(name, conds, n, m):
    lv = gen_rows(n, group_fn(max(1, n // 4 + 3)), 300 + n)
    rv = gen_rows(m, group_fn(max(1, m // 3 + 3), 2), 400 + m)
    want = N.matches([{c: lv[c][i] for c in lv} for i in range(n)], [{c: rv[c][j] for c in rv} for j in range(m)], conds)
    got = V.matches(lv, rv, conds, n, m, block_pairs=256)
    assert [g.tolist() for g in got] == want
    for kind in N.KINDS:
        assert V.rows_of(kind, got, m) == N.rows_of(kind, want, m), kind
