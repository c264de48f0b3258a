"""An exact model of ldb_gpu_table_setop (include/ldb_gpu.h, csrc/setop.cu), rule for rule:

- a row is a tuple of cells: Python ints (integers, raw decimals of any width, days, char(1) codes), floats, bytes for utf8, None for NULL;
- rows are equal when every cell is (IS NOT DISTINCT FROM): None equals None and nothing else, floats after -0.0 -> +0.0 and every NaN
  -> one NaN (canon), everything else by value;
- multiplicities, cL / cR a row's occurrences in left / right: DISTINCT and UNION 1, UNION ALL the rows of both sides unchanged,
  INTERSECT 1 if cL > 0 and cR > 0, EXCEPT 1 if cL > 0 and cR == 0, INTERSECT ALL min(cL, cR), EXCEPT ALL max(cL - cR, 0);
- order: each distinct row at the position of its first occurrence in left + right, its copies consecutive, its cells those of that
  first occurrence."""
import math

KINDS = ("distinct", "union_all", "union", "intersect", "intersect_all", "except", "except_all")
_NAN = object()


def canon_cell(v):
    """the equality key of one cell"""
    if isinstance(v, float):
        if math.isnan(v):
            return _NAN
        return 0.0 if v == 0.0 else v  # -0.0 == 0.0 already; the key makes it explicit
    return v


def canon(row) -> tuple:
    return tuple(canon_cell(v) for v in row)


def setop(kind: str, left: list, right=None) -> list:
    """the result rows of `kind` over lists of row tuples, in the call's order"""
    if kind == "distinct":
        assert right is None
        right = []
    if kind == "union_all":
        return list(left) + list(right)
    cl, cr, first = {}, {}, {}
    for r in left:
        k = canon(r)
        cl[k] = cl.get(k, 0) + 1
        first.setdefault(k, r)
    for r in right:
        k = canon(r)
        cr[k] = cr.get(k, 0) + 1
        if kind in ("distinct", "union"):
            first.setdefault(k, r)
    out = []
    for k, r in first.items():  # dict order: first occurrence in left + right
        a, b = cl.get(k, 0), cr.get(k, 0)
        times = {"distinct": 1, "union": 1, "intersect": int(a > 0 and b > 0), "except": int(a > 0 and b == 0),
                 "intersect_all": min(a, b), "except_all": max(a - b, 0)}[kind]
        out.extend([r] * times)
    return out


def same_cells(a, b) -> bool:
    """two result rows cell for cell, float zeros by sign and NaN equal to NaN"""
    if len(a) != len(b):
        return False
    for x, y in zip(a, b):
        if isinstance(x, float) and isinstance(y, float):
            if math.isnan(x) and math.isnan(y):
                continue
            if x != y or math.copysign(1.0, x) != math.copysign(1.0, y):
                return False
        elif x != y or type(x) is not type(y):
            return False
    return True
