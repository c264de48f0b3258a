"""An exact model of ldb_gpu_table_nl_join (include/ldb_gpu.h, csrc/nljoin.cu), rule for rule:

- a row is a dict of cells: Python ints (integers, raw decimals of any width, days, char(1) codes), floats, None for NULL;
- a condition is (left column, op, right column[, constant]) with one column None to compare the other with the constant
  ((None, op, c, v) reads  v OP right.c); a condition is TRUE only when no operand is NULL or NaN and the comparison holds (the ordered
  float predicates: NaN is never TRUE, not even for "!=", and -0.0 == +0.0 as Python compares them);
- a pair matches when every condition is TRUE; no conditions: every pair;
- rows, as (left id, right id) with None for the NULL-extended side: INNER the matching pairs in left row order, then right row order;
  LEFT / FULL also (left id, None) for a left row without a match at its place; RIGHT / FULL then (None, right id) for every unmatched
  right row in right row order; SEMI / ANTI the left ids with / without a match; MARK (left id, 0 / 1); COUNT (left id, matches)."""
import math

KINDS = ("inner", "left", "right", "full", "semi", "anti", "mark", "count")
OPS = {"=": lambda a, b: a == b, "!=": lambda a, b: a != b, "<": lambda a, b: a < b, "<=": lambda a, b: a <= b,
       ">": lambda a, b: a > b, ">=": lambda a, b: a >= b}


def _usable(v) -> bool:
    return v is not None and not (isinstance(v, float) and math.isnan(v))


def cond_true(a, op: str, b) -> bool:
    """one condition on two operands: UNKNOWN (NULL) and NaN operands are not TRUE"""
    return _usable(a) and _usable(b) and OPS[op](a, b)


def _split(conds):
    pairs, lsingle, rsingle = [], [], []
    for c in conds:
        lc, op, rc = c[0], c[1], c[2]
        v = c[3] if len(c) > 3 else None
        if lc is not None and rc is not None:
            pairs.append((lc, op, rc))
        elif lc is not None:
            lsingle.append((lc, op, v))
        else:
            rsingle.append((rc, op, v))
    return pairs, lsingle, rsingle


def matches(left: list, right: list, conds) -> list:
    """per left row, the ids of the right rows it matches, ascending"""
    pairs, lsingle, rsingle = _split(conds)
    lok = [all(cond_true(r[c], op, v) for c, op, v in lsingle) and all(_usable(r[c]) for c, _, _ in pairs) for r in left]
    rok = [j for j, r in enumerate(right) if all(cond_true(v, op, r[c]) for c, op, v in rsingle) and all(_usable(r[c]) for _, _, c in pairs)]
    fns = [(lc, OPS[op], rc) for lc, op, rc in pairs]
    out = []
    for i, lr in enumerate(left):
        if not lok[i]:
            out.append([])
            continue
        out.append([j for j in rok if all(f(lr[lc], right[j][rc]) for lc, f, rc in fns)])
    return out


def nl_join(kind: str, left: list, right: list, conds) -> list:
    """the result rows of `kind` (see the module's docstring), in order"""
    return rows_of(kind, matches(left, right, conds), len(right))


def rows_of(kind: str, m: list, n_right: int) -> list:
    """the result rows of `kind` from the per-left-row matches `m` over n_right right rows"""
    if kind == "semi":
        return [i for i, js in enumerate(m) if js]
    if kind == "anti":
        return [i for i, js in enumerate(m) if not js]
    if kind == "mark":
        return [(i, int(bool(js))) for i, js in enumerate(m)]
    if kind == "count":
        return [(i, len(js)) for i, js in enumerate(m)]
    out = []
    for i, js in enumerate(m):
        out.extend((i, j) for j in js)
        if not js and kind in ("left", "full"):
            out.append((i, None))
    if kind in ("right", "full"):
        hit = set(j for js in m for j in js)
        out.extend((None, j) for j in range(n_right) if j not in hit)
    return out
