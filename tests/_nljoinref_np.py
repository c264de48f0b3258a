"""A vectorised twin of the nested-loop join model (tests/_nljoinref.py) for sides too large for the pure-Python model.

The sides are dicts of columns (lists of cells as _nljoinref reads them: ints, floats, None for NULL); conditions are _nljoinref's.
`matches` returns per left row the ascending ids of the right rows it matches, `rows_of` the result rows of a kind, both equal to
_nljoinref's (tests/test_nljoinref_np.py pins them on seeded tables)."""
import math

import numpy as np

import _nljoinref as N

OPS = {"=": np.equal, "!=": np.not_equal, "<": np.less, "<=": np.less_equal, ">": np.greater, ">=": np.greater_equal}
_I64 = (-(1 << 63), (1 << 63) - 1)


def _usable(vals) -> np.ndarray:
    return np.array([v is not None and not (isinstance(v, float) and math.isnan(v)) for v in vals], bool)


def _values(vals, usable: np.ndarray) -> np.ndarray:
    """the cells as one array: float64 for floats, int64 for integers that fit it, else Python ints (16-byte decimals)"""
    present = [v for v, u in zip(vals, usable) if u]
    if any(isinstance(v, float) for v in present):
        return np.array([float(v) if u else 0.0 for v, u in zip(vals, usable)], np.float64)
    if all(_I64[0] <= v <= _I64[1] for v in present):
        return np.array([v if u else 0 for v, u in zip(vals, usable)], np.int64)
    return np.array([v if u else 0 for v, u in zip(vals, usable)], object)


def _side_ok(side: dict, n: int, singles, pair_cols) -> np.ndarray:
    ok = np.ones(n, bool)
    for c, op, v, const_left in singles:
        u = _usable(side[c])
        x = _values(side[c], u)
        cu = v is not None and not (isinstance(v, float) and math.isnan(v))
        if not cu:
            ok[:] = False
            continue
        with np.errstate(invalid="ignore"):
            ok &= u & (OPS[op](v, x) if const_left else OPS[op](x, v))
    for c in pair_cols:
        ok &= _usable(side[c])
    return ok


def matches(left: dict, right: dict, conds, n: int, m: int, block_pairs: int = 1 << 22) -> list:
    """per left row, the ascending ids of the right rows it matches"""
    pairs, lsingle, rsingle = N._split(conds)
    lok = _side_ok(left, n, [(c, op, v, False) for c, op, v in lsingle], [p[0] for p in pairs])
    rok = _side_ok(right, m, [(c, op, v, True) for c, op, v in rsingle], [p[2] for p in pairs])
    lv = [_values(left[lc], _usable(left[lc])) for lc, _, _ in pairs]
    rv = [_values(right[rc], _usable(right[rc])) for _, _, rc in pairs]
    out = []
    b = max(1, block_pairs // max(m, 1))
    for a in range(0, n, b):
        e = min(n, a + b)
        M = lok[a:e, None] & rok[None, :]
        for (lc, op, rc), x, y in zip(pairs, lv, rv):
            M &= OPS[op](x[a:e, None], y[None, :])
        out.extend(np.flatnonzero(row) for row in M)
    return out


def rows_of(kind: str, m: list, n_right: int) -> list:
    """_nljoinref.rows_of over the per-left-row matches `m` (arrays of right ids)"""
    lens = np.array([len(js) for js in m], np.int64)
    ids = np.arange(len(m))
    if kind == "semi":
        return ids[lens > 0].tolist()
    if kind == "anti":
        return ids[lens == 0].tolist()
    if kind == "mark":
        return list(zip(ids.tolist(), (lens > 0).astype(int).tolist()))
    if kind == "count":
        return list(zip(ids.tolist(), lens.tolist()))
    outer = kind in ("left", "full")
    per = np.where(outer & (lens == 0), 1, lens)
    li = np.repeat(ids, per)
    ri = np.full(len(li), -1, np.int64)
    matched = np.concatenate([js for js in m]) if m else np.zeros(0, np.int64)
    starts = np.concatenate([[0], np.cumsum(per)[:-1]]) if len(per) else np.zeros(0, np.int64)
    pos = np.repeat(starts, lens) + (np.arange(len(matched)) - np.repeat(np.concatenate([[0], np.cumsum(lens)[:-1]]) if len(lens) else lens, lens))
    ri[pos] = matched
    out = [(i, None if j < 0 else j) for i, j in zip(li.tolist(), ri.tolist())]
    if kind in ("right", "full"):
        hit = np.zeros(n_right, bool)
        hit[matched.astype(np.int64)] = True
        out.extend((None, j) for j in np.flatnonzero(~hit).tolist())
    return out
