"""An exact model of ldb_gpu_table_window (include/ldb_gpu.h, csrc/window.cu), rule for rule:

- rows in window order: partition keys ascending, then the order keys (a NULL greater than any value, DESC swaps), then source row;
- partitions: runs of rows equal on every partition key, NULL equal to NULL;
- ROWS frame [frm, to] (None = unbounded): a finite bound of the row at position j of a partition of length n is min(n - 1, max(0, j +
  offset)), as the reference clamps it; UNBOUNDED FOLLOWING is the partition end (the SQL meaning, not the reference's i64 wrap);
- ROW_NUMBER = i - lo + 1, COUNT_STAR = hi - lo + 1, COUNT = the non-NULL values of [lo, hi]; SUM, MIN, MAX over the non-NULL values,
  None when there are none; SUM wraps to a signed 128-bit integer.

Values are Python ints (raw decimals, days, char(1) codes), bytes for utf8, None for NULL."""
from functools import cmp_to_key

M128 = (1 << 128) - 1


def wrap128(v: int) -> int:
    v &= M128
    return v - (1 << 128) if v >> 127 else v


def _cmp_key(a, b, desc: bool) -> int:
    if a is None or b is None:
        c = (a is None) - (b is None)  # NULL greater than any value
    else:
        c = (a > b) - (a < b)
    return -c if desc else c


def window_order(cols: dict, partition_by: list, order_by: list) -> list:
    """the source row numbers in window order"""
    keys = [(c, False) for c in partition_by] + [(c, bool(d)) for c, d in order_by]
    n = len(next(iter(cols.values()))) if cols else 0

    def cmp(i, j):
        for c, d in keys:
            r = _cmp_key(cols[c][i], cols[c][j], d)
            if r:
                return r
        return 0
    return sorted(range(n), key=cmp_to_key(cmp))  # stable: ties keep source row order


def frame_bounds(s: int, e: int, i: int, frm, to) -> tuple:
    """[lo, hi] of row i of the partition [s, e] (window positions)"""
    n, j = e - s + 1, i - s
    lo = s if frm is None else s + min(n - 1, max(0, j + frm))
    hi = e if to is None else s + min(n - 1, max(0, j + to))
    return lo, hi


def window(cols: dict, partition_by: list, order_by: list, frame: tuple, funcs: list) -> tuple:
    """(order, {function name: values in window order}); funcs: [(kind, column, name)] with the kinds of capi.WIN"""
    order = window_order(cols, partition_by, order_by)
    n = len(order)
    parts = []  # [s, e] of each partition
    for i in range(n):
        if i == 0 or any(cols[c][order[i]] != cols[c][order[i - 1]] for c in partition_by):
            parts.append([i, i])
        else:
            parts[-1][1] = i
    frm, to = frame
    bounds = [None] * n
    for s, e in parts:
        for i in range(s, e + 1):
            bounds[i] = (s, e) + frame_bounds(s, e, i, frm, to)
    out = {}
    for kind, column, name in funcs:
        if kind in ("row_number", "rank"):
            out[name] = [i - b[2] + 1 for i, b in enumerate(bounds)]
            continue
        if kind == "count_star":
            out[name] = [b[3] - b[2] + 1 for b in bounds]
            continue
        v = [cols[column][r] for r in order]
        if kind in ("sum", "count"):
            ps, pc = [0], [0]
            for x in v:
                ps.append(ps[-1] + (x if kind == "sum" and x is not None else 0))
                pc.append(pc[-1] + (x is not None))
            cnt = [pc[b[3] + 1] - pc[b[2]] for b in bounds]
            if kind == "count":
                out[name] = cnt
            else:
                out[name] = [wrap128(ps[b[3] + 1] - ps[b[2]]) if c else None for b, c in zip(bounds, cnt)]
            continue
        pick = min if kind == "min" else max

        def better(a, x):
            return x if a is None else a if x is None else pick(a, x)
        res = [None] * n
        for s, e in parts:
            pre, suf = [None] * (e - s + 1), [None] * (e - s + 1)
            acc = None
            for i in range(s, e + 1):
                acc = better(acc, v[i])
                pre[i - s] = acc
            acc = None
            for i in range(e, s - 1, -1):
                acc = better(acc, v[i])
                suf[i - s] = acc
            for i in range(s, e + 1):
                lo, hi = bounds[i][2], bounds[i][3]
                if lo == s:
                    res[i] = pre[hi - s]
                elif hi == e:
                    res[i] = suf[lo - s]
                else:
                    acc = None
                    for x in v[lo:hi + 1]:
                        acc = better(acc, x)
                    res[i] = acc
        out[name] = res
    return order, out
