"""An exact model of ldb_gpu_table_window_ex (include/ldb_gpu.h, csrc/window.cu): RANGE frames and the ranking, offset and value
functions, standard SQL as PostgreSQL implements it, on top of _windowref's order and ROWS frames.

- peers: rows of a partition equal on every order key, NULL equal to NULL; without order keys the whole partition;
- ROWS frames: _windowref.frame_bounds (the reference's clamping, never empty);
- RANGE frames, per bound: None = the partition end, 0 = the first / last peer, an offset the rows of the partition's non-NULL keys
  whose key lies in [key + frm, key + to] (DESC: [key - to, key - frm], read in the order's direction).  As PostgreSQL walks its frame
  head and tail, a non-NULL row's offset bound stops at the edge of the partition's non-NULL run: a head past every key is the first
  row after the run, a tail before every key the last row before it.  A NULL-key row takes its NULL peers for an offset bound.  The
  frame is the positions [lo, hi], empty when lo > hi;
- functions over the frame: count_star, count, sum, min, max as in _windowref (0 / None over an empty frame), first_value,
  last_value, nth_value(n) (None past the frame);
- functions over the partition (row at position j of a partition of len rows): row_number (RANGE: j + 1), sql_rank, dense_rank,
  percent_rank, cume_dist, ntile(n), lag(n) / lead(n) with their default.

Values are Python ints (raw decimals, days, char(1) codes), floats, bytes for utf8, None for NULL."""
import bisect
import collections

import _windowref as W

VALUE_KINDS = ("lag", "lead", "first_value", "last_value", "nth_value")


def _parts(cols: dict, order: list, keys: list) -> list:
    """[s, e] of each run of rows equal on `keys` (NULL equal to NULL), in window positions"""
    runs = []
    for i in range(len(order)):
        if i == 0 or any(cols[c][order[i]] != cols[c][order[i - 1]] for c in keys):
            runs.append([i, i])
        else:
            runs[-1][1] = i
    return runs


def _range_bounds(i, s, e, ps, pe, key, run, desc, frm, to):
    """[lo, hi] of the RANGE frame of row i: partition [s, e], peers [ps, pe], key[p] the order key at position p; run = (ns, ne, ks)
    the partition's non-NULL keys at [ns, ne] and ks those keys ascending (negated under DESC)"""
    k = key[i] if key is not None else None  # no key words without an offset bound: only UNBOUNDED and CURRENT ROW read below
    ns, ne, ks = run if run is not None else (s, e, [])

    def head(off):  # the first row whose key is at or past key + off in the order's direction, else the row after the run
        return ns + bisect.bisect_left(ks, -(k - off) if desc else k + off)

    def tail(off):  # the last row whose key is at or before key + off in the order's direction, else the row before the run
        return ns + bisect.bisect_right(ks, -(k - off) if desc else k + off) - 1
    if frm is None:
        lo = s
    elif frm == 0 or k is None:
        lo = ps
    else:
        lo = head(frm)
    if to is None:
        hi = e
    elif to == 0 or k is None:
        hi = pe
    else:
        hi = tail(to)
    return lo, hi


def _extreme(v: list, bounds: list, parts: list, pick) -> list:
    """min / max of the non-NULL values of each frame: lo and hi never decrease within a partition, so one sliding deque each"""
    res = [None] * len(v)
    for s, e in parts:
        dq, r = collections.deque(), s
        for i in range(s, e + 1):
            lo, hi = bounds[i]
            while r <= hi:
                if v[r] is not None:
                    while dq and pick(v[r], v[dq[-1]]) == v[r] and v[r] != v[dq[-1]]:
                        dq.pop()
                    dq.append(r)
                r += 1
            while dq and dq[0] < lo:
                dq.popleft()
            res[i] = v[dq[0]] if dq and lo <= hi else None
    return res


def _ntile(j: int, size: int, n: int) -> int:
    q, r = divmod(size, n)
    big = r * (q + 1)
    return j // (q + 1) + 1 if j < big else r + (j - big) // q + 1


def window_ex(cols: dict, partition_by: list, order_by: list, frame: tuple, funcs: list, mode: str = "rows") -> tuple:
    """(order, {function name: values in window order}); funcs: [(kind, column, name[, n[, default]])] with the kinds of capi.WIN"""
    order = W.window_order(cols, partition_by, order_by)
    n = len(order)
    okeys = [c for c, _ in order_by]
    part = [None] * n  # (s, e)
    parts = _parts(cols, order, partition_by)
    for s, e in parts:
        for i in range(s, e + 1):
            part[i] = (s, e)
    peer, group = [None] * n, [0] * n  # (ps, pe); the 1-based peer group within the partition
    for s, e in _parts(cols, order, partition_by + okeys):
        for i in range(s, e + 1):
            peer[i] = (s, e)
            group[i] = group[s - 1] + 1 if s > 0 and part[s - 1][0] == part[s][0] else 1
    frm, to = frame
    offsets = mode == "range" and any(b not in (None, 0) for b in frame)  # one integer, date or decimal order key
    key = [cols[okeys[0]][r] for r in order] if offsets else None
    desc = bool(order_by and order_by[0][1])
    runs = {}
    if key is not None:
        for s, e in parts:
            nn = [p for p in range(s, e + 1) if key[p] is not None]
            runs[s] = (nn[0], nn[-1], [-key[p] if desc else key[p] for p in nn]) if nn else (s, s - 1, [])
    bounds = []
    for i in range(n):
        s, e = part[i]
        if mode == "rows":
            bounds.append(W.frame_bounds(s, e, i, frm, to))
        else:
            bounds.append(_range_bounds(i, s, e, peer[i][0], peer[i][1], key, runs.get(s), desc, frm, to))
    out = {}
    for f in funcs:
        kind, column, name = f[0], f[1], f[2]
        m = f[3] if len(f) > 3 and f[3] is not None else (1 if kind in ("lag", "lead") else 0)
        default = f[4] if len(f) > 4 else None
        v = [cols[column][r] for r in order] if column is not None else None
        if kind in ("min", "max"):
            out[name] = _extreme(v, bounds, parts, min if kind == "min" else max)
            continue
        if kind in ("count", "sum"):
            pc, psum = [0], [0]
            for x in v:
                pc.append(pc[-1] + (x is not None))
                psum.append(psum[-1] + (x if kind == "sum" and x is not None else 0))
        res = []
        for i in range(n):
            s, e = part[i]
            size, j = e - s + 1, i - s
            ps, pe = peer[i]
            lo, hi = bounds[i]
            cnt = pc[hi + 1] - pc[lo] if kind in ("count", "sum") and lo <= hi else 0
            if kind in ("row_number", "rank"):
                res.append(j + 1 if mode == "range" else i - lo + 1)
            elif kind == "count_star":
                res.append(max(0, hi - lo + 1))
            elif kind == "count":
                res.append(cnt)
            elif kind == "sum":
                res.append(W.wrap128(psum[hi + 1] - psum[lo]) if cnt else None)
            elif kind == "sql_rank":
                res.append(ps - s + 1)
            elif kind == "dense_rank":
                res.append(group[i])
            elif kind == "percent_rank":
                res.append((ps - s) / (size - 1) if size > 1 else 0.0)
            elif kind == "cume_dist":
                res.append((pe - s + 1) / size)
            elif kind == "ntile":
                res.append(_ntile(j, size, m))
            elif kind in ("lag", "lead"):
                p = i - m if kind == "lag" else i + m
                res.append(v[p] if s <= p <= e else default)
            elif kind == "first_value":
                res.append(v[lo] if lo <= hi else None)
            elif kind == "last_value":
                res.append(v[hi] if lo <= hi else None)
            elif kind == "nth_value":
                res.append(v[lo + m - 1] if lo <= hi and m - 1 <= hi - lo else None)
            else:
                raise ValueError(kind)
        out[name] = res
    return order, out
