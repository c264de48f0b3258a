"""The sorted-ranges path of nested-loop joins (csrc/nljoin_sorted.cu) against the exact model, through the vectorised twin
(tests/_nljoinref_np.py) where the sides are too large for the pure-Python model:

1. which path runs, from the per-family launch counts: the sorted ranges for a range, bands, equality plus range, equality only and
   equality with residuals in both orientations; the loop for a cross product, <> only, constants only and fewer than
   kNljSortMinPairs pairs; the sorted count, then the loop, for joins whose candidates exceed n m / kNljCandidateRatio;
2. every kind over every key shape, with residuals and constants in ON, over every operand family with NULLs, NaN and signed zeros,
   on ragged, bit-offset and single-batch HOST tables, result tables and a self join, each on the sorted path and matching rows;
3. ties and order: one key for every row, keys in row order (the order sort skipped) against shuffled keys (the order sort run),
   unmatched right rows under RIGHT and FULL;
4. extremes: int64, 16-byte decimal and infinite keys and bounds, < against <= at equal values;
5. the loop on a left slice against the matching rows of the sorted result over the whole left side;
6. scale against numpy: 2^22 x 2^22 COUNT / SEMI / ANTI / MARK, a 2^22-event band join against 2^16 windows in both orientations,
   equality plus range, RIGHT and FULL markers at 2^20;
7. the 2^40-row refusal after the sorted count."""
import numpy as np
import pytest

import _nljoinref as N
import _nljoinref_np as V
from lingodb_b200 import capi
from test_gpu_nljoin import LEFT_CARRY, RIGHT_CARRY, expected, out_layout, run_join
from test_gpu_setop import COLUMNS, PHYS, RIGHT_COLUMNS, check_against_model, gen_rows, group_fn, read_rows, stage

SIDE = 4100  # 4100^2 pairs: past kNljSortMinPairs (2^24)


def path_of(ctx, fn):
    """fn's result and the path it ran: "sort", "loop", "sort, then loop" (the candidates were too many for the sorted path) or "none"
    (an empty side)"""
    ctx.kernel_time_reset(True)
    out = fn()
    sort, loop = ctx.kernel_time("nljoin_search")[1], ctx.kernel_time("nljoin_count")[1]
    ctx.kernel_time_reset(False)
    return out, "sort, then loop" if sort and loop else "sort" if sort else "loop" if loop else "none"


def table(ctx, cols: dict, layout="single", seed=1, types=None):
    spec = [(c, (types or {}).get(c, "int64"), 0, 0) for c in cols]
    return stage(ctx, {c: list(v) for c, v in cols.items()}, spec, layout, seed)


def layout(kind, lcarry, rcarry):
    """test_gpu_nljoin.out_layout for columns of either test's tables (this file's are int64)"""
    left_only = kind in ("semi", "anti", "mark", "count")
    names = list(lcarry) + ([] if left_only else ["r_" + c for c in rcarry])
    phys = [PHYS.get(c, "int64") for c in list(lcarry) + ([] if left_only else list(rcarry))]
    if kind in ("mark", "count"):
        names, phys = names + ["v"], phys + ["int32" if kind == "mark" else "int64"]
    return names, phys


def check(out, kind, lv, rv, n, m, conds, lcarry, rcarry, what):
    names, phys = layout(kind, lcarry, rcarry)
    want = expected(kind, lv, rv, n, m, conds, lcarry, rcarry, [list(x) for x in V.matches(lv, rv, conds, n, m)])
    check_against_model(out, names, phys, want, what)


def ints(rng, n, lo, hi, null=0.0):
    v = rng.integers(lo, hi, n).tolist()
    return [None if null and rng.random() < null else x for x in v]


# ---------------------------------------------------------------------------------------------------- 1. which path runs
@pytest.mark.gpu
def test_path_taken():
    from lingodb_b200 import runtime
    rng = np.random.default_rng(1)
    big, small = 8192, 2048
    with runtime.Context(0) as ctx:
        def side(n, seed):  # b = a + a width below 64: narrow bands
            a = ints(rng, n, 0, 1 << 20)
            return {"a": a, "b": [x + int(w) for x, w in zip(a, rng.integers(0, 64, n))], "c": ints(rng, n, 0, 1024)}
        sides = {k: side(k, k) for k in (big, small, 1024)}
        T = {k: table(ctx, v, seed=k) for k, v in sides.items()}
        sort_cases = [
            ("range", "count", [("a", "<", "a")]),
            ("band", "inner", [("a", "<=", "b"), ("b", ">", "b")]),         # right b bounded by two left columns
            ("band_left", "inner", [("a", ">=", "a"), ("a", "<", "b")]),    # left a bounded by two right columns
            ("eq_range", "inner", [("c", "=", "c"), ("a", "<", "a")]),
            ("eq_only", "semi", [("c", "=", "c")]),
            ("eq_overlap", "inner", [("c", "=", "c"), ("b", ">=", "a"), ("a", "<=", "b")]),  # a key, a bound and a residual
        ]
        for n, m in ((big, small), (small, big)):  # the smaller side is sorted on a tie, so both orientations run
            for name, kind, conds in sort_cases:
                out, path = path_of(ctx, lambda: run_join(T[n], T[m], kind, conds, ["a"], ["a"]))
                assert path == "sort", (name, n, m)
                check(out, kind, sides[n], sides[m], n, m, conds, ["a"], ["a"], (name, n, m))
                out.destroy()
        loop_cases = [
            ("cross", "count", [], big, small, "loop"),
            ("ne", "count", [("a", "!=", "a")], big, small, "loop"),
            ("constants", "count", [("a", ">", None, 5), (None, "<", "b", 9)], big, small, "loop"),
            ("few_pairs", "count", [("a", "<", "a")], 1024, 1024, "loop"),
            # c <= c keys the sort, about n m / 2 candidates: the loop runs over the same words; the overlap residuals keep the rows few
            ("many_candidates", "inner", [("c", "<=", "c"), ("b", ">=", "a"), ("a", "<=", "b")], big, big, "sort, then loop"),
            ("many_candidates", "left", [("c", "<=", "c"), ("b", ">=", "a"), ("a", "<=", "b")], big, big, "sort, then loop"),
            ("many_candidates", "count", [("c", "<=", "c"), ("a", "!=", "b")], big, big, "sort, then loop"),
        ]
        for name, kind, conds, n, m, want in loop_cases:
            out, path = path_of(ctx, lambda: run_join(T[n], T[m], kind, conds, ["a"], ["a"]))
            assert path == want, (name, kind, path)
            check(out, kind, sides[n], sides[m], n, m, conds, ["a"], ["a"], (name, kind))
            out.destroy()


# ---------------------------------------------------------------------------------------------------- 2. kinds, shapes, families
SHAPES = [
    ("range", [("i32", "<", "i32")]),
    ("band_two_probe", [("i32", "<=", "i32"), ("j32", ">", "i32")]),
    ("eq_range", [("i8", "=", "i8"), ("dt", "<", "dt")]),
    ("eq_only", [("fs", "=", "fs")]),
    ("eq_residual_ne", [("i8", "=", "i8"), ("i64", "!=", "j64")]),
    ("eq_residual_range", [("fs", "=", "fs"), ("i32", "<", "i32"), ("f8", ">=", "f4")]),
    ("decimals", [("i8", "=", "i8"), ("dn", "<", "dw")]),
    ("decimals_eq", [("dw", "=", "dn")]),
    ("floats", [("fs", "=", "fs"), ("f4", "<", "f8")]),
    ("ints_mixed", [("i8", "=", "i8"), ("i16", ">=", "k16")]),
    ("constants", [("i8", ">", None, -20), (None, "<=", "i16", -30000), ("i8", "=", "i8"), ("i32", ">", "i32")]),
]
PAIR_KINDS = ("inner", "left", "right", "full")


def shaped_rows(n, m):
    """seeded rows of every type, reshaped so that every shape above matches some pairs and stays below n m / 256 candidates (the
    sorted path all the way): j32 = i32 + a width below 12 (bands a few groups wide), a quarter of the right dn cells equal to some
    left dw cell (16-byte equality), and most right char(1) codes absent on the left (equality on 95 codes alone is n m / 95)"""
    import random
    lv, rv = gen_rows(n, group_fn(1500), 71), gen_rows(m, group_fn(1700, 40), 72)
    rng = random.Random(73)
    lv["j32"] = [None if x is None else x + rng.randrange(12) for x in lv["i32"]]
    dws = [x for x in lv["dw"] if x is not None]
    rv["dn"] = [rng.choice(dws) if rng.random() < 0.25 else x for x in rv["dn"]]
    rv["fs"] = [x if x is None or rng.random() < 0.2 else 127 for x in rv["fs"]]
    return lv, rv


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["ragged", "offset", "single"])
def test_kinds_and_shapes_against_the_model(layout):
    from lingodb_b200 import runtime
    n, m = SIDE, SIDE + 3
    lv, rv = shaped_rows(n, m)
    with runtime.Context(0) as ctx:
        L = stage(ctx, lv, COLUMNS, layout, 1)
        Rt = stage(ctx, rv, RIGHT_COLUMNS, {"ragged": "single", "offset": "ragged", "single": "offset"}[layout], 2)
        empty = stage(ctx, gen_rows(0, group_fn(1), 0), COLUMNS, "single", 3)
        for si, (name, conds) in enumerate(SHAPES):
            src = L.setop(empty, "union_all", name="copy") if si % 3 == 2 else L  # a result table as the left side
            matched = [list(x) for x in V.matches(lv, rv, conds, n, m)]
            assert sum(map(len, matched)) > 0, name
            for kind in N.KINDS:
                if kind in PAIR_KINDS and name == "range":  # half of all pairs: the loop's ground (test_gpu_nljoin.py)
                    continue
                out, path = path_of(ctx, lambda: run_join(src, Rt, kind, conds, LEFT_CARRY, RIGHT_CARRY))
                assert path == "sort", (layout, name, kind, path)
                names, phys = out_layout(kind, LEFT_CARRY, RIGHT_CARRY)
                check_against_model(out, names, phys, expected(kind, lv, rv, n, m, conds, LEFT_CARRY, RIGHT_CARRY, matched), (layout, name, kind))
                out.destroy()
            if src is not L:
                src.destroy()


@pytest.mark.gpu
def test_self_join_and_null_keys():
    from lingodb_b200 import runtime
    rng = np.random.default_rng(5)
    n = SIDE
    v = {"a": ints(rng, n, 0, 3000, 0.1), "b": ints(rng, n, 0, 1 << 16, 0.1), "c": ints(rng, n, 0, 2000, 0.1)}
    with runtime.Context(0) as ctx:
        t = table(ctx, v, "ragged", 9)
        for conds in ([("b", ">", "b")], [("c", "=", "c"), ("b", "<=", "b")], [("a", "=", "a")]):
            for kind in N.KINDS:
                if kind in PAIR_KINDS and conds[0][1] != "=":
                    continue
                out, path = path_of(ctx, lambda: t.nl_join(t, kind, conds, columns=["a", "b"], other_columns=None if kind in ("semi", "anti", "mark", "count") else ["b"],
                                                           other_names=None if kind in ("semi", "anti", "mark", "count") else ["r_b"],
                                                           value_name="v" if kind in ("mark", "count") else None))
                assert path == "sort", (conds, kind)
                check(out, kind, v, v, n, n, conds, ["a", "b"], [] if kind in ("semi", "anti", "mark", "count") else ["b"], (conds, kind))
                out.destroy()


# ---------------------------------------------------------------------------------------------------- 3. ties and order
@pytest.mark.gpu
def test_ties_and_order():
    from lingodb_b200 import runtime
    n, m = 8192, 4096
    rng = np.random.default_rng(11)
    with runtime.Context(0) as ctx:
        # every right row on one key: each left row's range is the whole right side or nothing
        lv = {"a": ints(rng, n, -2000, 3)}
        rv = {"a": [0] * m}
        L, Rt = table(ctx, lv, "ragged", 1), table(ctx, rv, "single", 2)
        for kind in N.KINDS:
            conds = [("a", ">", "a")]
            out, path = path_of(ctx, lambda: run_join(L, Rt, kind, conds, ["a"], ["a"]))
            assert path == "sort", kind
            check(out, kind, lv, rv, n, m, conds, ["a"], ["a"], kind)
            out.destroy()
        # windows [lo, lo + 40) of events: keys in row order (no descent, no order sort) against shuffled keys (the order sort)
        ev = np.arange(n, dtype=np.int64) * 3
        for shuffled in (False, True):
            ts = rng.permutation(ev) if shuffled else ev
            lo = np.sort(rng.integers(0, 3 * n, 2048))
            lv = {"lo": lo.tolist(), "hi": (lo + 40).tolist()}
            rv = {"ts": ts.tolist()}
            W, E = table(ctx, lv, "single", 3), table(ctx, rv, "ragged", 4)
            conds = [("lo", "<=", "ts"), ("hi", ">", "ts")]
            for kind in ("inner", "left", "right", "full"):
                ctx.kernel_time_reset(True)
                out = run_join(W, E, kind, conds, ["lo"], ["ts"])
                searched, ordered = ctx.kernel_time("nljoin_search")[1], ctx.kernel_time("nljoin_order")[1]
                ctx.kernel_time_reset(False)
                assert searched and bool(ordered) == shuffled, (shuffled, kind)
                check(out, kind, lv, rv, 2048, n, conds, ["lo"], ["ts"], (shuffled, kind))
                out.destroy()


# ---------------------------------------------------------------------------------------------------- 4. extremes
@pytest.mark.gpu
def test_extremes():
    from lingodb_b200 import runtime
    lo64, hi64 = -(1 << 63), (1 << 63) - 1
    big = (1 << 127) - 1
    rng = np.random.default_rng(13)
    n = m = SIDE
    base = [lo64, lo64 + 1, -1, 0, 1, hi64 - 1, hi64]
    lv = {"a": [base[i % 7] if i % 3 else int(x) for i, x in enumerate(rng.integers(-5, 5, n))],
          "d": [[-big, -(1 << 64), -1, 0, 1 << 64, big][i % 6] for i in range(n)],
          "f": [[float("-inf"), -1.5, -0.0, 0.0, 2.5, float("inf"), float("nan")][i % 7] for i in range(n)]}
    rv = {"a": [base[(j * 5) % 7] if j % 2 else int(x) for j, x in enumerate(rng.integers(-5, 5, m))],
          "d": [[-big, -1, 0, 1, (1 << 64) + 1, big][(j * 7) % 6] for j in range(m)],
          "f": [[float("inf"), 0.0, -0.0, -1.5, float("-inf"), 1e300][(j * 3) % 6] for j in range(m)]}
    with runtime.Context(0) as ctx:
        cols = [("a", "int64", 0, 0), ("d", "decimal128", 38, 0), ("f", "float64", 0, 0)]
        L, Rt = stage(ctx, lv, cols, "single", 1), stage(ctx, rv, cols, "ragged", 2)
        for conds in ([("a", "<", "a")], [("a", "<=", "a")], [("a", ">", "a")], [("a", ">=", "a")], [("d", "<", "d")], [("d", "<=", "d")],
                      [("f", "<", "f")], [("f", "<=", "f")], [("f", "=", "f")], [("a", "=", "a"), ("d", ">=", "d")]):
            for kind in ("count", "semi", "anti", "mark"):
                out, path = path_of(ctx, lambda: run_join(L, Rt, kind, conds, ["a"], []))
                assert path == "sort", (conds, kind)
                check(out, kind, lv, rv, n, m, conds, ["a"], [], (conds, kind))
                out.destroy()


# ---------------------------------------------------------------------------------------------------- 5. loop against sort
@pytest.mark.gpu
def test_loop_slice_against_sorted_rows():
    """rows of left rows [a, a + 800) come from the loop (800 x SIDE < 2^24 pairs) and must equal the matching contiguous rows of the
    sorted path's result over the whole left side"""
    from lingodb_b200 import runtime
    rng = np.random.default_rng(17)
    n, m = SIDE, SIDE
    lv = {"a": ints(rng, n, 0, 1 << 14, 0.05), "c": ints(rng, n, 0, 1000)}
    rv = {"a": ints(rng, m, 0, 1 << 14, 0.05), "c": ints(rng, m, 0, 1000)}
    a0, k = 1000, 800
    sl = {c: v[a0:a0 + k] for c, v in lv.items()}
    with runtime.Context(0) as ctx:
        L, S, Rt = table(ctx, lv, "ragged", 1), table(ctx, sl, "single", 3), table(ctx, rv, "single", 2)
        for conds in ([("c", "=", "c"), ("a", "<", "a")], [("c", "=", "c"), ("a", ">=", "a"), ("a", "!=", "a")]):
            for kind in ("inner", "left", "semi", "anti", "mark", "count"):
                whole, p1 = path_of(ctx, lambda: run_join(L, Rt, kind, conds, ["a", "c"], ["a"]))
                part, p2 = path_of(ctx, lambda: run_join(S, Rt, kind, conds, ["a", "c"], ["a"]))
                assert p2 == "loop"
                names, phys = layout(kind, ["a", "c"], ["a"])
                w, p = read_rows(whole, names, phys), read_rows(part, names, phys)
                # the whole result's rows of the slice: located through the twin's per-left-row row counts
                per = V.matches(lv, rv, conds, n, m)
                if kind in ("semi", "anti"):
                    keep = [(len(x) > 0) == (kind == "semi") for x in per]
                    start, cnt = sum(keep[:a0]), sum(keep[a0:a0 + k])
                elif kind in ("mark", "count"):
                    start, cnt = a0, k
                else:
                    sizes = [max(len(x), 1 if kind == "left" else 0) for x in per]
                    start, cnt = sum(sizes[:a0]), sum(sizes[a0:a0 + k])
                assert p1 == "sort" and p == w[start:start + cnt], (conds, kind, p1)
                whole.destroy()
                part.destroy()


# ---------------------------------------------------------------------------------------------------- 6. scale
@pytest.mark.gpu
def test_scale_against_numpy():
    import torch
    from lingodb_b200 import runtime
    from lingodb_b200 import program as P
    from lingodb_b200.datagen import ColumnSpec
    from test_gpu_window import read_fixed
    rng = np.random.default_rng(19)

    def dev(ctx, name, cols):
        t = runtime.Table(ctx, name, [ColumnSpec(c, "int64") for c in cols])
        n = len(next(iter(cols.values())))
        t.append_device({c: torch.from_numpy(v).to("cuda:0") for c, v in cols.items()}, n)
        torch.cuda.synchronize()
        return t, P.RawTable(ctx, t.h)

    with runtime.Context(0) as ctx:
        n = 1 << 22
        a = rng.integers(-(1 << 40), 1 << 40, n)
        b = rng.integers(-(1 << 40), 1 << 40, n)
        ta, A = dev(ctx, "a", {"x": a})
        tb, B = dev(ctx, "b", {"x": b})
        want = np.searchsorted(np.sort(b), a, side="left")  # b < a
        for kind in ("count", "mark", "semi", "anti"):
            out, path = path_of(ctx, lambda: A.nl_join(B, kind, [("x", ">", "x")], columns=["x"], value_name="v" if kind in ("count", "mark") else None))
            assert path == "sort"
            if kind == "count":
                assert np.array_equal(np.array(read_fixed(out, "v", 8)), want)
            elif kind == "mark":
                assert np.array_equal(np.array(read_fixed(out, "v", 4)), (want > 0).astype(int))
            else:
                assert np.array_equal(np.array(read_fixed(out, "x", 8)), a[(want > 0) == (kind == "semi")])
            out.destroy()
        # a band join of 2^22 events against 2^16 windows, both orientations (the windows sorted, then the events)
        ts = rng.integers(0, 1 << 34, n)
        wlo = rng.integers(0, 1 << 34, 1 << 16)
        wl = rng.integers(0, 1 << 10, 1 << 16)
        te, Ev = dev(ctx, "e", {"ts": ts, "id": np.arange(n)})
        tw, Wi = dev(ctx, "w", {"lo": wlo, "hi": wlo + wl, "wid": np.arange(1 << 16)})
        order = np.argsort(ts, kind="stable")
        st = ts[order]
        first = np.searchsorted(st, wlo, side="left")
        last = np.searchsorted(st, wlo + wl, side="right")  # lo <= ts <= hi
        pairs = sorted((int(w), int(order[k])) for w in range(1 << 16) for k in range(first[w], last[w]))
        for left_windows in (True, False):
            if left_windows:
                out, path = path_of(ctx, lambda: Wi.nl_join(Ev, "inner", [("lo", "<=", "ts"), ("hi", ">=", "ts")], columns=["wid"], other_columns=["id"], other_names=["eid"]))
                got = list(zip(read_fixed(out, "wid", 8), read_fixed(out, "eid", 8)))
                assert got == pairs
            else:
                out, path = path_of(ctx, lambda: Ev.nl_join(Wi, "inner", [("ts", ">=", "lo"), ("ts", "<=", "hi")], columns=["id"], other_columns=["wid"], other_names=["wid2"]))
                got = list(zip(read_fixed(out, "id", 8), read_fixed(out, "wid2", 8)))
                assert got == sorted((e, w) for w, e in pairs)
            assert path == "sort"
            out.destroy()
        # equality plus range: same key, right value below the left one
        k1, k2 = rng.integers(0, 1 << 12, n), rng.integers(0, 1 << 12, n)
        tk1, K1 = dev(ctx, "k1", {"k": k1, "x": a})
        tk2, K2 = dev(ctx, "k2", {"k": k2, "x": b})
        out, path = path_of(ctx, lambda: K1.nl_join(K2, "count", [("k", "=", "k"), ("x", ">", "x")], columns=[], value_name="v"))
        assert path == "sort"
        key2 = k2 * (1 << 42) + (b + (1 << 40))
        want = np.searchsorted(np.sort(key2), k1 * (1 << 42) + (a + (1 << 40)), side="left") - np.searchsorted(np.sort(k2), k1, side="left")
        assert np.array_equal(np.array(read_fixed(out, "v", 8)), want)
        out.destroy()
        # RIGHT and FULL markers at 2^20: a narrow band, so most rows are unmatched on both sides
        m = 1 << 20
        x, y = rng.integers(0, 1 << 30, m), rng.integers(0, 1 << 30, m)
        tx, X = dev(ctx, "x", {"x": x, "x2": x + 200})
        ty, Y = dev(ctx, "y", {"y": y})
        sy = np.sort(y)
        order = np.argsort(y, kind="stable")
        first, last = np.searchsorted(sy, x, side="right"), np.searchsorted(sy, x + 200, side="left")
        sx = np.sort(x)
        has = np.searchsorted(sx, y, side="left") - np.searchsorted(sx, y - 200, side="right") > 0  # some x < y < x + 200
        for kind in ("right", "full"):
            out, path = path_of(ctx, lambda: X.nl_join(Y, kind, [("x", "<", "y"), ("x2", ">", "y")], columns=["x"], other_columns=["y"], other_names=["ry"]))
            assert path == "sort"
            want = []
            for i in range(m):
                if first[i] < last[i]:
                    want.extend((int(x[i]), int(y[j])) for j in np.sort(order[first[i]:last[i]]))
                elif kind == "full":
                    want.append((int(x[i]), None))
            want.extend((None, int(v)) for v in y[~has])
            assert list(zip(read_fixed(out, "x", 8), read_fixed(out, "ry", 8))) == want, kind
            out.destroy()
        for t in (ta, tb, te, tw, tk1, tk2, tx, ty):
            t.clear()


# ---------------------------------------------------------------------------------------------------- 7. errors
@pytest.mark.gpu
def test_refusal_after_the_sorted_count():
    """2^20 x 2^20 rows on one key: every pair matches a <=, 2^40 rows, refused with LDB_ERR_CAPACITY after the sorted count"""
    import torch
    from lingodb_b200 import runtime
    from lingodb_b200 import program as P
    from lingodb_b200.datagen import ColumnSpec
    n = 1 << 20
    with runtime.Context(0) as ctx:
        t = runtime.Table(ctx, "t", [ColumnSpec("x", "int64")])
        t.append_device({"x": torch.zeros(n, device="cuda:0", dtype=torch.int64)}, n)
        torch.cuda.synchronize()
        T = P.RawTable(ctx, t.h)
        ctx.kernel_time_reset(True)
        with pytest.raises(capi.LdbRuntimeError) as e:
            T.nl_join(T, "inner", [("x", "<=", "x")], columns=[], other_columns=[])
        assert e.value.code == capi.LDB_ERR_CAPACITY and str(1 << 40) in str(e.value)
        assert ctx.kernel_time("nljoin_search")[1] > 0 and ctx.kernel_time("nljoin_count")[1] == 0
        ctx.kernel_time_reset(False)
        out = T.nl_join(T, "count", [("x", "<=", "x")], columns=[], value_name="c")
        assert out.num_rows == n
        t.clear()
