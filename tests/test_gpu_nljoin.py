"""Nested-loop joins on the device (ldb_gpu_table_nl_join, RawTable.nl_join) against the exact model in tests/_nljoinref.py:

1. seeded tables of every physical type with NULLs, NaNs, signed zeros and garbage under NULL cells, cell for cell in order, every kind
   over column-to-column conditions of each operand family (mixed-width integers, dates, char(1), an 8-byte against a 16-byte decimal,
   float32 against float64), a band join, single-side conditions in ON, a cross product and carried utf8 columns, at sizes around the
   left tile (1024 rows) and the right tile and chunk (512 / 1024 rows), over ragged, bit-offset and single-batch layouts and result
   tables as input;
2. contention: every pair matches, so every right marker is set;
3. 2^16 x 2^16 COUNT / SEMI / ANTI / MARK against numpy searchsorted counts;
4. a self join through COUNT and through LEFT OUTER followed by a program aggregation;
5. sharded composition: the right side broadcast with ldb_gpu_table_exchange over 2 and 3 in-process ranks, a local join per rank;
6. every documented error, the capture refusal included, with nothing launched, and the capacity refusal of a 2^40-row result;
7. the reference's answers (tests/golden/nljoins.json): the select1-3.test count subqueries through a COUNT self join and through a
   LEFT OUTER self join followed by a program aggregation, and the unnesting.test / join.test queries as their joins."""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import _nljoinref as N
from lingodb_b200 import capi
from test_gpu_setop import COLUMNS, PHYS, RIGHT_COLUMNS, gen_rows, group_fn, read_rows, check_against_model, stage

# (name, conditions): every operand family, a band, single-side conditions and a cross product
CONDS = [
    ("ints", [("i32", "<", "i64")]),
    ("ints_mixed", [("i8", ">=", "k16"), ("i64", "!=", "j64")]),
    ("dates", [("dt", "<=", "dt")]),
    ("chars", [("fs", ">", "fs")]),
    ("decimals", [("dn", "<", "dw")]),
    ("decimals_eq", [("dw", "=", "dn")]),
    ("floats", [("f4", "<", "f8")]),
    ("floats_ne", [("f8", "!=", "e8")]),
    ("band", [("i32", ">=", "j32"), ("i16", "<", "k16")]),
    ("in_on", [("i8", ">", None, -20), (None, "<=", "i16", 0), ("i32", ">", "i32")]),
    ("four", [("i64", "<", "i64"), ("dt", "!=", "dt"), ("f8", ">=", "f4"), ("fs", "<=", "fs")]),
    ("cross", []),
]
LEFT_CARRY = ["i64", "s", "dw", "f8"]
RIGHT_CARRY = ["i32", "s", "dn"]


def match_lists(lv, rv, n, m, conds):
    return N.matches([{c: lv[c][i] for c in lv} for i in range(n)], [{c: rv[c][j] for c in rv} for j in range(m)], conds)


def expected(kind, lv, rv, n, m, conds, lcarry, rcarry, matched=None):
    got = N.rows_of(kind, match_lists(lv, rv, n, m, conds) if matched is None else matched, m)
    if kind in ("semi", "anti"):
        return [tuple(lv[c][i] for c in lcarry) for i in got]
    if kind in ("mark", "count"):
        return [tuple(lv[c][i] for c in lcarry) + (v,) for i, v in got]
    return [tuple(None if i is None else lv[c][i] for c in lcarry) + tuple(None if j is None else rv[c][j] for c in rcarry) for i, j in got]


def out_layout(kind, lcarry, rcarry):
    names = list(lcarry) + ([] if kind in ("semi", "anti", "mark", "count") else ["r_" + c for c in rcarry])
    phys = [PHYS[c] for c in lcarry] + ([] if kind in ("semi", "anti", "mark", "count") else [PHYS[c] for c in rcarry])
    if kind == "mark":
        names, phys = names + ["v"], phys + ["int32"]
    if kind == "count":
        names, phys = names + ["v"], phys + ["int64"]
    return names, phys


def run_join(L, Rt, kind, conds, lcarry, rcarry):
    pairs = kind not in ("semi", "anti", "mark", "count")
    return L.nl_join(Rt, kind, conds, columns=lcarry, other_columns=rcarry if pairs else None,
                     other_names=["r_" + c for c in rcarry] if pairs else None, value_name="v" if kind in ("mark", "count") else None)


# ---------------------------------------------------------------------------------------------------- 1. seeded tables
# around the left tile (1024 rows), the right tile (512) and the smallest chunk (1024), the other side kept small so the model stays fast
SIZES = [(0, 0), (1, 1), (0, 7), (7, 0), (1, 1025), (2, 1023), (1023, 1), (1025, 33), (33, 511), (31, 513), (2049, 65)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,m", SIZES)
def test_device_equals_the_model(n, m):
    from lingodb_b200 import runtime
    with runtime.Context(0) as ctx:
        lv = gen_rows(n, group_fn(max(1, n // 3 + 5)), 100 + n)
        rv = gen_rows(m, group_fn(max(1, m // 2 + 5), 3), 200 + m)
        layouts = ["ragged", "offset", "single"]
        L = stage(ctx, lv, COLUMNS, layouts[n % 3], 1)
        Rt = stage(ctx, rv, RIGHT_COLUMNS, layouts[(m + 1) % 3], 2)
        empty = stage(ctx, gen_rows(0, group_fn(1), 0), COLUMNS, "single", 3)
        for ci, (cname, conds) in enumerate(CONDS):
            # a result table as the left side for every third condition set: validity bytes, 16-byte decimals
            src = L.setop(empty, "union_all", name="copy") if ci % 3 == 2 else L
            matched = match_lists(lv, rv, n, m, conds)
            for kind in N.KINDS:
                out = run_join(src, Rt, kind, conds, LEFT_CARRY, RIGHT_CARRY)
                names, phys = out_layout(kind, LEFT_CARRY, RIGHT_CARRY)
                check_against_model(out, names, phys, expected(kind, lv, rv, n, m, conds, LEFT_CARRY, RIGHT_CARRY, matched), (n, m, cname, kind))
                out.destroy()
            if src is not L:
                src.destroy()


@pytest.mark.gpu
def test_results_feed_the_next_join():
    """a join result (NULL-extended cells included) is the left side of the next join"""
    from lingodb_b200 import runtime
    n, m = 300, 200
    lv, rv = gen_rows(n, group_fn(40), 5), gen_rows(m, group_fn(40, 10), 6)
    with runtime.Context(0) as ctx:
        L, Rt = stage(ctx, lv, COLUMNS, "ragged", 5), stage(ctx, rv, RIGHT_COLUMNS, "offset", 6)
        first = L.nl_join(Rt, "full", [("i32", "<", "i64")], columns=["i32", "s"], other_columns=["i64", "dn"], other_names=["r_i64", "r_dn"])
        want1 = expected("full", lv, rv, n, m, [("i32", "<", "i64")], ["i32", "s"], ["i64", "dn"])
        check_against_model(first, ["i32", "s", "r_i64", "r_dn"], ["int32", "utf8", "int64", "decimal128"], want1, "first")
        second = first.nl_join(Rt, "count", [("r_i64", ">", "i64")], columns=["i32", "r_i64"], value_name="c")
        fv = {"i32": [r[0] for r in want1], "r_i64": [r[2] for r in want1]}
        left = [{"i32": a, "r_i64": b} for a, b in zip(fv["i32"], fv["r_i64"])]
        right = [{"i64": v} for v in rv["i64"]]
        want2 = [(left[i]["i32"], left[i]["r_i64"], c) for i, c in N.nl_join("count", left, right, [("r_i64", ">", "i64")])]
        check_against_model(second, ["i32", "r_i64", "c"], ["int32", "int64", "int64"], want2, "second")


@pytest.mark.gpu
def test_pair_kinds_over_several_tiles_and_chunks():
    """two left tiles by two right chunks: every (left row, chunk) offset of the write pass, cell for cell"""
    from lingodb_b200 import runtime
    n, m = 1025, 1537
    lv, rv = gen_rows(n, group_fn(300), 31), gen_rows(m, group_fn(300, 50), 32)
    with runtime.Context(0) as ctx:
        L, Rt = stage(ctx, lv, COLUMNS, "ragged", 31), stage(ctx, rv, RIGHT_COLUMNS, "offset", 32)
        for cname, conds in (("ints", [("i32", "<", "i64")]), ("band", [("i32", ">=", "j32"), ("i16", "<", "k16")])):
            matched = match_lists(lv, rv, n, m, conds)
            for kind in ("inner", "left", "right", "full"):
                out = run_join(L, Rt, kind, conds, LEFT_CARRY, RIGHT_CARRY)
                names, phys = out_layout(kind, LEFT_CARRY, RIGHT_CARRY)
                check_against_model(out, names, phys, expected(kind, lv, rv, n, m, conds, LEFT_CARRY, RIGHT_CARRY, matched), (cname, kind))
                out.destroy()


@pytest.mark.gpu
def test_constants_of_either_kind():
    """an int constant against a float column, a float one against a float column; a non-integral float against an integer column
    is refused rather than read as 0"""
    from lingodb_b200 import runtime
    n, m = 200, 150
    lv, rv = gen_rows(n, group_fn(60), 41), gen_rows(m, group_fn(60, 7), 42)
    with runtime.Context(0) as ctx:
        L, Rt = stage(ctx, lv, COLUMNS, "single", 41), stage(ctx, rv, RIGHT_COLUMNS, "ragged", 42)
        for conds in ([("f8", "<", None, -5000), ("i32", "<", "i64")], [(None, ">", "f4", 2.5), ("i32", "<", "i64")],
                      [("i64", ">=", None, 3.0), ("i32", "<", "i64")]):
            out = run_join(L, Rt, "count", conds, ["i64"], [])
            check_against_model(out, ["i64", "v"], ["int64", "int64"], expected("count", lv, rv, n, m, conds, ["i64"], []), conds)
            out.destroy()
        with pytest.raises(capi.LdbRuntimeError) as e:
            run_join(L, Rt, "count", [("i64", "<", None, 2.5)], ["i64"], [])
        assert e.value.code == capi.LDB_ERR_INVALID and "fvalue" in str(e.value)


# ---------------------------------------------------------------------------------------------------- 2. contention
@pytest.mark.gpu
def test_every_pair_matches():
    from lingodb_b200 import runtime
    n, m = 1500, 1100
    with runtime.Context(0) as ctx:
        vals = {"i64": list(range(n))}
        rvals = {"i64": [10 ** 9 + j for j in range(m)]}
        cols = [c for c in COLUMNS if c[0] == "i64"]
        L, Rt = stage(ctx, vals, cols, "single", 1), stage(ctx, rvals, cols, "ragged", 2)
        for kind in ("full", "right", "count", "mark"):
            out = run_join(L, Rt, kind, [("i64", "<", "i64")], ["i64"], ["i64"])
            if kind in ("full", "right"):
                assert out.num_rows == n * m  # no unmatched right row: every marker set
                got = read_rows(out, ["i64", "r_i64"], ["int64", "int64"])
                assert got[:3] == [(0, 10 ** 9), (0, 10 ** 9 + 1), (0, 10 ** 9 + 2)] and got[-1] == (n - 1, 10 ** 9 + m - 1)
            else:
                got = read_rows(out, ["v"], ["int64" if kind == "count" else "int32"])
                assert got == [(m if kind == "count" else 1,)] * n
            out.destroy()


# ---------------------------------------------------------------------------------------------------- 3. large sizes
@pytest.mark.gpu
def test_large_counts_against_numpy():
    from lingodb_b200 import runtime
    from test_gpu_window import read_fixed
    n = m = 1 << 16
    rng = np.random.default_rng(7)
    a = rng.integers(-(1 << 20), 1 << 20, n)
    b = rng.integers(-(1 << 20), 1 << 20, m)
    cols = [("i64", "int64", 0, 0)]
    with runtime.Context(0) as ctx:
        L = stage(ctx, {"i64": a.tolist()}, cols, "ragged", 3)
        Rt = stage(ctx, {"i64": b.tolist()}, cols, "single", 4)
        want = np.searchsorted(np.sort(b), a, side="left")  # right values < left value
        cnt = L.nl_join(Rt, "count", [("i64", ">", "i64")], columns=[], value_name="v")
        assert np.array_equal(np.array(read_fixed(cnt, "v", 8)), want)
        mark = L.nl_join(Rt, "mark", [("i64", ">", "i64")], columns=[], value_name="v")
        assert np.array_equal(np.array(read_fixed(mark, "v", 4)), (want > 0).astype(int))
        semi = L.nl_join(Rt, "semi", [("i64", ">", "i64")], columns=["i64"])
        assert np.array_equal(np.array(read_fixed(semi, "i64", 8)), a[want > 0])
        anti = L.nl_join(Rt, "anti", [("i64", ">", "i64")], columns=["i64"])
        assert np.array_equal(np.array(read_fixed(anti, "i64", 8)), a[want == 0])


# ---------------------------------------------------------------------------------------------------- 4. self joins
@pytest.mark.gpu
def test_self_join_count_and_left_outer_aggregation():
    """(SELECT count(*) FROM t1 AS x WHERE x.b < t1.b): the COUNT join, and the LEFT OUTER join grouped by a program afterwards"""
    from lingodb_b200 import runtime
    from lingodb_b200 import program as P
    from test_gpu_window import read_fixed
    rng = np.random.default_rng(3)
    n = 700
    bvals = [None if rng.random() < 0.1 else int(v) for v in rng.integers(90, 250, n)]
    avals = list(range(n))
    cols = [("a", "int64", 0, 0), ("b", "int64", 0, 0)]
    want = [sum(1 for y in bvals if y is not None and x is not None and y < x) for x in bvals]
    with runtime.Context(0) as ctx:
        from _progref import to_table_data
        t = P.RawTable(ctx, ctx.table_from_host(to_table_data("t1", {"a": avals, "b": bvals}, cols, [100, 400])).h)
        cnt = t.nl_join(t, "count", [("b", ">", "b")], columns=["a"], value_name="n")
        assert read_fixed(cnt, "n", 8) == want
        lo = t.nl_join(t, "left", [("b", ">", "b")], columns=["a"], other_columns=["a"], other_names=["xa"])
        st = P.group_by(ctx, lo, [("col", "a")], [("count", ("col", "xa"))])
        got = {k[0]: v[0] for k, v in P.decode_groups(P.read_groups(ctx, st, 2048), 1, 1).items()}
        assert got == {a: w for a, w in zip(avals, want)}
        ctx.L.ldb_gpu_state_destroy(st)


# ---------------------------------------------------------------------------------------------------- 5. sharded composition
@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_broadcast_composition(world):
    """each rank holds a slice of the left side; the right side is broadcast to every rank, then each rank joins locally: the ranks'
    rows together are the model's"""
    from test_gpu_exchange import ranks
    from lingodb_b200 import program as P
    import _progref as R
    n, m = 5000, 1500
    lv, rv = gen_rows(n, group_fn(900), 21), gen_rows(m, group_fn(900, 100), 22)
    names = ["i64", "i32", "f8"]
    cols = [c for c in COLUMNS if c[0] in names]
    conds = [("i32", "<", "i32"), ("f8", ">=", "f8")]
    with ranks(world, user_bytes=64 << 20) as (ctxs, comms):
        def shard(values, r, k):
            idx = [i for i in range(k) if (i // 500) % world == r]
            return {c: [values[c][i] for i in idx] for c in names}, idx
        Ls = [P.RawTable(c, c.table_from_host(R.to_table_data("l", shard(lv, r, n)[0], cols, [])).h) for r, c in enumerate(ctxs)]
        Rs = [P.RawTable(c, c.table_from_host(R.to_table_data("r", shard(rv, r, m)[0], cols, [])).h) for r, c in enumerate(ctxs)]

        def run(r):
            rx = comms[r].table_exchange_varlen(Rs[r], [], names, name="rx", recv_offset=0, recv_bytes=32 << 20)
            out = Ls[r].nl_join(rx, "count", conds, columns=["i64"], value_name="v")
            return read_rows(out, ["i64", "v"], ["int64", "int64"])
        with ThreadPoolExecutor(world) as ex:
            res = list(ex.map(run, range(world)))
        got = sorted((x for rank in res for x in rank), key=repr)
        want = sorted((tuple(w) for w in expected("count", lv, rv, n, m, conds, ["i64"], [])), key=repr)
        assert got == want


# ---------------------------------------------------------------------------------------------------- 6. errors
@pytest.mark.gpu
def test_documented_errors():
    from lingodb_b200 import runtime
    from lingodb_b200 import program as P
    vals = gen_rows(40, group_fn(5), 9)
    inv, uns = capi.LDB_ERR_INVALID, capi.LDB_ERR_UNSUPPORTED
    with runtime.Context(0) as ctx:
        L, Rt = stage(ctx, vals, COLUMNS, "single", 1), stage(ctx, vals, RIGHT_COLUMNS, "ragged", 2)
        other = runtime.Context(0)
        Lo = stage(other, vals, COLUMNS, "single", 3)
        e = capi.Error()
        enc = lambda xs: None if xs is None else (C.c_char_p * max(1, len(xs)))(*[x.encode() if x is not None else None for x in xs])

        def cond(lc, op, rc, v=0):
            return capi.JoinCond(None if lc is None else lc.encode(), op, None if rc is None else rc.encode(), capi.I128(v, 0), 0.0)

        def rc(lh, rh, kind, cs, lcols=None, rcols=None, rnames=None, value=None, nl=None, nr=None):
            arr = (capi.JoinCond * max(1, len(cs)))(*cs)
            out = C.c_void_p()
            code = ctx.L.ldb_gpu_table_nl_join(lh, rh, kind, len(cs), arr, len(lcols) if nl is None and lcols else (nl or 0), enc(lcols),
                                               len(rcols) if nr is None and rcols else (nr or 0), enc(rcols), enc(rnames),
                                               None if value is None else value.encode(), b"x", C.byref(out), C.byref(e))
            return code
        ok = [cond("i64", 2, "i64")]
        one = ["i64"]
        before = ctx.launch_count()
        assert rc(None, Rt.h, 1, ok, one, one) == inv
        assert rc(L.h, None, 1, ok, one, one) == inv
        for k in (0, 9, -1):
            assert rc(L.h, Rt.h, k, ok, one, one) == inv, k
        assert rc(L.h, Rt.h, 1, [cond("nope", 2, "i64")], one, one) == inv and "nope" in e.message.decode()
        assert rc(L.h, Rt.h, 1, [cond("i64", 2, "nope")], one, one) == inv
        assert rc(L.h, Rt.h, 1, [cond("i64", 6, "i64")], one, one) == inv  # unknown op
        assert rc(L.h, Rt.h, 1, [cond(None, 2, None)], one, one) == inv  # no column
        assert rc(L.h, Rt.h, 1, [cond("i64", 2, None)] * 9, one, one) == inv  # 9 conditions
        assert rc(L.h, Rt.h, 1, [cond("i64", 2, "i64")] * 5, one, one) == inv  # 5 column-to-column conditions
        assert rc(L.h, Rt.h, 1, ok, ["i8"] * 17, one) == inv  # 17 carried columns
        assert rc(L.h, Rt.h, 1, ok, one, ["nope"]) == inv
        assert rc(L.h, Lo.h, 1, ok, one, one) == inv  # different contexts
        assert rc(L.h, Rt.h, 7, ok, one) == inv  # MARK without value_name
        assert rc(L.h, Rt.h, 8, ok, one) == inv  # COUNT without value_name
        assert rc(L.h, Rt.h, 5, ok, one, one) == inv  # right columns for SEMI
        assert rc(L.h, L.h, 1, ok, None, None) == inv and "i8" in e.message.decode()  # self join without right_names
        assert rc(L.h, Rt.h, 8, ok, one, None, None, "i64") == inv  # value column named like a carried one
        assert rc(L.h, Rt.h, 1, [cond("s", 2, "s")], one, one) == uns and "s" in e.message.decode()  # utf8
        assert rc(L.h, Rt.h, 1, [cond("s", 2, None)], one, one) == uns
        assert rc(L.h, Rt.h, 1, [cond("i64", 2, "f8")], one, one) == uns and "f8" in e.message.decode()  # integer vs float
        assert rc(L.h, Rt.h, 1, [cond("dt", 2, "i32")], one, one) == uns  # date vs integer
        assert rc(L.h, Rt.h, 1, [cond("fs", 2, "i8")], one, one) == uns  # char(1) vs integer
        assert ctx.launch_count() == before
        ctx.graph_begin()
        try:
            code = rc(L.h, Rt.h, 1, ok, one, one, ["r"])
            msg = e.message.decode()
        finally:
            ctx.graph_end()
        assert code == uns and "captured" in msg
        assert ctx.launch_count() == before
        # and the tables still work afterwards
        out = L.nl_join(Rt, "count", [("i64", "<", "i64")], columns=["i64"], value_name="v")
        assert out.num_rows == 40
        other.close()


@pytest.mark.gpu
def test_result_past_device_memory_is_refused():
    """a 2^20 x 2^20 cross product has 2^40 rows: counted, then refused with LDB_ERR_CAPACITY naming the count, nothing written"""
    import torch
    from lingodb_b200 import runtime
    from lingodb_b200 import program as P
    from lingodb_b200.datagen import ColumnSpec
    n = 1 << 20
    with runtime.Context(0) as ctx:
        x = torch.arange(n, device="cuda:0", dtype=torch.int64)
        t = runtime.Table(ctx, "t", [ColumnSpec("x", "int64")])
        t.append_device({"x": x}, n)
        torch.cuda.synchronize()
        T = P.RawTable(ctx, t.h)
        with pytest.raises(capi.LdbRuntimeError) as e:
            T.nl_join(T, "inner", [], columns=[], other_columns=[])
        assert e.value.code == capi.LDB_ERR_CAPACITY and str(1 << 40) in str(e.value)
        out = T.nl_join(T, "count", [("x", ">", "x")], columns=[], value_name="c")  # the context still works
        assert out.num_rows == n
        t.clear()


# ---------------------------------------------------------------------------------------------------- 7. the reference's answers
@pytest.mark.gpu
def test_reference_answers_on_the_device():
    from lingodb_b200 import runtime
    from lingodb_b200 import program as P
    from test_gpu_window import read_fixed
    from _progref import to_table_data
    from test_nljoin_model import answer_matches, golden, run_query, small_answer, small_joins
    g = golden()
    cols = [(c, "int64", 0, 0) for c in ("rid", "a", "b", "c", "d", "e")]
    with runtime.Context(0) as ctx:
        checked = 0
        for f, v in g["files"].items():
            t1 = v["t1"]
            vals = {"rid": list(range(len(t1)))}
            vals.update({c: [r[k] for r in t1] for k, c in enumerate("abcde")})
            t = P.RawTable(ctx, ctx.table_from_host(to_table_data("t1", vals, cols, [7, 19])).h)
            # t1 AS x: a COUNT self join on t1.b > x.b
            cnt = t.nl_join(t, "count", [("b", ">", "b")], columns=["rid"], value_name="n")
            by_count = read_fixed(cnt, "n", 8)
            # and a LEFT OUTER self join grouped by the left row, counting the matched x rows
            lo = t.nl_join(t, "left", [("b", ">", "b")], columns=["rid"], other_columns=["rid"], other_names=["xrid"])
            st = P.group_by(ctx, lo, [("col", "rid")], [("count", ("col", "xrid"))], expected_groups=64)
            grouped = {k[0]: w[0] for k, w in P.decode_groups(P.read_groups(ctx, st, 64), 1, 1).items()}
            ctx.L.ldb_gpu_state_destroy(st)
            assert [grouped[i] for i in range(len(t1))] == by_count, f
            for q in v["queries"]:
                assert answer_matches(q, run_query(q["sql"], t1, by_count)), (f, q["line"])
                checked += 1
        assert checked == 154
        small = g["small"]
        for q in small["queries"]:
            key = (q["file"], q["line"])
            lv, rv, kind, conds = small_joins(small["integers"])[key]
            L = P.RawTable(ctx, ctx.table_from_host(to_table_data("l", {"v": lv, "lid": list(range(len(lv)))}, [("v", "int64", 0, 0), ("lid", "int64", 0, 0)], [])).h)
            R = P.RawTable(ctx, ctx.table_from_host(to_table_data("r", {"v": rv}, [("v", "int64", 0, 0)], [])).h)
            if kind == "count":
                per = read_fixed(L.nl_join(R, "count", conds, columns=[], value_name="n"), "n", 8)
            elif kind == "mark":
                per = [bool(x) for x in read_fixed(L.nl_join(R, "mark", conds, columns=[], value_name="n"), "n", 4)]
            elif kind == "semi":
                kept = set(read_fixed(L.nl_join(R, "semi", conds, columns=["lid"]), "lid", 8))
                per = [i in kept for i in range(len(lv))]
            else:  # left outer: the matched right values per left row, NULL-extended rows carry none
                out = L.nl_join(R, "left", conds, columns=["lid"], other_columns=["v"], other_names=["rv"])
                per = [[] for _ in lv]
                for lid, x in zip(read_fixed(out, "lid", 8), read_fixed(out, "rv", 8)):
                    if x is not None:
                        per[lid].append(x)
            assert small_answer(key, lv, per) == q["rows"], key
