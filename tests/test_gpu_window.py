"""Window functions on the device (ldb_gpu_table_window, RawTable.window) against the exact model in tests/_windowref.py: the reference's
uni.test window answers, seeded random tables (every key type, NULL keys and arguments, ASC / DESC order keys with ties, every frame
shape and all six kinds, carried fixed-width and utf8 columns), dbgen lineitem at SF1 in one batch against numpy, and every documented
error, the capture refusal included."""
import ctypes as C
import os
import random
import struct

import numpy as np
import pytest

import _progref as R
import _windowref as W
from lingodb_b200 import capi

WIDTH = {"int8": 1, "int16": 2, "int32": 4, "date32": 4, "fsb4": 4, "float32": 4, "int64": 8, "float64": 8, "decimal128": 16}

COLUMNS = [("p32", "int32", 0, 0), ("p64", "int64", 0, 0), ("pdn", "decimal128", 18, 2), ("pdw", "decimal128", 38, 2), ("pdt", "date32", 0, 0),
           ("ps", "utf8", 0, 0), ("o32", "int32", 0, 0), ("os", "utf8", 0, 0), ("a64", "int64", 0, 0), ("adw", "decimal128", 38, 2),
           ("adn", "decimal128", 18, 2), ("a8", "int8", 0, 0), ("adt", "date32", 0, 0), ("afs", "fsb4", 0, 0), ("cname", "utf8", 0, 0),
           ("c16", "int16", 0, 0), ("cf8", "float64", 0, 0)]
PHYS = {n: p for n, p, _, _ in COLUMNS}
KEYS = ["p32", "p64", "pdn", "pdw", "pdt", "ps"]
FRAMES = [(None, 0), (None, None), (-3, 2), (0, 0), (2, 5), (-5, -2), (None, 3), (-2, None)]
ORDERS = [[("o32", False)], [("os", True)], [("o32", True), ("os", False)], []]
FUNCS = [
    [("row_number", None, "rn"), ("count_star", None, "cs"), ("count", "a64", "cnt"), ("sum", "adw", "sw"), ("sum", "adn", "sn"), ("min", "a8", "m8"),
     ("max", "adt", "mdt"), ("max", "a64", "m64")],
    [("count", "cname", "cn"), ("sum", "a64", "s64"), ("sum", "a8", "s8"), ("min", "adw", "mw"), ("max", "adw", "xw"), ("min", "afs", "mfs"),
     ("min", "adn", "mn"), ("rank", None, "rk")],
]
CARRIED = ["cname", "c16", "cf8", "a64", "ps"]
OUT_PHYS = {"rn": "int64", "cs": "int64", "cnt": "int64", "cn": "int64", "rk": "int64", "sw": "decimal128", "sn": "decimal128",
            "s64": "decimal128", "s8": "decimal128"}


# ---------------------------------------------------------------------------------------------------- data
def key_value(phys: str, g: int):
    """the partition key of group g as a cell of the type (distinct groups, distinct values; utf8 with long shared prefixes)"""
    if phys == "int32":
        return g * 7 - 100000
    if phys == "int64":
        return g * (1 << 33) - (1 << 40)
    if phys == "decimal128":  # both widths: values beyond 64 bits only fit the wide column, so they stay below 10^17
        return g * 1000003 - 5 * 10 ** 16
    if phys == "date32":
        return g - 5000
    return b"shared/prefix/of/group/" * 2 + str(g).encode()


def gen(seed: int, n: int, card) -> dict:
    rng = random.Random(seed)
    groups = [None if (card and rng.random() < 0.05) else rng.randrange(card) if card else 0 for _ in range(n)]
    v = {}
    for k in KEYS:
        w = "decimal128" if PHYS[k] == "decimal128" else PHYS[k]
        v[k] = [None if g is None else key_value(w, g) for g in groups]
    mute = [g is not None and g % 5 == 1 for g in groups]  # every argument of these groups is NULL: all-NULL partitions

    def arg(fn, rate=0.2):
        return [None if (m or rng.random() < rate) else fn() for m in mute]
    carry = [(1 << 64) - 1, 1 << 63, -((1 << 64) - 1), (1 << 100) + 12345, -(1 << 100)]
    v["o32"] = [None if rng.random() < 0.1 else rng.randrange(max(1, n // 4)) for _ in range(n)]
    v["os"] = [None if rng.random() < 0.1 else b"ord/" * 3 + rng.choice([b"", b"a", b"ab", b"\xff", b"\x00"]) * rng.randrange(3) for _ in range(n)]
    v["a64"] = arg(lambda: rng.choice([rng.randrange(-(1 << 63), 1 << 63), rng.randrange(-1000, 1000)]))
    v["adw"] = arg(lambda: rng.choice(carry + [rng.randrange(-10 ** 30, 10 ** 30)]))
    v["adn"] = arg(lambda: rng.randrange(-10 ** 17, 10 ** 17))
    v["a8"] = arg(lambda: rng.randrange(-128, 128))
    v["adt"] = arg(lambda: rng.randrange(-20000, 20000))
    v["afs"] = arg(lambda: rng.randrange(32, 127))
    v["cname"] = [None if rng.random() < 0.1 else b"name-%d" % rng.randrange(10 ** 6) * rng.randrange(1, 4) for _ in range(n)]
    v["c16"] = [None if rng.random() < 0.1 else rng.randrange(-32768, 32768) for _ in range(n)]
    v["cf8"] = [None if rng.random() < 0.1 else rng.uniform(-1e9, 1e9) for _ in range(n)]
    return v


def stage(ctx, values: dict, cuts=()):
    from lingodb_b200 import program as P
    t = ctx.table_from_host(R.to_table_data("w", values, COLUMNS, list(cuts)))
    return P.RawTable(ctx, t.h)


def raw(phys: str, v):
    if v is None or phys != "float64":
        return v
    return struct.unpack("<q", struct.pack("<d", v))[0]


def read_fixed(t, column: str, cell: int) -> list:
    """every cell of a fixed-width column as the signed integer of its bytes (None for NULL), read in one call"""
    n = t.num_rows
    ids = np.arange(max(n, 1), dtype=np.int64)
    buf = np.zeros(max(n, 1) * cell, np.uint8)
    valid = np.zeros(max(n, 1), np.uint8)
    e = capi.Error()
    capi.check(t.ctx.L.ldb_gpu_table_gather(t.h, column.encode(), ids.ctypes.data_as(C.POINTER(C.c_int64)), n, buf.ctypes.data, valid.ctypes.data, C.byref(e)), e)
    if cell == 16:
        w = buf.view(np.uint64).reshape(-1, 2)[:n]
        vals = [R.wrap128(int(h) << 64 | int(lo)) for lo, h in zip(w[:, 0].tolist(), w[:, 1].tolist())]
    else:
        vals = buf.view({1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}[cell])[:n].tolist()
    return [x if ok else None for x, ok in zip(vals, valid[:n].tolist())]


def read_column(t, column: str, phys: str) -> list:
    if phys == "utf8":
        return t.gather_strings(column, list(range(t.num_rows)), decode=False)
    return read_fixed(t, column, WIDTH[phys])


def out_phys(name: str, funcs: list) -> str:
    if name in OUT_PHYS:
        return OUT_PHYS[name]
    return next(PHYS[c] for _, c, nm in funcs if nm == name)


def check_case(t, values: dict, part: list, order: list, frame: tuple, funcs: list, what: str):
    w = t.window(partition_by=part, order_by=order, frame=frame, funcs=funcs, columns=CARRIED)
    try:
        perm, want = W.window(values, part, order, frame, funcs)
        assert w.num_rows == len(perm), what
        for c in CARRIED:
            got = read_column(w, c, PHYS[c])
            exp = [raw(PHYS[c], values[c][r]) for r in perm]
            assert got == exp, (what, c)
        for _, _, name in funcs:
            got = read_column(w, name, out_phys(name, funcs))
            assert got == want[name], (what, name, next(i for i, (a, b) in enumerate(zip(got, want[name])) if a != b))
    finally:
        w.destroy()


# ---------------------------------------------------------------------------------------------------- 1. the reference's uni answers
@pytest.mark.gpu
def test_uni_window_answers_on_the_device():
    from lingodb_b200 import runtime
    from test_window_model import UNI, UNI_WINDOWS, expected_uni, studenten, uni_rows
    cols = [("matrnr", "int64", 0, 0), ("name", "utf8", 0, 0), ("semester", "int64", 0, 0)]
    values = studenten()
    with runtime.Context(0) as ctx:
        from lingodb_b200 import program as P
        t = P.RawTable(ctx, ctx.table_from_host(R.to_table_data("studenten", values, cols, [])).h)
        for q, (part, order, funcs) in UNI_WINDOWS.items():
            w = t.window(partition_by=part, order_by=order, funcs=funcs, columns=["matrnr", "semester"])
            out = {name: read_fixed(w, name, 16 if kind == "sum" else 8) for kind, _, name in funcs}
            got_cols = {"matrnr": read_fixed(w, "matrnr", 8), "semester": read_fixed(w, "semester", 8)}
            assert uni_rows(q, got_cols, list(range(w.num_rows)), out) == expected_uni(q), (q, UNI["queries"][q]["sql"])
            w.destroy()


# ---------------------------------------------------------------------------------------------------- 2. random tables against the model
def cards(n: int) -> list:
    out = []
    for c in [None, 7, n // 3, n]:
        if (c is None or c > 0) and c not in out:
            out.append(c)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 2, 1000, 100003, (1 << 20) + 7])
def test_device_equals_the_model(n):
    from lingodb_b200 import runtime
    with runtime.Context(0) as ctx:
        case = 0
        for ci, card in enumerate(cards(n)):
            values = gen(1000 * n + ci, n, card)
            t = stage(ctx, values)
            keys = [[]] if card is None else [[k] for k in KEYS]
            combos = [(k, f) for k in keys for f in FRAMES]
            if n > 1000:  # larger tables: every key type and frame once, spread over the cardinalities
                combos = combos[ci % len(combos)::max(1, len(combos) // (2 if n > 200000 else 8))]
            for part, frame in combos:
                if card is not None and part == ["pdt"]:
                    part = ["pdt", "ps"]  # two keys
                check_case(t, values, part, ORDERS[case % len(ORDERS)], frame, FUNCS[case % 2], (n, card, part, frame, case))
                case += 1


# ---------------------------------------------------------------------------------------------------- 3. lineitem at SF1 against numpy
@pytest.fixture(scope="module")
def lineitem():
    from lingodb_b200 import datagen, dbgen
    li = dbgen.tpch(1.0, chunk_rows=1 << 23)["lineitem"]
    assert len(li.chunks) == 1

    def col(c):
        return np.asarray(li.chunks[0][c])
    ok = col("l_orderkey").astype(np.int64)
    price = col("l_extendedprice").view(np.int64).reshape(len(ok), -1)[:, 0].copy()
    # l_linenumber: 1.. within each order (lineitem rows come order by order)
    first = np.r_[True, ok[1:] != ok[:-1]]
    starts = np.flatnonzero(first)
    line = (np.arange(len(ok)) - np.repeat(starts, np.diff(np.r_[starts, len(ok)])) + 1).astype(np.int32)
    cols = [datagen.ColumnSpec("l_orderkey", "int32"), datagen.ColumnSpec("l_linenumber", "int32"), datagen.ColumnSpec("l_suppkey", "int32"),
            datagen.ColumnSpec("l_extendedprice", "decimal128", 12, 2)]
    chunk = {"l_orderkey": col("l_orderkey"), "l_linenumber": line, "l_suppkey": col("l_suppkey"), "l_extendedprice": li.chunks[0]["l_extendedprice"]}
    return datagen.TableData("lineitem", cols, [chunk], [len(ok)]), ok, line.astype(np.int64), col("l_suppkey").astype(np.int64), price


@pytest.mark.gpu
def test_lineitem_sf1_against_numpy(lineitem):
    from lingodb_b200 import program as P, runtime
    td, ok, line, supp, price = lineitem
    n = len(ok)
    with runtime.Context(0) as ctx:
        t = P.RawTable(ctx, ctx.table_from_host(td).h)
        # partition by l_orderkey order by l_linenumber DESC: ROW_NUMBER counts the lines from the last, a running SUM of the price
        w = t.window(partition_by=["l_orderkey"], order_by=[("l_linenumber", True)], funcs=[("row_number", None, "rn"), ("sum", "l_extendedprice", "s")],
                     columns=["l_orderkey", "l_linenumber"])
        perm = np.lexsort((np.arange(n), -line, ok))
        assert np.array_equal(np.array(read_fixed(w, "l_orderkey", 4)), ok[perm])
        assert np.array_equal(np.array(read_fixed(w, "l_linenumber", 4)), line[perm])
        sp = ok[perm]
        head = np.r_[True, sp[1:] != sp[:-1]]
        pstart = np.maximum.accumulate(np.where(head, np.arange(n), 0))
        assert np.array_equal(np.array(read_fixed(w, "rn", 8)), np.arange(n) - pstart + 1)
        cs = np.cumsum(price[perm])
        assert np.array_equal(np.array(read_fixed(w, "s", 16)), cs - np.r_[0, cs][pstart])
        w.destroy()
        # partition by l_suppkey, ROWS BETWEEN 3 PRECEDING AND 3 FOLLOWING, MAX of the price
        w = t.window(partition_by=["l_suppkey"], order_by=[("l_orderkey", False), ("l_linenumber", False)], frame=(-3, 3),
                     funcs=[("max", "l_extendedprice", "m")], columns=[])
        perm = np.lexsort((np.arange(n), line, ok, supp))
        sp = supp[perm]
        head = np.r_[True, sp[1:] != sp[:-1]]
        idx = np.arange(n)
        s = np.maximum.accumulate(np.where(head, idx, 0))
        tail = np.r_[sp[1:] != sp[:-1], True]
        e = np.minimum.accumulate(np.where(tail, idx, n)[::-1])[::-1]
        pp = price[perm]
        want = np.max(np.stack([pp[np.clip(idx + d, s, e)] for d in range(-3, 4)]), axis=0)
        assert np.array_equal(np.array(read_fixed(w, "m", 16)), want)
        w.destroy()
        # no partition: a running SUM over all 6 M rows, across many scan tiles
        w = t.window(order_by=[("l_orderkey", False), ("l_linenumber", False)], funcs=[("sum", "l_extendedprice", "s"), ("count", "l_extendedprice", "c")], columns=[])
        perm = np.lexsort((np.arange(n), line, ok))
        assert np.array_equal(np.array(read_fixed(w, "s", 16)), np.cumsum(price[perm]))
        assert np.array_equal(np.array(read_fixed(w, "c", 8)), np.arange(1, n + 1))
        w.destroy()


# ---------------------------------------------------------------------------------------------------- 4. errors
@pytest.mark.gpu
def test_documented_errors():
    from lingodb_b200 import runtime
    values = gen(7, 50, 7)
    values["f4"] = [1.5] * 50
    cols = COLUMNS + [("f4", "float32", 0, 0)]
    with runtime.Context(0) as ctx:
        from lingodb_b200 import program as P
        t = P.RawTable(ctx, ctx.table_from_host(R.to_table_data("w", values, cols, [])).h)
        multi = P.RawTable(ctx, ctx.table_from_host(R.to_table_data("m", values, cols, [20])).h)
        ok = [("sum", "a64", "s")]

        def code(tab=t, **kw):
            kw.setdefault("funcs", ok)
            kw.setdefault("columns", [])
            with pytest.raises(capi.LdbRuntimeError) as ei:
                tab.window(**kw)
            return ei.value.code, str(ei.value)
        assert code(partition_by=["nope"])[0] == capi.LDB_ERR_INVALID
        assert code(funcs=[("sum", "nope", "s")])[0] == capi.LDB_ERR_INVALID
        assert code(columns=["nope"])[0] == capi.LDB_ERR_INVALID
        for f in [("sum", "f4", "s"), ("min", "cname", "s"), ("max", "f4", "s"), ("sum", "adt", "s")]:
            c, m = code(funcs=[f])
            assert c == capi.LDB_ERR_UNSUPPORTED and f[1] in m, (f, m)
        c, m = code(partition_by=["f4"])
        assert c == capi.LDB_ERR_UNSUPPORTED and "f4" in m
        assert code(tab=multi)[0] == capi.LDB_ERR_UNSUPPORTED
        for frame in [(3, 2), ((1 << 63) - 1, (1 << 63) - 1), (-(1 << 63), -(1 << 63))]:  # from > to, from UNBOUNDED FOLLOWING, to UNBOUNDED PRECEDING
            assert code(frame=frame)[0] == capi.LDB_ERR_INVALID, frame
        assert code(funcs=[])[0] == capi.LDB_ERR_INVALID
        assert code(funcs=ok * 9)[0] == capi.LDB_ERR_INVALID
        assert code(partition_by=KEYS[:5])[0] == capi.LDB_ERR_INVALID
        assert code(order_by=[(k, False) for k in KEYS[:5]])[0] == capi.LDB_ERR_INVALID
        assert code(columns=[n for n, *_ in COLUMNS])[0] == capi.LDB_ERR_INVALID  # 17 carried columns
        assert code(columns=None)[0] == capi.LDB_ERR_INVALID  # "all" is 18 columns here
        fs = (capi.WindowFunc * 1)(capi.WindowFunc(9, b"a64", b"x"))
        out, e = C.c_void_p(), capi.Error()
        assert ctx.L.ldb_gpu_table_window(t.h, 0, None, 0, None, None, -(1 << 63), 0, 1, fs, 0, None, None, C.byref(out), C.byref(e)) == capi.LDB_ERR_INVALID
        assert ctx.L.ldb_gpu_table_window(None, 0, None, 0, None, None, -(1 << 63), 0, 1, fs, 0, None, None, C.byref(out), C.byref(e)) == capi.LDB_ERR_INVALID
        # inside a captured query: refused before anything is enqueued
        before = ctx.launch_count()
        ctx.graph_begin()
        try:
            c, m = code()
        finally:
            ctx.graph_end().destroy()
        assert c == capi.LDB_ERR_UNSUPPORTED and "captured" in m
        assert ctx.launch_count() == before
        # and the table still works afterwards
        w = t.window(funcs=ok, columns=[])
        assert w.num_rows == 50
