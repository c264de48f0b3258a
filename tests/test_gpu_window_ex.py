"""RANGE frames and the ranking, offset and value window functions on the device (ldb_gpu_table_window_ex, RawTable.window with
mode="range" or the new kinds) against the exact model in tests/_windowref_ex.py: seeded tables of every key type with few and many
peers, NULLs, ASC and DESC, sizes on the 2048-row scan tiles and the 524 288-row chunks of tile totals; RANGE offsets of 0, past the
partition and at the int64 and 16-byte decimal extremes; LAG, LEAD, FIRST_VALUE, LAST_VALUE and NTH_VALUE over every carried type (utf8
and float bit patterns included) and defaults of every fixed-width type; the old and the new entry byte-identical in ROWS mode; window
results fed into a second window and a set operation; dbgen lineitem at SF1 against numpy; and every new error."""
import ctypes as C
import math
import random

import numpy as np
import pytest

import _progref as R
import _windowref_ex as X
from lingodb_b200 import capi
from test_gpu_window import FRAMES as ROWS_FRAMES, read_column, read_fixed

COLUMNS = [("p", "int32", 0, 0), ("k32", "int32", 0, 0), ("k64", "int64", 0, 0), ("kdt", "date32", 0, 0), ("kdn", "decimal128", 18, 2),
           ("kdw", "decimal128", 38, 0), ("kfs", "fsb4", 0, 0), ("ks", "utf8", 0, 0),
           ("v8", "int8", 0, 0), ("v16", "int16", 0, 0), ("v32", "int32", 0, 0), ("v64", "int64", 0, 0), ("vdt", "date32", 0, 0),
           ("vfs", "fsb4", 0, 0), ("vdn", "decimal128", 18, 2), ("vdw", "decimal128", 38, 0), ("vf4", "float32", 0, 0),
           ("vf8", "float64", 0, 0), ("vs", "utf8", 0, 0)]
PHYS = {n: p for n, p, _, _ in COLUMNS}
RANGE_KEYS = ["k32", "k64", "kdt", "kdn", "kdw"]  # the key types a RANGE offset takes
VALUES = ["v8", "v16", "v32", "v64", "vdt", "vfs", "vdn", "vdw", "vf4", "vf8", "vs"]
RANGE_FRAMES = [(None, 0), (None, None), (0, 0), (-3, 0), (-5, 5), (2, 7), (None, -2), (1, None)]
FLOATS = [0.0, -0.0, math.nan, -math.nan, math.inf, -math.inf, 5e-324, 1.5, -2.25, 1e300]
DEFAULTS = {"v8": -128, "v16": 32767, "v32": -5, "v64": -(1 << 63), "vdt": 19000, "vfs": 65, "vdn": 10 ** 18 - 1, "vdw": -(10 ** 38 - 1),
            "vf4": 2.5, "vf8": -0.0}
FUNCS = [
    [("sql_rank", None, "rk"), ("dense_rank", None, "dr"), ("percent_rank", None, "pr"), ("cume_dist", None, "cd"), ("ntile", None, "nt", 3),
     ("row_number", None, "rn"), ("count_star", None, "cs"), ("sum", "v64", "s")],
    [("lag", "v64", "lg"), ("lead", "vs", "ld", 2), ("first_value", "vf8", "fv"), ("last_value", "vdw", "lv"), ("nth_value", "vf4", "nv", 2),
     ("min", "v32", "mn"), ("max", "vdn", "mx"), ("count", "vs", "cn")],
    [("lag", "vdt", "lgd", 3, 19000), ("lead", "v8", "ldd", 1, -128), ("first_value", "vs", "fs"), ("last_value", "vf4", "lf"),
     ("nth_value", "v16", "n3", 3), ("lag", "vfs", "lfs"), ("sum", "vdw", "sw"), ("ntile", None, "nt7", 7)],
]
OUT_PHYS = {"rk": "int64", "dr": "int64", "nt": "int64", "nt7": "int64", "rn": "int64", "cs": "int64", "cn": "int64", "pr": "float64",
            "cd": "float64", "s": "decimal128", "sw": "decimal128"}


def out_phys(f) -> str:
    return OUT_PHYS.get(f[2]) or PHYS[f[1]]


def bits(phys: str, v):
    """a model value as the device cell reads back: floats as their bits"""
    if v is None:
        return None
    if phys == "float32":
        return int(np.array([v], np.float32).view(np.int32)[0])
    if phys == "float64":
        return int(np.array([v], np.float64).view(np.int64)[0])
    return v


# ---------------------------------------------------------------------------------------------------- data
def gen(seed: int, n: int, card, distinct) -> dict:
    """partitions: card (None: one), keys from `distinct` values per type (few: many peers; None: unique), 10 % NULL keys"""
    rng = random.Random(seed)
    v = {"p": [None if card and rng.random() < 0.05 else rng.randrange(card) if card else 0 for _ in range(n)]}
    pool = distinct or 3 * n + 1

    def key(scale):
        return [None if rng.random() < 0.1 else (rng.randrange(pool) - pool // 2) * scale for _ in range(n)]
    v["k32"], v["k64"], v["kdt"], v["kdn"], v["kdw"] = key(1), key(1 << 40), key(1), key(7), key(1 << 70)
    v["kfs"] = [None if rng.random() < 0.1 else 32 + rng.randrange(min(pool, 90)) for _ in range(n)]
    v["ks"] = [None if rng.random() < 0.1 else b"k/" + str(rng.randrange(pool)).encode() for _ in range(n)]

    def arg(fn):
        return [None if rng.random() < 0.15 else fn() for _ in range(n)]
    v["v8"] = arg(lambda: rng.randrange(-128, 128))
    v["v16"] = arg(lambda: rng.randrange(-32768, 32768))
    v["v32"] = arg(lambda: rng.randrange(-(1 << 31), 1 << 31))
    v["v64"] = arg(lambda: rng.randrange(-(1 << 63), 1 << 63))
    v["vdt"] = arg(lambda: rng.randrange(-30000, 30000))
    v["vfs"] = arg(lambda: rng.randrange(32, 127))
    v["vdn"] = arg(lambda: rng.randrange(-10 ** 17, 10 ** 17))
    v["vdw"] = arg(lambda: rng.randrange(-10 ** 37, 10 ** 37))
    v["vf4"] = arg(lambda: rng.choice(FLOATS[:-1] + [rng.uniform(-1e6, 1e6)]))
    v["vf8"] = arg(lambda: rng.choice(FLOATS + [rng.uniform(-1e9, 1e9)]))
    v["vs"] = arg(lambda: b"value-" * rng.randrange(0, 4) + str(rng.randrange(1000)).encode())
    return v


def stage(ctx, values: dict, cuts=()):
    from lingodb_b200 import program as P
    return P.RawTable(ctx, ctx.table_from_host(R.to_table_data("wx", values, COLUMNS, list(cuts))).h)


def check_case(t, values, part, order, frame, funcs, mode, what, carried=("vs", "v64")):
    w = t.window(partition_by=part, order_by=order, frame=frame, funcs=funcs, columns=list(carried), mode=mode)
    try:
        perm, want = X.window_ex(values, part, order, frame, funcs, mode)
        assert w.num_rows == len(perm), what
        for c in carried:
            assert read_column(w, c, PHYS[c]) == [values[c][r] for r in perm], (what, c)
        for f in funcs:
            ph = out_phys(f)
            got = read_column(w, f[2], ph)
            exp = [bits(ph, x) for x in want[f[2]]]
            assert got == exp, (what, f, next(i for i, (a, b) in enumerate(zip(got, exp)) if a != b))
    finally:
        w.destroy()


# ---------------------------------------------------------------------------------------------------- 1. device = model
@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 2, 1000, 2047, 2049, 100003, 524289, (1 << 20) + 7])
def test_device_equals_the_model(n):
    from lingodb_b200 import runtime
    big = n > 3000
    with runtime.Context(0) as ctx:
        case = 0
        shapes = [(None, 4), (7, None), (n // 3 or None, 3)] if not big else [(None, None), (1 << 10, 16)]
        for si, (card, distinct) in enumerate(shapes):
            values = gen(7919 * n + si, n, card, distinct)
            t = stage(ctx, values)
            part = [] if card is None else ["p"]
            combos = []
            for k in RANGE_KEYS + ["kfs", "ks"]:
                for desc in (False, True):
                    for frame in RANGE_FRAMES:
                        if k in ("kfs", "ks") and frame not in [(None, 0), (None, None), (0, 0)]:
                            continue  # RANGE offsets take integer, date and decimal keys
                        combos.append(([(k, desc)], frame, "range"))
            combos += [([("k32", False), ("ks", True)], (None, 0), "range"), ([], (None, None), "range"), ([("k64", True)], (-2, 3), "rows")]
            if big:  # larger tables: a spread of key types, directions and frames, different per shape and size
                combos = combos[(si + n) % 7::max(1, len(combos) // (2 if n > 200000 else 12))]
            for order, frame, mode in combos:
                check_case(t, values, part, order, frame, FUNCS[case % len(FUNCS)], mode, (n, card, distinct, order, frame, mode))
                case += 1


# ---------------------------------------------------------------------------------------------------- 2. extremes
@pytest.mark.gpu
def test_range_offsets_at_the_key_extremes():
    from lingodb_b200 import program as P, runtime
    i64 = (1 << 63) - 1
    w128 = (1 << 127) - 1
    k64 = [i64, i64 - 3, -i64 - 1, None, 0, -i64 - 1 + 2, i64 - 3, 5]
    kdw = [w128, w128 - 3, -w128 - 1, None, 0, -w128 + 1, w128 - 3, 5]
    x = list(range(1, len(k64) + 1))
    cols = [("p", "int32", 0, 0), ("k64", "int64", 0, 0), ("kdw", "decimal128", 38, 0), ("x", "int64", 0, 0)]
    values = {"p": [0] * 4 + [1] * 4, "k64": k64, "kdw": kdw, "x": x}
    frames = [(0, 5), (-5, 0), (-i64, 0), (0, i64 - 1), (-i64, i64 - 1), (1, i64 - 1), (-i64, -1), (-3, 3), (4, 9)]
    funcs = [("sum", "x", "s"), ("count_star", None, "c"), ("first_value", "x", "f"), ("last_value", "x", "l")]
    with runtime.Context(0) as ctx:
        t = P.RawTable(ctx, ctx.table_from_host(R.to_table_data("ext", values, cols, [])).h)
        for key in ("k64", "kdw"):
            for part in ([], ["p"]):
                for desc in (False, True):
                    for frame in frames:
                        w = t.window(partition_by=part, order_by=[(key, desc)], frame=frame, funcs=funcs, columns=["x"], mode="range")
                        perm, want = X.window_ex(values, part, [(key, desc)], frame, funcs, "range")
                        assert read_fixed(w, "x", 8) == [x[r] for r in perm]
                        for _, _, name in funcs:
                            assert read_fixed(w, name, 16 if name == "s" else 8) == want[name], (key, part, desc, frame, name)
                        w.destroy()


# ---------------------------------------------------------------------------------------------------- 3. values and defaults
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 37, 5000])
def test_value_functions_and_defaults_of_every_type(n):
    from lingodb_b200 import runtime
    values = gen(n + 5, n, 5, 6)
    with runtime.Context(0) as ctx:
        t = stage(ctx, values)
        for c in VALUES:
            funcs = [("lag", c, "a"), ("lead", c, "b", 2), ("first_value", c, "f"), ("last_value", c, "l"), ("nth_value", c, "t", 2),
                     ("lag", c, "z", 0)]
            if c in DEFAULTS:
                funcs += [("lag", c, "ad", 1, DEFAULTS[c]), ("lead", c, "bd", 3, DEFAULTS[c])]
            for mode, frame in (("rows", (-1, 1)), ("range", (-2, 2))):
                check_case(t, values, ["p"], [("k32", n % 2 == 0)], frame, funcs, mode, (n, c, mode), carried=())


# ---------------------------------------------------------------------------------------------------- 4. old entry = new entry in ROWS mode
def read_raw(t, column: str, cell: int):
    n = t.num_rows
    ids = np.arange(max(n, 1), dtype=np.int64)
    buf = np.zeros(max(n, 1) * cell, np.uint8)
    valid = np.zeros(max(n, 1), np.uint8)
    e = capi.Error()
    capi.check(t.ctx.L.ldb_gpu_table_gather(t.h, column.encode(), ids.ctypes.data_as(C.POINTER(C.c_int64)), n, buf.ctypes.data, valid.ctypes.data, C.byref(e)), e)
    return buf.tobytes(), valid.tobytes()


@pytest.mark.gpu
def test_old_and_new_entry_are_byte_identical_in_rows_mode():
    from lingodb_b200 import runtime
    values = gen(11, 3000, 9, 40)
    funcs = [("row_number", None, "rn"), ("count_star", None, "cs"), ("count", "vs", "cn"), ("sum", "vdw", "sw"), ("sum", "v8", "s8"),
             ("min", "vdn", "mn"), ("max", "vdt", "mx"), ("min", "vfs", "mf")]
    cells = {"rn": 8, "cs": 8, "cn": 8, "sw": 16, "s8": 16, "mn": 16, "mx": 4, "mf": 4}
    with runtime.Context(0) as ctx:
        t = stage(ctx, values)
        for frame in ROWS_FRAMES:
            for order in ([("k64", False)], [("ks", True), ("kdn", False)], []):
                old = t.window(partition_by=["p"], order_by=order, frame=frame, funcs=funcs, columns=["vs", "vf8"])
                new = t.window(partition_by=["p"], order_by=order, frame=frame, funcs=[f + (None,) for f in funcs], columns=["vs", "vf8"])
                try:
                    for name, cell in cells.items():
                        ro, rn = read_raw(old, name, cell), read_raw(new, name, cell)
                        vo = np.frombuffer(ro[1], np.uint8)
                        # the cells under a NULL are not part of the answer; the validity bytes and every other cell are
                        assert ro[1] == rn[1], (frame, order, name)
                        bo = np.frombuffer(ro[0], np.uint8).reshape(-1, cell)[vo.astype(bool)]
                        bn = np.frombuffer(rn[0], np.uint8).reshape(-1, cell)[vo.astype(bool)]
                        assert np.array_equal(bo, bn), (frame, order, name)
                    assert read_column(old, "vs", "utf8") == read_column(new, "vs", "utf8")
                    assert read_fixed(old, "vf8", 8) == read_fixed(new, "vf8", 8)
                finally:
                    old.destroy()
                    new.destroy()


# ---------------------------------------------------------------------------------------------------- 5. composition
@pytest.mark.gpu
def test_window_results_feed_a_second_window_and_a_set_operation():
    from lingodb_b200 import runtime
    values = gen(3, 4000, 6, 30)
    with runtime.Context(0) as ctx:
        t = stage(ctx, values)
        f1 = [("sql_rank", None, "rk"), ("lag", "vs", "prev"), ("sum", "v32", "run")]
        w1 = t.window(partition_by=["p"], order_by=[("k32", True)], funcs=f1, columns=["p", "k32", "vs"], mode="range")
        perm, want = X.window_ex(values, ["p"], [("k32", True)], (None, 0), f1, "range")
        mid = {"p": [values["p"][r] for r in perm], "k32": [values["k32"][r] for r in perm], "vs": [values["vs"][r] for r in perm]}
        mid.update(want)
        # a second window over the first one's output: DENSE_RANK by the rank, and a rolling RANGE SUM over the running sums' rank
        f2 = [("dense_rank", None, "dr"), ("count", "prev", "np"), ("lead", "prev", "nx"), ("max", "run", "mr")]
        w2 = w1.window(partition_by=["p"], order_by=[("rk", False)], frame=(-2, 0), funcs=f2, columns=["rk", "prev"], mode="range")
        perm2, want2 = X.window_ex(mid, ["p"], [("rk", False)], (-2, 0), f2, "range")
        assert read_fixed(w2, "rk", 8) == [mid["rk"][r] for r in perm2]
        assert read_column(w2, "prev", "utf8") == [mid["prev"][r] for r in perm2]
        for name, ph in (("dr", "int64"), ("np", "int64"), ("nx", "utf8"), ("mr", "decimal128")):
            assert read_column(w2, name, ph) == want2[name], name
        # and into a set operation: the distinct (p, rk) pairs, each at its first occurrence
        d = w1.distinct(columns=["p", "rk"])
        pairs = list(dict.fromkeys(zip(mid["p"], mid["rk"])))
        assert list(zip(read_fixed(d, "p", 4), read_fixed(d, "rk", 8))) == pairs
        for x in (d, w2, w1):
            x.destroy()


# ---------------------------------------------------------------------------------------------------- 6. lineitem at SF1 against numpy
@pytest.mark.gpu
def test_lineitem_sf1_against_numpy():
    from lingodb_b200 import datagen, dbgen, program as P, runtime
    li = dbgen.tpch(1.0, chunk_rows=1 << 23)["lineitem"]
    assert len(li.chunks) == 1
    ch = li.chunks[0]
    supp = np.asarray(ch["l_suppkey"]).astype(np.int64)
    partk = np.asarray(ch["l_partkey"]).astype(np.int64)
    ship = np.asarray(ch["l_shipdate"]).astype(np.int64)
    n = len(supp)
    price = np.asarray(ch["l_extendedprice"]).view(np.int64).reshape(n, -1)[:, 0].copy()
    qty = np.asarray(ch["l_quantity"]).view(np.int64).reshape(n, -1)[:, 0].copy()
    cols = [datagen.ColumnSpec("l_suppkey", "int32"), datagen.ColumnSpec("l_partkey", "int32"), datagen.ColumnSpec("l_shipdate", "date32"),
            datagen.ColumnSpec("l_extendedprice", "decimal128", 12, 2), datagen.ColumnSpec("l_quantity", "decimal128", 12, 2)]
    td = datagen.TableData("lineitem", cols, [{c.name: ch[c.name] for c in cols}], [n])
    idx = np.arange(n)
    with runtime.Context(0) as ctx:
        t = P.RawTable(ctx, ctx.table_from_host(td).h)
        # RANK and DENSE_RANK of l_extendedprice DESC per l_suppkey
        w = t.window(partition_by=["l_suppkey"], order_by=[("l_extendedprice", True)], funcs=[("sql_rank", None, "rk"), ("dense_rank", None, "dr")],
                     columns=["l_suppkey"], mode="range")
        perm = np.lexsort((idx, -price, supp))
        sp, pp = supp[perm], price[perm]
        head = np.r_[True, sp[1:] != sp[:-1]]
        peer = head | np.r_[True, pp[1:] != pp[:-1]]
        start = np.maximum.accumulate(np.where(head, idx, 0))
        pstart = np.maximum.accumulate(np.where(peer, idx, 0))
        groups = np.cumsum(peer)
        assert np.array_equal(np.array(read_fixed(w, "l_suppkey", 4)), sp)
        assert np.array_equal(np.array(read_fixed(w, "rk", 8)), pstart - start + 1)
        assert np.array_equal(np.array(read_fixed(w, "dr", 8)), groups - groups[start] + 1)
        w.destroy()
        # a 30-day rolling SUM(l_quantity) per l_partkey by l_shipdate: RANGE BETWEEN 29 PRECEDING AND CURRENT ROW
        w = t.window(partition_by=["l_partkey"], order_by=[("l_shipdate", False)], frame=(-29, 0), funcs=[("sum", "l_quantity", "q")],
                     columns=["l_partkey", "l_shipdate"], mode="range")
        perm = np.lexsort((idx, ship, partk))
        key = partk[perm] * (1 << 20) + ship[perm]  # shipdates are 8 000 .. 11 000 days: a partition's keys never reach the next one's
        lo = np.searchsorted(key, key - 29, "left")
        hi = np.searchsorted(key, key, "right")
        cs = np.r_[0, np.cumsum(qty[perm])]
        assert np.array_equal(np.array(read_fixed(w, "l_shipdate", 4)), ship[perm])
        assert np.array_equal(np.array(read_fixed(w, "q", 16)), cs[hi] - cs[lo])
        w.destroy()


# ---------------------------------------------------------------------------------------------------- 7. errors
@pytest.mark.gpu
def test_documented_errors():
    from lingodb_b200 import runtime
    values = gen(5, 60, 4, 10)
    cols = COLUMNS + [("f4", "float32", 0, 0)]
    values["f4"] = [1.5] * 60
    with runtime.Context(0) as ctx:
        from lingodb_b200 import program as P
        t = P.RawTable(ctx, ctx.table_from_host(R.to_table_data("e", values, cols, [])).h)
        multi = P.RawTable(ctx, ctx.table_from_host(R.to_table_data("m", values, cols, [30])).h)
        ok = [("sql_rank", None, "r")]

        def code(tab=t, **kw):
            kw.setdefault("funcs", ok)
            kw.setdefault("columns", [])
            kw.setdefault("order_by", [("k32", False)])
            kw.setdefault("mode", "range")
            with pytest.raises(capi.LdbRuntimeError) as ei:
                tab.window(**kw)
            return ei.value.code, str(ei.value)

        def raw_call(frame, funcs, order=("k32",), fn="ldb_gpu_table_window_ex"):
            out, e = C.c_void_p(), capi.Error()
            oc = (C.c_char_p * 1)(*[o.encode() for o in order])
            desc = (C.c_int32 * 1)(0)
            if fn == "ldb_gpu_table_window_ex":
                fs = (capi.WindowFuncEx * len(funcs))(*funcs)
                return ctx.L.ldb_gpu_table_window_ex(t.h, 0, None, len(order), oc, desc, frame, len(funcs), fs, 0, None, None, C.byref(out), C.byref(e))
            fs = (capi.WindowFunc * len(funcs))(*funcs)
            return ctx.L.ldb_gpu_table_window(t.h, 0, None, len(order), oc, desc, -(1 << 63), 0, len(funcs), fs, 0, None, None, C.byref(out), C.byref(e))

        before = ctx.launch_count()
        inv, uns = capi.LDB_ERR_INVALID, capi.LDB_ERR_UNSUPPORTED
        for f in [("lag", "v64", "x", -1), ("lead", "v64", "x", -1), ("ntile", None, "x", 0), ("nth_value", "v64", "x", 0), ("nth_value", "v64", "x", -5)]:
            assert code(funcs=[f])[0] == inv, f
        # defaults: outside the type, on another kind, value and fvalue disagreeing
        for c, d in [("v8", 128), ("v8", -129), ("v16", 1 << 15), ("v32", 1 << 31), ("vdt", -(1 << 31) - 1), ("vfs", 1 << 40), ("v64", 1 << 63),
                     ("vdn", 10 ** 18), ("vdw", -(10 ** 38)), ("vf4", 1e300), ("v64", 2.5)]:
            c_, m = code(funcs=[("lag", c, "x", 1, d)])
            assert c_ == inv, (c, d, m)
        assert code(funcs=[("first_value", "v64", "x", 1, 3)])[0] == inv
        bad = capi.WindowFuncEx(capi.WIN["lag"], 1, b"v64", b"x", 1, capi.I128(1, 0), 2.0)  # value 1, fvalue 2
        assert raw_call(C.byref(capi.WindowFrame(1, 0, -(1 << 63), 0)), [bad]) == inv
        bad = capi.WindowFuncEx(capi.WIN["lag"], 1, b"vf8", b"x", 1, capi.I128(3, 0), 2.5)  # a float argument reads fvalue
        assert raw_call(C.byref(capi.WindowFrame(1, 0, -(1 << 63), 0)), [bad]) == inv
        good = capi.WindowFuncEx(capi.WIN["sql_rank"], 0, None, b"x", 0, capi.I128(0, 0), 0.0)
        assert raw_call(C.byref(capi.WindowFrame(2, 0, -(1 << 63), 0)), [good]) == inv  # unknown mode
        assert raw_call(None, [good]) == inv  # no frame
        # the old entry refuses the new kinds
        for kind in range(7, 17):
            assert raw_call(None, [capi.WindowFunc(kind, b"v64", b"x")], fn="ldb_gpu_table_window") == inv, kind
        # bad frames, counts and names as before
        for frame in [(3, 2), ((1 << 63) - 1, (1 << 63) - 1), (-(1 << 63), -(1 << 63))]:
            assert code(frame=frame)[0] == inv
        assert code(funcs=ok * 9)[0] == inv
        assert code(funcs=[("sql_rank", None, "vs")], columns=["vs"])[0] == inv
        assert code(funcs=[("lag", "nope", "x")])[0] == inv
        # unsupported: RANGE offsets without exactly one integer, date or decimal order key, utf8 defaults, float SUM
        assert code(frame=(-1, 0), order_by=[])[0] == uns
        assert code(frame=(-1, 0), order_by=[("k32", False), ("k64", False)])[0] == uns
        for k in ("ks", "kfs"):
            c_, m = code(frame=(0, 2), order_by=[(k, False)])
            assert c_ == uns and k in m
        c_, m = code(funcs=[("lead", "vs", "x", 1, 0)])
        assert c_ == uns and "utf8" in m
        assert code(funcs=[("sum", "f4", "x")])[0] == uns
        assert code(tab=multi)[0] == uns
        assert ctx.launch_count() == before
        # inside a captured query: refused before anything is enqueued
        ctx.graph_begin()
        try:
            c_, m = code()
        finally:
            ctx.graph_end().destroy()
        assert c_ == uns and "captured" in m
        assert ctx.launch_count() == before
        # RANGE frames without offsets take any order keys; the table still works
        w = t.window(order_by=[("ks", False), ("kfs", True)], funcs=[("sum", "v64", "s"), ("cume_dist", None, "c")], columns=[], mode="range")
        assert w.num_rows == 60
        w.destroy()
