"""Window functions (ldb_gpu_table_window) over every kind of source table the header names, every key and argument type, the tile-scan
and segment-tree edges, extreme values, frames at the offset limits and sharded inputs, against the exact model in tests/_windowref.py
(and, for tables of a million rows, a vectorised numpy restatement of its rules, itself checked against the model):

1. sources: HOST batches under each staging mode (copied / packed, narrowed / 16-byte decimals) at bit offsets 0 and 3 with garbage
   under NULL cells, borrowed DEVICE batches at bit offsets 0, 3 and 7 with utf8 offsets past 0, materialised rows, exported groups
   (16-byte float cells), join-marker and dictionary tables, received and sorted tables, set-operation and window results;
2. every key type as a partition and an order key, ASC and DESC, and every argument type under every kind that takes it, with the
   result types of the header;
3. sizes on and next to the 2048-row scan tiles and the 524 288-row chunks of tile totals, powers of two (no padding leaves in the
   tree), and partition boundaries on, before and after tile edges;
4. partitions whose only values are the identities of the MIN / MAX tree, and SUMs that wrap past 2^127;
5. frames near the +-2^40 clamp and at +-2^63;
6. a table exchanged on its partition keys across 2 and 3 in-process ranks, then a local window per rank;
7. every documented error with nothing launched: the 2^32-row refusal and duplicate output names included."""
import ctypes as C
import random
import struct
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import _progref as R
import _setopref as S
import _windowref as W
from lingodb_b200 import capi
from test_gpu_result_reads import BASE_COLUMNS, STAGING, base_values, cells_of, device_table, host_table
from test_gpu_setop import COLUMNS, NAMES, PHYS, raw, stage
from test_gpu_window import read_column

KEY_PHYS = ("int32", "date32", "fsb4", "int64", "decimal128", "utf8")
SUM_PHYS = ("int8", "int16", "int32", "int64", "decimal128")
MM_PHYS = SUM_PHYS + ("date32", "fsb4")
FRAMES = [(None, 0), (-2, 3), (None, None), (0, None), (-5, -1), (1, 4)]
I64_MIN, I64_MAX, I128_MIN, I128_MAX = -(1 << 63), (1 << 63) - 1, -(1 << 127), (1 << 127) - 1


# ---------------------------------------------------------------------------------------------------- checking one table
def funcs_for(cols: dict) -> list:
    """ROW_NUMBER, COUNT(*), and every kind over every column of `cols` that takes it"""
    fs = [("row_number", None, "w_rn"), ("count_star", None, "w_cs")]
    for c, (p, _) in cols.items():
        if p in SUM_PHYS:
            fs.append(("sum", c, "w_sum_" + c))
        if p in MM_PHYS:
            fs += [("min", c, "w_min_" + c), ("max", c, "w_max_" + c)]
        fs.append(("count", c, "w_cnt_" + c))
    return fs


def out_phys(kind: str, arg_phys) -> str:
    return "int64" if kind in ("row_number", "rank", "count_star", "count") else "decimal128" if kind == "sum" else arg_phys


def check_window(t, cols: dict, part: list, order: list, frame: tuple, funcs=None, carried=None, what=None, model=None):
    """the window of table `t` (cols: {column: (phys, cells in row order)}) against the model, eight functions per call: the carried
    columns (default: every column, passed as columns = NULL; they ride on the first call) cell for cell in window order, then every
    function's value.  Returns the model's (order, values)."""
    vals = {c: cells for c, (_, cells) in cols.items()}
    funcs = funcs_for(cols) if funcs is None else funcs
    perm, want = model if model is not None else W.window(vals, part, order, frame, funcs)
    every = carried is None
    carried = list(cols) if every else list(carried)
    wrong = []
    for k in range(0, len(funcs), 8):
        chunk = funcs[k:k + 8]
        w = t.window(partition_by=part, order_by=order, frame=frame, funcs=chunk, columns=(None if every else carried) if k == 0 else [])
        try:
            assert w.num_rows == len(perm), (what, w.num_rows, len(perm))
            for c in carried if k == 0 else []:
                p = cols[c][0]
                if read_column(w, c, p) != [raw(p, vals[c][r]) for r in perm]:
                    wrong.append(("carried", c))
            for kind, c, name in chunk:
                got = read_column(w, name, out_phys(kind, cols[c][0] if c else None))
                if got != want[name]:
                    i = next(i for i, (a, b) in enumerate(zip(got, want[name])) if a != b)
                    wrong.append((name, i, got[i], want[name][i]))
        finally:
            w.destroy()
    assert not wrong, (what, part, order, frame, wrong[:8])
    return perm, want


def combos(keys: list, count: int, seed: int) -> list:
    """`count` (partition keys, order keys, frame) cases over the key columns: one, two or no partition keys, one or two order keys of
    either direction, the frames in turn"""
    rng = random.Random(seed)
    out = []
    for i in range(count):
        part = rng.sample(keys, min([1, 2, 0][i % 3], len(keys)))
        rest = [k for k in keys if k not in part] or keys
        order = [(k, rng.random() < 0.5) for k in rng.sample(rest, min(1 + i % 2, len(rest)))]
        out.append((part, order, FRAMES[(i + seed) % len(FRAMES)]))
    return out


def key_columns(cols: dict) -> list:
    return [c for c, (p, _) in cols.items() if p in KEY_PHYS]


# ---------------------------------------------------------------------------------------------------- seeded values over every type
def f32(x: float) -> float:
    return struct.unpack("<f", struct.pack("<f", x))[0]


def typed(name: str, k: int, rng: random.Random):
    """value k of a small per-column domain (heavy ties, negatives), or now and then a value at the type's edges"""
    p = PHYS[name]
    edge = rng.random() < 0.15
    if p == "int8":
        return rng.choice([-128, 127, -1]) if edge else (k * 37) % 256 - 128
    if p == "int16":
        return rng.choice([-32768, 32767]) if edge else (k * 4099) % 65536 - 32768
    if p == "int32":
        return rng.choice([-(1 << 31), (1 << 31) - 1]) if edge else k * 7919 - 40000 if name == "i32" else rng.randrange(-(1 << 31), 1 << 31)
    if p == "date32":
        return rng.choice([-719162, 2932896]) if edge else k * 3 - 300
    if p == "fsb4":
        return 32 + (k * 13) % 224  # char(1) codes 0x20..0xFF: compared as the int32 of the cell
    if p == "int64":
        return rng.choice([I64_MIN, I64_MAX]) if edge else k * (1 << 40) - (1 << 62) if name == "i64" else rng.randrange(I64_MIN, I64_MAX + 1)
    if name == "dn":
        return rng.choice([-(10 ** 18 - 1), 10 ** 18 - 1]) if edge else k * 1000003 - 5 * 10 ** 16
    if name == "dw":  # two values near 10^38 already wrap a SUM past 2^127
        return rng.choice([-(10 ** 38 - 1), 10 ** 38 - 1, 1 << 100, -(1 << 64)]) if edge else k * 10 ** 30 - 10 ** 32
    if p == "float32":
        return rng.choice([-0.0, float("nan")]) if edge else f32(k * 0.5 - 3)
    if p == "float64":
        return rng.choice([-0.0, float("inf")]) if edge else k * 0.25 - 1e3
    return b"a long shared prefix of this column's strings/" + str(k).encode() if k % 5 else b""  # utf8


def gen(seed: int, n: int, card: int, null: float = 0.1) -> dict:
    rng = random.Random(seed)
    return {c: [None if rng.random() < null else typed(c, rng.randrange(card), rng) for _ in range(n)] for c in NAMES}


def typed_cols(values: dict) -> dict:
    return {c: (PHYS[c], values[c]) for c in NAMES}


# ---------------------------------------------------------------------------------------------------- 1. every source kind
@pytest.fixture(scope="module", params=list(STAGING))
def staged_ctx(request):
    """a context made under one HOST staging mode: below 65 536 rows a batch is copied (decimals narrowed to 8 bytes unless narrowing
    is off), from 65 536 rows on packed (unless packing is off)"""
    from lingodb_b200 import runtime
    packed, narrow = STAGING[request.param]
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("LDB_PACKED_STAGING", packed)
        mp.setenv("LDB_NARROW_STAGING", narrow)
        ctx = runtime.Context(0)
    yield ctx
    ctx.close()


_BASE_MODELS = {}  # (n, case): the model's answer, shared by every staging mode and offset of one table


def base_cols(data) -> dict:
    return {c: (p, cells_of(p, *data[c])) for c, p, _, _ in BASE_COLUMNS}


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 3])
@pytest.mark.parametrize("n", [65535, 65536])
def test_host_batches_under_each_staging_mode(staged_ctx, n, offset):
    """one HOST batch (random bytes under NULL cells, utf8 NULL cells with their strings): copied at 65 535 rows, packed at 65 536"""
    from lingodb_b200 import program as P
    data = base_values(n, n)
    t = host_table(staged_ctx, f"h{n}_{offset}", data, n, offset)
    cols = base_cols(data)
    for i, (part, order, frame) in enumerate(combos(key_columns(cols), 2, n)):
        funcs = funcs_for(cols)
        key = (n, i)
        if key not in _BASE_MODELS:
            _BASE_MODELS[key] = W.window({c: v for c, (_, v) in cols.items()}, part, order, frame, funcs)
        check_window(P.RawTable(staged_ctx, t.h), cols, part, order, frame, funcs, what=("host", n, offset, i), model=_BASE_MODELS[key])
    t.clear()


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 3, 7])
def test_device_batches_at_bit_offsets(gpu_ctx, offset):
    from lingodb_b200 import program as P
    n = 5003
    data = base_values(100 + offset, n)
    t = device_table(gpu_ctx, f"d{offset}", data, n, offset)
    cols = base_cols(data)
    for i, (part, order, frame) in enumerate(combos(key_columns(cols), 3, offset)):
        check_window(P.RawTable(gpu_ctx, t.h), cols, part, order, frame, what=("device", offset, i))
    t.clear()


@pytest.mark.gpu
def test_materialized_rows(gpu_ctx):
    """decimal128 16-byte cells with validity bytes: a left outer probe_each's side column (NULL without a match), a NULL-propagating
    sum and a CASE over a full-range i128 column, so SUMs wrap"""
    from lingodb_b200 import program as P, runtime
    from test_gpu_result_reads import _ints, _wide, arrow
    col, const = (lambda x: ("col", x)), (lambda v: ("const", v))
    rng = np.random.default_rng(21)
    nb, n = 300, 4000
    bk = (rng.permutation(nb) * 2).astype(np.int32)
    bv, bnull = _ints(rng, nb, 64), rng.random(nb) < 0.2
    bt = runtime.Table(gpu_ctx, "wbuild", R.specs_of([("bk", "int32", 0, 0), ("bv", "int64", 0, 0)]))
    bt.append_host({"bk": bk, "bv": bv, "bv$valid": arrow("int64", bv, bnull, 0)[1]}, nb)
    spec = [("k", "int32", 0, 0), ("x", "int64", 0, 0), ("y", "int32", 0, 0), ("z", "decimal128", 38, 0)]
    rawv = {"k": (rng.integers(0, 2 * nb, n).astype(np.int32), np.zeros(n, bool)), "x": (_ints(rng, n, 64) >> 1, rng.random(n) < 0.2),
            "y": (rng.integers(-3, 4, n).astype(np.int32), rng.random(n) < 0.2), "z": (_wide(rng, n), rng.random(n) < 0.3)}
    pt = runtime.Table(gpu_ctx, "wprobe", R.specs_of(spec))
    chunk = {}
    for c, phys, _, _ in spec:
        chunk[c], chunk[c + "$valid"] = arrow(phys, *rawv[c], 0)
    pt.append_host(chunk, n)
    jt = runtime.join_table(gpu_ctx, nb)
    P.build_join(gpu_ctx, bt, jt, col("bk"), payload=("rowid",))
    m = ("probe_each", jt, col("k"), "outer")
    outs = [("rowid",), ("fetch", bt, m, "bv"), ("add", col("x"), col("y")), ("case", ("cmp", ">", col("y"), const(0)), col("x"), col("z")), col("y")]
    mt = P.RawTable(gpu_ctx, P.materialize(gpu_ctx, pt, outs))
    rows = mt.num_rows
    cols = {f"c{j}": ("decimal128", mt.gather(f"c{j}", list(range(rows)))) for j in range(5)}
    assert sorted(cols["c0"][1]) == list(range(n)) and all(None in cols[f"c{j}"][1] for j in (1, 2, 3))
    for i, (part, order, frame) in enumerate([(["c4"], [("c3", True)], (None, 0)), (["c1"], [("c0", False)], (-3, 3)),
                                              (["c4", "c1"], [("c2", False), ("c0", True)], (0, None)), ([], [("c3", False)], (None, 0))]):
        check_window(mt, cols, part, order, frame, what=("materialized", i))
    mt.destroy()
    runtime.state_destroy(gpu_ctx, jt)
    bt.clear()
    pt.clear()


@pytest.mark.gpu
def test_exported_groups(gpu_ctx):
    """int64 keys in 8-byte cells, decimal aggregates and a float64 aggregate in 16-byte cells (carried, and COUNT's argument)"""
    from lingodb_b200 import program as P, runtime
    from test_gpu_result_reads import _ints, arrow, read
    col = lambda x: ("col", x)
    rng = np.random.default_rng(22)
    n = 20000
    g = rng.integers(-40, 40, n).astype(np.int32)
    h = rng.integers(0, 6, n).astype(np.int32)
    v = _ints(rng, n, 64) >> 2
    spec = [("g", "int32", 0, 0), ("h", "int32", 0, 0), ("v", "int64", 0, 0)]
    rawv = {"g": (g, rng.random(n) < 0.1), "h": (h, rng.random(n) < 0.1), "v": (v, (np.abs(g) % 7 == 0) | (rng.random(n) < 0.2))}
    t = runtime.Table(gpu_ctx, "wgsrc", R.specs_of(spec))
    chunk = {}
    for c, phys, _, _ in spec:
        chunk[c], chunk[c + "$valid"] = arrow(phys, *rawv[c], 0)
    t.append_host(chunk, n)
    st = P.group_by(gpu_ctx, t, [col("g"), col("h")], [("sum", col("v")), ("max", col("v")), ("min_f64", ("i2f", col("v"))), ("count", col("v"))],
                    expected_groups=1024)
    gt = P.groups_table(gpu_ctx, st)
    m = gt.num_rows
    phys = {"k0": "int64", "k1": "int64", "a0": "decimal128", "a1": "decimal128", "a2": "float64", "a3": "decimal128"}
    cols = {c: (p, read(gt, c, p, list(range(m)))) for c, p in phys.items()}
    assert None in cols["a2"][1] and None in cols["k0"][1]
    for i, (part, order, frame) in enumerate([(["k0"], [("k1", True)], (None, 0)), (["k1"], [("a0", False), ("k0", True)], (-2, 2)),
                                              ([], [("a1", True)], (None, None)), (["k0", "k1"], [], (None, None))]):
        check_window(gt, cols, part, order, frame, what=("groups", i))
    gt.destroy()
    runtime.state_destroy(gpu_ctx, st)
    t.clear()


@pytest.mark.gpu
def test_join_marker_and_dictionary_tables(gpu_ctx):
    from lingodb_b200 import program as P, runtime
    from test_gpu_result_reads import _strings, arrow, read
    col, const = (lambda x: ("col", x)), (lambda v: ("const", v))
    rng = np.random.default_rng(23)
    nb = 5000
    bk = rng.choice(np.arange(-20_000, 20_000), nb, replace=False).astype(np.int32)
    bt = runtime.Table(gpu_ctx, "wkb", R.specs_of([("bk", "int32", 0, 0)]))
    bt.append_host({"bk": bk}, nb)
    pk = rng.integers(-20_000, 20_000, 8000).astype(np.int32)
    pt = runtime.Table(gpu_ctx, "wkp", R.specs_of([("pk", "int32", 0, 0)]))
    pt.append_host({"pk": pk}, len(pk))
    jt = runtime.join_table(gpu_ctx, nb)
    P.build_join(gpu_ctx, bt, jt, col("bk"), payload=("rowid",))
    P.run_effects(gpu_ctx, pt, [("mark", ("probe", jt, col("pk")), ("cmp", ">", col("pk"), const(-5000)))])
    mt = P.join_marks(gpu_ctx, jt, P.ALL)
    phys = {"key": "int64", "payload": "int64", "marked": "int32"}
    cols = {c: (p, read(mt, c, p, list(range(mt.num_rows)))) for c, p in phys.items()}
    assert set(cols["marked"][1]) == {0, 1}
    for i, (part, order, frame) in enumerate([(["marked"], [("key", True)], (None, 0)), (["marked"], [("payload", False)], (-4, 1)),
                                              ([], [("marked", False), ("key", False)], (0, 0))]):
        check_window(mt, cols, part, order, frame, what=("marks", i))
    # the dictionary table: "str" (utf8) partitions, "rank" (int32) orders
    n = 20000
    s = _strings(rng, n)
    t = runtime.Table(gpu_ctx, "wdsrc", R.specs_of([("s", "utf8", 0, 0)]))
    buf, bitmap = arrow("utf8", s, rng.random(n) < 0.1, 0)
    t.append_host({"s": buf, "s$valid": bitmap}, n)
    d = P.dict_state(gpu_ctx, 8192, 1 << 20)
    P.run_effects(gpu_ctx, t, [("strcode", d, "s")])
    dt = P.dict_table(gpu_ctx, d)
    m = dt.num_rows
    strs = dt.gather_strings("str", list(range(m)), decode=False)
    cols = {"str": ("utf8", strs), "rank": ("int32", dt.gather("rank", list(range(m)), cell_bytes=4))}
    for i,(part, order, frame) in enumerate([(["str"], [("rank", False)], (None, 0)), ([], [("rank", True)], (-1, 1)),
                                              ([], [("str", True)], (None, 0))]):
        check_window(dt, cols, part, order, frame, what=("dictionary", i))
    dt.destroy()
    mt.destroy()
    runtime.state_destroy(gpu_ctx, d)
    runtime.state_destroy(gpu_ctx, jt)
    for tab in (bt, pt, t):
        tab.clear()


@pytest.mark.gpu
def test_received_and_sorted_tables():
    """rank 0 / 1 of a table_exchange_varlen (validity bytes, utf8 offsets from 0) and of a sort_exchange, each modelled over the rows
    that rank holds"""
    from test_gpu_exchange import ranks
    from lingodb_b200 import program as P
    world, n = 2, 6000
    values = gen(31, n, 400)
    with ranks(world, user_bytes=64 << 20) as (ctxs, comms):
        srcs = [P.RawTable(c, c.table_from_host(R.to_table_data("x", {k: v[r::world] for k, v in values.items()}, COLUMNS, [])).h)
                for r, c in enumerate(ctxs)]
        half = 32 << 20

        def run(r):
            rx = comms[r].table_exchange_varlen(srcs[r], ["i64", "dt"], NAMES, name="rx", recv_offset=0, recv_bytes=half)
            sx, _, _ = comms[r].sort_exchange(srcs[r], [("dn", True), ("i32", False)], NAMES, name="sx", recv_offset=half, recv_bytes=half)
            return rx, sx
        with ThreadPoolExecutor(world) as ex:
            tabs = list(ex.map(run, range(world)))
        seen = 0
        for r, (rx, sx) in enumerate(tabs):
            for kind, tab in (("received", rx), ("sorted", sx)):
                m = tab.num_rows
                seen += m
                cols = {c: (PHYS[c], read_column(tab, c, PHYS[c])) for c in NAMES}
                cols = {c: (p, [None if v is None else struct.unpack("<f" if p == "float32" else "<d", struct.pack("<i" if p == "float32" else "<q", v))[0]
                                for v in cells]) if p.startswith("float") else (p, cells) for c, (p, cells) in cols.items()}
                for i, (part, order, frame) in enumerate(combos(key_columns(cols), 2, 40 + r)):
                    check_window(tab, cols, part, order, frame, carried=NAMES, what=(kind, r, i))
        assert seen == 2 * n


@pytest.mark.gpu
def test_setop_and_window_results(gpu_ctx):
    """a DISTINCT result (validity bytes, 16-byte decimals) as the source; then a window result as the source of a second window,
    partitioned by the first one's SUM (16-byte decimal with validity bytes) and its MIN over a narrowed decimal (8-byte cells)"""
    n = 3000
    values = gen(41, n, 60)
    t = stage(gpu_ctx, values, COLUMNS, "single", 41)
    names = ["i8", "i32", "dt", "fs", "dn", "dw", "s", "f8"]
    d = t.distinct(names)
    rows = S.setop("distinct", list(zip(*[values[c] for c in names])))
    dcols = {c: (PHYS[c], [r[j] for r in rows]) for j, c in enumerate(names)}
    for i, (part, order, frame) in enumerate(combos(key_columns(dcols), 3, 41)):
        check_window(d, dcols, part, order, frame, what=("distinct", i))
    d.destroy()
    # the first window, partitioned by a tied int32 so its SUM and MIN repeat within partitions
    first = [("sum", "dw", "s1"), ("min", "dn", "m1"), ("max", "fs", "x1"), ("row_number", None, "r1")]
    carry = ["i64", "s", "i16", "dn"]
    w1 = t.window(partition_by=["i32"], order_by=[], frame=(None, None), funcs=first, columns=carry)
    perm, want = W.window(values, ["i32"], [], (None, None), first)
    cols = {c: (PHYS[c], [values[c][r] for r in perm]) for c in carry}
    cols.update({"s1": ("decimal128", want["s1"]), "m1": ("decimal128", want["m1"]), "x1": ("fsb4", want["x1"]), "r1": ("int64", want["r1"])})
    check_window(w1, cols, ["s1", "m1"], [("i64", True), ("s", False)], (None, 0), what="window of a window")
    check_window(w1, cols, ["m1"], [("s1", False), ("r1", True)], (-1, 1), carried=["i16", "s1"], what="window of a window, carried")
    w1.destroy()


# ---------------------------------------------------------------------------------------------------- 2. every key and argument type
TYPE_KEYS = ["i32", "dt", "fs", "i64", "dn", "dw", "s"]


@pytest.mark.gpu
def test_every_key_and_argument_type(gpu_ctx):
    n = 3000
    values = gen(51, n, 40)
    t = stage(gpu_ctx, values, COLUMNS, "single", 51)  # random bytes under the NULL cells
    cols = typed_cols(values)
    cases = []
    for i, k in enumerate(TYPE_KEYS):
        other = TYPE_KEYS[(i + 3) % len(TYPE_KEYS)]
        cases += [([k], [(other, i % 2 == 1)], FRAMES[i % len(FRAMES)]), ([other], [(k, True)], FRAMES[(i + 1) % len(FRAMES)]),
                  ([], [(k, False)], (None, 0))]
    for part, order, frame in cases:
        check_window(t, cols, part, order, frame, carried=NAMES if part and part[0] == "i32" else [], what="types")
    # result types: SUM is decimal128(38, the argument's scale), MIN / MAX the argument's type; a set operation refuses mismatched
    # types and scales, so a union with a one-row table of the expected type succeeds and one of another type fails
    funcs = [f for f in funcs_for(cols) if f[0] in ("sum", "min", "max")]
    probes = {}
    from lingodb_b200 import program as P
    for p, scale in [("int8", 0), ("int16", 0), ("int32", 0), ("int64", 0), ("date32", 0), ("fsb4", 0), ("decimal128", 2), ("decimal128", 0)]:
        probes[(p, scale)] = P.RawTable(gpu_ctx, gpu_ctx.table_from_host(R.to_table_data(f"p{p}{scale}", {"x": [1]}, [("x", p, 38, scale)], [])).h)
    for k in range(0, len(funcs), 8):
        chunk = funcs[k:k + 8]
        w = t.window(partition_by=["fs"], funcs=chunk, columns=[])
        for kind, c, name in chunk:
            p = PHYS[c]
            scale = 2 if p == "decimal128" else 0
            want = ("decimal128", scale) if kind == "sum" else (p, scale)
            u = w.setop(probes[want], "union_all", [name], ["x"])
            assert u.num_rows == n + 1, (name, want)
            u.destroy()
            wrong = ("int16", 0) if want[0] != "int16" else ("int8", 0)
            with pytest.raises(capi.LdbRuntimeError) as ei:
                w.setop(probes[wrong], "union_all", [name], ["x"])
            assert ei.value.code == capi.LDB_ERR_UNSUPPORTED, name
            if want[0] == "decimal128":
                with pytest.raises(capi.LdbRuntimeError):
                    w.setop(probes[("decimal128", 2 - scale)], "union_all", [name], ["x"])
        w.destroy()
    for pr in probes.values():
        pr.destroy()


# ---------------------------------------------------------------------------------------------------- 3. scan and tree edges
def np_window(v: np.ndarray, null: np.ndarray, key: np.ndarray, frame: tuple) -> dict:
    """the model's rules, vectorised, for a table already in window order: partitions are runs of equal `key` (int64, None as
    NULL is not used here), `v` int64 values small enough that no prefix sum leaves int64.  Returns {kind: (values, valid)}."""
    n = len(v)
    idx = np.arange(n)
    head = np.r_[True, key[1:] != key[:-1]] if n else np.zeros(0, bool)
    tail = np.r_[key[1:] != key[:-1], True] if n else np.zeros(0, bool)
    s = np.maximum.accumulate(np.where(head, idx, 0))
    e = np.minimum.accumulate(np.where(tail, idx, n)[::-1])[::-1]
    ln, j = e - s + 1, idx - s
    frm, to = frame
    lo = s if frm is None else s + np.minimum(ln - 1, np.maximum(0, j + frm))
    hi = e if to is None else s + np.minimum(ln - 1, np.maximum(0, j + to))
    pc = np.r_[0, np.cumsum(~null)]
    cnt = pc[hi + 1] - pc[lo]
    ps = np.r_[0, np.cumsum(np.where(null, 0, v))]
    out = {"row_number": (idx - lo + 1, np.ones(n, bool)), "count_star": (hi - lo + 1, np.ones(n, bool)), "count": (cnt, np.ones(n, bool)),
           "sum": (np.where(cnt > 0, ps[hi + 1] - ps[lo], 0), cnt > 0)}
    for kind, ident, pick in (("min", I64_MAX, np.minimum), ("max", I64_MIN, np.maximum)):
        # a sparse table: level k holds the pick over [i, i + 2^k); [lo, hi] is two overlapping blocks of the largest fitting level
        levels = [np.where(null, ident, v)]
        while (1 << len(levels)) <= max(n, 1):
            a, half = levels[-1], 1 << (len(levels) - 1)
            levels.append(pick(a, np.r_[a[half:], np.full(half, ident)]))
        width = hi - lo + 1
        lvl = np.floor(np.log2(np.maximum(width, 1))).astype(np.int64)
        res = np.empty(n, np.int64)
        for k in np.unique(lvl):
            m = lvl == k
            res[m] = pick(levels[k][lo[m]], levels[k][hi[m] - (1 << int(k)) + 1])
        out[kind] = (np.where(cnt > 0, res, 0), cnt > 0)
    return out


def read_np(t, column: str, cell: int):
    """(values as int64, validity) of a fixed-width column; 16-byte cells must hold values of 64 bits"""
    n = t.num_rows
    ids = np.arange(max(n, 1), dtype=np.int64)
    buf = np.zeros(max(n, 1) * cell, np.uint8)
    valid = np.zeros(max(n, 1), np.uint8)
    e = capi.Error()
    capi.check(t.ctx.L.ldb_gpu_table_gather(t.h, column.encode(), ids.ctypes.data_as(C.POINTER(C.c_int64)), n, buf.ctypes.data, valid.ctypes.data, C.byref(e)), e)
    if cell == 16:
        w = buf.view(np.int64).reshape(-1, 2)[:n]
        assert np.array_equal(w[:, 1], w[:, 0] >> 63), column  # the high word is the low word's sign
        vals = w[:, 0].copy()
    else:
        vals = buf.view({4: np.int32, 8: np.int64}[cell])[:n].astype(np.int64)
    return vals, valid[:n].astype(bool)


EDGE_FUNCS = [("row_number", None, "rn"), ("count_star", None, "cs"), ("count", "v", "cnt"), ("sum", "v", "sm"), ("min", "v", "mn"), ("max", "v", "mx"),
              ("min", "w", "mnw"), ("max", "w", "mxw")]


def check_np(w, v, null, key, frame, what):
    want = np_window(v, null, key, frame)
    for kind, c, name in EDGE_FUNCS:
        got, ok = read_np(w, name, 16 if kind == "sum" or c == "w" else 8)
        exp, eok = want[kind]
        assert np.array_equal(ok, eok), (what, name, frame, int(np.argmax(ok != eok)))
        bad = np.flatnonzero((got != exp) & eok)
        assert not len(bad), (what, name, frame, int(bad[0]), int(got[bad[0]]), int(exp[bad[0]]))


def edge_table(ctx, key, v, null):
    """source order is window order: `key` ascending (int32 partition key), "v" int64 and "w" decimal128(38) 16-byte cells of the same
    values, NULL where `null`"""
    from lingodb_b200 import datagen
    from lingodb_b200 import program as P
    n = len(v)
    bm = np.packbits(~null, bitorder="little")
    wide = np.stack([v.view(np.uint64), (v >> 63).view(np.uint64)], axis=1).view(np.uint8).reshape(-1, 16)
    spec = [datagen.ColumnSpec("p", "int32"), datagen.ColumnSpec("v", "int64"), datagen.ColumnSpec("w", "decimal128", 38, 0)]
    chunk = {"p": key.astype(np.int32), "v": v, "v$valid": bm, "w": wide, "w$valid": bm}
    tab = ctx.table_from_host(datagen.TableData("edge", spec, [chunk], [n]))  # holds the host buffers the staging reads
    return tab, P.RawTable(ctx, tab.h)


def test_numpy_reference_equals_the_model():
    """the vectorised restatement used for the large tables gives the model's answers on small ones (no GPU)"""
    rng = np.random.default_rng(61)
    for n in (0, 1, 7, 300):
        key = np.sort(rng.integers(0, max(1, n // 20), n)).astype(np.int64)
        v = rng.integers(-1000, 1000, n).astype(np.int64)
        null = rng.random(n) < 0.3
        cells = {"p": key.tolist(), "v": [None if z else int(x) for x, z in zip(v, null)]}
        for frame in [(-1, 1), (None, 0), (0, None), (-3000, 3000), (2, 5), (-5, -2), (None, None)]:
            funcs = [(k, None if k in ("row_number", "count_star") else "v", k) for k in ("row_number", "count_star", "count", "sum", "min", "max")]
            perm, want = W.window(cells, ["p"], [], frame, funcs)
            assert perm == list(range(n))
            got = np_window(v, null, key, frame)
            for k, _, _ in funcs:
                vals, ok = got[k]
                assert [int(x) if o else None for x, o in zip(vals, ok)] == want[k], (n, frame, k)


def edge_values(n: int, seed: int):
    rng = np.random.default_rng(seed)
    v = rng.integers(-(1 << 40), 1 << 40, n).astype(np.int64)
    null = rng.random(n) < 0.2
    null[:3] = True  # the running MIN / MAX starts on NULLs
    return v, null


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2047, 2048, 2049, 4095, 4096, 4097, 65536, 524288, 524289, 1 << 20])
def test_one_running_scan_across_every_tile(gpu_ctx, n):
    """no partition key: one partition whose running frames cross every 2048-row tile and every chunk of 256 tiles; powers of two
    leave the segment tree without padding leaves"""
    v, null = edge_values(n, n)
    key = np.zeros(n, np.int64)
    tab, t = edge_table(gpu_ctx, key, v, null)
    for frame in [(None, 0), (-1, 1), (0, None), (-3000, 3000)]:
        w = t.window(frame=frame, funcs=EDGE_FUNCS, columns=[])
        check_np(w, v, null, key, frame, ("scan", n))
        w.destroy()
    tab.clear()


def run_lengths(total: int) -> list:
    """partition runs of `total` rows in all: a first run of 1 row, then boundaries one row before, on and one row after the 2048-row
    tile edges in turn (all three at every fourth edge), so runs of 1, 2046..2049 rows"""
    cuts, k = {1}, 1
    while k * 2048 + 1 < total:
        cuts.update({k * 2048 + d for d in ((-1, 0, 1) if k % 4 == 0 else ((k % 3) - 1,))})
        k += 1
    return np.diff([0] + sorted(cuts) + [total]).tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("total", [20000, 530000])
def test_partition_runs_across_tile_edges(gpu_ctx, total):
    runs = run_lengths(total)
    key = np.repeat(np.arange(len(runs)), runs).astype(np.int64)
    n = len(key)
    starts = np.r_[0, np.cumsum(runs)[:-1]]
    assert all((starts % 2048 == d % 2048).sum() >= 3 for d in (-1, 0, 1))
    v, null = edge_values(n, total)
    null[starts[2]:starts[3]] = True  # a whole partition without a value
    tab, t = edge_table(gpu_ctx, key, v, null)
    for frame in [(-1, 1), (None, 0), (0, None), (-3000, 3000)]:
        w = t.window(partition_by=["p"], frame=frame, funcs=EDGE_FUNCS, columns=[])
        check_np(w, v, null, key, frame, ("runs", total))
        w.destroy()
    if total < 100000:  # and the model itself over the small one
        cells = {"p": key.tolist(), "v": [None if z else int(x) for x, z in zip(v, null)]}
        cols = {"p": ("int32", cells["p"]), "v": ("int64", cells["v"])}
        check_window(t, cols, ["p"], [], (-1, 1), funcs=[f for f in EDGE_FUNCS if f[1] != "w"], carried=["p", "v"], what="runs model")
    tab.clear()


# ---------------------------------------------------------------------------------------------------- 4. extreme values and wrap
@pytest.mark.gpu
def test_identity_values_and_wrapping_sums(gpu_ctx):
    """partitions whose only values are INT64_MIN / INT64_MAX (8- and 16-byte cells) or -2^127 / 2^127 - 1 (16-byte cells), between NULLs:
    MIN / MAX return them valid and NULL only where the frame holds no value; int8 / int16 extremes; SUMs past 2^64 (int64) and past
    2^127 (decimal(38), wrapping)"""
    from lingodb_b200 import program as P
    spec = [("p", "int32", 0, 0), ("o", "int32", 0, 0), ("e64", "int64", 0, 0), ("ew", "decimal128", 38, 0), ("e8", "int8", 0, 0),
            ("e16", "int16", 0, 0), ("dw", "decimal128", 38, 2)]
    extremes = [(I64_MIN, I64_MIN, -128, -32768), (I64_MAX, I64_MAX, 127, 32767), (I64_MIN, I128_MIN, -128, 32767), (I64_MAX, I128_MAX, 127, -32768)]
    rng = random.Random(71)
    values = {c: [] for c, *_ in spec}
    for g in range(40):
        size = rng.choice([1, 2, 5, 17])
        e64, ew, e8, e16 = extremes[g % 4]
        for i in range(size):
            has = g % 5 != 4 and rng.random() < 0.4  # every fifth partition has no value at all
            values["p"].append(g)
            values["o"].append(rng.randrange(size))
            values["e64"].append(e64 if has else None)
            values["ew"].append(ew if has else None)
            values["e8"].append(e8 if has else None)
            values["e16"].append(e16 if has else None)
            values["dw"].append(rng.choice([10 ** 38 - 1, 10 ** 38 - 2, -(10 ** 38 - 1)]) if g % 3 else None)
    t = P.RawTable(gpu_ctx, gpu_ctx.table_from_host(R.to_table_data("ext", values, spec, [])).h)
    cols = {c: (p, values[c]) for c, p, _, _ in spec}
    for frame in [(0, 0), (-1, 1), (None, 0), (None, None), (1, 2)]:
        _, want = check_window(t, cols, ["p"], [("o", False)], frame, what=("extremes", frame))
        if frame == (None, None):
            assert {I64_MIN, I64_MAX} <= set(want["w_min_e64"]) and {I128_MIN, I128_MAX} <= set(want["w_max_ew"]) and None in want["w_max_ew"]
            assert any(x is not None and (x > I64_MAX or x < I64_MIN) for x in want["w_sum_e64"])  # past 2^64
            exact = {}
            for g, x in zip(values["p"], values["dw"]):
                exact[g] = exact.get(g, 0) + (x or 0)
            assert max(exact.values()) > I128_MAX  # some partition's SUM wraps past 2^127


# ---------------------------------------------------------------------------------------------------- 5. frames at the limits
LIMIT_FRAMES = [(-(1 << 40) - 1, -(1 << 40) + 1), ((1 << 40), (1 << 40)), (-(1 << 63) + 1, (1 << 63) - 2), ((1 << 62), None), (None, -(1 << 62)),
                (5, None), (-(1 << 63) + 1, -(1 << 63) + 1), ((1 << 63) - 2, (1 << 63) - 2), (-(1 << 40), 1 << 40), (3, 3)]


@pytest.mark.gpu
def test_frames_at_the_offset_limits(gpu_ctx):
    """offsets past the +-2^40 clamp and near +-2^63: ROW_NUMBER is i - lo + 1, which is <= 0 when the frame starts after the row"""
    n = 600
    values = gen(81, n, 30)
    t = stage(gpu_ctx, values, COLUMNS, "single", 81)
    cols = {c: (PHYS[c], values[c]) for c in ["i32", "i64", "dn", "dw", "i8", "fs", "s"]}
    for i, frame in enumerate(LIMIT_FRAMES):
        part = [["i32"], [], ["s", "fs"]][i % 3]
        _, want = check_window(t, cols, part, [("i64", i % 2 == 0)], frame, what=("limits", frame))
        if frame[0] is not None and frame[0] > 0:
            assert min(want["w_rn"]) <= 0, frame


# ---------------------------------------------------------------------------------------------------- 6. sharded composition
@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_composition(world):
    """a table sharded by batch-sized slices, exchanged on its fixed-width partition keys (NULL keys included), then a local window
    per rank ordered last by a unique row id: every row keyed by its id equals the single-table model, and every partition sits on one
    rank"""
    from test_gpu_exchange import ranks
    from lingodb_b200 import program as P
    n = 12000
    values = gen(91, n, 150)
    values["rid"] = list(range(n))
    names = ["i64", "dn", "dt", "j32", "s", "dw", "j64", "i8", "f4", "i16", "fs", "rid"]  # the exchange ships up to 16 columns
    cols_spec = [c for c in COLUMNS if c[0] in names] + [("rid", "int64", 0, 0)]
    configs = [(["i64"], [("j32", True), ("rid", False)], (-2, 2)), (["dn", "dt"], [("s", False), ("rid", True)], (None, 0))]
    funcs = [("row_number", None, "w_rn"), ("sum", "dw", "w_sum"), ("min", "j64", "w_min"), ("max", "i8", "w_max"), ("count", "f4", "w_cnt"),
             ("count_star", None, "w_cs"), ("sum", "i16", "w_s16"), ("max", "fs", "w_mfs")]
    outs = [("int64", "w_rn"), ("decimal128", "w_sum"), ("int64", "w_min"), ("int8", "w_max"), ("int64", "w_cnt"), ("int64", "w_cs"),
            ("decimal128", "w_s16"), ("fsb4", "w_mfs")]
    with ranks(world, user_bytes=96 << 20) as (ctxs, comms):
        def shard(r):
            idx = [i for i in range(n) if (i // 1000) % world == r]
            return P.RawTable(ctxs[r], ctxs[r].table_from_host(R.to_table_data("sh", {c: [values[c][i] for i in idx] for c in names}, cols_spec, [])).h)
        srcs = [shard(r) for r in range(world)]
        half = 48 << 20
        for ci, (part, order, frame) in enumerate(configs):
            def run(r):
                rx = comms[r].table_exchange_varlen(srcs[r], part, names, name="rx", recv_offset=ci * half, recv_bytes=half)
                w = rx.window(partition_by=part, order_by=order, frame=frame, funcs=funcs, columns=["rid"] + part)
                got = {"rid": read_column(w, "rid", "int64")}
                for c in part:
                    got[c] = read_column(w, c, PHYS[c])
                for p, name in outs:
                    got[name] = read_column(w, name, p)
                w.destroy()
                rx.destroy()
                return got
            with ThreadPoolExecutor(world) as ex:
                res = list(ex.map(run, range(world)))
            perm, want = W.window(values, part, order, frame, funcs)
            exp = {values["rid"][r]: tuple(want[name][i] for _, name in outs) for i, r in enumerate(perm)}
            got, owner = {}, {}
            for r, g in enumerate(res):
                for i, rid in enumerate(g["rid"]):
                    assert rid not in got, (ci, rid)
                    got[rid] = tuple(g[name][i] for _, name in outs)
                    pk = tuple(g[c][i] for c in part)
                    assert owner.setdefault(pk, r) == r, (ci, pk)  # one partition, one rank
            assert len(got) == n and got == exp, (ci, next((k for k in exp if got.get(k) != exp[k]), None))
            assert len(set(owner.values())) == world, ci


# ---------------------------------------------------------------------------------------------------- 7. errors, nothing launched
@pytest.mark.gpu
def test_errors_launch_nothing():
    import torch
    from lingodb_b200 import datagen, runtime
    from lingodb_b200 import program as P
    from test_gpu_window import COLUMNS as WCOLUMNS, KEYS as WKEYS, gen as wgen
    values = wgen(7, 50, 7)
    values["f4"] = [1.5] * 50
    cols = WCOLUMNS + [("f4", "float32", 0, 0)]
    with runtime.Context(0) as ctx:
        t = P.RawTable(ctx, ctx.table_from_host(R.to_table_data("w", values, cols, [])).h)
        multi = P.RawTable(ctx, ctx.table_from_host(R.to_table_data("m", values, cols, [20])).h)
        small = P.RawTable(ctx, ctx.table_from_host(R.to_table_data("s", {c: values[c] for c in ("a64", "p32", "cname")},
                                                                    [c for c in WCOLUMNS if c[0] in ("a64", "p32", "cname")], [])).h)
        ok = [("sum", "a64", "s")]
        before = ctx.launch_count()

        def code(tab=t, **kw):
            kw.setdefault("funcs", ok)
            kw.setdefault("columns", [])
            with pytest.raises(capi.LdbRuntimeError) as ei:
                tab.window(**kw)
            assert ctx.launch_count() == before, kw
            return ei.value.code, str(ei.value)
        inv, uns = capi.LDB_ERR_INVALID, capi.LDB_ERR_UNSUPPORTED
        assert code(partition_by=["nope"])[0] == inv
        assert code(funcs=[("sum", "nope", "s")])[0] == inv
        assert code(columns=["nope"])[0] == inv
        for f in [("sum", "f4", "s"), ("min", "cname", "s"), ("max", "f4", "s"), ("sum", "adt", "s"), ("min", "cf8", "s"), ("max", "cname", "s")]:
            c, m = code(funcs=[f])
            assert c == uns and f[1] in m, (f, m)
        for k in ("f4", "a8", "c16", "cf8"):
            c, m = code(partition_by=[k])
            assert c == uns and k in m, k
            c, m = code(order_by=[(k, True)])
            assert c == uns and k in m, k
        assert code(tab=multi)[0] == uns
        for frame in [(3, 2), ((1 << 63) - 1, (1 << 63) - 1), (-(1 << 63), -(1 << 63)), (None, -(1 << 63)), ((1 << 63) - 1, None)]:
            assert code(frame=frame)[0] == inv, frame
        assert code(funcs=[])[0] == inv
        assert code(funcs=ok * 9)[0] == inv
        assert code(partition_by=WKEYS[:5])[0] == inv
        assert code(order_by=[(k, False) for k in WKEYS[:5]])[0] == inv
        assert code(columns=[n for n, *_ in WCOLUMNS])[0] == inv  # 17 carried columns
        assert code(columns=None)[0] == inv  # "all" is 18 columns here
        # duplicate output names: a function named like a carried column (named, or every column of a small table), two functions of
        # one name, a column carried twice
        for kw, clash in [(dict(funcs=[("sum", "a64", "a64")], columns=["p32", "a64"]), "a64"), (dict(tab=small, funcs=[("sum", "a64", "a64")], columns=None), "a64"),
                          (dict(tab=small, funcs=[("count", "p32", "cname")], columns=None), "cname"),
                          (dict(funcs=[("sum", "a64", "x"), ("row_number", None, "y"), ("count", "a64", "x")]), "x"),
                          (dict(columns=["a64", "p32", "a64"]), "a64"), (dict(funcs=[("row_number", None, "p32")], columns=["p32"]), "p32")]:
            c, m = code(**kw)
            assert c == inv and clash in m, (kw, m)
        fs = (capi.WindowFunc * 1)(capi.WindowFunc(9, b"a64", b"x"))
        out, e = C.c_void_p(), capi.Error()
        assert ctx.L.ldb_gpu_table_window(t.h, 0, None, 0, None, None, -(1 << 63), 0, 1, fs, 0, None, None, C.byref(out), C.byref(e)) == inv
        assert ctx.L.ldb_gpu_table_window(None, 0, None, 0, None, None, -(1 << 63), 0, 1, fs, 0, None, None, C.byref(out), C.byref(e)) == inv
        fs = (capi.WindowFunc * 1)(capi.WindowFunc(capi.WIN["sum"], b"a64", None))
        assert ctx.L.ldb_gpu_table_window(t.h, 0, None, 0, None, None, -(1 << 63), 0, 1, fs, 0, None, None, C.byref(out), C.byref(e)) == inv
        assert ctx.launch_count() == before
        # inside a captured query
        ctx.graph_begin()
        try:
            c, m = code()
        finally:
            ctx.graph_end().destroy()
        assert c == uns and "captured" in m
        # 2^32 rows: one borrowed DEVICE batch of 2^32 int8 rows over a 4 GiB tensor (a batch's row count is an int64, so one batch
        # reaches it); refused before the sort is sized or anything launched
        buf = torch.empty(1 << 32, dtype=torch.int8, device="cuda:0")
        huge = ctx.table("huge", [datagen.ColumnSpec("i8", "int8")])
        huge.append_device({"i8": buf}, 1 << 32)
        hr = P.RawTable(ctx, huge.h)
        assert hr.num_rows == 1 << 32
        c, m = code(tab=hr, funcs=[("sum", "i8", "s")])
        assert c == uns and "2^32" in m, m
        c, m = code(tab=hr, funcs=[("row_number", None, "r")], columns=None)
        assert c == uns and "2^32" in m, m
        huge.clear()
        del buf
        # and the tables still work afterwards
        w = t.window(funcs=ok, columns=[])
        assert w.num_rows == 50
        w.destroy()
        w = small.window(funcs=[("sum", "a64", "total")], columns=None)
        assert w.num_rows == 50
        w.destroy()
