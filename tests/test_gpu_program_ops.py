"""The program interpreter (csrc/program.cu) opcode by opcode, layout by layout and sink by sink, against the exact reference evaluator
of tests/_progref.py.  Materialized cells are compared bit for bit (validity included; any NaN equals any NaN), aligned to their source
rows through a ROWID output because the materialize sink appends in no fixed order."""
import math
import random

import numpy as np
import pytest

import _progref as R
from lingodb_b200 import capi, datagen, program as P, runtime

pytestmark = pytest.mark.gpu

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))
N_SWEEP = 3000


# ---------------------------------------------------------------------------------------------------- helpers
def _stage(ctx, name, values, columns=R.SWEEP_COLUMNS, cuts=()):
    return ctx.table_from_host(R.to_table_data(name, values, columns, cuts))


def _read(ctx, h, n_cols):
    """every column of a library-made single-batch table (c0..cN), one list per column (None = NULL)"""
    t = P.RawTable(ctx, h)
    n = t.num_rows
    cols = [t.gather(f"c{i}", list(range(n))) for i in range(n_cols)]
    t.destroy()
    return cols


def _materialize(ctx, tab, exprs, where=None):
    h = P.materialize(ctx, tab, list(exprs), where=where)
    return _read(ctx, h, len(exprs))


def _check_batch(ctx, tab, ev, batch, what=""):
    """materialize [ROWID] + the batch's expressions; every cell equals the evaluator's value for that row"""
    exprs = [e for _, e in batch]
    got = _materialize(ctx, tab, [("rowid",)] + exprs)
    want = ev.run(exprs)[0]
    assert sorted(got[0]) == list(range(ev.n)), what
    for j, e in enumerate(exprs):
        for rid, g in zip(got[0], got[j + 1]):
            w = want[j][rid - ev.first_row]
            assert R.same_cell(g, w), (what, e, rid, g, w)


def _check_where(ctx, tab, ev, pred, what=""):
    got = _materialize(ctx, tab, [("rowid",)], where=pred)[0]
    want = ev.run([("rowid",)], where=pred)[0][0]
    assert sorted(got) == want, (what, pred)


def _check_programs(ctx, tab, ev, progs, what=""):
    for batch in R.pack(progs):
        _check_batch(ctx, tab, ev, batch, what)
    for ty, e in progs:
        if ty == "bool":
            _check_where(ctx, tab, ev, e, what)


@pytest.fixture(scope="module")
def sweep(gpu_ctx):
    values = R.gen_values(101, N_SWEEP)
    tab = _stage(gpu_ctx, "sweep", values, cuts=(1000,))
    return tab, values, R.Evaluator(values)


# ---------------------------------------------------------------------------------------------------- 1. opcodes
def _edge_programs():
    """every opcode on the edge rows of the sweep table (the first rows of every column hold its edge values)"""
    ints = [col(c) for c in R.INT_COLUMNS]
    out = []
    for c in ints:
        out += [("int", ("neg", c)), ("int", ("mul", c, c)), ("int", ("mul", c, const(R.I64_MAX))), ("int", ("add", c, const(R.I128_MAX))),
                ("int", ("sub", c, const(1))), ("float", ("i2f", c)), ("bool", ("isnull", c)), ("int", ("mul", c, const((1 << 64) + 1)))]
        out += [("int", ("div", c, const(k))) for k in (2, -2, 0, 7, -(1 << 64), R.I128_MAX)]
        out += [("int", ("div", const(k), ("case", ("cmp", "=", c, const(-1)), const(1), c))) for k in (-7, R.I128_MAX, 1 << 100)]
        out += [("bool", ("cmp", op, c, const(k))) for op in R.CMP_OPS for k in (0, -1, R.I64_MAX, 1 << 64)]
    out += [("int", ("div", col("i64"), col("i32"))), ("int", ("div", col("dn"), ("case", ("cmp", "=", col("i16"), const(-1)), const(3), col("i16"))))]
    out += [("bool", ("cmp", op, col("dw"), col("dn"))) for op in R.CMP_OPS]  # values that differ only in the high word
    out += [("int", ("year", col("dt")))] + [("int", ("year", const(d))) for d in (-719163, R.I32_MAX, R.I32_MIN)]
    out += [("bool", ("cmp", op, col("dt"), const(11016))) for op in R.CMP_OPS]
    for a, b in (("f8", "f4"), ("f4", "f8"), ("f8", "f8")):
        out += [("float", (op, col(a), col(b))) for op in ("fadd", "fsub", "fmul", "fdiv")]
        out += [("bool", ("fcmp", op, col(a), col(b))) for op in R.CMP_OPS]
    out += [("float", ("fdiv", col("f8"), ("f64", z))) for z in (0.0, -0.0, math.inf)]
    out += [("float", ("i2f", const(v))) for v in (2**53 + 1, 2**64 - 1, R.I128_MIN, -(2**53 + 3), (1 << 100) + 1)]
    for s in R.STRING_COLUMNS:
        out += [("int", ("strkey8", s)), ("bool", ("isnull", ("strkey8", s)))]
        out += [("bool", ("strcmp", op, s, p)) for op in R.CMP_OPS for p in R.PATTERNS]
        out += [("bool", ("like", k, s, p)) for k in ("prefix", "suffix", "contains") for p in R.PATTERNS]
    a, b = ("cmp", ">", col("i32"), const(0)), ("fcmp", "<", col("f8"), ("f64", 0.0))  # both NULL on some rows
    out += [("bool", ("and", a, b)), ("bool", ("or", a, b)), ("bool", ("not", a)), ("bool", ("not", ("isnull", a))),
            ("int", ("case", a, col("dw"), col("i8"))), ("float", ("case", b, col("f4"), ("f64", -1.5))), ("bool", ("between", col("i16"), const(-5), const(5)))]
    return out


def test_every_opcode_on_edge_values(gpu_ctx, sweep):
    tab, _, ev = sweep
    _check_programs(gpu_ctx, tab, ev, _edge_programs(), "edges")


@pytest.mark.parametrize("seed", range(6))
def test_random_programs(gpu_ctx, sweep, seed):
    tab, _, ev = sweep
    _check_programs(gpu_ctx, tab, ev, R.programs(1000 + seed, 50), f"seed {seed}")


# ---------------------------------------------------------------------------------------------------- 2. layouts
LAYOUT_PROGRAMS = R.programs(77, 40)


def test_ragged_batches(gpu_ctx):
    values = R.gen_values(5, 1 + 31 + 33 + 4097 + 50)
    tab = _stage(gpu_ctx, "ragged", values, cuts=(1, 32, 65, 4162))
    _check_programs(gpu_ctx, tab, R.Evaluator(values), LAYOUT_PROGRAMS, "ragged")


def test_device_resident_batch(gpu_ctx):
    import torch
    values = R.gen_values(6, 2500)
    td = R.to_table_data("dev", values)
    tab = runtime.Table(gpu_ctx, "dev", td.columns)
    ch = td.chunks[0]
    dev = {}
    for k, v in ch.items():
        if isinstance(v, tuple):
            dev[k] = (torch.from_numpy(v[0]).cuda(), torch.from_numpy(v[1]).cuda())
        else:
            dev[k] = torch.from_numpy(np.ascontiguousarray(v)).cuda()
    torch.cuda.synchronize()
    tab.append_device(dev, td.chunk_rows[0])
    _check_programs(gpu_ctx, tab, R.Evaluator(values), LAYOUT_PROGRAMS, "device")


@pytest.mark.parametrize("offset", range(1, 8))
def test_bitmaps_at_array_offsets(gpu_ctx, offset):
    """Arrow slices: every buffer and validity bitmap starts `offset` rows in, so row 0's validity bit sits mid-byte"""
    values = R.gen_values(10 + offset, 700)
    specs = R.specs_of()
    tab = runtime.Table(gpu_ctx, f"off{offset}", specs)
    ch = {}
    for name, phys, _, _ in R.SWEEP_COLUMNS:
        buf, bm = R.column_buffers(phys, values[name], offset)
        ch[name] = buf
        if bm is not None:
            bm = bm.copy()
            bm[0] |= (1 << offset) - 1  # the filler rows before the slice read as valid: a reader that ignores the offset sees them
            ch[name + "$valid"] = bm
    tab.append_host(ch, 700, offset=offset)
    _check_programs(gpu_ctx, tab, R.Evaluator(values), LAYOUT_PROGRAMS[:12], f"offset {offset}")


def test_large_host_batch_through_compressed_staging(gpu_ctx):
    """a HOST batch of >= 65 536 rows takes the packed staging path; checked through keyless SUM / COUNT / MIN / MAX of each output"""
    n = 70_000
    values = R.gen_values(8, n)
    tab = _stage(gpu_ctx, "big", values)
    ev = R.Evaluator(values)
    progs = [p for p in R.programs(78, 40) if p[0] in ("int", "bool", "date")][:12]
    for ty, e in progs:
        aggs = [("sum", e), ("count", e), ("count_star", None), ("min", e), ("max", e)]
        st = P.group_by(gpu_ctx, tab, [], aggs)
        got = P.decode_groups(P.read_groups(gpu_ctx, st, 4), 0, len(aggs))[()]
        gpu_ctx.L.ldb_gpu_state_destroy(st)
        vals = ev.eval(e)
        want = R.group_by(n, [], [(k, None if x is None else vals) for k, x in aggs])[()]
        assert got == want, e


def test_validity_bytes_of_a_materialized_source(gpu_ctx, sweep):
    """a materialized table (16-byte cells, one validity byte per row) fed back in as a program's source"""
    tab, values, _ = sweep
    names = [c for c in R.INT_COLUMNS if c != "k"] + ["dt"]  # the materialize sink's limit: 8 outputs
    src = P.RawTable(gpu_ctx, P.materialize(gpu_ctx, tab, [col(c) for c in names]))
    rename = {c: f"c{i}" for i, c in enumerate(names)}
    # the materialize sink's row order is not the source's: align the evaluator's columns to the materialized rows
    got = [src.gather(f"c{i}", list(range(src.num_rows))) for i in range(len(names))]
    ev = R.Evaluator({rename[c]: got[i] for i, c in enumerate(names)})
    assert sorted(map(repr, zip(*got))) == sorted(map(repr, zip(*[values[c] for c in names])))

    def uses_only(e):
        if not isinstance(e, tuple):
            return True
        if e[0] == "col":
            return e[1] in rename
        if e[0] in ("strkey8", "strcmp", "like", "fcmp", "f64", "i2f", "fadd", "fsub", "fmul", "fdiv"):
            return False
        return all(uses_only(x) for x in e[1:])

    def ren(e):
        if isinstance(e, tuple) and e and e[0] == "col":
            return ("col", rename[e[1]])
        return tuple(ren(x) for x in e) if isinstance(e, tuple) else e

    progs = [(t, ren(e)) for t, e in R.programs(79, 200) if t in ("int", "bool", "date") and uses_only(e)][:25]
    assert len(progs) >= 10
    _check_programs(gpu_ctx, P.RawTable(gpu_ctx, src.h), ev, progs, "validity bytes")
    src.destroy()


def test_side_columns_over_a_multi_batch_side_table(gpu_ctx, sweep):
    """FETCH of every column type of a 4-batch side table, at row numbers that include NULL, negative and out-of-range ones"""
    _, values, _ = sweep
    side = _stage(gpu_ctx, "side", values, cuts=(7, 1500, 1501))
    rows = R.gen_values(33, 1200, columns=[("r", "int32", 0, 0)], null_rate=0.1)
    rng = random.Random(4)
    rows["r"] = [None if v is None else rng.choice([rng.randrange(N_SWEEP), -1, N_SWEEP, N_SWEEP - 1, 0, 1499, 1500, 1501, R.I32_MAX]) for v in rows["r"]]
    probe = _stage(gpu_ctx, "rows", rows, columns=[("r", "int32", 0, 0)])
    ev = R.Evaluator(rows, sides={side.h.value: R.Side(values)})
    f = lambda c: ("fetch", side, col("r"), c)
    progs = [("int", f(c)) for c in R.INT_COLUMNS + ["dt"]] + [("float", f(c)) for c in R.FLOAT_COLUMNS]
    progs += [("int", ("strkey8", f(c))) for c in R.STRING_COLUMNS] + [("bool", ("like", "contains", f("s"), "a")), ("bool", ("strcmp", ">=", f("u"), "é"))]
    progs += [("int", ("add", f("dw"), f("i8"))), ("bool", ("isnull", f("dn")))]
    _check_programs(gpu_ctx, probe, ev, progs, "side columns")


# ---------------------------------------------------------------------------------------------------- 3. aggregates
AGG_COLUMNS = [("g0", "int32", 0, 0), ("g1", "int64", 0, 0), ("g2", "int8", 0, 0), ("g3", "int16", 0, 0), ("v", "decimal128", 38, 0), ("f", "float64", 0, 0),
               ("w", "int64", 0, 0)]
BIG = [R.I64_MIN - 5, R.I64_MAX + 9, -(3 << 70), (5 << 90) + 1, R.I128_MIN + 1, R.I128_MAX - 1, -1, -7, 12, 0]


@pytest.fixture(scope="module")
def agg_table(gpu_ctx):
    rng = random.Random(21)
    n = 5000
    vals = {c: [] for c, *_ in AGG_COLUMNS}
    for i in range(n):
        g = [rng.choice([0, 1, 2, None]) for _ in range(4)]
        for k in range(4):
            vals[f"g{k}"].append(g[k])
        vals["v"].append(None if g[0] == 2 or rng.random() < 0.1 else rng.choice(BIG + [rng.randrange(-(1 << 100), 1 << 100), rng.randrange(-50, 50)]))
        vals["f"].append(None if (g[0] == 1 and g[1] == 0) or rng.random() < 0.1 else rng.randrange(-2**20, 2**20) / 8.0)  # sums exact in any order
        vals["w"].append(None if rng.random() < 0.2 else rng.choice([R.I64_MIN, R.I64_MAX, -3, rng.randrange(-1000, 1000)]))
    return _stage(gpu_ctx, "agg", vals, columns=AGG_COLUMNS, cuts=(1, 2000)), vals, n


AGG_SETS = [[("sum", "v"), ("count", "v"), ("count_star", None), ("min", "v"), ("max", "v"), ("any", "w"), ("min", "w"), ("max", "w")],
            [("sum_f64", "f"), ("min_f64", "f"), ("max_f64", "f"), ("count", "f")]]


@pytest.mark.parametrize("n_keys", range(5))
@pytest.mark.parametrize("aggset", range(len(AGG_SETS)))
def test_aggregates_every_kind_and_key_count(gpu_ctx, agg_table, n_keys, aggset):
    tab, vals, n = agg_table
    aggs = AGG_SETS[aggset]
    keys = [f"g{k}" for k in range(n_keys)]
    st = P.group_by(gpu_ctx, tab, [col(k) for k in keys], [(k, None if c is None else col(c)) for k, c in aggs], expected_groups=256)
    f64 = tuple(i for i, (k, _) in enumerate(aggs) if k.endswith("_f64"))
    got = P.decode_groups(P.read_groups(gpu_ctx, st, 1024), n_keys, len(aggs), f64_aggs=f64)
    want = R.group_by(n, [vals[k] for k in keys], [(k, None if c is None else vals[c]) for k, c in aggs])
    assert set(got) == set(want)
    any_at = [i for i, (k, _) in enumerate(aggs) if k == "any"]
    for g, w in want.items():
        for i, (kind, _) in enumerate(aggs):
            gv = got[g][i]
            if kind == "any":
                assert (gv is None and w[i] is None) or gv in w[i], (g, kind)
            else:
                assert gv == w[i], (g, kind, gv, w[i])
    assert any(w[0] is None for w in want.values()) or n_keys == 0 or aggset == 1  # groups whose inputs are all NULL
    # the same groups through the exported table: every key and aggregate column read back by a second program
    gt = P.groups_table(gpu_ctx, st)
    outs = [col(f"k{k}") for k in range(n_keys)]
    idx = [i for i in range(len(aggs)) if i not in any_at]
    got2 = {}
    for part in range(0, len(idx), 8 - n_keys):  # <= 8 outputs per materialize; the key columns align the parts
        cols = idx[part:part + 8 - n_keys]
        rows = _materialize(gpu_ctx, gt, outs + [col(f"a{i}") for i in cols])
        for r in zip(*rows):
            got2.setdefault(tuple(r[:n_keys]), []).extend(R.bits_f64(v) if v is not None and j in f64 else v for j, v in zip(cols, r[n_keys:]))
    assert got2 == {g: [w[i] for i in idx] for g, w in want.items()}
    # HAVING over the exported aggregates: a sign test on MIN / MAX, a comparison on the float aggregates
    for i, (kind, _) in enumerate(aggs):
        if kind in ("min", "max"):
            pred = ("cmp", "<", col(f"a{i}"), const(0))
            test = lambda x: x is not None and x < 0
        elif kind in ("sum_f64", "min_f64", "max_f64"):
            pred = ("fcmp", ">", col(f"a{i}"), ("f64", 100.5))
            test = lambda x: x is not None and x > 100.5
        else:
            continue
        kept = _materialize(gpu_ctx, gt, outs[:n_keys] + [col(f"a{i}")], where=pred)
        got_keys = sorted(map(repr, zip(*kept[:n_keys]))) if n_keys else ["()"] * len(kept[0])
        want_keys = sorted(repr(g) for g, w in want.items() if test(w[i])) if n_keys else ["()"] * sum(test(w[i]) for w in want.values())
        assert got_keys == want_keys, (kind, i)
    gt.destroy()
    gpu_ctx.L.ldb_gpu_state_destroy(st)


def test_keyless_aggregate_over_no_rows(gpu_ctx, agg_table):
    tab, _, _ = agg_table
    aggs = [("sum", col("v")), ("count", col("v")), ("count_star", None), ("min", col("v")), ("max", col("w")), ("sum_f64", col("f")),
            ("max_f64", col("f")), ("any", col("w"))]
    st = P.group_by(gpu_ctx, tab, [], aggs, where=("cmp", "=", col("g0"), const(7)))
    assert P.decode_groups(P.read_groups(gpu_ctx, st, 4), 0, 8, f64_aggs=(5, 6)) == {(): [None, 0, 0, None, None, None, None, None]}
    gt = P.groups_table(gpu_ctx, st)
    assert _materialize(gpu_ctx, gt, [col(f"a{i}") for i in range(8)]) == [[None], [0], [0], [None], [None], [None], [None], [None]]
    gt.destroy()
    gpu_ctx.L.ldb_gpu_state_destroy(st)


# ---------------------------------------------------------------------------------------------------- 4. joins
JOIN_COLUMNS = [("k", "int64", 0, 0), ("p", "int64", 0, 0)]


def test_join_build_rejects_keys_and_payloads_outside_int32(gpu_ctx):
    for k, p in (((1 << 32) + 7, 1), (R.I32_MAX + 1, 1), (R.I32_MIN - 1, 2), (7, 1 << 32), (7, R.I32_MIN - 1)):
        src = _stage(gpu_ctx, "bad", {"k": [1, 2, k, None], "p": [1, 2, p, 3]}, columns=JOIN_COLUMNS)
        jt = runtime.join_table(gpu_ctx, 64, unique=False)
        with pytest.raises(capi.LdbRuntimeError) as ex:
            P.build_join(gpu_ctx, src, jt, col("k"), payload=col("p"))
        assert ex.value.code == 2  # LDB_ERR_UNSUPPORTED
        gpu_ctx.L.ldb_gpu_state_destroy(jt)
    # the int32 extremes and a NULL payload are stored (the NULL payload as 0)
    src = _stage(gpu_ctx, "ok", {"k": [R.I32_MIN, R.I32_MAX, -1, 5], "p": [R.I32_MAX, R.I32_MIN, 4, None]}, columns=JOIN_COLUMNS)
    jt = runtime.join_table(gpu_ctx, 64, unique=False)
    P.build_join(gpu_ctx, src, jt, col("k"), payload=col("p"))
    assert runtime.join_count(gpu_ctx, jt) == 4
    got = _materialize(gpu_ctx, src, [col("k"), ("probe", jt, col("k"))])
    assert sorted(zip(*got)) == sorted([(R.I32_MIN, R.I32_MAX), (R.I32_MAX, R.I32_MIN), (-1, 4), (5, 0)])
    gpu_ctx.L.ldb_gpu_state_destroy(jt)


def test_join_build_fails_when_rows_cannot_be_stored(gpu_ctx):
    n = 40_000
    src = _stage(gpu_ctx, "many", {"k": list(range(n)), "p": list(range(n))}, columns=JOIN_COLUMNS)
    jt = runtime.join_table(gpu_ctx, 16, unique=False)  # far smaller than the build side
    with pytest.raises(capi.LdbRuntimeError) as ex:
        P.build_join(gpu_ctx, src, jt, col("k"), payload=col("p"))
    assert ex.value.code == 4  # LDB_ERR_CAPACITY
    gpu_ctx.L.ldb_gpu_state_destroy(jt)
    pair = _stage(gpu_ctx, "pair", {"k": [1, -1], "p": [1, -1]}, columns=JOIN_COLUMNS)  # (key -1, payload -1) is the empty-slot pattern
    jt = runtime.join_table(gpu_ctx, 16, unique=False)
    with pytest.raises(capi.LdbRuntimeError):
        P.build_join(gpu_ctx, pair, jt, col("k"), payload=col("p"))
    gpu_ctx.L.ldb_gpu_state_destroy(jt)


PROBE_KEYS = [-1, R.I32_MIN, R.I32_MAX, 0, 1, 5, 39, 40, -10, -11, (1 << 32) - 1, 1 << 32, R.I32_MAX + 1, R.I32_MIN - 1, None]


@pytest.fixture(scope="module")
def join_tables(gpu_ctx):
    """hashed unique, hashed multimap and direct-address tables over keys that include -1, INT32_MIN and INT32_MAX, and their multimaps"""
    rng = random.Random(9)
    uk = [-1, R.I32_MIN, R.I32_MAX, 0, 5, 40] + rng.sample(range(-10**6, 10**6), 300)
    uk = list(dict.fromkeys(uk))
    up = [rng.randrange(-2**31, 2**31) for _ in uk]
    mk = [rng.choice([-1, R.I32_MIN, R.I32_MAX, 0, 5, 39, 1]) for _ in range(200)] + [None] * 5
    mp = [rng.randrange(-2**31, 2**31) for _ in mk]
    tabs, maps = {}, {}
    for name, keys, pays, unique in (("unique", uk, up, True), ("multi", mk, mp, False)):
        src = _stage(gpu_ctx, name, {"k": keys, "p": pays}, columns=JOIN_COLUMNS, cuts=(3,))
        jt = runtime.join_table(gpu_ctx, len(keys), unique=unique)
        P.build_join(gpu_ctx, src, jt, col("k"), payload=col("p"))
        mm = {}
        for k, p in zip(keys, pays):
            if k is not None:
                mm.setdefault(k, []).append(p)
        tabs[name], maps[jt.value] = jt, mm
    dk = list(range(-10, 41))
    dp = [rng.randrange(0, 2**31 - 1) for _ in dk]
    dtab = runtime.Table(gpu_ctx, "direct_src", [datagen.ColumnSpec("k", "int32"), datagen.ColumnSpec("p", "int32")])
    dtab.append_host({"k": np.array(dk, np.int32), "p": np.array(dp, np.int32)}, len(dk))
    jt = runtime.join_table_direct(gpu_ctx, -10, 40)
    runtime.run_pipeline(gpu_ctx, "scan_build", dtab, build_key="k", build_payload="p", sink=jt)
    tabs["direct"], maps[jt.value] = jt, {k: [p] for k, p in zip(dk, dp)}
    yield tabs, maps
    for jt in tabs.values():
        gpu_ctx.L.ldb_gpu_state_destroy(jt)


@pytest.mark.parametrize("kind", ["unique", "multi", "direct"])
def test_probe_and_probe_each_against_a_multimap(gpu_ctx, join_tables, kind):
    tabs, maps = join_tables
    jt = tabs[kind]
    rng = random.Random(3)
    keys = PROBE_KEYS * 3 + [rng.choice(PROBE_KEYS[:10]) for _ in range(500)]
    probe = _stage(gpu_ctx, "probe", {"k": keys, "p": list(range(len(keys)))}, columns=JOIN_COLUMNS, cuts=(17,))
    ev = R.Evaluator({"k": keys, "p": list(range(len(keys)))}, joins=maps)
    if kind != "multi":  # PROBE's payload is determined only for a key with one match
        _check_programs(gpu_ctx, probe, ev, [("int", ("probe", jt, col("k"))), ("bool", ("isnull", ("probe", jt, col("k"))))], kind)
    for outer in (False, True):
        m = ("probe_each", jt, col("k")) + (("outer",) if outer else ())
        exprs = [("rowid",), m, ("add", m, col("p"))]
        got = _materialize(gpu_ctx, probe, exprs)
        want = ev.run(exprs)[0]
        assert sorted(map(repr, zip(*got))) == sorted(map(repr, zip(*want))), (kind, outer)
        # the same join under a WHERE on the payload
        pred = ("cmp", ">", m, const(0))
        got = _materialize(gpu_ctx, probe, [("rowid",), m], where=pred)
        want = ev.run([("rowid",), m], where=pred)[0]
        assert sorted(map(repr, zip(*got))) == sorted(map(repr, zip(*want))), (kind, outer, "where")


# ---------------------------------------------------------------------------------------------------- 5. ORDER BY
ORDER_COLUMNS = [("i32", "int32", 0, 0), ("i64", "int64", 0, 0), ("dt", "date32", 0, 0), ("dn", "decimal128", 18, 2)]


@pytest.mark.parametrize("n", [0, 1, 4095, 4096, 4097, 3 * 4096 + 1, 1_000_003])
def test_order_by_is_a_stable_sort(gpu_ctx, n):
    rng = np.random.default_rng(n)
    small = rng.integers(-3, 3, n)  # heavy ties
    vals = {"i32": small.astype(np.int32), "i64": np.where(rng.random(n) < 0.5, small, rng.integers(-2**63, 2**63 - 1, n)).astype(np.int64),
            "dt": rng.integers(-800_000, 3_000_000, n).astype(np.int32) // 997 * 997,
            "dn": np.where(rng.random(n) < 0.7, small * 10**17, rng.integers(-10**18 + 1, 10**18, n)).astype(np.int64)}
    dcells = np.zeros((n, 2), np.int64)
    dcells[:, 0], dcells[:, 1] = vals["dn"], vals["dn"] >> 63
    tab = runtime.Table(gpu_ctx, f"ord{n}", R.specs_of(ORDER_COLUMNS))
    tab.append_host({"i32": vals["i32"], "i64": vals["i64"], "dt": vals["dt"], "dn": dcells.view(np.uint8).reshape(n, 16)}, n)
    raw = P.RawTable(gpu_ctx, tab.h)
    for c in vals:
        v = vals[c]
        asc = np.argsort(v, kind="stable")
        desc = np.argsort(~v, kind="stable")  # ~v = -v - 1: reverses the order without overflow
        for descending, order in ((False, asc), (True, desc)):
            for limit in sorted({0, 1, n, n + 5}):
                ids = raw.order_by(c, descending=descending, limit=limit)
                assert ids == order[:limit].tolist(), (c, descending, limit)
