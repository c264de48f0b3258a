"""Join-table markers in program pipelines (LDB_OP_MARK, ldb_gpu_join_table_marks / _clear_marks): reversed semi, anti and mark joins
and right / full outer joins over four build sides (a multimap with duplicate and NULL keys, a unique table, a direct-address table and a
2-key key-tuple multimap, all with ROWID payloads), exact against a plain-Python model on seeded data; the edge cases of the markers'
lifetime; the rejections; and Q21 and Q22 in the reference's reversed shape on the dbgen-faithful SF1 tables, against the reference's
own answers."""
import json
import os
from collections import Counter

import numpy as np
import pytest

from lingodb_b200 import capi, datagen, dbgen, program as P, runtime

pytestmark = pytest.mark.gpu

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_kats.json")))["tpch_sf1"]
NB, NA = 3000, 5000


def _table(ctx, name, cols, valid=None, cuts=()):
    """int32 columns cut into batches at `cuts`, with Arrow validity bitmaps for the columns in `valid`"""
    valid = valid or {}
    td = datagen.TableData(name, [datagen.ColumnSpec(k, "int32") for k in cols])
    n = len(next(iter(cols.values())))
    edges = [0] + list(cuts) + [n]
    for a, b in zip(edges, edges[1:]):
        ch = {k: np.ascontiguousarray(v[a:b]) for k, v in cols.items()}
        for k, v in valid.items():
            ch[k + "$valid"] = np.packbits(v[a:b], bitorder="little")
        td.chunks.append(ch)
        td.chunk_rows.append(b - a)
    return ctx.table_from_host(td)


def _rows(ctx, h, cells):
    """the rows of a library-made table: `cells` = [(column, cell bytes)]"""
    t = P.RawTable(ctx, h) if not isinstance(h, P.RawTable) else h
    ids = list(range(t.num_rows))
    out = list(zip(*[t.gather(c, ids, cell_bytes=w) for c, w in cells])) if ids else []
    t.destroy()
    return out


def _marks(ctx, js, which, n_keys=1):
    names = ["key"] if n_keys == 1 else [f"k{j}" for j in range(n_keys)]
    cells = [(c, 8) for c in names] + [("payload", 8)] + ([("marked", 4)] if which == P.ALL else [])
    return Counter(_rows(ctx, P.join_marks(ctx, js, which), cells))


@pytest.fixture(scope="module")
def sides(gpu_ctx):
    """the build tables, the probe table and the four join tables with their models (entries: (key tuple, build row))"""
    ctx = gpu_ctx
    rng = np.random.default_rng(2024)
    bk = rng.integers(0, 800, NB).astype(np.int32)  # duplicates
    bk2 = rng.integers(0, 3, NB).astype(np.int32)
    bv = rng.integers(0, 4, NB).astype(np.int32)
    bvalid = rng.random(NB) > 0.1
    B = _table(ctx, "b", {"k": bk, "k2": bk2, "v": bv}, {"k": bvalid}, (NB // 3,))
    uk = rng.permutation(3000)[:2000].astype(np.int32)  # unique, no NULLs
    uv = rng.integers(0, 4, 2000).astype(np.int32)
    U = _table(ctx, "u", {"k": uk, "v": uv, "rid": np.arange(2000, dtype=np.int32)})
    ak = rng.integers(0, 1000, NA).astype(np.int32)
    ak2 = rng.integers(0, 3, NA).astype(np.int32)
    av = rng.integers(0, 4, NA).astype(np.int32)
    ac = rng.integers(0, 2, NA).astype(np.int32)
    avalid, cvalid = rng.random(NA) > 0.1, rng.random(NA) > 0.3
    cuts = (NA // 7, NA // 2, NA - NA // 5)
    A = _table(ctx, "a", {"pk": ak, "pk2": ak2, "pv": av, "c": ac}, {"pk": avalid, "c": cvalid}, cuts)
    multi = runtime.join_table(ctx, NB, unique=False)
    P.build_join(ctx, B, multi, col("k"), payload=("rowid",))
    uniq = runtime.join_table(ctx, 2000)
    P.build_join(ctx, U, uniq, col("k"), payload=("rowid",))
    direct = runtime.join_table_direct(ctx, 0, 2999)
    runtime.run_pipeline(ctx, "scan_build", U, build_key="k", build_payload="rid", sink=direct)
    tup = runtime.join_table_keys(ctx, 2, NB, unique=False)
    P.build_join(ctx, B, tup, [col("k"), col("k2")], payload=("rowid",))
    b_entries = [((int(bk[i]),), i) for i in range(NB) if bvalid[i]]
    u_entries = [((int(uk[i]),), i) for i in range(2000)]
    t_entries = [((int(bk[i]), int(bk2[i])), i) for i in range(NB) if bvalid[i]]
    probe = dict(pk=[int(x) if v else None for x, v in zip(ak, avalid)], pk2=ak2.tolist(), pv=av.tolist(), c=[int(x) if v else None for x, v in zip(ac, cvalid)])
    s = {
        "multi": dict(js=multi, src=B, v=bv, entries=b_entries, keys=[col("pk")], n=1, each=True),
        "unique": dict(js=uniq, src=U, v=uv, entries=u_entries, keys=[col("pk")], n=1, each=False),
        "direct": dict(js=direct, src=U, v=uv, entries=u_entries, keys=[col("pk")], n=1, each=False),
        "tuple": dict(js=tup, src=B, v=bv, entries=t_entries, keys=[col("pk"), col("pk2")], n=2, each=True),
    }
    yield dict(sides=s, A=A, probe=probe, B=B, U=U)
    for x in s.values():
        runtime.state_destroy(ctx, x["js"])
    for t in (A, B, U):
        t.clear()


def _pkey(probe, i, n):
    k = (probe["pk"][i],) if n == 1 else (probe["pk"][i], probe["pk2"][i])
    return None if None in k else k


def _model(sd, probe, rows, cond):
    """qualifying (probe row, build row) pairs and the marked entries' build rows"""
    by = {}
    for k, r in sd["entries"]:
        by.setdefault(k, []).append(r)
    pairs, marked = [], set()
    for i in rows:
        k = _pkey(probe, i, sd["n"])
        for r in by.get(k, []) if k else []:
            if cond(i, r):
                pairs.append((i, r))
                marked.add(r)
    return pairs, marked


def _expect(sd, marked, which):
    out = Counter()
    for k, r in sd["entries"]:
        m = r in marked
        if which == P.ALL:
            out[k + (r, int(m))] += 1
        elif m == (which == P.MARKED):
            out[k + (r,)] += 1
    return out


def _probe(sd, outer=False):
    if sd["each"] or outer:
        return ("probe_each", sd["js"], *sd["keys"], *(["outer"] if outer else []))
    return ("probe", sd["js"], *sd["keys"])


@pytest.mark.parametrize("side", ["multi", "unique", "direct", "tuple"])
def test_reversed_semi_anti_and_mark_joins(gpu_ctx, sides, side):
    """the probe side marks the entries it matches under the residual fetch(v) <> pv; the marked entries are the semi join, the unmarked
    ones the anti join, all with their flag the mark join"""
    ctx, sd, probe = gpu_ctx, sides["sides"][side], sides["probe"]
    js = sd["js"]
    P.clear_marks(ctx, js)
    m = _probe(sd)
    residual = ("cmp", "!=", ("fetch", sd["src"], m, "v"), col("pv"))
    P.run_effects(ctx, sides["A"], [("mark", m, residual)])
    _, marked = _model(sd, probe, range(NA), lambda i, r: int(sd["v"][r]) != probe["pv"][i])
    assert marked and len(marked) < len(sd["entries"])
    for which in (P.MARKED, P.UNMARKED, P.ALL):
        assert _marks(ctx, js, which, sd["n"]) == _expect(sd, marked, which), which


@pytest.mark.parametrize("side", ["multi", "unique", "direct", "tuple"])
def test_right_and_full_outer_joins(gpu_ctx, sides, side):
    """right outer: the inner PROBE_EACH pairs under the residual, each marking its entry, then the unmarked entries with a NULL probe
    row.  Full outer: a left-outer PROBE_EACH marking every match, then the unmarked entries."""
    ctx, sd, probe = gpu_ctx, sides["sides"][side], sides["probe"]
    js = sd["js"]
    # ---- right outer
    P.clear_marks(ctx, js)
    m = ("probe_each", js, *sd["keys"])
    residual = ("cmp", "!=", ("fetch", sd["src"], m, "v"), col("pv"))
    got = Counter(_rows(ctx, P.materialize(ctx, sides["A"], [("rowid",), m], where=("mark", m, residual)), [("c0", 16), ("c1", 16)]))
    for row in _marks(ctx, js, P.UNMARKED, sd["n"]).elements():
        got[(None, row[-1])] += 1
    pairs, marked = _model(sd, probe, range(NA), lambda i, r: int(sd["v"][r]) != probe["pv"][i])
    want = Counter(pairs) + Counter((None, r) for _, r in sd["entries"] if r not in marked)
    assert got == want
    # ---- full outer
    P.clear_marks(ctx, js)
    mo = ("probe_each", js, *sd["keys"], "outer")
    got = Counter((i, r) for i, r, _ in _rows(ctx, P.materialize(ctx, sides["A"], [("rowid",), mo, ("mark", mo, const(1))]), [("c0", 16), ("c1", 16), ("c2", 16)]))
    for row in _marks(ctx, js, P.UNMARKED, sd["n"]).elements():
        got[(None, row[-1])] += 1
    pairs, marked = _model(sd, probe, range(NA), lambda i, r: True)
    matched = {i for i, _ in pairs}
    want = Counter(pairs) + Counter((i, None) for i in range(NA) if i not in matched) + Counter((None, r) for _, r in sd["entries"] if r not in marked)
    assert got == want


def test_mark_values_null_and_false_conditions(gpu_ctx, sides):
    """dst is TRUE exactly when the condition is TRUE and the probe matched, never NULL; a NULL or FALSE condition marks nothing"""
    ctx, sd, probe = gpu_ctx, sides["sides"]["multi"], sides["probe"]
    js = sd["js"]
    P.clear_marks(ctx, js)
    m = ("probe_each", js, col("pk"), "outer")
    cond = ("cmp", "=", col("c"), const(1))
    rows = _rows(ctx, P.materialize(ctx, sides["A"], [("rowid",), m, ("mark", m, cond)]), [("c0", 16), ("c1", 16), ("c2", 16)])
    assert all(x in (0, 1) for _, _, x in rows)
    assert Counter((i, r) for i, r, x in rows if x) == Counter(_model(sd, probe, range(NA), lambda i, r: probe["c"][i] == 1)[0])
    _, marked = _model(sd, probe, range(NA), lambda i, r: probe["c"][i] == 1)
    assert _marks(ctx, js, P.ALL) == _expect(sd, marked, P.ALL)


def test_marks_accumulate_clear_and_later_inserts(gpu_ctx, sides):
    """two probe programs accumulate; clear_marks unmarks all; an empty probe side and a never-marked table mark nothing; entries
    inserted after marking come back unmarked while the earlier marks stay"""
    ctx, probe = gpu_ctx, sides["probe"]
    sd = sides["sides"]["unique"]
    js = sd["js"]
    P.clear_marks(ctx, js)
    half = NA // 2
    pk = np.array([x if x is not None else 0 for x in probe["pk"]], np.int32)
    pv = np.array([x is not None for x in probe["pk"]])
    A1 = _table(ctx, "a1", {"pk": pk[:half]}, {"pk": pv[:half]})
    A2 = _table(ctx, "a2", {"pk": pk[half:]}, {"pk": pv[half:]}, (100,))
    for t in (A1, A2):
        P.run_effects(ctx, t, [("mark", ("probe", js, col("pk")), const(1))])
    _, marked = _model(sd, probe, range(NA), lambda i, r: True)
    assert _marks(ctx, js, P.ALL) == _expect(sd, marked, P.ALL)
    P.clear_marks(ctx, js)
    assert _marks(ctx, js, P.MARKED) == Counter()
    assert _marks(ctx, js, P.UNMARKED) == _expect(sd, set(), P.UNMARKED)
    E = _table(ctx, "empty", {"pk": np.zeros(0, np.int32)})
    P.run_effects(ctx, E, [("mark", ("probe", js, col("pk")), const(1))])
    assert _marks(ctx, js, P.ALL) == _expect(sd, set(), P.ALL)
    # never marked: no markers at all
    fresh = runtime.join_table(ctx, 4000, unique=False)
    P.build_join(ctx, sides["U"], fresh, col("k"), payload=("rowid",))
    assert _marks(ctx, fresh, P.ALL) == _expect(sd, set(), P.ALL)
    P.clear_marks(ctx, fresh)
    # marked, then more rows inserted
    P.run_effects(ctx, A1, [("mark", ("probe", fresh, col("pk")), const(1))])
    _, marked = _model(sd, probe, range(half), lambda i, r: True)
    P.build_join(ctx, sides["U"], fresh, ("add", col("k"), const(5000)), payload=("add", ("rowid",), const(2000)))
    want = _expect(sd, marked, P.ALL) + Counter((k + 5000, r + 2000, 0) for (k,), r in sd["entries"])
    assert _marks(ctx, fresh, P.ALL) == want
    runtime.state_destroy(ctx, fresh)
    for t in (A1, A2, E):
        t.clear()


def _raises(code, fn, text):
    with pytest.raises(capi.LdbRuntimeError) as ei:
        fn()
    assert ei.value.code == code and text in str(ei.value), str(ei.value)


def test_rejections(gpu_ctx, sides):
    ctx = gpu_ctx
    B = sides["B"]
    INV, UNS = capi.LDB_ERR_INVALID, capi.LDB_ERR_UNSUPPORTED
    own = runtime.join_table(ctx, NB, unique=False)
    _raises(INV, lambda: P.build_join(ctx, B, own, col("k"), where=("mark", ("probe", own, col("k")), const(1))), "may not mark the join table it builds")
    pair = runtime.join_table_pair(ctx, 64)
    gj = runtime.join_table(ctx, 64, n_side=1)
    for js in (pair, gj):
        _raises(INV, lambda: P.run_effects(ctx, B, [("mark", ("probe", js, col("k")), const(1))]), "MARK takes a plain single-key")
        _raises(INV, lambda: P.join_marks(ctx, js, P.ALL), "not pair tables or group-join maps")
        _raises(INV, lambda: P.clear_marks(ctx, js), "not pair tables or group-join maps")
    _raises(INV, lambda: P.join_marks(ctx, own, 2), "which is 1")
    # a MARK whose table no earlier probe reads
    b = P.Builder()
    b.expr(const(1))
    b.tables.append(own)
    b.instr.append((P.OPS["mark"], b._reg(), 0, 0, 0))
    d, keep = P._desc(ctx, B, b, -1)
    d.sink_kind = P.SINK_NONE
    _raises(INV, lambda: P._run(ctx, d, b), "no earlier PROBE / PROBE_EACH")
    b2 = P.Builder()
    b2.expr(const(1))
    d2, keep2 = P._desc(ctx, B, b2, -1)
    d2.sink_kind, d2.sink = P.SINK_NONE, own
    _raises(INV, lambda: P._run(ctx, d2, b2), "LDB_SINK_NONE takes no sink state")
    ctx.graph_begin()
    try:
        _raises(UNS, lambda: P.run_effects(ctx, B, [("mark", ("probe", sides["sides"]["multi"]["js"], col("k")), const(1))]), "not part of captured queries")
        _raises(UNS, lambda: P.join_marks(ctx, own, P.ALL), "not part of captured queries")
    finally:
        ctx.graph_end().destroy()
    for js in (own, pair, gj):
        runtime.state_destroy(ctx, js)


# ---------------------------------------------------------------- Q21 and Q22 on the SF1 tables, reversed as the reference lowers them
def _dec(v: int, scale: int) -> str:
    s = "-" if v < 0 else ""
    v = abs(v)
    return f"{s}{v // 10**scale}.{v % 10**scale:0{scale}d}"


@pytest.fixture(scope="module")
def sf1(gpu_ctx):
    t = dbgen.tpch(1.0, extended=True, attributes=True)
    tabs = {k: gpu_ctx.table_from_host(t[k]) for k in ("lineitem", "orders", "supplier")}
    cat = lambda n, k: np.concatenate([c[k] for c in t[n].chunks])
    cu = datagen.TableData("customer22", [datagen.ColumnSpec("c_custkey", "int32"), datagen.ColumnSpec("c_nationkey", "int32"),
                                          datagen.ColumnSpec("c_acctbal", "decimal128", 12, 2)])
    cu.chunks.append({"c_custkey": cat("customer", "c_custkey"), "c_nationkey": cat("customer", "c_nationkey"),
                      "c_acctbal": dbgen._dec128(dbgen.balances_and_quantities(1.0)["c_acctbal"])})
    cu.chunk_rows.append(len(cu.chunks[0]["c_custkey"]))
    tabs["customer"] = gpu_ctx.table_from_host(cu)
    yield tabs
    for x in tabs.values():
        x.clear()


def test_q21_reversed_exists_and_not_exists(gpu_ctx, sf1):
    """F orders: the unmarked entries of an orders table probed by the lines whose l_linestatus <> 'F'.  The l1 candidates (late lines of
    Saudi suppliers in F orders) form a row-id multimap; EXISTS l2 keeps its entries marked by a line of another supplier; NOT EXISTS l3
    keeps the entries of a second multimap built from those that no late line of another supplier marks."""
    ctx, t = gpu_ctx, sf1
    li = t["lineitem"]
    names = [n for n, _ in datagen.NATIONS]
    notnull = lambda e: ("not", ("isnull", e))
    late = ("cmp", ">", col("l_receiptdate"), col("l_commitdate"))
    states, tables = [], []

    def table(expected, unique=True):
        states.append(runtime.join_table(ctx, expected, unique=unique))
        return states[-1]

    orders = table(1_600_000)
    P.build_join(ctx, t["orders"], orders, col("o_orderkey"), payload=("rowid",))
    P.run_effects(ctx, li, [("mark", ("probe", orders, col("l_orderkey")), ("cmp", "!=", col("l_linestatus"), const(ord("F"))))])
    f_orders = P.join_marks(ctx, orders, P.UNMARKED)
    tables.append(f_orders)
    f_set = table(f_orders.num_rows)
    P.build_join(ctx, f_orders, f_set, col("key"))
    saudi = table(4096)
    P.build_join(ctx, t["supplier"], saudi, col("s_suppkey"), where=("cmp", "=", col("s_nationkey"), const(names.index("SAUDI ARABIA"))))
    l1 = table(400_000, unique=False)
    P.build_join(ctx, li, l1, col("l_orderkey"), payload=("rowid",),
                 where=("and", late, ("and", notnull(("probe", saudi, col("l_suppkey"))), notnull(("probe", f_set, col("l_orderkey"))))))
    e2 = ("probe_each", l1, col("l_orderkey"))
    P.run_effects(ctx, li, [("mark", e2, ("cmp", "!=", col("l_suppkey"), ("fetch", li, e2, "l_suppkey")))])
    exists = P.join_marks(ctx, l1, P.MARKED)
    tables.append(exists)
    l1b = table(max(exists.num_rows, 1), unique=False)
    P.build_join(ctx, exists, l1b, col("key"), payload=col("payload"))
    e3 = ("probe_each", l1b, col("l_orderkey"))
    P.run_effects(ctx, li, [("mark", e3, ("and", late, ("cmp", "!=", col("l_suppkey"), ("fetch", li, e3, "l_suppkey"))))])
    wait = P.join_marks(ctx, l1b, P.UNMARKED)
    tables.append(wait)
    st = P.group_by(ctx, wait, [("fetch", li, col("payload"), "l_suppkey")], [("count_star", None)], expected_groups=4096)
    states.append(st)
    got = P.decode_groups(P.read_groups(ctx, st, 4096), 1, 1)
    top = sorted((("Supplier#%09d" % k, v[0]) for (k,), v in got.items()), key=lambda kv: (-kv[1], kv[0]))[:100]
    assert [[n, str(v)] for n, v in top] == GOLD["q21_rows"]
    for x in tables:
        x.destroy()
    for s_ in states:
        runtime.state_destroy(ctx, s_)


def test_q22_reversed_not_exists(gpu_ctx, sf1):
    """the keyless average balance of the listed country codes (code = 10 + nation in the generator), the customers above it as the build
    side, marked by every order's o_custkey; the unmarked ones grouped by country code"""
    ctx, t = gpu_ctx, sf1
    cu = t["customer"]
    codes = [13, 31, 23, 29, 30, 18, 17]
    code = ("add", col("c_nationkey"), const(10))
    listed = ("cmp", "=", code, const(codes[0]))
    for c in codes[1:]:
        listed = ("or", listed, ("cmp", "=", code, const(c)))
    st = P.group_by(ctx, cu, [], [("sum", col("c_acctbal")), ("count_star", None)], where=("and", listed, ("cmp", ">", col("c_acctbal"), const(0))))
    total, n = P.decode_groups(P.read_groups(ctx, st, 4), 0, 2)[()]
    runtime.state_destroy(ctx, st)
    rich = runtime.join_table(ctx, 160_000)
    P.build_join(ctx, cu, rich, col("c_custkey"), payload=("rowid",), where=("and", listed, ("cmp", ">", ("mul", col("c_acctbal"), const(n)), const(total))))
    P.run_effects(ctx, t["orders"], [("mark", ("probe", rich, col("o_custkey")), const(1))])
    no_orders = P.join_marks(ctx, rich, P.UNMARKED)
    row = col("payload")
    st = P.group_by(ctx, no_orders, [("add", ("fetch", cu, row, "c_nationkey"), const(10))], [("count_star", None), ("sum", ("fetch", cu, row, "c_acctbal"))], expected_groups=64)
    got = P.decode_groups(P.read_groups(ctx, st, 64), 1, 2)
    runtime.state_destroy(ctx, st)
    no_orders.destroy()
    runtime.state_destroy(ctx, rich)
    assert [[str(c), str(v[0]), _dec(v[1], 2)] for (c,), v in sorted(got.items())] == GOLD["q22_rows"]
