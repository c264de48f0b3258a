"""Multi-column equi-joins through key-tuple join tables, against the reference's own answers (tests/golden/reference_kats.json) on the
dbgen-faithful SF1 tables with their attribute columns: Q20 probes the exported (part, supplier) groups with the partsupp row's own
(ps_partkey, ps_suppkey), and Q9 runs as a program — (l_partkey, l_suppkey) probes a key-tuple table whose payload is ps_supplycost."""
import datetime
import json
import os

import pytest

from lingodb_b200 import datagen, dbgen, program as P, runtime

pytestmark = pytest.mark.gpu

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_kats.json")))["tpch_sf1"]
NAMES = [n for n, _ in datagen.NATIONS]
col, const = (lambda n: ("col", n)), (lambda v: ("const", v))


def dec(v: int, scale: int) -> str:
    s = "-" if v < 0 else ""
    v = abs(v)
    return f"{s}{v // 10**scale}.{v % 10**scale:0{scale}d}"


def day(s: str) -> int:
    return (datetime.date.fromisoformat(s) - datetime.date(1970, 1, 1)).days


def notnull(e):
    return ("not", ("isnull", e))


@pytest.fixture(scope="module")
def db(gpu_ctx):
    t = dbgen.tpch(1.0, extended=True, attributes=True)
    tabs = {k: gpu_ctx.table_from_host(t[k]) for k in ("lineitem", "orders", "supplier", "part", "partsupp")}
    states = []
    yield dict(t=tabs, states=states)
    for s in states:
        runtime.state_destroy(gpu_ctx, s)


def test_q20_with_a_composite_probe(gpu_ctx, db):
    """1994 lineitem groups keyed by (l_partkey, l_suppkey), exported, then keyed by both columns in a unique key-tuple table of row ids:
    each partsupp row probes its own (ps_partkey, ps_suppkey) — no residual supplier predicate."""
    ctx, t = gpu_ctx, db["t"]
    ps = t["partsupp"]
    st = P.group_by(ctx, t["lineitem"], [col("l_partkey"), col("l_suppkey")], [("sum", col("l_quantity"))],
                    where=("and", ("cmp", ">=", col("l_shipdate"), const(day("1994-01-01"))), ("cmp", "<", col("l_shipdate"), const(day("1995-01-01")))),
                    expected_groups=1_000_000)
    db["states"].append(st)
    pairs = P.groups_table(ctx, st)
    kt = runtime.join_table_keys(ctx, 2, pairs.num_rows)
    db["states"].append(kt)
    P.build_join(ctx, pairs, kt, [col("k0"), col("k1")], payload=("rowid",))
    assert runtime.join_count(ctx, kt) == pairs.num_rows
    forest = runtime.join_table(ctx, 210_000)
    db["states"].append(forest)
    P.build_join(ctx, t["part"], forest, col("p_partkey"), where=("like", "prefix", "p_name", "forest"))
    canada = runtime.join_table(ctx, 16_000)
    db["states"].append(canada)
    P.build_join(ctx, t["supplier"], canada, col("s_suppkey"), where=("cmp", "=", col("s_nationkey"), const(NAMES.index("CANADA"))))
    g = ("probe", kt, col("ps_partkey"), col("ps_suppkey"))
    where = ("and", ("and", notnull(("probe", forest, col("ps_partkey"))), notnull(("probe", canada, col("ps_suppkey")))),
             ("and", notnull(g), ("cmp", ">", ("mul", col("ps_availqty"), const(200)), ("fetch", pairs, g, "a0"))))
    st = P.group_by(ctx, ps, [col("ps_suppkey")], [("count_star", None)], where=where, expected_groups=4096)
    got = P.decode_groups(P.read_groups(ctx, st, 4096), 1, 1)
    runtime.state_destroy(ctx, st)
    pairs.destroy()
    assert [["Supplier#%09d" % k] for (k,) in sorted(got)] == GOLD["q20_rows"]


def q9_program(ctx, t, states):
    """Q9 as program pipelines: p_name LIKE '%green%' as a part semi-join; the green parts' partsupp rows in a key-tuple table
    (ps_partkey, ps_suppkey) → ps_supplycost; o_orderdate and s_nationkey fetched through row-id joins.  Returns {(nation, year): sum}."""
    def keep(s):
        states.append(s)
        return s

    green = keep(runtime.join_table(ctx, 210_000))
    P.build_join(ctx, t["part"], green, col("p_partkey"), where=("like", "contains", "p_name", "green"))
    is_green = lambda k: notnull(("probe", green, col(k)))
    cost = keep(runtime.join_table_keys(ctx, 2, 800_000))
    P.build_join(ctx, t["partsupp"], cost, [col("ps_partkey"), col("ps_suppkey")], payload=col("ps_supplycost"), where=is_green("ps_partkey"))
    orows = keep(runtime.join_table(ctx, 1_500_000))
    P.build_join(ctx, t["orders"], orows, col("o_orderkey"), payload=("rowid",))
    srows = keep(runtime.join_table(ctx, 10_000))
    P.build_join(ctx, t["supplier"], srows, col("s_suppkey"), payload=("rowid",))
    c = ("probe", cost, col("l_partkey"), col("l_suppkey"))
    amount = ("sub", ("mul", col("l_extendedprice"), ("sub", const(100), col("l_discount"))), ("mul", c, col("l_quantity")))
    year = ("year", ("fetch", t["orders"], ("probe", orows, col("l_orderkey")), "o_orderdate"))
    nation = ("fetch", t["supplier"], ("probe", srows, col("l_suppkey")), "s_nationkey")
    st = keep(P.group_by(ctx, t["lineitem"], [nation, year], [("sum", amount)], where=("and", is_green("l_partkey"), notnull(c)), expected_groups=256))
    return {k: v[0] for k, v in P.decode_groups(P.read_groups(ctx, st, 256), 2, 1).items()}


def test_q9_as_a_program(gpu_ctx, db):
    got = q9_program(gpu_ctx, db["t"], db["states"])
    rows = sorted(((NAMES[n], y, v) for (n, y), v in got.items()), key=lambda r: (r[0], -r[1]))
    assert len(rows) == 175
    assert [[n, str(y), dec(v, 4)] for n, y, v in rows] == GOLD["q9_rows"]
