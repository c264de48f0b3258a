"""Q2, Q8, Q11, Q14, Q17, Q19 and Q20 as program pipelines on the dbgen-faithful SF1 tables with their attribute columns, against the
reference's own answers (tests/golden/reference_kats.json, the rows test_reference_answers_sf1.py reproduces in numpy), formatted the
same way.  Build-side attributes are read as side columns through ROWID joins; ratios are computed on the host from the device's exact
sums and truncated to six decimals as the reference prints them."""
import datetime
import json
import os
from fractions import Fraction

import pytest

from lingodb_b200 import datagen, dbgen, program as P, runtime

pytestmark = pytest.mark.gpu

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_kats.json")))["tpch_sf1"]
NAMES = [n for n, _ in datagen.NATIONS]
col, const = (lambda n: ("col", n)), (lambda v: ("const", v))
REV = ("mul", col("l_extendedprice"), ("sub", const(100), col("l_discount")))


def dec(v: int, scale: int) -> str:
    s = "-" if v < 0 else ""
    v = abs(v)
    return f"{s}{v // 10**scale}.{v % 10**scale:0{scale}d}"


def trunc6(f: Fraction) -> str:
    return dec(int(f * 10**6), 6)


def day(s: str) -> int:
    return (datetime.date.fromisoformat(s) - datetime.date(1970, 1, 1)).days


def in_region(r: str):
    return [i for i, (_, reg) in enumerate(datagen.NATIONS) if reg == datagen.REGIONS.index(r)]


def any_of(e, values):
    out = ("cmp", "=", e, const(values[0]))
    for v in values[1:]:
        out = ("or", out, ("cmp", "=", e, const(v)))
    return out


def notnull(e):
    return ("not", ("isnull", e))


@pytest.fixture(scope="module")
def db(gpu_ctx):
    t = dbgen.tpch(1.0, extended=True, attributes=True)
    tabs = {k: gpu_ctx.table_from_host(t[k]) for k in ("lineitem", "orders", "customer", "supplier", "part", "partsupp")}
    assert len(t["orders"].chunks) > 1  # Q8 reads orders columns across batches
    states = []

    def table(expected, unique=True):
        states.append(runtime.join_table(gpu_ctx, expected, unique=unique))
        return states[-1]

    def rowids(source, key, expected, where=None, unique=True):
        """join table key → row id of `source` (the side-column row of that table)"""
        jt = table(expected, unique)
        P.build_join(gpu_ctx, tabs[source] if isinstance(source, str) else source, jt, col(key), payload=("rowid",), where=where)
        return jt

    tabs["part_rows"] = rowids("part", "p_partkey", 210_000)
    yield dict(t=tabs, table=table, rowids=rowids, states=states)
    for s_ in states:
        gpu_ctx.L.ldb_gpu_state_destroy(s_)


def _one(ctx, table, aggs, where):
    st = P.group_by(ctx, table, [], aggs, where=where)
    got = P.decode_groups(P.read_groups(ctx, st, 4), 0, len(aggs))[()]
    ctx.L.ldb_gpu_state_destroy(st)
    return got


def test_q14_q17_q19(gpu_ctx, db):
    """Q14: CASE on LIKE 'PROMO%' over the fetched p_type.  Q17: per-part sum and count of l_quantity as an exported group table, read
    back through a unique row-id join (two values of one group row).  Q19: the part-side conjunctions of the three branches build one
    row-id join table; the residual OR checks the fetched p_brand with each branch's quantity range."""
    t, pa = db["t"], db["t"]["part"]
    li = t["lineitem"]
    prow = ("probe", t["part_rows"], col("l_partkey"))
    # ---- Q14
    promo = ("like", "prefix", ("fetch", pa, prow, "p_type"), "PROMO")
    total, promo_rev = _one(gpu_ctx, li, [("sum", REV), ("sum", ("case", promo, REV, const(0)))],
                            ("and", ("cmp", ">=", col("l_shipdate"), const(day("1995-09-01"))), ("cmp", "<", col("l_shipdate"), const(day("1995-10-01")))))
    assert [[trunc6(Fraction(100 * promo_rev, total))]] == GOLD["q14_rows"]
    # ---- Q17
    med23 = ("and", ("strcmp", "=", ("fetch", pa, prow, "p_brand"), "Brand#23"), ("strcmp", "=", ("fetch", pa, prow, "p_container"), "MED BOX"))
    st = P.group_by(gpu_ctx, li, [col("l_partkey")], [("sum", col("l_quantity")), ("count_star", None)], where=med23, expected_groups=1024)
    per_part = P.groups_table(gpu_ctx, st)
    db["states"].append(st)
    g = ("probe", db["rowids"](per_part, "k0", 1024), col("l_partkey"))
    small = ("cmp", "<", ("mul", ("mul", const(5), col("l_quantity")), ("fetch", per_part, g, "a1")), ("fetch", per_part, g, "a0"))
    (s17,) = _one(gpu_ctx, li, [("sum", col("l_extendedprice"))], ("and", notnull(g), small))
    assert [[trunc6(Fraction(s17, 700))]] == GOLD["q17_rows"]
    per_part.destroy()
    # ---- Q19
    branches = ((12, ("SM CASE", "SM BOX", "SM PACK", "SM PKG"), 1, 5), (23, ("MED BAG", "MED BOX", "MED PKG", "MED PACK"), 10, 10),
                (34, ("LG CASE", "LG BOX", "LG PACK", "LG PKG"), 20, 15))
    parts19 = db["table"](4096)
    for brand, containers, _, size_max in branches:
        cont = ("strcmp", "=", "p_container", containers[0])
        for c in containers[1:]:
            cont = ("or", cont, ("strcmp", "=", "p_container", c))
        P.build_join(gpu_ctx, pa, parts19, col("p_partkey"), payload=("rowid",),
                     where=("and", ("and", ("strcmp", "=", "p_brand", "Brand#%d" % brand), cont), ("between", col("p_size"), const(1), const(size_max))))
    r19 = ("probe", parts19, col("l_partkey"))
    residual = None
    for brand, _, q_lo, _ in branches:
        b = ("and", ("strcmp", "=", ("fetch", pa, r19, "p_brand"), "Brand#%d" % brand), ("between", col("l_quantity"), const(100 * q_lo), const(100 * (q_lo + 10))))
        residual = b if residual is None else ("or", residual, b)
    where = ("and", ("and", ("or", ("strcmp", "=", "l_shipmode", "AIR"), ("strcmp", "=", "l_shipmode", "AIR REG")), ("strcmp", "=", "l_shipinstruct", "DELIVER IN PERSON")),
             ("and", notnull(r19), residual))
    (s19,) = _one(gpu_ctx, li, [("sum", REV)], where)
    assert [[dec(s19, 4)]] == GOLD["q19_rows"]


def test_q8(gpu_ctx, db):
    """Market share per year: o_orderdate and o_custkey fetched from the multi-batch orders table, c_nationkey through a row-id join
    keyed by the fetched o_custkey, the string predicate on the fetched p_type."""
    t = db["t"]
    orow = ("probe", db["rowids"]("orders", "o_orderkey", 1_600_000), col("l_orderkey"))
    crow = ("probe", db["rowids"]("customer", "c_custkey", 160_000), ("fetch", t["orders"], orow, "o_custkey"))
    srow = ("probe", db["rowids"]("supplier", "s_suppkey", 16_000), col("l_suppkey"))
    odate = ("fetch", t["orders"], orow, "o_orderdate")
    steel = ("strcmp", "=", ("fetch", t["part"], ("probe", t["part_rows"], col("l_partkey")), "p_type"), "ECONOMY ANODIZED STEEL")
    where = ("and", steel, ("and", ("between", odate, const(day("1995-01-01")), const(day("1996-12-31"))), any_of(("fetch", t["customer"], crow, "c_nationkey"), in_region("AMERICA"))))
    brazil = ("cmp", "=", ("fetch", t["supplier"], srow, "s_nationkey"), const(NAMES.index("BRAZIL")))
    st = P.group_by(gpu_ctx, t["lineitem"], [("year", odate)], [("sum", REV), ("sum", ("case", brazil, REV, const(0)))], where=where, expected_groups=16)
    got = P.decode_groups(P.read_groups(gpu_ctx, st, 16), 1, 2)
    gpu_ctx.L.ldb_gpu_state_destroy(st)
    assert sorted(got) == [(1995,), (1996,)]
    assert [[str(y), trunc6(Fraction(got[(y,)][1], got[(y,)][0]))] for y in (1995, 1996)] == GOLD["q8_rows"]


def test_q2_and_q11(gpu_ctx, db):
    """Q2: the per-part minimum cost over European suppliers as an exported group table, fetched back through a unique row-id join to
    pick the cheapest partsupp rows; s_acctbal, s_nationkey and p_mfgr are side columns.  Q11: HAVING against a keyless total."""
    t = db["t"]
    ps, su, pa = t["partsupp"], t["supplier"], t["part"]
    # ---- Q2
    eu = db["rowids"]("supplier", "s_suppkey", 16_000, where=any_of(col("s_nationkey"), in_region("EUROPE")))
    srow = ("probe", eu, col("ps_suppkey"))
    prow = ("probe", t["part_rows"], col("ps_partkey"))
    brass15 = ("and", ("cmp", "=", ("fetch", pa, prow, "p_size"), const(15)), ("like", "suffix", ("fetch", pa, prow, "p_type"), "BRASS"))
    st = P.group_by(gpu_ctx, ps, [col("ps_partkey")], [("min", col("ps_supplycost"))], where=("and", notnull(srow), brass15), expected_groups=8192)
    mincost = P.groups_table(gpu_ctx, st)
    db["states"].append(st)
    g = ("probe", db["rowids"](mincost, "k0", 8192), col("ps_partkey"))
    mfgr = const(0)
    for m in range(5, 0, -1):
        mfgr = ("case", ("strcmp", "=", ("fetch", pa, prow, "p_mfgr"), "Manufacturer#%d" % m), const(m), mfgr)
    where = ("and", ("and", notnull(g), notnull(srow)), ("cmp", "=", col("ps_supplycost"), ("fetch", mincost, g, "a0")))
    mt = P.RawTable(gpu_ctx, P.materialize(gpu_ctx, ps, [("fetch", su, srow, "s_acctbal"), ("fetch", su, srow, "s_nationkey"), col("ps_suppkey"), col("ps_partkey"), mfgr], where=where))
    ids = list(range(mt.num_rows))
    bal, nat, supp, part, mf = (mt.gather(f"c{i}", ids) for i in range(5))
    rows = sorted((-b, NAMES[n], "Supplier#%09d" % s_, p, f) for b, n, s_, p, f in zip(bal, nat, supp, part, mf))[:100]
    assert [[dec(-b, 2), sn, nn, str(p), "Manufacturer#%d" % f] for b, nn, sn, p, f in rows] == GOLD["q2_rows"]
    mt.destroy()
    mincost.destroy()
    # ---- Q11
    german = db["table"](16_000)
    P.build_join(gpu_ctx, su, german, col("s_suppkey"), where=("cmp", "=", col("s_nationkey"), const(NAMES.index("GERMANY"))))
    value, w = ("mul", col("ps_supplycost"), col("ps_availqty")), notnull(("probe", german, col("ps_suppkey")))
    (total,) = _one(gpu_ctx, ps, [("sum", value)], w)
    st = P.group_by(gpu_ctx, ps, [col("ps_partkey")], [("sum", value)], where=w, expected_groups=65_536)
    per_part = P.groups_table(gpu_ctx, st)
    db["states"].append(st)
    hv = P.RawTable(gpu_ctx, P.materialize(gpu_ctx, per_part, [col("k0"), col("a0")], where=("cmp", ">", ("mul", col("a0"), const(10_000)), const(total))))
    ids = list(range(hv.num_rows))
    rows = sorted(zip(hv.gather("c0", ids), hv.gather("c1", ids)), key=lambda kv: (-kv[1], kv[0]))
    assert [[str(k), dec(v, 2)] for k, v in rows] == GOLD["q11_rows"]
    hv.destroy()
    per_part.destroy()


def test_q20(gpu_ctx, db):
    """1994 lineitem groups keyed by (l_partkey, l_suppkey) in a non-unique join table keyed by the part alone; PROBE_EACH by ps_partkey
    walks a part's groups, and the residual predicate on the fetched k1 / a0 keeps the group of the row's own supplier whose half-sum
    is below ps_availqty."""
    t = db["t"]
    ps = t["partsupp"]
    st = P.group_by(gpu_ctx, t["lineitem"], [col("l_partkey"), col("l_suppkey")], [("sum", col("l_quantity"))],
                    where=("and", ("cmp", ">=", col("l_shipdate"), const(day("1994-01-01"))), ("cmp", "<", col("l_shipdate"), const(day("1995-01-01")))),
                    expected_groups=1_000_000)
    pairs = P.groups_table(gpu_ctx, st)
    db["states"].append(st)
    m = ("probe_each", db["rowids"](pairs, "k0", pairs.num_rows, unique=False), col("ps_partkey"))
    forest = db["table"](210_000)
    P.build_join(gpu_ctx, t["part"], forest, col("p_partkey"), where=("like", "prefix", "p_name", "forest"))
    canada = db["table"](16_000)
    P.build_join(gpu_ctx, t["supplier"], canada, col("s_suppkey"), where=("cmp", "=", col("s_nationkey"), const(NAMES.index("CANADA"))))
    where = ("and", ("and", notnull(("probe", forest, col("ps_partkey"))), notnull(("probe", canada, col("ps_suppkey")))),
             ("and", ("cmp", "=", ("fetch", pairs, m, "k1"), col("ps_suppkey")), ("cmp", ">", ("mul", col("ps_availqty"), const(200)), ("fetch", pairs, m, "a0"))))
    st = P.group_by(gpu_ctx, ps, [col("ps_suppkey")], [("count_star", None)], where=where, expected_groups=4096)
    got = P.decode_groups(P.read_groups(gpu_ctx, st, 4096), 1, 1)
    gpu_ctx.L.ldb_gpu_state_destroy(st)
    assert [["Supplier#%09d" % k] for (k,) in sorted(got)] == GOLD["q20_rows"]
    pairs.destroy()
