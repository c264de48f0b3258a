"""Program join build and probe times: the plain int32 join table against key-tuple join tables (LDB_STATE_KEY_JOIN), and Q9 as a
program against the specialised ldb_tpch_q9.

  python tools/keyjoin_sweep.py [--build-rows 16M] [--probe-rows 128M] [--sf 10] [--reps 5] [--out result.json]

1. Build side: `build-rows` distinct keys k (a permutation of 0..n-1, int32); probe side: `probe-rows` keys uniform in 0..2n-1 (half
   hit).  Three tables over the same keys: the plain int32 table (key k), a 1-key tuple table (key k) and a 2-key tuple table
   (k >> 12, k & 4095: correlated components), each with a row-id payload.  The build is one JOIN_BUILD program into a fresh table;
   the probe is one program that probes every row and keeps none (WHERE payload = -1), so its sink costs nothing.  The match
   counts are checked once outside the timings.
2. Q9 at scale factor `sf` (datagen tables with parts): the program (a part semi-join on '%green%', a (ps_partkey, ps_suppkey) key-tuple
   table with ps_supplycost payloads, row-id joins for o_orderdate and s_nationkey, a two-key hash aggregation), builds included, against
   ldb_tpch_q9; both results must agree.
The cases alternate within each repetition; every number is the median of `reps` runs timed with CUDA events on the context's compute
stream, reported with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lingodb_b200 import datagen, program as P, runtime  # noqa: E402
from lingodb_b200.datagen import ColumnSpec, TableData  # noqa: E402

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def rows_arg(s):
    s = s.upper()
    return int(float(s[:-1]) * (1 << 20)) if s.endswith("M") else int(s)


def int32_table(ctx, name, cols, batch_rows=1 << 24):
    n = len(next(iter(cols.values())))
    td = TableData(name, [ColumnSpec(k, "int32") for k in cols])
    for b in range(0, n, batch_rows):
        td.chunks.append({k: np.ascontiguousarray(v[b:b + batch_rows]) for k, v in cols.items()})
        td.chunk_rows.append(min(batch_rows, n - b))
    return ctx.table_from_host(td)


def timed(ctx, fn):
    ctx.synchronize()
    ctx.timer_start()
    fn()
    return ctx.timer_stop()


def q9_program(ctx, t, states):
    """Q9 as program pipelines; {(nationkey, year): sum_profit}"""
    def keep(s):
        states.append(s)
        return s

    notnull = lambda e: ("not", ("isnull", e))
    green = keep(runtime.join_table(ctx, t["part"].num_rows))
    P.build_join(ctx, t["part"], green, col("p_partkey"), where=("like", "contains", "p_name", "green"))
    is_green = lambda k: notnull(("probe", green, col(k)))
    cost = keep(runtime.join_table_keys(ctx, 2, t["partsupp"].num_rows // 8))
    P.build_join(ctx, t["partsupp"], cost, [col("ps_partkey"), col("ps_suppkey")], payload=col("ps_supplycost"), where=is_green("ps_partkey"))
    orows = keep(runtime.join_table(ctx, t["orders"].num_rows))
    P.build_join(ctx, t["orders"], orows, col("o_orderkey"), payload=("rowid",))
    srows = keep(runtime.join_table(ctx, t["supplier"].num_rows))
    P.build_join(ctx, t["supplier"], srows, col("s_suppkey"), payload=("rowid",))
    c = ("probe", cost, col("l_partkey"), col("l_suppkey"))
    amount = ("sub", ("mul", col("l_extendedprice"), ("sub", const(100), col("l_discount"))), ("mul", c, col("l_quantity")))
    year = ("year", ("fetch", t["orders"], ("probe", orows, col("l_orderkey")), "o_orderdate"))
    nation = ("fetch", t["supplier"], ("probe", srows, col("l_suppkey")), "s_nationkey")
    st = keep(P.group_by(ctx, t["lineitem"], [nation, year], [("sum", amount)], where=("and", is_green("l_partkey"), notnull(c)), expected_groups=256))
    return {k: v[0] for k, v in P.decode_groups(P.read_groups(ctx, st, 256), 2, 1).items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-rows", type=rows_arg, default=16 << 20)
    ap.add_argument("--probe-rows", type=rows_arg, default=128 << 20)
    ap.add_argument("--sf", type=float, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"card": card(), "build_rows": a.build_rows, "probe_rows": a.probe_rows, "sf": a.sf, "reps": a.reps}
    nb, na = a.build_rows, a.probe_rows
    rng = np.random.default_rng(5)
    k = rng.permutation(nb).astype(np.int32)
    q = rng.integers(0, 2 * nb, na, dtype=np.int64).astype(np.int32)
    with runtime.Context(0) as ctx:
        B = int32_table(ctx, "build", {"k": k, "hi": k >> 12, "lo": k & 4095})
        A = int32_table(ctx, "probe", {"k": q, "hi": q >> 12, "lo": q & 4095})
        del k, q
        cases = {
            "int32": (lambda: runtime.join_table(ctx, nb), col("k"), [col("k")]),
            "tuple1": (lambda: runtime.join_table_keys(ctx, 1, nb), [col("k")], [col("k")]),
            "tuple2": (lambda: runtime.join_table_keys(ctx, 2, nb), [col("hi"), col("lo")], [col("hi"), col("lo")]),
        }
        built = {}
        for name, (make, bkey, pkeys) in cases.items():  # correctness once, untimed
            jt = make()
            P.build_join(ctx, B, jt, bkey, payload=("rowid",))
            assert runtime.join_count(ctx, jt) == nb, name
            st = P.group_by(ctx, A, [], [("count", ("probe", jt, *pkeys))])
            res.setdefault("matches", {})[name] = P.decode_groups(P.read_groups(ctx, st, 4), 0, 1)[()][0]
            runtime.state_destroy(ctx, st)
            built[name] = jt
        assert len(set(res["matches"].values())) == 1, res["matches"]
        times = {f"{n}_{w}": [] for n in cases for w in ("build_ms", "probe_ms")}
        for _ in range(a.reps):
            for name, (make, bkey, pkeys) in cases.items():
                jt = make()
                times[f"{name}_build_ms"].append(timed(ctx, lambda: P.build_join(ctx, B, jt, bkey, payload=("rowid",))))
                runtime.state_destroy(ctx, jt)

                def probe():
                    p = ("probe", built[name], *pkeys)
                    st = P.group_by(ctx, A, [], [("count_star", None)], where=("cmp", "=", p, const(-1)))
                    runtime.state_destroy(ctx, st)

                times[f"{name}_probe_ms"].append(timed(ctx, probe))
        res.update({n: float(np.median(v)) for n, v in times.items()})
        for jt in built.values():
            runtime.state_destroy(ctx, jt)
        B.clear()
        A.clear()

        t = datagen.tpch(a.sf, with_parts=True)
        tabs = {n: ctx.table_from_host(v) for n, v in t.items()}
        g = runtime.Tpch(ctx, tabs)
        states = []
        prog = q9_program(ctx, tabs, states)
        spec = g.q9()
        nat = {n: i for i, n in enumerate(g.nation_names)}
        assert prog == {(nat[r["nation"]], r["o_year"]): r["sum_profit"] for r in spec}, "Q9 as a program differs from ldb_tpch_q9"
        for s in states:
            runtime.state_destroy(ctx, s)
        qt = {"q9_program_ms": [], "q9_specialised_ms": []}
        for _ in range(a.reps):
            st = []
            qt["q9_program_ms"].append(timed(ctx, lambda: q9_program(ctx, tabs, st)))
            for s in st:
                runtime.state_destroy(ctx, s)
            qt["q9_specialised_ms"].append(timed(ctx, g.q9))
        res.update({n: float(np.median(v)) for n, v in qt.items()})
        res["q9_groups"] = len(prog)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
