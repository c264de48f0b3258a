"""Probe-side EXISTS (LDB_OP_EXISTS) in program joins: EXISTS without and with a residual, Q21 as one EXISTS program against its reversed
marker version, and the plain JOIN_BUILD / PROBE / PROBE_EACH program times of this build against a baseline build of the library, in one
process.

  python tools/existsjoin_sweep.py [--build-rows 16M] [--probe-rows 128M] [--reps 5] [--baseline-lib other/libldb_gpu.so] [--no-q21]
                                   [--out result.json]

Build side: `build-rows` distinct int32 keys (a permutation of 0..n-1) and a value column v, loaded into a plain multimap and a unique
table with row-id payloads; probe side: `probe-rows` keys uniform in 0..2n-1 (half hit) and a value column.  The probe programs keep no
row (their WHERE compares a boolean with 2), so their sink costs nothing:
  exists_ms            EXISTS without a residual on the multimap
  exists_unique_ms     the same on the unique table
  probe_unique_ms      NOT ISNULL(PROBE) on the unique table (what a semi join without a residual took before)
  exists_residual_ms   EXISTS on the multimap with the residual fetch(v) <> v (one side-column read per match)
  probe_residual_ms    the same semi join through PROBE on the unique table: NOT ISNULL(PROBE) AND fetch(v at the probe) <> v
  each_residual_ms     PROBE_EACH on the multimap with fetch(v at the match) <> v in WHERE (a verdict per match, not per row)
  q21_exists_ms        Q21 at SF1 as one program over lineitem with three EXISTS (builds of its four tables excluded)
  q21_reversed_ms      Q21 in the reversed marker shape (the programs after the orders build, marks scans and their builds included)
  build_ms / probe_ms / probe_each_ms   JOIN_BUILD into a fresh table, PROBE, PROBE_EACH; with --baseline-lib the same three again on a
                       context of the baseline library ("base_" prefix), the two alternating within each repetition
Verdict counts and Q21's groups are checked once outside the timings.  Every number is the median of `reps` runs timed with CUDA events on
the context's compute stream (the host waits for the stream), reported with the card's name and power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lingodb_b200 import datagen, dbgen, program as P, runtime  # noqa: E402
from tools.markjoin_sweep import card, context_of, count_where, int32_table, rows_arg, timed  # noqa: E402

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))


def q21_tables(ctx, t):
    """the four tables of the one-program Q21: Saudi suppliers, lineitem by orderkey, its late lines, its lines not yet 'F'"""
    li = t["lineitem"]
    late = ("cmp", ">", col("l_receiptdate"), col("l_commitdate"))
    saudi = runtime.join_table(ctx, 4096)
    P.build_join(ctx, t["supplier"], saudi, col("s_suppkey"), where=("cmp", "=", col("s_nationkey"), const([n for n, _ in datagen.NATIONS].index("SAUDI ARABIA"))))
    out = [saudi]
    for expected, where in ((6_100_000, None), (4_000_000, late), (3_100_000, ("cmp", "!=", col("l_linestatus"), const(ord("F"))))):
        js = runtime.join_table(ctx, expected, unique=False)
        P.build_join(ctx, li, js, col("l_orderkey"), payload=("rowid",), where=where)
        out.append(js)
    return out


def q21_exists(ctx, t, tabs):
    li = t["lineitem"]
    saudi, lines, late_lines, open_lines = tabs
    late = ("cmp", ">", col("l_receiptdate"), col("l_commitdate"))
    other = lambda js: ("cmp", "!=", ("fetch", li, ("match", js), "l_suppkey"), col("l_suppkey"))
    where = ("and", ("and", ("not", ("isnull", ("probe", saudi, col("l_suppkey")))), late),
             ("and", ("and", ("not", ("exists", open_lines, col("l_orderkey"), None)), ("exists", lines, col("l_orderkey"), other(lines))),
                     ("not", ("exists", late_lines, col("l_orderkey"), other(late_lines)))))
    st = P.group_by(ctx, li, [col("l_suppkey")], [("count_star", None)], where=where, expected_groups=4096)
    got = P.decode_groups(P.read_groups(ctx, st, 4096), 1, 1)
    runtime.state_destroy(ctx, st)
    return got


def q21_reversed(ctx, t, orders, saudi):
    """the reversed marker shape: F orders = the unmarked entries of `orders` probed by the non-F lines, the l1 candidates as a row-id
    multimap marked by the lines of another supplier, a second multimap of those left unmarked by the late lines of another supplier"""
    li = t["lineitem"]
    late = ("cmp", ">", col("l_receiptdate"), col("l_commitdate"))
    notnull = lambda e: ("not", ("isnull", e))
    states, tables = [], []
    P.clear_marks(ctx, orders)
    P.run_effects(ctx, li, [("mark", ("probe", orders, col("l_orderkey")), ("cmp", "!=", col("l_linestatus"), const(ord("F"))))])
    f_orders = P.join_marks(ctx, orders, P.UNMARKED)
    tables.append(f_orders)
    f_set = runtime.join_table(ctx, f_orders.num_rows)
    states.append(f_set)
    P.build_join(ctx, f_orders, f_set, col("key"))
    l1 = runtime.join_table(ctx, 400_000, unique=False)
    states.append(l1)
    P.build_join(ctx, li, l1, col("l_orderkey"), payload=("rowid",),
                 where=("and", late, ("and", notnull(("probe", saudi, col("l_suppkey"))), notnull(("probe", f_set, col("l_orderkey"))))))
    e2 = ("probe_each", l1, col("l_orderkey"))
    P.run_effects(ctx, li, [("mark", e2, ("cmp", "!=", col("l_suppkey"), ("fetch", li, e2, "l_suppkey")))])
    exists = P.join_marks(ctx, l1, P.MARKED)
    tables.append(exists)
    l1b = runtime.join_table(ctx, max(exists.num_rows, 1), unique=False)
    states.append(l1b)
    P.build_join(ctx, exists, l1b, col("key"), payload=col("payload"))
    e3 = ("probe_each", l1b, col("l_orderkey"))
    P.run_effects(ctx, li, [("mark", e3, ("and", late, ("cmp", "!=", col("l_suppkey"), ("fetch", li, e3, "l_suppkey"))))])
    wait = P.join_marks(ctx, l1b, P.UNMARKED)
    tables.append(wait)
    st = P.group_by(ctx, wait, [("fetch", li, col("payload"), "l_suppkey")], [("count_star", None)], expected_groups=4096)
    states.append(st)
    got = P.decode_groups(P.read_groups(ctx, st, 4096), 1, 1)
    for x in tables:
        x.destroy()
    for s_ in states:
        runtime.state_destroy(ctx, s_)
    return got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-rows", type=rows_arg, default=16 << 20)
    ap.add_argument("--probe-rows", type=rows_arg, default=128 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--baseline-lib")
    ap.add_argument("--no-q21", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"card": card(), "build_rows": a.build_rows, "probe_rows": a.probe_rows, "reps": a.reps, "baseline": bool(a.baseline_lib)}
    nb, na = a.build_rows, a.probe_rows
    rng = np.random.default_rng(5)
    k = rng.permutation(nb).astype(np.int32)
    bv = rng.integers(0, 4, nb).astype(np.int32)
    q = rng.integers(0, 2 * nb, na, dtype=np.int64).astype(np.int32)
    qv = rng.integers(0, 4, na).astype(np.int32)
    ctxs = {"": runtime.Context(0)}
    if a.baseline_lib:
        ctxs["base_"] = context_of(a.baseline_lib)
    data = {p: (int32_table(c, "build", {"k": k, "v": bv}), int32_table(c, "probe", {"k": q, "v": qv})) for p, c in ctxs.items()}
    ctx = ctxs[""]
    B, A = data[""]
    multi = runtime.join_table(ctx, nb, unique=False)
    P.build_join(ctx, B, multi, col("k"), payload=("rowid",))
    uniq = runtime.join_table(ctx, nb)
    P.build_join(ctx, B, uniq, col("k"), payload=("rowid",))
    never = lambda e: ("cmp", "=", e, const(2))
    ex = ("exists", multi, col("k"), None)
    ex_u = ("exists", uniq, col("k"), None)
    hit_u = ("not", ("isnull", ("probe", uniq, col("k"))))
    ex_r = ("exists", multi, col("k"), ("cmp", "!=", ("fetch", B, ("match", multi), "v"), col("v")))
    pr = ("probe", uniq, col("k"))
    pr_r = ("and", ("not", ("isnull", pr)), ("cmp", "!=", ("fetch", B, pr, "v"), col("v")))
    each_r = ("cmp", "!=", ("fetch", B, ("probe_each", multi, col("k")), "v"), col("v"))
    # correctness once, untimed
    hit = q < nb
    res["hits"] = int(hit.sum())
    assert count_where(ctx, A, ex) == count_where(ctx, A, ex_u) == count_where(ctx, A, hit_u) == res["hits"]
    res["residual_hits"] = count_where(ctx, A, ex_r)
    assert count_where(ctx, A, pr_r) == count_where(ctx, A, each_r) == res["residual_hits"]
    r = np.argsort(k)[np.where(hit, q, 0)]  # k is a permutation: the build row of key x is argsort(k)[x]
    assert res["residual_hits"] == int((hit & (bv[r] != qv)).sum())
    del r
    del k, bv, q, qv, hit
    names = ["exists_ms", "exists_unique_ms", "probe_unique_ms", "exists_residual_ms", "probe_residual_ms", "each_residual_ms"]
    q21 = None
    if not a.no_q21:
        t = dbgen.tpch(1.0, extended=True, attributes=True)
        q21 = {n: ctx.table_from_host(t[n]) for n in ("lineitem", "orders", "supplier")}
        del t
        tabs = q21_tables(ctx, q21)
        orders = runtime.join_table(ctx, 1_600_000)
        P.build_join(ctx, q21["orders"], orders, col("o_orderkey"), payload=("rowid",))
        a1, a2 = q21_exists(ctx, q21, tabs), q21_reversed(ctx, q21, orders, tabs[0])
        assert a1 == a2 and len(a1) > 0
        res["q21_groups"] = len(a1)
        names += ["q21_exists_ms", "q21_reversed_ms"]
    times = {n: [] for n in names}
    times.update({f"{p}{n}": [] for p in ctxs for n in ("build_ms", "probe_ms", "probe_each_ms")})
    for _ in range(a.reps):
        times["exists_ms"].append(timed(ctx, lambda: count_where(ctx, A, never(ex))))
        times["exists_unique_ms"].append(timed(ctx, lambda: count_where(ctx, A, never(ex_u))))
        times["probe_unique_ms"].append(timed(ctx, lambda: count_where(ctx, A, never(hit_u))))
        times["exists_residual_ms"].append(timed(ctx, lambda: count_where(ctx, A, never(ex_r))))
        times["probe_residual_ms"].append(timed(ctx, lambda: count_where(ctx, A, never(pr_r))))
        times["each_residual_ms"].append(timed(ctx, lambda: count_where(ctx, A, never(each_r))))
        if q21:
            times["q21_exists_ms"].append(timed(ctx, lambda: q21_exists(ctx, q21, tabs)))
            times["q21_reversed_ms"].append(timed(ctx, lambda: q21_reversed(ctx, q21, orders, tabs[0])))
        for p, c in ctxs.items():
            b_, a_ = data[p]
            fresh = runtime.join_table(c, nb)
            times[f"{p}build_ms"].append(timed(c, lambda: P.build_join(c, b_, fresh, col("k"), payload=("rowid",))))
            times[f"{p}probe_ms"].append(timed(c, lambda: count_where(c, a_, ("cmp", "=", ("probe", fresh, col("k")), const(-1)))))
            times[f"{p}probe_each_ms"].append(timed(c, lambda: count_where(c, a_, ("cmp", "=", ("probe_each", fresh, col("k")), const(-1)))))
            runtime.state_destroy(c, fresh)
    res.update({n: float(np.median(v)) for n, v in times.items()})
    for js in (multi, uniq):
        runtime.state_destroy(ctx, js)
    if q21:
        for js in tabs + [orders]:
            runtime.state_destroy(ctx, js)
        for x in q21.values():
            x.clear()
    for p, c in ctxs.items():
        for t_ in data[p]:
            t_.clear()
        c.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
