"""The generic program pipeline (csrc/program.cu) through the C-ABI: arbitrary expressions, nullable columns, strings, float/int64
operands, SUM/COUNT/MIN/MAX/ANY with SQL null semantics over ANY number of groups, semi joins and ORDER BY — against the CPU
oracle where it has the query (nullable scans: the reference's own Restrictions with the NOTNULL filters its pushdown adds,
test_nullable_scans_match_the_reference_filters), against an independent numpy evaluation for the rest (NULL handling inside
aggregates and boolean connectives: the three-valued-logic rules of the SQL standard, restated in numpy)."""
import ctypes as C

import numpy as np
import pytest

from lingodb_b200 import datagen

pytestmark = pytest.mark.gpu

col = lambda n: ("col", n)
const = lambda v: ("const", v)


def _lo64(a):
    return a[:, :8].copy().view(np.int64).reshape(-1)


def test_q1_and_q6_as_programs_match_the_oracle(gpu_ctx, oracle):
    """The two scan pipelines of BASELINE configs 0/1 written as register programs (db.mul/sub/add over decimals, date compare,
    BETWEEN): same exact i64/i128 sums as the oracle (the specialised kernels' results), here over ragged batches."""
    from lingodb_b200 import program as P
    t = datagen.tpch(0.05, seed=77, chunk_rows=30_011)
    li = gpu_ctx.table_from_host(t["lineitem"])
    oh = oracle.table(t["lineitem"])
    ext, disc, tax = col("l_extendedprice"), col("l_discount"), col("l_tax")
    one = const(100)
    disc_price = ("mul", ext, ("sub", one, disc))
    aggs = [("sum", col("l_quantity")), ("sum", ext), ("sum", disc_price), ("sum", ("mul", disc_price, ("add", one, tax))), ("sum", disc), ("count_star", None)]
    d = oracle.lib.oracle_parse_date(b"1998-09-02")
    st = P.group_by(gpu_ctx, li, [col("l_returnflag"), col("l_linestatus")], aggs, where=("cmp", "<=", col("l_shipdate"), const(d)), expected_groups=16)
    got = P.decode_groups(P.read_groups(gpu_ctx, st, 64), 2, 6)
    want = oracle.q1(oh)[0]
    assert len(got) == len(want) == 4
    for r in want:  # decode_groups returns signed 128-bit python ints
        g = got[(r["l_returnflag"], r["l_linestatus"])]
        assert [g[0], g[1], g[2], g[3], g[5]] == [r["sum_qty"], r["sum_base_price"], r["sum_disc_price"], r["sum_charge"], r["count_order"]]
    gpu_ctx.L.ldb_gpu_state_destroy(st)
    # Q6: keyless sum(ext * disc) under shipdate range, discount BETWEEN, quantity <
    lo, hi = oracle.lib.oracle_parse_date(b"1994-01-01"), oracle.lib.oracle_parse_date(b"1995-01-01")
    where = ("and", ("and", ("cmp", ">=", col("l_shipdate"), const(lo)), ("cmp", "<", col("l_shipdate"), const(hi))),
             ("and", ("between", disc, const(5), const(7)), ("cmp", "<", col("l_quantity"), const(2400))))
    st = P.group_by(gpu_ctx, li, [], [("sum", ("mul", ext, disc))], where=where)
    got = P.decode_groups(P.read_groups(gpu_ctx, st, 4), 0, 1)
    assert got[()][0] == oracle.q6(oh)[0]["revenue"]
    gpu_ctx.L.ldb_gpu_state_destroy(st)


def test_nullable_columns_types_and_every_aggregate(gpu_ctx):
    """Validity bitmaps on int32 / int64 / decimal(38) / float64 / utf8 columns, a nullable group key (NULLs form one group),
    three-valued WHERE, SUM / COUNT / COUNT(*) / MIN / MAX / ANY / float aggregates that skip NULLs and stay NULL on empty input."""
    from lingodb_b200 import program as P
    rng = np.random.default_rng(5)
    n = 150_001
    a = rng.integers(-1000, 1000, n).astype(np.int32)
    b = rng.integers(-2**40, 2**40, n).astype(np.int64)
    dlo = rng.integers(-10**15, 10**15, n).astype(np.int64)
    d = np.zeros((n, 2), np.int64)
    d[:, 0], d[:, 1] = dlo, dlo >> 63
    d[::1000, 1] += 3  # some values beyond 64 bits: decimal(38) cells are read whole
    f = rng.normal(size=n)
    g = rng.integers(0, 40, n).astype(np.int32)
    words = [b"alpha", b"beta", b"gamma", b"abacus", b"zeta", b""]
    sidx = rng.integers(0, len(words), n)
    offs = np.zeros(n + 1, np.int32)
    offs[1:] = np.cumsum([len(words[i]) for i in sidx])
    sbytes = np.frombuffer(b"".join(words[i] for i in sidx), np.uint8).copy()
    valid = {k: rng.random(n) > p for k, p in (("a", 0.1), ("b", 0.2), ("d", 0.15), ("f", 0.3), ("g", 0.05), ("s", 0.1))}
    valid["d"][g == 7] = False  # one group whose SUM(d) has no input at all
    bits = {k: np.packbits(v, bitorder="little") for k, v in valid.items()}
    specs = [datagen.ColumnSpec("a", "int32"), datagen.ColumnSpec("b", "int64"), datagen.ColumnSpec("d", "decimal128", 38, 2), datagen.ColumnSpec("f", "float64"),
             datagen.ColumnSpec("g", "int32"), datagen.ColumnSpec("s", "utf8")]
    td = datagen.TableData("t", specs)
    td.chunks.append({"a": a, "b": b, "d": d.view(np.uint8).reshape(n, 16), "f": f, "g": g, "s": (offs, sbytes), **{k + "$valid": v for k, v in bits.items()}})
    td.chunk_rows.append(n)
    tab = gpu_ctx.table_from_host(td)
    # WHERE (a > 100 OR b IS NULL) AND NOT (s LIKE 'a%')   — NULL a with non-NULL b → NULL OR false = NULL → dropped; NULL s → dropped
    where = ("and", ("or", ("cmp", ">", col("a"), const(100)), ("isnull", col("b"))), ("not", ("like", "prefix", "s", "a")))
    aggs = [("sum", col("d")), ("count", col("b")), ("count_star", None), ("min", col("a")), ("max", col("b")), ("sum_f64", col("f")), ("min_f64", col("f")), ("any", col("a"))]
    st = P.group_by(gpu_ctx, tab, [col("g")], aggs, where=where, expected_groups=64)
    got = P.decode_groups(P.read_groups(gpu_ctx, st, 256), 1, 8, f64_aggs=(5, 6))
    gpu_ctx.L.ldb_gpu_state_destroy(st)
    # ---- numpy restatement of the SQL semantics
    starts_a = np.array([w.startswith(b"a") for w in words])[sidx]
    cond_or_true = (valid["a"] & (a > 100)) | ~valid["b"]
    keep = cond_or_true & valid["s"] & ~starts_a
    dfull = [(int(d[i, 1]) << 64) | (int(d[i, 0]) & 0xFFFFFFFFFFFFFFFF) for i in range(n)]
    sgn = lambda v: v - (1 << 128) if v >> 127 else v
    want = {}
    for key in list(range(40)) + [None]:
        m = keep & (~valid["g"] if key is None else (valid["g"] & (g == key)))
        if not m.any():
            continue
        idx = np.flatnonzero(m)
        dv = [dfull[i] for i in idx if valid["d"][i]]
        av, bv, fv = a[idx][valid["a"][idx]], b[idx][valid["b"][idx]], f[idx][valid["f"][idx]]
        want[(key,)] = [sgn(sum(dv) & ((1 << 128) - 1)) if dv else None, len(bv), len(idx), int(av.min()) if len(av) else None, int(bv.max()) if len(bv) else None,
                        float(fv.sum()) if len(fv) else None, float(fv.min()) if len(fv) else None, set(av.tolist())]
    assert set(got) == set(want)
    assert (7,) in want and want[(7,)][0] is None  # the all-NULL input group exists and its SUM is NULL
    for k, w in want.items():
        gk = got[k]
        assert gk[0] == w[0], (k, "sum(d)")
        assert gk[1] == w[1] and gk[2] == w[2], (k, "counts")
        s64 = lambda v: None if v is None else ((v & 0xFFFFFFFFFFFFFFFF) ^ (1 << 63)) - (1 << 63)
        assert gk[3] == w[3] and gk[4] == w[4], (k, "min/max")  # signed 128-bit results, read whole
        if w[5] is None:
            assert gk[5] is None and gk[6] is None
        else:
            assert abs(gk[5] - w[5]) <= 1e-6 * max(1.0, abs(w[5])) and gk[6] == w[6], (k, "float aggregates")  # north_star: 1e-6 relative
        assert (gk[7] is None and not w[7]) or s64(gk[7]) in w[7], (k, "any")
    # string ordering and equality against constants (VarLen32Filter<Lt…>): count(*) WHERE s < 'beta' / s = 'zeta' / s >= ''
    for op, k in (("<", "beta"), ("=", "zeta"), (">=", ""), ("!=", "gamma")):
        st = P.group_by(gpu_ctx, tab, [], [("count_star", None)], where=("strcmp", op, "s", k))
        cnt = P.decode_groups(P.read_groups(gpu_ctx, st, 4), 0, 1)[()][0]
        gpu_ctx.L.ldb_gpu_state_destroy(st)
        wk = np.array([{"<": w < k.encode(), "=": w == k.encode(), ">=": w >= k.encode(), "!=": w != k.encode()}[op] for w in words])[sidx]
        assert cnt == int((wk & valid["s"]).sum()), (op, k)


def test_nullable_scans_match_the_reference_filters(gpu_ctx, oracle):
    """WHERE predicates over nullable generator columns, evaluated by the program pipeline with SQL three-valued logic, keep exactly
    the rows the reference's scan keeps with the filter lists its pushdown writes for nullable columns ([NOTNULL, cmp…],
    Pushdown.cpp:346-372 → Restrictions.cpp:67-162), and SUM skips the same NULL cells: count and sum bit-exact against the oracle
    (the reference-compiled Restrictions when oracle/_ref is built)."""
    from lingodb_b200 import program as P
    from _nullable import cases, nullable_lineitem
    li, _ = nullable_lineitem()
    tab = gpu_ctx.table_from_host(li)
    oh = oracle.table(li)
    date = lambda s: oracle.lib.oracle_parse_date(s.encode())
    for filters, where, sum_column in cases(date):
        aggs = [("count_star", None)] + ([("sum", col(sum_column))] if sum_column else [])
        st = P.group_by(gpu_ctx, tab, [], aggs, where=where)
        got = P.decode_groups(P.read_groups(gpu_ctx, st, 4), 0, len(aggs))[()]
        gpu_ctx.L.ldb_gpu_state_destroy(st)
        want_n, want_sum = oracle.scan_count_sum(oh, filters, sum_column)
        assert got[0] == want_n, filters
        if sum_column:
            assert got[1] == want_sum, filters
    oracle.free(oh)


def test_large_domain_group_by_having_and_order_by(gpu_ctx):
    """One group per order (the Q18 sub-query shape: 75 000 groups here, millions at scale), HAVING through the exported groups table,
    ORDER BY … LIMIT through the device radix sort — against numpy."""
    from lingodb_b200 import program as P
    s = datagen.scale(0.05, seed=3)
    li = datagen.lineitem(s, ["l_orderkey", "l_quantity"], chunk_rows=70_000)
    keys = np.concatenate([c["l_orderkey"] for c in li.chunks])
    qty = np.concatenate([_lo64(c["l_quantity"]) for c in li.chunks])
    tab = gpu_ctx.table_from_host(li)
    st = P.group_by(gpu_ctx, tab, [col("l_orderkey")], [("sum", col("l_quantity")), ("count_star", None), ("max", col("l_quantity"))], expected_groups=s.n_orders + 1000)
    n = C.c_int64()
    from lingodb_b200 import capi
    e = capi.Error()
    capi.check(gpu_ctx.L.ldb_gpu_hashagg_count(st, C.byref(n), C.byref(e)), e)
    uk, inv = np.unique(keys, return_inverse=True)
    assert n.value == len(uk)
    sums = np.bincount(inv, weights=qty.astype(np.float64)).astype(np.int64)
    got = P.decode_groups(P.read_groups(gpu_ctx, st, len(uk) + 16), 1, 3)
    assert len(got) == len(uk)
    mx = np.zeros(len(uk), np.int64)
    np.maximum.at(mx, inv, qty)
    cnt = np.bincount(inv)
    for i in range(0, len(uk), 97):
        assert got[(int(uk[i]),)] == [int(sums[i]), int(cnt[i]), int(mx[i])]
    # HAVING sum(l_quantity) > 200.00 → ORDER BY sum desc LIMIT 10
    gt = P.groups_table(gpu_ctx, st)
    hv = P.RawTable(gpu_ctx, P.materialize(gpu_ctx, gt, [col("k0"), col("a0")], where=("cmp", ">", col("a0"), const(20000))))
    sel = sums > 20000
    assert hv.num_rows == int(sel.sum())
    ids = hv.order_by("c1", descending=True, limit=10)
    top_sums = hv.gather("c1", ids)
    assert top_sums == sorted(sums[sel].tolist(), reverse=True)[:10]
    top_keys = hv.gather("c0", ids)
    for k, v in zip(top_keys, top_sums):
        assert int(sums[np.searchsorted(uk, k)]) == v
    # ascending over an int32 column of a base table, full sort
    od = gpu_ctx.table_from_host(datagen.orders(s, chunk_rows=1 << 20))
    raw = P.RawTable(gpu_ctx, od.h)
    ids = raw.order_by("o_custkey")
    ck = np.concatenate([c["o_custkey"] for c in datagen.orders(s).chunks])
    assert len(ids) == len(ck) and (np.diff(ck[np.array(ids)]) >= 0).all() and sorted(ids) == list(range(len(ck)))
    for t in (hv, gt):
        t.destroy()
    gpu_ctx.L.ldb_gpu_state_destroy(st)
