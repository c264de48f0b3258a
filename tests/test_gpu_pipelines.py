"""Every specialised pipeline (K1/K2, K3, K4, K5 + top-k, K8, K9 — csrc/kernels.cu) against the exact reference of tests/_piperef.py,
bit for bit: negative, wide and warp-mixed values, every group-by signature, hash-colliding / extreme / dense / sparse keys, partial
tiles, ragged and offset batches, DEVICE next to narrowed HOST batches, compressed staging, every filter op, every tile pipeline
(`ldb_gpu_set_tuning`), both filter forms (`ldb_gpu_set_filter_specialisation`) and every documented error."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import _piperef as P
import _progref as R

pytestmark = pytest.mark.gpu
COLS = P.PIPE_COLUMNS + [("d", "decimal128", 18, 2), ("k2", "int32", 0, 0)]
SCHEMA = P.schema_of(COLS)
HERE = os.path.dirname(os.path.abspath(__file__))


# ---------------------------------------------------------------------------------------------------- helpers
def rt():
    from lingodb_b200 import runtime
    return runtime


def capi():
    from lingodb_b200 import capi as c
    return c


def values(seed: int, n: int, mix: str, key_domain: int = 4) -> dict:
    """seeded rows: keys k (key_domain values) and k2, int32/date/fsb4/utf8 columns from the generator, decimals by `mix`:
    tpch (the 32-bit fast path), negative, wide (|v| up to 10^18) or mixed (TPC-H with one operand in [2^31, 2^32) every 32 rows)"""
    v = P.gen_table(seed, n, COLS, key_domain=key_domain)
    rng = np.random.default_rng(seed)
    v["k2"] = [int(x) for x in rng.integers(0, 3, n)]
    dec = {"tpch": lambda: (rng.integers(0, 10**7, n), rng.integers(0, 11, n), rng.integers(0, 9, n), rng.integers(0, 10**5, n)),
           "negative": lambda: tuple(rng.integers(-10**7, 10**7, n) for _ in range(4)),
           "wide": lambda: tuple(rng.integers(-10**18 + 1, 10**18, n) for _ in range(4))}
    if mix == "mixed":
        a, b, c, d = dec["tpch"]()
        for arr in (a, b, c, d):
            arr[7::32] = rng.integers(1 << 31, 1 << 32, len(arr[7::32]))
            arr[19::96] = (1 << 31) - 1 - arr[19::96] % 3
    else:
        a, b, c, d = dec[mix]()
    for name, arr in zip("abcd", (a, b, c, d)):
        v[name] = [int(x) for x in arr]
    return v


def table(ctx, name, vals, cuts=(), offset=0, device=(), columns=COLS):
    """a runtime Table of `vals` cut into batches at `cuts`; batches whose index is in `device` are borrowed DEVICE buffers, the rest
    HOST batches staged from Arrow buffers with `offset` leading rows (ArrayView.offset)"""
    import torch
    t = rt().Table(ctx, name, R.specs_of(columns))
    n = len(next(iter(vals.values())))
    edges = [0] + list(cuts) + [n]
    for bi, (a, b) in enumerate(zip(edges, edges[1:])):
        if bi in device:
            ch = {}
            for cname, phys, _, _ in columns:
                buf, _ = R.column_buffers(phys, vals[cname][a:b])
                if phys == "utf8":
                    ch[cname] = (torch.from_numpy(buf[0]).cuda(ctx.device), torch.from_numpy(buf[1]).cuda(ctx.device))
                else:
                    ch[cname] = torch.from_numpy(np.ascontiguousarray(buf)).cuda(ctx.device)
            t.append_device(ch, b - a)
        else:
            ch = {cname: R.column_buffers(phys, vals[cname][a:b], offset)[0] for cname, phys, _, _ in columns}
            t.append_host(ch, b - a, offset)
    ctx.synchronize()
    return t


def expect_error(code, fn, *a, **kw):
    with pytest.raises(capi().LdbRuntimeError) as e:
        fn(*a, **kw)
    assert e.value.code == code, str(e.value)


def gpu_groupby(ctx, src, keys, aggs, filters=(), capacity=64):
    run = rt()
    c = capi()
    if not keys:
        s, e = C.c_void_p(), c.Error()
        c.check(ctx.L.ldb_gpu_simple_state_create(ctx.h, len(aggs), C.byref(s), C.byref(e)), e)
        try:
            run.run_pipeline(ctx, "scan_reduce", src, filters=filters, aggs=aggs, sink=s)
            out = (c.I128 * 8)()
            c.check(ctx.L.ldb_gpu_simple_state_read(s, out, C.byref(e)), e)
            return {(): [out[i].value() for i in range(len(aggs))]}
        finally:
            run.state_destroy(ctx, s)
    s = run.groupby_state(ctx, len(keys), len(aggs), capacity)
    try:
        run.run_pipeline(ctx, "scan_groupby", src, filters=filters, keys=keys, aggs=aggs, sink=s)
        return read_groups(ctx, s, len(aggs))
    finally:
        run.state_destroy(ctx, s)


def read_groups(ctx, s, n_aggs):
    c = capi()
    rows = (c.GroupRow * 4096)()
    n, e = C.c_int32(), c.Error()
    c.check(ctx.L.ldb_gpu_groupby_read(s, rows, 4096, C.byref(n), C.byref(e)), e)
    assert n.value <= 4096
    return {(r.keys[0], r.keys[1]): [r.aggs[i].value() for i in range(n_aggs)] for r in rows[: n.value]}


def sig_aggs(sig):
    """a signature of _piperef.SIGNATURES over the value columns a, b, c, d"""
    nk, aggs = sig
    return ["k", "k2"][:nk], [(e, ["abcd"[p] for p in pos]) for e, pos in aggs]


def _env_int(name, dflt, lo, hi):
    try:
        v = int(os.environ.get(name, dflt))
    except ValueError:
        v = 0  # atoi
    return min(max(v, lo), hi)


def env_tuning():
    """the configuration the process started with (kernels.cu tuningStorage: LDB_STAGES_* / LDB_RPT_BUILD / LDB_SPECIALISE /
    LDB_*_SLEEP_NS, else the tuned defaults): (set_tuning arguments, specialisation, poll pauses)"""
    stages = tuple(_env_int("LDB_STAGES_" + k, d, 2, 4) for k, d in (("BUILD", 3), ("PROBE_AGG", 3), ("PROBE2", 3), ("STAR", 2)))
    rpt = _env_int("LDB_RPT_BUILD", 2, 1, 4)
    return (stages + (2 if rpt == 3 else rpt,), _env_int("LDB_SPECIALISE", 1, 0, 1),
            (_env_int("LDB_PRODUCER_SLEEP_NS", 0, 0, 2000), _env_int("LDB_CONSUMER_SLEEP_NS", 0, 0, 2000)))


DEFAULT_TUNING = env_tuning()[0]


class tuned:
    """ldb_gpu_set_tuning / _filter_specialisation / _poll_pause for a block; the process's configuration comes back in `finally`"""

    def __init__(self, ctx, tuning=None, spec=None, pause=None):
        base, base_spec, base_pause = env_tuning()
        self.ctx, self.tuning = ctx, tuning or base
        self.spec = base_spec if spec is None else spec
        self.pause = pause or base_pause

    def __enter__(self):
        self.ctx.L.ldb_gpu_set_tuning(*self.tuning)
        self.ctx.L.ldb_gpu_set_filter_specialisation(self.spec)
        self.ctx.L.ldb_gpu_set_poll_pause(*self.pause)

    def __exit__(self, *a):
        base, base_spec, base_pause = env_tuning()
        self.ctx.L.ldb_gpu_set_tuning(*base)
        self.ctx.L.ldb_gpu_set_filter_specialisation(base_spec)
        self.ctx.L.ldb_gpu_set_poll_pause(*base_pause)


def filter_cases(sets, rotate: int, specialised: bool):
    """every filter set in the cells that launch the filter-shape instantiations (none / one compare / range), one of them (rotating)
    elsewhere"""
    return sets if specialised else [sets[rotate % len(sets)]]


TUNINGS = [(s, r) for s in (2, 3, 4) for r in (1, 2, 4)]  # (stages, rows per thread of a build tile)


def build_table(ctx, ref: P.JoinTable):
    run = rt()
    if ref.kind == "pair":
        return run.join_table_pair(ctx, ref.expected_rows, ref.unique)
    if ref.kind == "direct":
        return run.join_table_direct(ctx, ref.key_min, ref.key_max)
    return run.join_table(ctx, ref.expected_rows, ref.unique, ref.n_side, ref.n_aggs)


def new_table(kind="hash", expected_rows=1024, **kw) -> P.JoinTable:
    t = P.JoinTable(kind, expected_rows, **kw)
    t.expected_rows = expected_rows
    return t


def gpu_payloads(ctx, table_state, keys: list):
    """K8 with a $payload probe of every key in `keys`: sorted (key, payload) pairs — the contents of a plain table"""
    import torch
    run = rt()
    cols = [("pk", "int32", 0, 0)]
    src = table(ctx, "probe_keys", {"pk": keys}, columns=cols)
    cap = 4 * len(keys) + 64
    out_k = torch.zeros(cap, dtype=torch.int32, device="cuda")
    out_p = torch.zeros(cap, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    run.run_pipeline(ctx, "scan_materialize", src, probes=[(table_state, "pk")], out_columns=["pk", "$payload"],
                     out_buffers=[out_k.data_ptr(), out_p.data_ptr()], out_capacity=cap, out_count=C.c_void_p(cnt.data_ptr()))
    ctx.synchronize()
    n = int(cnt.item())
    assert n <= cap
    return sorted(zip(out_k[:n].tolist(), out_p[:n].tolist()))


def ref_payloads(ref: P.JoinTable, keys: list):
    idx = ref.index()
    return sorted((k, e[1]) for k in keys for e in idx.get(k, []))


# key patterns of a join build side (n rows)
def keys_of(pattern: str, n: int, seed: int) -> list:
    rng = random.Random(seed)
    if pattern == "dense":
        return list(range(n))
    if pattern == "sparse":
        return rng.sample(range(-(1 << 31), 1 << 31), n)
    if pattern == "negative":
        return [-1 - i * 7 for i in range(n)]
    if pattern == "extremes":
        base = [P.I32_MIN, P.I32_MAX, 0, -1, 1, P.I32_MIN + 1, P.I32_MAX - 1]
        return base + rng.sample(range(-10**6, 10**6), n - len(base))
    if pattern == "colliding":  # one directory slot near the end of a 4096-slot table: long runs that wrap around
        return P.colliding_keys(16, 4093, n)
    raise ValueError(pattern)


# ---------------------------------------------------------------------------------------------------- K1 / K2
@pytest.mark.parametrize("mix", ["tpch", "negative", "wide", "mixed"])
def test_every_groupby_signature(gpu_ctx, mix):
    vals = values(11, 9000, mix)
    src = table(gpu_ctx, "t", vals, cuts=(4097, 4098, 8000))
    for sig in P.SIGNATURES:
        keys, aggs = sig_aggs(sig)
        assert gpu_groupby(gpu_ctx, src, keys, aggs) == P.scan_groupby(vals, SCHEMA, [], keys, aggs), (mix, sig)


@pytest.mark.parametrize("n_groups", [1, 4, 5, 16, 17, 1000])
def test_groupby_key_patterns(gpu_ctx, n_groups):
    """register-resident (<= 4), shared-memory (<= 16) and HBM groups; key (0, 0), negative and extreme keys"""
    rng = random.Random(n_groups)
    pool = [(0, 0), (P.I32_MIN, P.I32_MAX), (-1, -1), (P.I32_MAX, 0), (-1, 0)] + [(rng.randrange(-(1 << 31), 1 << 31), rng.randrange(-3, 3)) for _ in range(n_groups)]
    pool = list(dict.fromkeys(pool))[:n_groups]
    vals = values(5, 12000, "mixed")
    pick = [pool[rng.randrange(len(pool))] if i >= len(pool) else pool[i] for i in range(12000)]
    vals["k"], vals["k2"] = [p[0] for p in pick], [p[1] for p in pick]
    src = table(gpu_ctx, "t", vals, cuts=(3000,))
    for sig in (P.SIGNATURES[0], P.SIGNATURES[8], P.SIGNATURES[7]):
        keys, aggs = sig_aggs(sig)
        want = P.scan_groupby(vals, SCHEMA, [], keys, aggs, capacity=2048)
        assert gpu_groupby(gpu_ctx, src, keys, aggs, capacity=2048) == want


def test_groupby_batch_layouts(gpu_ctx):
    """partial tiles (tiles are 256 x 2 rows), ragged batches, Arrow offsets (plain loads), DEVICE batches with 16-byte decimals next
    to narrowed HOST batches"""
    sizes = [1, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025]
    vals = values(3, sum(sizes), "mixed")
    cuts = list(np.cumsum(sizes)[:-1])
    keys, aggs = sig_aggs(P.SIGNATURES[0])
    want = P.scan_groupby(vals, SCHEMA, [("i", "!=", 12345)], keys, aggs)
    for offset in (0, 1, 2, 3):
        src = table(gpu_ctx, "t", vals, cuts=cuts, offset=offset)
        assert gpu_groupby(gpu_ctx, src, keys, aggs, [("i", "!=", 12345)]) == want, offset
    # a 16-byte DEVICE batch beside narrowed HOST batches
    src = table(gpu_ctx, "t", vals, cuts=cuts, device=(1, 4, 9))
    assert gpu_groupby(gpu_ctx, src, keys, aggs, [("i", "!=", 12345)]) == want
    keys1, aggs1 = sig_aggs(P.SIGNATURES[3])
    assert gpu_groupby(gpu_ctx, src, keys1, aggs1) == P.scan_groupby(vals, SCHEMA, [], keys1, aggs1)


def test_groupby_without_narrow_staging_and_with_compressed_staging(gpu_ctx):
    vals = values(9, 70_000, "mixed")
    keys, aggs = sig_aggs(P.SIGNATURES[0])
    want = P.scan_groupby(vals, SCHEMA, [], keys, aggs)
    assert gpu_groupby(gpu_ctx, table(gpu_ctx, "big", vals), keys, aggs) == want  # one >= 65 536-row HOST batch: compressed staging
    old = os.environ.get("LDB_NARROW_STAGING")
    os.environ["LDB_NARROW_STAGING"] = "0"  # read when a context is created
    try:
        ctx2 = rt().Context(0)
    finally:
        if old is None:
            del os.environ["LDB_NARROW_STAGING"]
        else:
            os.environ["LDB_NARROW_STAGING"] = old
    try:
        small = {k: v[:5000] for k, v in vals.items()}
        assert gpu_groupby(ctx2, table(ctx2, "t", small, cuts=(777,)), keys, aggs) == P.scan_groupby(small, SCHEMA, [], keys, aggs)
    finally:
        ctx2.close()


FILTER_SETS = [
    [("i", "=", 5)], [("i", "!=", 5)], [("i", "<", 0)], [("i", "<=", -1)], [("i", ">", 100)], [("i", ">=", P.I32_MIN)], [("i", "notnull", 0)],
    [("i", "in", [5])], [("i", "in", [0, 1, -1, 2, 3, P.I32_MIN, P.I32_MAX, 99])], [("i", ">", -50), ("i", "<=", 50)],
    [("i", "<", 1 << 40)], [("i", ">", -(1 << 40)), ("i", "<", 1 << 35)],
    [("dt", ">=", "1994-01-01"), ("dt", "<", "1995-01-01")], [("dt", "<", "1970-01-01")], [("dt", "in", ["1970-01-01", "2000-02-29"])],
    [("fs", "=", "A")], [("fs", "!=", "")], [("fs", ">", "B")], [("fs", "in", ["A", "\x7f"])],
    [("a", ">=", "0.05"), ("a", "<=", "0.07")], [("a", "<", 0)], [("a", ">", "-1.5")], [("a", "in", ["0", "0.01", "-0.01"])], [("a", "!=", "0")],
    [("s", "=", "")], [("s", "!=", "")], [("s", "=", "ab")], [("s", "contains", "")], [("s", "contains", "a")], [("s", "contains", "é")],
    [("s", "contains", "\x7f")], [("s", "=", "é")],
    [("i", ">", -(1 << 30)), ("dt", ">", "1900-01-01"), ("a", "<", "1000000000"), ("s", "contains", "a")],
]


def test_every_filter_op_on_every_type(gpu_ctx):
    vals = values(21, 6000, "negative")
    vals["i"] = [x if j % 3 else (j % 200) - 100 for j, x in enumerate(vals["i"])]
    src = table(gpu_ctx, "t", vals, cuts=(2049,))
    aggs = [("col", ["a"]), ("one", [])]
    for f in FILTER_SETS:
        want = P.scan_groupby(vals, SCHEMA, f, [], aggs)
        assert gpu_groupby(gpu_ctx, src, [], aggs, f) == want, f


# ---------------------------------------------------------------------------------------------------- K3 + K8
@pytest.mark.parametrize("pattern", ["dense", "sparse", "negative", "extremes", "colliding"])
@pytest.mark.parametrize("unique", [True, False])
def test_build_then_materialize(gpu_ctx, pattern, unique):
    n = 600
    keys = keys_of(pattern, n, 7)
    if not unique:
        keys = keys + keys[: n // 3] + keys[: 17]
    rng = random.Random(1)
    m = len(keys)
    vals = values(2, m, "negative")
    vals["k"] = keys
    vals["i"] = [rng.randrange(-(1 << 31), 1 << 31) for _ in range(m)]
    vals["i"] = [x if not (k == -1 and x == -1) else 0 for k, x in zip(keys, vals["i"])]
    probe = keys[::2] + [k ^ 0x55 for k in keys[:50]] + [P.I32_MIN, P.I32_MAX]
    filters_all = [[], [("dt", ">", "1950-01-01")], [("dt", ">", "1950-01-01"), ("dt", "<", "2050-01-01")], [("a", ">", 0)]]
    for stages, rpt in TUNINGS:
        for spec in (0, 1):
            filters = filters_all[(stages + rpt + spec) % len(filters_all)]
            ref = new_table(expected_rows=2048, unique=unique)
            P.scan_build(vals, SCHEMA, filters, ref, "k", payload="i")
            with tuned(gpu_ctx, (stages, 3, 3, 2, rpt), spec, pause=(0, 200) if stages == 4 else (0, 0)):
                src = table(gpu_ctx, "b", vals, cuts=(m // 3 + 1,))
                st = build_table(gpu_ctx, ref)
                rt().run_pipeline(gpu_ctx, "scan_build", src, filters=filters, build_key="k", build_payload="i", sink=st)
                assert rt().join_count(gpu_ctx, st) == ref.count()
                assert gpu_payloads(gpu_ctx, st, probe) == ref_payloads(ref, probe), (stages, rpt, spec, filters)
                rt().state_destroy(gpu_ctx, st)


def test_build_with_a_parent_probe_and_year_payloads(gpu_ctx):
    rng = random.Random(4)
    parent_keys = list(range(0, 400, 2))
    pvals = values(1, len(parent_keys) * 2, "tpch")
    pvals["k"] = parent_keys + parent_keys  # a multimap parent: two entries per key
    pvals["i"] = [rng.randrange(0, 1000) for _ in pvals["k"]]
    n = 1500
    vals = values(8, n, "tpch")
    vals["k"] = list(range(n))
    vals["k2"] = [rng.randrange(0, 450) for _ in range(n)]
    vals["dt"] = [rng.choice([0, -1, 10957, P.I32_MAX, P.I32_MIN, P.I32_MAX - 719468, P.I32_MAX - 719467, P.I32_MIN + 1, 2932896, -719163]) for _ in range(n)]
    for spec in (0, 1):
        with tuned(gpu_ctx, spec=spec):
            pref = new_table(expected_rows=512, unique=False)
            P.scan_build(pvals, SCHEMA, [], pref, "k", payload="i")
            psrc = table(gpu_ctx, "p", pvals)
            pst = build_table(gpu_ctx, pref)
            rt().run_pipeline(gpu_ctx, "scan_build", psrc, build_key="k", build_payload="i", sink=pst)
            src = table(gpu_ctx, "c", vals, cuts=(700,))
            for payload, expr in ((None, "column"), ("dt", "year")):
                ref = new_table(expected_rows=4096, unique=False)
                P.scan_build(vals, SCHEMA, [("i", "!=", 3)], ref, "k", payload=payload, payload_expr=expr, probe=(pref, "k2"))
                st = build_table(gpu_ctx, ref)
                rt().run_pipeline(gpu_ctx, "scan_build", src, filters=[("i", "!=", 3)], build_key="k", build_payload=payload,
                                  build_payload_expr=expr, probes=[(pst, "k2")], sink=st)
                assert rt().join_count(gpu_ctx, st) == ref.count()
                assert gpu_payloads(gpu_ctx, st, vals["k"]) == ref_payloads(ref, vals["k"]), (spec, expr)
                rt().state_destroy(gpu_ctx, st)
            rt().state_destroy(gpu_ctx, pst)


def test_year_payload_for_every_int32_day(gpu_ctx):
    days = [0, -1, 1, 10957, 11016, -719162, -719163, 2932896, 2932897, P.I32_MAX, P.I32_MIN, P.I32_MAX - 719468, P.I32_MAX - 719467,
            P.I32_MIN + 719468, -1 - 146097 * 5000] + [random.Random(2).randrange(-(1 << 31), 1 << 31) for _ in range(500)]
    vals = values(3, len(days), "tpch")
    vals["k"], vals["dt"] = list(range(len(days))), days
    ref = new_table(expected_rows=len(days))
    P.scan_build(vals, SCHEMA, [], ref, "k", payload="dt", payload_expr="year")
    st = build_table(gpu_ctx, ref)
    rt().run_pipeline(gpu_ctx, "scan_build", table(gpu_ctx, "y", vals), build_key="k", build_payload="dt", build_payload_expr="year", sink=st)
    assert gpu_payloads(gpu_ctx, st, vals["k"]) == ref_payloads(ref, vals["k"])
    rt().state_destroy(gpu_ctx, st)


# ---------------------------------------------------------------------------------------------------- K5 + top-k
def _group_join(gpu_ctx, n_groups, unique, agg, vals, filters, stages, spec, k):
    keys = keys_of("sparse", n_groups, 5) if n_groups > 64 else list(range(-20, n_groups - 20))
    bvals = values(6, len(keys), "tpch")
    # side0 = i // 3: three entries share each side0 (the copies of a multimap key never share one), so groups with equal sums are
    # ordered by side0 and then by key
    bvals["k"], bvals["k2"] = keys, [x % 5 for x in range(len(keys))]
    if not unique:
        bvals = {c: v + v[: len(v) // 2] for c, v in bvals.items()}
    bvals["i"] = [x // 3 for x in range(len(bvals["k"]))]
    ref = new_table(expected_rows=2 * len(bvals["k"]), unique=unique, n_side=2, n_aggs=1)
    P.scan_build(bvals, SCHEMA, [], ref, "k", payload="k2", side=["i", "k2"])
    vals = dict(vals)
    rng = random.Random(n_groups)
    ties = keys[:3]  # one side0 group: the same two rows each, so equal sums and equal side0
    probed = keys[3:]
    vals["k"] = [rng.choice(probed) if j % 4 else rng.randrange(-(1 << 31), 1 << 31) for j in range(len(vals["k"]))]
    for t in ties:
        for j in (0, 1):
            for c in vals:
                vals[c] = vals[c] + [t if c == "k" else vals[c][j]]
    P.probe_agg(vals, SCHEMA, filters, ref, "k", agg)
    with tuned(gpu_ctx, (3, stages, 3, 2, 2), spec):
        st = build_table(gpu_ctx, ref)
        rt().run_pipeline(gpu_ctx, "scan_build", table(gpu_ctx, "b", bvals), build_key="k", build_payload="k2", side=["i", "k2"], sink=st)
        src = table(gpu_ctx, "p", vals, cuts=(1001, 2500), device=(1,))  # 16-byte DEVICE decimals between narrowed HOST batches
        rt().run_pipeline(gpu_ctx, "scan_probe_agg", src, filters=filters, aggs=[agg], probes=[(st, "k")], sink=st)
        c = capi()
        rows, n, e = (c.TopKRow * 64)(), C.c_int32(), c.Error()
        c.check(gpu_ctx.L.ldb_gpu_join_table_topk(st, k, rows, C.byref(n), C.byref(e)), e)
        got = [(r.key, r.side[0], r.side[1], r.agg.value()) for r in rows[: n.value]]
        assert rt().join_count(gpu_ctx, st) == ref.count()
        rt().state_destroy(gpu_ctx, st)
    return got, P.topk(ref, k)


@pytest.mark.parametrize("agg", [("col", ["a"]), ("mul", ["a", "b"]), ("mul_1minus", ["a", "b"]), ("mul_1minus_1plus", ["a", "b", "c"])])
@pytest.mark.parametrize("mix", ["negative", "mixed", "wide"])
def test_probe_aggregate_topk(gpu_ctx, agg, mix):
    vals = values(31, 4000, mix)
    sets = [[], [("i", ">", -(1 << 30))], [("i", ">", -(1 << 30)), ("i", "<", 1 << 30)], [("a", ">=", 0)]]  # the last stages a decimal
    for stages in (2, 3, 4):
        for spec in (0, 1):
            for filters in filter_cases(sets, stages + spec, stages == 3 and spec == 1):  # shapes: 3 stages, specialisation on
                for n_groups, unique, k in ((40, True, 64), (3000, True, 10), (40, False, 64)):
                    got, want = _group_join(gpu_ctx, n_groups, unique, agg, vals, filters, stages, spec, k)
                    assert got == want, (stages, spec, filters, n_groups, unique)


# ---------------------------------------------------------------------------------------------------- K4
@pytest.mark.parametrize("agg", [("col", ["a"]), ("mul_1minus", ["a", "b"]), ("mul_1minus_1plus", ["a", "b", "c"])])
def test_probe_probe_groupby(gpu_ctx, agg):
    rng = random.Random(3)
    a_keys = keys_of("extremes", 300, 1)
    b_keys = keys_of("colliding", 200, 0)
    avals, bvals = values(1, 300, "tpch"), values(2, 200, "tpch")
    avals["k"], avals["i"] = a_keys, [rng.randrange(-3, 6) for _ in a_keys]
    bvals["k"], bvals["i"] = b_keys, [rng.randrange(-3, 6) for _ in b_keys]
    vals = values(7, 5000, "mixed")
    vals["k"] = [rng.choice(a_keys) for _ in range(5000)]
    vals["k2"] = [rng.choice(b_keys) for _ in range(5000)]
    sets = [[], [("dt", ">", "1900-01-01")], [("i", ">", -(1 << 30)), ("i", "<", 1 << 30)], [("a", ">=", 0)]]  # the last stages a decimal
    for stages in (2, 3, 4):
        for spec in (0, 1):
            for filters in filter_cases(sets, stages + spec, stages == 3 and spec == 1):  # shapes: 3 stages, specialisation on
                refs, sts = [], []
                with tuned(gpu_ctx, (3, 3, stages, 2, 2), spec):
                    for v, unique in ((avals, True), (bvals, False)):
                        ref = new_table(expected_rows=2048, unique=unique)
                        P.scan_build(v, SCHEMA, [], ref, "k", payload="i")
                        st = build_table(gpu_ctx, ref)
                        rt().run_pipeline(gpu_ctx, "scan_build", table(gpu_ctx, "b", v), build_key="k", build_payload="i", sink=st)
                        refs.append(ref)
                        sts.append(st)
                    want = P.probe2_groupby(vals, SCHEMA, filters, refs[0], "k", refs[1], "k2", agg)
                    g = rt().groupby_state(gpu_ctx, 1, 1, 64)
                    src = table(gpu_ctx, "p", vals, cuts=(2500,), device=(stages % 2,))  # one 16-byte DEVICE batch
                    rt().run_pipeline(gpu_ctx, "scan_probe2_groupby", src, filters=filters, aggs=[agg], probes=[(sts[0], "k"), (sts[1], "k2")], sink=g)
                    assert read_groups(gpu_ctx, g, 1) == want, (stages, spec, filters)
                    for s in sts + [g]:
                        rt().state_destroy(gpu_ctx, s)


def test_probe_probe_groupby_drops_only_the_marker_of_a_wide_table(gpu_ctx):
    """payload 5 in a table with side lanes must not match payload 5 | 2^31 of a plain table"""
    run = rt()
    a = run.join_table(gpu_ctx, 16, True, 1, 0)
    b = run.join_table(gpu_ctx, 16, True, 0, 0)
    ref_a, ref_b = new_table(expected_rows=16, n_side=1), new_table(expected_rows=16)
    for st, ref, pay in ((a, ref_a, [5, 6]), (b, ref_b, [5 - (1 << 31), 6])):
        v = values(1, 2, "tpch")
        v["k"], v["i"] = [1, 2], pay
        P.scan_build(v, SCHEMA, [], ref, "k", payload="i", side=["i"] if ref.n_side else ())
        run.run_pipeline(gpu_ctx, "scan_build", table(gpu_ctx, "b", v), build_key="k", build_payload="i", side=["i"] if ref.n_side else (), sink=st)
    vals = values(2, 10, "tpch")
    vals["k"], vals["k2"] = [1, 2] * 5, [1, 2] * 5
    g = run.groupby_state(gpu_ctx, 1, 1, 16)
    run.run_pipeline(gpu_ctx, "scan_probe2_groupby", table(gpu_ctx, "p", vals), aggs=[("col", ["a"])], probes=[(a, "k"), (b, "k2")], sink=g)
    assert read_groups(gpu_ctx, g, 1) == P.probe2_groupby(vals, SCHEMA, [], ref_a, "k", ref_b, "k2", ("col", ["a"]))
    for st in (a, b, g):
        run.state_destroy(gpu_ctx, st)


# ---------------------------------------------------------------------------------------------------- K9
def _star_case(gpu_ctx, seed, s_direct, o_direct, filters):
    """P: composite key (k, k2) → decimal payload; S on i → g0; O on fs → g1 (> 256 groups, including (-1, -1))"""
    rng = random.Random(seed)
    run = rt()
    pvals = values(seed, 700, "negative")
    pairs = list(dict.fromkeys((rng.randrange(-50, 50), rng.randrange(-3, 3)) for _ in range(700)))
    pairs = [p for p in pairs if p != (-1, -1)]
    pvals = {c: v[: len(pairs)] for c, v in pvals.items()}
    pvals["k"], pvals["k2"] = [p[0] for p in pairs], [p[1] for p in pairs]
    s_keys, o_keys = list(range(0, 40)), list(range(-30, 0))
    svals, ovals = values(seed + 1, len(s_keys), "tpch"), values(seed + 2, len(o_keys), "tpch")
    svals["i"], svals["k"] = s_keys, [-1 if x == 0 else x % 23 for x in s_keys]
    ovals["fs"], ovals["k"] = o_keys, [-1 if x == -30 else x % 17 for x in o_keys]
    refs, sts = [], []
    for v, kind, key, payload, k2 in ((pvals, "pair", "k", "a", "k2"), (svals, "direct" if s_direct else "hash", "i", "k", None),
                                     (ovals, "direct" if o_direct else "hash", "fs", "k", None)):
        ref = new_table(kind, expected_rows=1024, key_min=min(v[key]), key_max=max(v[key]))
        P.scan_build(v, SCHEMA, [], ref, key, payload=payload, key2=k2)
        st = build_table(gpu_ctx, ref)
        run.run_pipeline(gpu_ctx, "scan_build", table(gpu_ctx, "b", v, cuts=(257,) if kind == "pair" else ()), build_key=key, build_key2=k2,
                         build_payload=payload, sink=st)
        assert run.join_count(gpu_ctx, st) == ref.count()
        refs.append(ref)
        sts.append(st)
    vals = values(seed + 3, 6000, "mixed")
    vals["k"] = [rng.choice(pairs)[0] if j % 3 else rng.randrange(-60, 60) for j in range(6000)]
    vals["k2"] = [rng.choice(pairs)[1] if j % 3 else rng.randrange(-3, 3) for j in range(6000)]
    for j in range(0, 6000, 3):
        p = rng.choice(pairs)
        vals["k"][j], vals["k2"][j] = p
    vals["i"] = [rng.choice(s_keys) if j % 50 else 0 for j in range(6000)]  # every 50th row lands in the (-1, -1) group
    vals["fs"] = [rng.choice(o_keys) if j % 50 else -30 for j in range(6000)]
    want = P.star_probe_groupby(vals, SCHEMA, filters, refs[0], ("k", "k2"), refs[1], "i", refs[2], "fs", ("a", "b", "d"))
    g = run.groupby_state(gpu_ctx, 2, 1, 1024)
    run.run_pipeline(gpu_ctx, "scan_star_probe_groupby", table(gpu_ctx, "p", vals, cuts=(1025, 2049), device=(1,)), filters=filters,
                     aggs=[("mul_1minus_minus_paymul", ["a", "b", "d"])], probes=[(sts[0], "k", "k2"), (sts[1], "i"), (sts[2], "fs")], sink=g)
    got = read_groups(gpu_ctx, g, 1)
    for s in sts + [g]:
        run.state_destroy(gpu_ctx, s)
    return got, want


def test_star_probe_groupby(gpu_ctx):
    sets = [[], [("dt", ">", "1900-01-01")], [("k2", ">", -3), ("k2", "<=", 1)]]
    for stages in (2, 3, 4):
        for spec in (0, 1):
            for s_direct, o_direct in ((False, False), (True, True), (True, False)):
                # shapes: 2 stages, specialisation on (and 2 rows per thread, the default of LDB_RPT_STAR)
                for filters in filter_cases(sets, stages + spec + s_direct, stages == 2 and spec == 1):
                    with tuned(gpu_ctx, DEFAULT_TUNING[:3] + (stages,) + DEFAULT_TUNING[4:], spec):
                        got, want = _star_case(gpu_ctx, stages * 10 + spec, s_direct, o_direct, filters)
                    assert len(want) > 256 and (-1, -1) in want
                    assert got == want, (stages, spec, s_direct, o_direct, filters)


@pytest.mark.parametrize("rpt", ["1", "4"])
def test_star_probe_rows_per_thread(rpt):
    """K9's rows per thread is read from LDB_RPT_STAR once per process: the star cases again in a child process"""
    if os.environ.get("LDB_RPT_STAR"):
        pytest.skip("already inside the child process")
    env = dict(os.environ, LDB_RPT_STAR=rpt)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu", os.path.join(HERE, "test_gpu_pipelines.py") + "::test_star_probe_groupby"],
                       env=env, cwd=os.path.dirname(HERE), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "1 passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------- errors
def test_documented_errors(gpu_ctx):
    c, run = capi(), rt()
    vals = values(1, 40, "tpch")
    vals["k"], vals["i"] = list(range(40)), list(range(40))
    src = table(gpu_ctx, "e", vals)
    cases = [  # (table, build kwargs, rows override, code)
        (new_table(expected_rows=8), {}, {}, c.LDB_ERR_CAPACITY),  # 16 slots, 40 keys: full
        (new_table(expected_rows=64), {}, {"k": [3] * 40}, c.LDB_ERR_INVALID),  # duplicate in a unique table
        (new_table(expected_rows=64, unique=False), {}, {"k": [-1] * 40, "i": [-1] * 40}, c.LDB_ERR_UNSUPPORTED),  # (-1, -1)
        (new_table(expected_rows=64, n_side=1, n_aggs=1), {"side": ["i"]}, {"i": [x - 20 for x in range(40)]}, c.LDB_ERR_UNSUPPORTED),  # negative payload
        (new_table("direct", key_min=0, key_max=30), {}, {}, c.LDB_ERR_INVALID),  # key out of range
        (new_table("direct", key_min=0, key_max=50), {}, {"k": [x % 20 for x in range(40)]}, c.LDB_ERR_INVALID),  # duplicate direct key
    ]
    for ref, kw, over, code in cases:
        v = dict(vals, **over)
        P.scan_build(v, SCHEMA, [], ref, "k", payload="i", side=kw.get("side", ()))
        with pytest.raises(P.PipeError) as e:
            ref.count()
        assert e.value.code == code
        st = build_table(gpu_ctx, ref)
        run.run_pipeline(gpu_ctx, "scan_build", table(gpu_ctx, "e", v), build_key="k", build_payload="i", sink=st, **kw)
        expect_error(code, run.join_count, gpu_ctx, st)
        if ref.n_side:
            rows, n, err = (c.TopKRow * 4)(), C.c_int32(), c.Error()
            assert gpu_ctx.L.ldb_gpu_join_table_topk(st, 4, rows, C.byref(n), C.byref(err)) == code  # no partial answer either
        run.state_destroy(gpu_ctx, st)
    # group-by capacity: 17 groups in a 16-group state
    v = dict(vals, k=[x % 17 for x in range(40)])
    with pytest.raises(P.PipeError) as e:
        P.scan_groupby(v, SCHEMA, [], ["k"], [("col", ["a"]), ("one", [])], capacity=16)
    assert e.value.code == c.LDB_ERR_CAPACITY
    expect_error(c.LDB_ERR_CAPACITY, gpu_groupby, gpu_ctx, table(gpu_ctx, "g", v), ["k"], [("col", ["a"]), ("one", [])], capacity=16)
    # an aggregate signature no kernel is compiled for, and a filter constant beyond 64 bits
    for fn in (lambda: gpu_groupby(gpu_ctx, src, ["k"], [("mul", ["a", "b"])]),
               lambda: gpu_groupby(gpu_ctx, src, [], [("col", ["a"]), ("one", [])], [("a", "<", 1 << 62)]),
               lambda: gpu_groupby(gpu_ctx, src, [], [("col", ["a"]), ("one", [])], [("a", ">", -(1 << 61))])):
        expect_error(c.LDB_ERR_UNSUPPORTED, fn)
    with pytest.raises(P.PipeError):
        P.scan_groupby(vals, SCHEMA, [], ["k"], [("mul", ["a", "b"])])
    with pytest.raises(P.PipeError):
        P.filter_rows(vals, SCHEMA, [("a", "<", 1 << 62)])
    # a group-join map sums at one width: a 128-bit expression after a 64-bit COL is refused, and the COL lane stays readable
    ref = new_table(expected_rows=64, n_side=1, n_aggs=1)
    P.scan_build(vals, SCHEMA, [], ref, "k", payload="i", side=["i"])
    st = build_table(gpu_ctx, ref)
    run.run_pipeline(gpu_ctx, "scan_build", src, build_key="k", build_payload="i", side=["i"], sink=st)
    P.probe_agg(vals, SCHEMA, [], ref, "k", ("col", ["a"]))
    run.run_pipeline(gpu_ctx, "scan_probe_agg", src, aggs=[("col", ["a"])], probes=[(st, "k")], sink=st)
    with pytest.raises(P.PipeError) as e:
        P.probe_agg(vals, SCHEMA, [], ref, "k", ("mul", ["a", "b"]))
    assert e.value.code == c.LDB_ERR_UNSUPPORTED
    expect_error(c.LDB_ERR_UNSUPPORTED, run.run_pipeline, gpu_ctx, "scan_probe_agg", src, aggs=[("mul", ["a", "b"])], probes=[(st, "k")], sink=st)
    rows, n, err = (c.TopKRow * 64)(), C.c_int32(), c.Error()
    c.check(gpu_ctx.L.ldb_gpu_join_table_topk(st, 64, rows, C.byref(n), C.byref(err)), err)
    assert [(r.key, r.side[0], r.side[1], r.agg.value()) for r in rows[: n.value]] == P.topk(ref, 64)
    run.state_destroy(gpu_ctx, st)
