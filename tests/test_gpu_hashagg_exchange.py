"""The partitioned merge of program hash aggregations across ranks (ldb_gpu_hashagg_exchange, parallel.Comm.hashagg_exchange) against the
exact model of tests/_progref.py: every rank runs its shard's program into `local`, the exchange folds each group into `owned` on the
rank that owns its key hash, and the union of the ranks' `owned` states must be the aggregation over the whole input, bit for bit,
with no group on two ranks.  Also: skew, the receive capacity and its overflow, every documented error, and Q18 / Q6 at SF1 over
sharded lineitem against the reference's own answers.

Ranks are contexts of this process on device 0 wired by parallel.Comm.local_group.  The exchange waits for its peers on the host, so
each rank calls it from a thread of its own."""
import ctypes as C
import random
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import _progref as R
from lingodb_b200 import capi, datagen, dbgen, program as P, runtime
from test_gpu_exchange import SENTINEL, heap_fill, heap_read, ranks

pytestmark = pytest.mark.gpu
col, const = (lambda n: ("col", n)), (lambda v: ("const", v))
ENTRY_TAIL = 2 * 8 * 8  # cursors + counts behind the receive region

COLUMNS = [("k", "int32", 0, 0), ("g0", "int32", 0, 0), ("g1", "int64", 0, 0), ("g2", "int8", 0, 0), ("g3", "int16", 0, 0), ("v", "decimal128", 38, 0),
           ("w", "int64", 0, 0), ("f", "float64", 0, 0)]
# all nine aggregate kinds over two aggregate sets (at most eight aggregates per state)
AGG_SETS = [[("sum", "v"), ("count", "v"), ("count_star", None), ("min", "v"), ("max", "v"), ("any", "w"), ("sum_f64", "f"), ("min_f64", "f")],
            [("max_f64", "f"), ("count", "f"), ("min", "w"), ("max", "w"), ("sum", "w")]]


def gen(seed: int, n: int, domain: str) -> dict:
    """gen_values columns with nullable keys g0..g3 over a small ("small") or a wide ("wide") domain and integer-valued doubles f (their
    sums are exact in any order)"""
    v = R.gen_values(seed, n, COLUMNS, null_rate=0.12)
    rng = random.Random(seed)
    for k in range(4):
        g = v[f"g{k}"]
        if domain == "small":
            v[f"g{k}"] = [None if x is None else x % (2 + k) for x in g]
    v["f"] = [None if x is None else float(rng.randrange(-2**20, 2**20)) for x in v["f"]]
    return v


def stage(ctx, name, values, columns=COLUMNS, cuts=()):
    return ctx.table_from_host(R.to_table_data(name, values, columns, cuts))


def shard_bounds(n: int, world: int, seed: int) -> list:
    """ragged row ranges [lo, hi) of `world` ranks; with more than one rank, one of them is empty"""
    rng = random.Random(seed)
    b = [0] + sorted(rng.randrange(n + 1) for _ in range(world - 1)) + [n]
    if world > 1:
        e = rng.randrange(world)
        if e + 1 < world:
            b[e + 1] = b[e]
        else:
            b[e] = n
    return list(zip(b, b[1:]))


def slice_values(v: dict, lo: int, hi: int) -> dict:
    return {c: x[lo:hi] for c, x in v.items()}


def exchange_all(comms, locals_, owneds, capacity=None, recv_offset=0):
    """every rank's exchange, one thread per rank; returns each rank's exception (None = success)"""
    def one(r):
        try:
            comms[r].hashagg_exchange(locals_[r], owneds[r], capacity=capacity, recv_offset=recv_offset)
            return None
        except capi.LdbRuntimeError as e:
            return e
    with ThreadPoolExecutor(len(comms)) as ex:
        return list(ex.map(one, range(len(comms))))


def exchange_ok(comms, locals_, owneds, **kw):
    errs = exchange_all(comms, locals_, owneds, **kw)
    assert errs == [None] * len(comms), [str(e) for e in errs]


def count(ctx, st) -> int:
    n, e = C.c_int64(), capi.Error()
    capi.check(ctx.L.ldb_gpu_hashagg_count(st, C.byref(n), C.byref(e)), e)
    return n.value


def read(ctx, st, n_keys, aggs):
    f64 = tuple(i for i, (k, _) in enumerate(aggs) if k.endswith("_f64"))
    return P.decode_groups(P.read_groups(ctx, st, max(count(ctx, st), 1)), n_keys, len(aggs), f64_aggs=f64)


def assert_rows(got: dict, want: dict, aggs, what=""):
    assert set(got) == set(want), what
    for g, w in want.items():
        for i, (kind, _) in enumerate(aggs):
            if kind == "any":
                assert (got[g][i] is None and w[i] is None) or got[g][i] in w[i], (what, g, kind)
            else:
                assert got[g][i] == w[i], (what, g, kind, got[g][i], w[i])


def run_ranks(ctxs, comms, shards, keys, aggs, expected, capacity=None, destroy=True):
    """each rank's program into its `local`, then the exchange; returns (locals, owneds, per-rank owned groups)"""
    locals_, owneds = [], []
    for r, (c, tab) in enumerate(zip(ctxs, shards)):
        st = P.hashagg_state(c, len(keys), [k for k, _ in aggs], expected)
        if tab is not None:
            P.group_by(c, tab, [col(k) for k in keys], [(k, None if x is None else col(x)) for k, x in aggs], state=st)
        locals_.append(st)
        owneds.append(P.hashagg_state(c, len(keys), [k for k, _ in aggs], expected))
    exchange_ok(comms, locals_, owneds, capacity=capacity)
    got = [read(c, o, len(keys), aggs) for c, o in zip(ctxs, owneds)]
    if destroy:
        for c, a, b in zip(ctxs, locals_, owneds):
            c.L.ldb_gpu_state_destroy(a)
            c.L.ldb_gpu_state_destroy(b)
    return locals_, owneds, got


def union_disjoint(parts: list) -> dict:
    out = {}
    for p in parts:
        for g, row in p.items():
            assert g not in out, ("group on two ranks", g)
            out[g] = row
    return out


def want_of(v: dict, keys, aggs) -> dict:
    n = len(v["k"])
    return R.group_by(n, [v[k] for k in keys], [(k, None if x is None else v[x]) for k, x in aggs])


# ---------------------------------------------------------------------------------------------------- 1. exact against the model
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_exchange_matches_the_model(world):
    n = 2400 if world < 8 else 4000
    with ranks(world, user_bytes=8 << 20) as (ctxs, comms):
        for domain in ("small", "wide"):
            v = gen(70 + world, n, domain)
            bounds = shard_bounds(n, world, world * 13 + len(domain))
            shards = [stage(c, f"s{r}", slice_values(v, lo, hi), cuts=((hi - lo) // 3,) if hi - lo > 3 else ()) if hi > lo else None
                      for r, (c, (lo, hi)) in enumerate(zip(ctxs, bounds))]
            assert world == 1 or any(s is None for s in shards)
            for n_keys in range(5):
                keys = [f"g{k}" for k in range(n_keys)]
                for aggs in AGG_SETS:
                    want = want_of(v, keys, aggs)
                    _, _, got = run_ranks(ctxs, comms, shards, keys, aggs, expected=n)
                    what = (world, domain, n_keys, aggs[0][0])
                    if n_keys == 0:
                        for g in got:  # the keyless row on every rank
                            assert_rows(g, want, aggs, what)
                    else:
                        assert_rows(union_disjoint(got), want, aggs, what)
                        if domain == "wide" and world > 1:
                            assert sum(1 for g in got if g) > 1, what  # the groups really spread over the ranks
                    if n_keys == 2 and aggs is AGG_SETS[0]:
                        assert any(None in g for g in want), what  # NULL keys
                        assert domain == "small" or any(w[0] is None for w in want.values()), what  # NULL aggregates


def test_through_the_all_gather_of_the_counts():
    """without a capacity and without the in-process host barrier, the ranks share their group counts with the small all-gather"""
    world = 3
    with ranks(world, user_bytes=8 << 20) as (ctxs, comms):
        v = gen(5, 3000, "wide")
        shards = [stage(c, f"s{r}", slice_values(v, lo, hi)) for r, (c, (lo, hi)) in enumerate(zip(ctxs, [(0, 1000), (1000, 2500), (2500, 3000)]))]
        for cm in comms:
            cm._local = None
        keys, aggs = ["g0", "g1"], AGG_SETS[0]
        _, _, got = run_ranks(ctxs, comms, shards, keys, aggs, expected=3000)
        assert_rows(union_disjoint(got), want_of(v, keys, aggs), aggs)


# ---------------------------------------------------------------------------------------------------- 2. spread and skew
def test_every_rank_holds_every_group_and_a_second_exchange_accumulates():
    world, aggs = 4, AGG_SETS[0]
    with ranks(world, user_bytes=8 << 20) as (ctxs, comms):
        vs = []
        for r in range(world):
            v = gen(200 + r, 1500, "small")
            v["g0"] = [i % 300 for i in range(1500)]  # all 300 groups on every rank
            vs.append(v)
        whole = {c: sum((v[c] for v in vs), []) for c in vs[0]}
        shards = [stage(c, f"s{r}", v) for r, (c, v) in enumerate(zip(ctxs, vs))]
        locals_, owneds, got = run_ranks(ctxs, comms, shards, ["g0"], aggs, expected=512, destroy=False)
        assert_rows(union_disjoint(got), want_of(whole, ["g0"], aggs), aggs)
        exchange_ok(comms, locals_, owneds)  # the same partial states once more: counts and sums double, MIN / MAX / ANY stay
        twice = {c: x + x for c, x in whole.items()}
        got2 = union_disjoint([read(c, o, 1, aggs) for c, o in zip(ctxs, owneds)])
        assert_rows(got2, want_of(twice, ["g0"], aggs), aggs)
        for c, a, b in zip(ctxs, locals_, owneds):
            c.L.ldb_gpu_state_destroy(a)
            c.L.ldb_gpu_state_destroy(b)


def test_one_key_goes_to_one_owner():
    world, aggs = 3, AGG_SETS[1]
    with ranks(world) as (ctxs, comms):
        vs = [gen(300 + r, 800, "small") for r in range(world)]
        for v in vs:
            v["g1"] = [-12345] * 800
        whole = {c: sum((v[c] for v in vs), []) for c in vs[0]}
        _, _, got = run_ranks(ctxs, comms, [stage(c, f"s{r}", v) for r, (c, v) in enumerate(zip(ctxs, vs))], ["g1"], aggs, expected=8)
        assert sorted(len(g) for g in got) == [0, 0, 1]
        assert_rows(union_disjoint(got), want_of(whole, ["g1"], aggs), aggs)


def test_owner_bits_are_uniform_over_1_5_million_keys():
    world, n = 3, 1_500_000
    with ranks(world, user_bytes=64 << 20) as (ctxs, comms):
        locals_, owneds = [], []
        for r, c in enumerate(ctxs):
            td = datagen.TableData(f"keys{r}", [datagen.ColumnSpec("key", "int64", 0, 0)])
            lo, hi = n * r // world, n * (r + 1) // world
            td.chunks.append({"key": np.arange(lo, hi, dtype=np.int64) * 7919 + 3})
            td.chunk_rows.append(hi - lo)
            tab = c.table_from_host(td)
            locals_.append(P.group_by(c, tab, [col("key")], [("count_star", None)], expected_groups=hi - lo))
            owneds.append(P.hashagg_state(c, 1, ["count_star"], n // 2))
        exchange_ok(comms, locals_, owneds, capacity=n // world // 2)
        shares = [count(c, o) / n for c, o in zip(ctxs, owneds)]
        assert abs(sum(shares) - 1.0) < 1e-12
        assert all(0.32 <= s <= 0.347 for s in shares), shares


# ---------------------------------------------------------------------------------------------------- 3. capacity and errors
def test_capacity_overflow_keeps_the_heap_outside_the_claimed_ranges_and_a_retry_succeeds():
    world, aggs, recv = 3, AGG_SETS[0], 4096
    entry = 48 + 16 * len(aggs)
    with ranks(world, user_bytes=8 << 20) as (ctxs, comms):
        vs = [gen(400 + r, 900, "wide") for r in range(world)]
        whole = {c: sum((v[c] for v in vs), []) for c in vs[0]}
        shards = [stage(c, f"s{r}", v) for r, (c, v) in enumerate(zip(ctxs, vs))]
        keys = ["g1", "g3"]

        def fresh(expected):
            return [P.hashagg_state(c, 2, [k for k, _ in aggs], expected) for c in ctxs]
        locals_ = fresh(2048)
        for c, tab, st in zip(ctxs, shards, locals_):
            P.group_by(c, tab, [col(k) for k in keys], [(k, None if x is None else col(x)) for k, x in aggs], state=st)
        named = lambda e: int(re.search(r"retry with capacity (\d+)", str(e)).group(1))
        errs = exchange_all(comms, locals_, fresh(2048), capacity=0, recv_offset=recv)  # everybody received something: every rank fails
        assert all(e is not None and e.code == capi.LDB_ERR_CAPACITY for e in errs), errs
        need = max(named(e) for e in errs)
        cap = need - 1
        region = world * cap * entry
        for cm in comms:
            heap_fill(cm, recv - 1024, 1024 + region + ENTRY_TAIL + 4096)
        errs = exchange_all(comms, locals_, fresh(2048), capacity=cap, recv_offset=recv)
        failed = [r for r, e in enumerate(errs) if e is not None]
        assert failed and all(errs[r].code == capi.LDB_ERR_CAPACITY and named(errs[r]) == need for r in failed), errs
        for d, cm in enumerate(comms):  # every byte outside the claimed ranges (and the cursors / counts) still holds the sentinel
            raw = np.frombuffer(heap_read(cm, recv - 1024, 1024 + region + ENTRY_TAIL + 4096), dtype=np.uint32).copy()
            counts = np.frombuffer(heap_read(cm, recv + region + 64, 8 * world), dtype=np.uint64)
            base = 1024 // 4
            for s in range(world):
                at = base + s * cap * entry // 4
                raw[at: at + min(int(counts[s]), cap) * entry // 4] = SENTINEL
            raw[base + region // 4: base + (region + ENTRY_TAIL) // 4] = SENTINEL
            assert (raw == SENTINEL).all(), d
            assert (max(int(x) for x in counts) > cap) == (d in failed)
        owneds = fresh(2048)
        exchange_ok(comms, locals_, owneds, capacity=need, recv_offset=recv)
        got = union_disjoint([read(c, o, 2, aggs) for c, o in zip(ctxs, owneds)])
        assert_rows(got, want_of(whole, keys, aggs), aggs)


def test_an_owned_state_too_small_fails_through_its_count():
    world = 2
    with ranks(world) as (ctxs, comms):
        v = gen(9, 3000, "wide")
        v["g1"] = list(range(3000))
        tabs = [stage(c, f"s{r}", slice_values(v, 1500 * r, 1500 * (r + 1))) for r, c in enumerate(ctxs)]
        locals_ = [P.group_by(c, t, [col("g1")], [("count_star", None)], expected_groups=2048) for c, t in zip(ctxs, tabs)]
        owneds = [P.hashagg_state(c, 1, ["count_star"], 8) for c in ctxs]
        exchange_ok(comms, locals_, owneds)
        for c, o in zip(ctxs, owneds):
            with pytest.raises(capi.LdbRuntimeError) as e:
                count(c, o)
            assert e.value.code == capi.LDB_ERR_CAPACITY and "full" in str(e.value)


def test_documented_errors():
    with ranks(2, user_bytes=1 << 20) as (ctxs, comms):
        c, cm = ctxs[0], comms[0]
        L = c.L
        mk = lambda ctx, nk, kinds: P.hashagg_state(ctx, nk, kinds, 64)
        a = mk(c, 1, ["sum", "count"])
        others = {"key count": mk(c, 2, ["sum", "count"]), "aggregate count": mk(c, 1, ["sum"]), "aggregate kinds": mk(c, 1, ["sum", "count_star"]),
                  "same state": a, "other context": mk(ctxs[1], 1, ["sum", "count"]), "not a hash aggregation": runtime.join_table(c, 64, unique=True)}

        def call(local, owned, off=0, cap=16, comm=cm):
            e = capi.Error()
            return L.ldb_gpu_hashagg_exchange(local, owned, comm.h, off, cap, C.byref(e)), e
        for what, o in others.items():
            rc, e = call(a, o)
            assert rc == capi.LDB_ERR_INVALID, (what, e.message)
            if what not in ("same state",):
                rc, e = call(o, a)
                assert rc == capi.LDB_ERR_INVALID, (what, "swapped", e.message)
        b = mk(c, 1, ["sum", "count"])
        user = cm.heap()[1]
        for off, cap in ((user, 1), (user - 64, 1), (8, 1), (-16, 1), (0, -1), (0, user // 64), (0, 1 << 62)):
            rc, e = call(a, b, off, cap)
            assert rc == capi.LDB_ERR_INVALID, (off, cap, e.message)
        c.graph_begin()
        rc, e = call(a, b)
        c.graph_end().destroy()
        assert rc == capi.LDB_ERR_UNSUPPORTED, e.message
        rc, e = call(None, b)
        assert rc == capi.LDB_ERR_INVALID


# ---------------------------------------------------------------------------------------------------- 4. Q18 and Q6 at SF1
@pytest.fixture(scope="module")
def sf1():
    return dbgen.tpch(1.0, extended=True)


def _chunks(td, idx, name):
    out = datagen.TableData(name, td.columns)
    for i in idx:
        out.chunks.append(td.chunks[i])
        out.chunk_rows.append(td.chunk_rows[i])
    return out


@pytest.mark.parametrize("world", [2, 3])
def test_q18_and_q6_over_sharded_lineitem_reproduce_the_reference(sf1, oracle, world):
    from test_reference_answers_sf1 import GOLD, day, dec
    li = sf1["lineitem"]
    okeys = [c["l_orderkey"] for c in li.chunks]
    # batches cut lineitem inside orders: the same order's lines sit on two ranks, so the exchange merges partial sums
    assert sum(1 for i in range(1, len(okeys)) if okeys[i][0] == okeys[i - 1][-1]) > world
    with ranks(world, user_bytes=256 << 20) as (ctxs, comms):
        lis = [c.table_from_host(_chunks(li, range(r, len(li.chunks), world), f"li{r}")) for r, c in enumerate(ctxs)]
        ods = [c.table_from_host(sf1["orders"]) for c in ctxs]  # replicated
        locals_ = [P.group_by(c, t, [col("l_orderkey")], [("sum", col("l_quantity"))], expected_groups=1_600_000) for c, t in zip(ctxs, lis)]
        owneds = [P.hashagg_state(c, 1, ["sum"], 1_600_000) for c in ctxs]
        exchange_ok(comms, locals_, owneds)
        assert sum(count(c, o) for c, o in zip(ctxs, owneds)) == 1_500_000
        rows = []
        for c, o, od in zip(ctxs, owneds, ods):  # HAVING on the owned partition, semi join with the replicated orders, per-rank top 100
            groups = P.groups_table(c, o)
            big = runtime.join_table(c, 4096, unique=True)
            P.build_join(c, groups, big, col("k0"), payload=col("a0"), where=("cmp", ">", col("a0"), const(30000)))
            pb = ("probe", big, col("o_orderkey"))
            mt = P.RawTable(c, P.materialize(c, od, [col("o_custkey"), col("o_orderkey"), col("o_orderdate"), col("o_totalprice"), pb], where=("not", ("isnull", pb))))
            ids = mt.order_by("c3", descending=True)
            rows += list(zip(*[mt.gather(f"c{i}", ids) for i in range(5)]))
            mt.destroy()
            groups.destroy()
            c.L.ldb_gpu_state_destroy(big)
        rows.sort(key=lambda r: (-r[3], r[2]))
        got18 = [["Customer#%09d" % r[0], str(r[0]), str(r[1]), day(r[2]), dec(r[3], 2), dec(r[4], 2)] for r in rows[:100]]
        assert got18 == GOLD["q18_rows"]
        # Q6 as a keyless program over the same shards: every rank's owned row is the whole answer
        lo, hi = oracle.lib.oracle_parse_date(b"1994-01-01"), oracle.lib.oracle_parse_date(b"1995-01-01")
        where = ("and", ("and", ("cmp", ">=", col("l_shipdate"), const(lo)), ("cmp", "<", col("l_shipdate"), const(hi))),
                 ("and", ("between", col("l_discount"), const(5), const(7)), ("cmp", "<", col("l_quantity"), const(2400))))
        aggs = [("sum", ("mul", col("l_extendedprice"), col("l_discount")))]
        q6l = [P.group_by(c, t, [], aggs, where=where) for c, t in zip(ctxs, lis)]
        q6o = [P.hashagg_state(c, 0, ["sum"], 1) for c in ctxs]
        exchange_ok(comms, q6l, q6o)
        want = oracle.q6(oracle.table(li))[0]["revenue"]
        assert dec(want, 4) == GOLD["q6"]
        for c, o in zip(ctxs, q6o):
            assert P.decode_groups(P.read_groups(c, o, 4), 0, 1)[()][0] == want
        assert all(P.decode_groups(P.read_groups(c, s, 4), 0, 1)[()][0] != want for c, s in zip(ctxs, q6l))  # no rank had it alone
