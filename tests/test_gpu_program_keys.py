"""Key-tuple join tables in program pipelines (LDB_STATE_KEY_JOIN, csrc/program.cu): 1-4 int64 keys → int64 payload, built by the
JOIN_BUILD sink and read by PROBE / PROBE_EACH — against a plain-Python multimap model, on ragged multi-batch tables with NULLs in every
key position on both sides, int64 edge keys and payloads, tuples that differ in one component only (with colliding hash tags), and every
documented failure."""
import ctypes as C
import json
import random
import time
from collections import Counter

import numpy as np
import pytest

import _keyhash as K

from lingodb_b200 import capi, datagen, parallel, program as P, runtime

pytestmark = pytest.mark.gpu

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
EDGE = [I64_MIN, -1, 0, 1 << 31, I64_MAX]
M64 = (1 << 64) - 1


class Multimap:
    """The model: key tuple → payloads of its build rows.  A tuple with a NULL component is never stored and never matches; a unique
    table keeps one of its duplicates' payloads (which one is unspecified)."""

    def __init__(self, unique):
        self.unique, self.d = unique, {}

    def insert(self, key, payload):
        if None not in key:
            self.d.setdefault(key, []).append(payload)

    def count(self):
        return len(self.d) if self.unique else sum(map(len, self.d.values()))

    def matches(self, key):
        return [] if None in key else self.d.get(key, [])


def _table(ctx, name, cols, valid, cuts):
    """int64 columns cut into ragged batches at `cuts`, with Arrow validity bitmaps for the columns in `valid`"""
    td = datagen.TableData(name, [datagen.ColumnSpec(k, "int64") for k in cols])
    n = len(next(iter(cols.values())))
    edges = [0] + list(cuts) + [n]
    for a, b in zip(edges, edges[1:]):
        ch = {k: np.ascontiguousarray(v[a:b]) for k, v in cols.items()}
        for k, v in valid.items():
            ch[k + "$valid"] = np.packbits(v[a:b], bitorder="little")
        td.chunks.append(ch)
        td.chunk_rows.append(b - a)
    return ctx.table_from_host(td)


def _cuts(n):
    return (n // 7, n // 2, n - n // 5)


def _keys_of(cols, valid, n_keys, i):
    return tuple(int(cols[f"k{j}"][i]) if valid[f"k{j}"][i] else None for j in range(n_keys))


def _read(ctx, out_h, n_cols):
    out = P.RawTable(ctx, out_h)
    ids = list(range(out.num_rows))
    rows = list(zip(*[out.gather(f"c{c}", ids) for c in range(n_cols)])) if ids else []
    out.destroy()
    return rows


def _tuple_hash(cols):
    """the table's placement hash (csrc/keyhash.cuh keyTupleHash, seed 0) over int64 key columns, vectorised"""
    return K.key_tuple_hash_np([np.asarray(c).astype(np.int64) for c in cols])


def _tag_twins(prefix, rng):
    """two values v1 != v2 such that the tuples prefix + (v1,) and prefix + (v2,) share their 32-bit hash tag and their slot in a
    16-slot directory: a probe for one meets the other's entry with an equal tag, so only a compare of the LAST component tells them
    apart"""
    n = 1 << 21
    last = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
    cols = [np.full(n, v, dtype=np.int64) for v in prefix] + [last]
    h = _tuple_hash(cols)
    sig = (h >> np.uint64(32)) * np.uint64(16) + (h & np.uint64(15))
    order = np.argsort(sig, kind="stable")
    s = sig[order]
    dup = np.flatnonzero((s[1:] == s[:-1]) & (last[order[1:]] != last[order[:-1]]))
    assert len(dup), "no tag twins found"
    i = dup[0]
    return int(last[order[i]]), int(last[order[i + 1]])


def _probe_runs(h, cap):
    """linear probing of entries with placement hashes h into `cap` slots (the order of inserts does not change it): the longest
    displacement of an entry from its home slot, and the longest run of occupied slots (what a probe for an absent tuple walks)"""
    n = np.bincount((h & np.uint64(cap - 1)).astype(np.int64), minlength=cap)
    n = np.concatenate([n, n])  # two laps: runs that wrap past the last slot
    s = np.cumsum(n - 1)
    carry = s - np.minimum(np.minimum.accumulate(s), 0)  # entries still waiting for a slot after slot i (Lindley's recursion)
    occ = np.concatenate([[0], carry[:-1]]) + n > 0
    d = np.diff(np.concatenate([[0], occ.astype(np.int8), [0]]))
    return int(carry.max()), int((np.flatnonzero(d == -1) - np.flatnonzero(d == 1)).max())


def _edge_data(n_keys, seed):
    """build and probe sides over edge values: base tuples with 1-5 duplicates, tuples that share every component but one with a
    present tuple, NULLs in each key position (over cells that hold a present tuple's values) on both sides"""
    rng = np.random.default_rng(seed)
    pyr = random.Random(seed)

    def value():
        return pyr.choice(EDGE) if pyr.random() < 0.6 else int(rng.integers(-(1 << 40), 1 << 40))

    base = list({tuple(value() for _ in range(n_keys)) for _ in range(400)})
    near = []
    for t in base[:150]:
        for j in range(n_keys):
            v = list(t)
            v[j] = value() if pyr.random() < 0.5 else (t[j] + 1 if t[j] != I64_MAX else t[j] - 1)
            near.append(tuple(v))
    present = base + near[::2]
    absent = near[1::2]
    brows = []
    for t in present:
        brows += [t] * pyr.randint(1, 5)
    pyr.shuffle(brows)
    prows = [pyr.choice(present) for _ in range(3000)] + absent * 3
    pyr.shuffle(prows)

    def side(rows, null_rate):
        n = len(rows)
        cols = {f"k{j}": np.array([r[j] for r in rows], dtype=np.int64) for j in range(n_keys)}
        valid = {f"k{j}": rng.random(n) > null_rate for j in range(n_keys)}
        return cols, valid

    bcols, bvalid = side(brows, 0.04)
    pcols, pvalid = side(prows, 0.04)
    pays = np.array([pyr.choice(EDGE + [int(rng.integers(I64_MIN, I64_MAX))]) for _ in brows], dtype=np.int64)
    return bcols, bvalid, pays, pcols, pvalid


@pytest.mark.parametrize("unique", [True, False], ids=["unique", "multimap"])
@pytest.mark.parametrize("n_keys", [1, 2, 3, 4])
def test_edge_keys_payloads_and_nulls(gpu_ctx, n_keys, unique):
    ctx = gpu_ctx
    bcols, bvalid, pays, pcols, pvalid = _edge_data(n_keys, 100 + n_keys)
    nb, na = len(pays), len(pcols["k0"])
    B = _table(ctx, "b", dict(bcols, pay=pays), bvalid, _cuts(nb))
    A = _table(ctx, "a", pcols, pvalid, _cuts(na))
    keys = [col(f"k{j}") for j in range(n_keys)]
    model, rows_model = Multimap(unique), Multimap(unique)
    for i in range(nb):
        k = _keys_of(bcols, bvalid, n_keys, i)
        model.insert(k, int(pays[i]))
        rows_model.insert(k, i)
    kt = runtime.join_table_keys(ctx, n_keys, nb, unique=unique)
    P.build_join(ctx, B, kt, keys, payload=col("pay"))
    kr = runtime.join_table_keys(ctx, n_keys, nb, unique=unique, bloom=False)
    P.build_join(ctx, B, kr, keys, payload=("rowid",))
    try:
        assert runtime.join_count(ctx, kt) == model.count() and runtime.join_count(ctx, kr) == model.count()
        probe_keys = [_keys_of(pcols, pvalid, n_keys, i) for i in range(na)]
        # PROBE: one payload of the tuple, NULL when absent
        for r, (row, got) in enumerate(sorted(_read(ctx, P.materialize(ctx, A, [("rowid",), ("probe", kt, *keys)]), 2))):
            assert row == r
            want = model.matches(probe_keys[r])
            assert (got is None) if not want else got in want, (probe_keys[r], got, want)
        # PROBE_EACH over the row-id table: the build rows of every match, each with exactly the probe's tuple
        got = Counter(_read(ctx, P.materialize(ctx, A, [("rowid",), ("probe_each", kr, *keys)]), 2))
        if unique:
            assert sum(got.values()) == sum(1 for k in probe_keys if model.matches(k))
            for (r, b), c in got.items():
                assert c == 1 and b in rows_model.matches(probe_keys[r])
        else:
            assert got == Counter((r, b) for r, k in enumerate(probe_keys) for b in rows_model.matches(k))
        # PROBE_EACH over the payload table, outer: every payload of a match, one NULL tuple for a row without any
        got = Counter(_read(ctx, P.materialize(ctx, A, [("rowid",), ("probe_each", kt, *keys, "outer")]), 2))
        want = Counter()
        for r, k in enumerate(probe_keys):
            m = model.matches(k)
            if not m:
                want[(r, None)] += 1
            elif not unique:
                for v in m:
                    want[(r, v)] += 1
        if unique:
            assert Counter(k for k in got.elements() if k[1] is None) == want
            assert all(c == 1 and v in model.matches(probe_keys[r]) for (r, v), c in got.items() if v is not None)
            assert sum(got.values()) == na
        else:
            assert got == want
    finally:
        for s in (kt, kr):
            runtime.state_destroy(ctx, s)
        A.clear()
        B.clear()


@pytest.mark.parametrize("n_keys", [1, 2, 3, 4])
def test_tag_twins_are_told_apart_by_their_last_component(gpu_ctx, n_keys):
    """a 16-slot table holding prefix + (a,) probed for prefix + (b,), where both tuples have the same tag and home slot: the probe meets
    the entry with its own tag, and only the compare of the last key rejects it"""
    ctx = gpu_ctx
    rng = np.random.default_rng(40 + n_keys)
    prefix = tuple(EDGE[:n_keys - 1])
    a, b = _tag_twins(prefix, rng)
    rows = [prefix + (a,), prefix + (b,), prefix + (a,)]
    cols = {f"k{j}": np.array([r[j] for r in rows], dtype=np.int64) for j in range(n_keys)}
    T = _table(ctx, "t", dict(cols, pay=np.array([11, 22, 33], dtype=np.int64)), {}, ())
    keys = [col(f"k{j}") for j in range(n_keys)]
    for unique in (True, False):
        kt = runtime.join_table_keys(ctx, n_keys, 8, unique=unique)  # 16 slots
        P.build_join(ctx, T, kt, keys, payload=col("pay"), where=("cmp", "!=", col("pay"), const(22)))
        assert runtime.join_count(ctx, kt) == (1 if unique else 2)
        got = sorted(_read(ctx, P.materialize(ctx, T, [("rowid",), ("probe", kt, *keys)]), 2))
        assert got[1] == (1, None) and got[0][1] in (11, 33) and got[2][1] in (11, 33)
        each = Counter(_read(ctx, P.materialize(ctx, T, [("rowid",), ("probe_each", kt, *keys, "outer")]), 2))
        assert each[(1, None)] == 1 and sum(c for (r, _), c in each.items() if r == 1) == 1
        runtime.state_destroy(ctx, kt)
    T.clear()


def test_probe_each_duplicates_outer_and_regrow(gpu_ctx):
    """2 keys, 1-40 duplicates per tuple, NULL keys on both sides, ragged batches; inner and outer PROBE_EACH whose materialize regrows
    far past the probe side's rows; row-id payloads read back as side columns"""
    ctx = gpu_ctx
    rng = np.random.default_rng(7)
    tuples = np.unique(rng.integers(0, 400, (2600, 2)), axis=0)[:2000] * np.array([1 << 33, -3], dtype=np.int64)
    dup = rng.integers(1, 41, len(tuples))
    rows = np.repeat(tuples, dup, axis=0)
    rows = rows[rng.permutation(len(rows))]
    nb = len(rows)
    bcols = {"k0": rows[:, 0].copy(), "k1": rows[:, 1].copy(), "pay": rng.integers(I64_MIN, I64_MAX, nb, dtype=np.int64)}
    bvalid = {"k0": rng.random(nb) > 0.03, "k1": rng.random(nb) > 0.03}
    na = 20_011
    pick = tuples[rng.integers(0, len(tuples), na)]
    pick[rng.random(na) < 0.2, 1] += 1  # misses that share key 0 with a present tuple
    pcols = {"k0": pick[:, 0].copy(), "k1": pick[:, 1].copy()}
    pvalid = {"k0": rng.random(na) > 0.05, "k1": rng.random(na) > 0.05}
    B = _table(ctx, "b", bcols, bvalid, _cuts(nb))
    A = _table(ctx, "a", pcols, pvalid, (1, 4_999, 17_000))
    kt = runtime.join_table_keys(ctx, 2, nb, unique=False)
    P.build_join(ctx, B, kt, [col("k0"), col("k1")], payload=("rowid",))
    model = Multimap(False)
    for i in range(nb):
        model.insert(_keys_of(bcols, bvalid, 2, i), i)
    pk = [_keys_of(pcols, pvalid, 2, i) for i in range(na)]
    try:
        assert runtime.join_count(ctx, kt) == model.count()
        for outer in (False, True):
            m = ("probe_each", kt, col("k0"), col("k1"), *(("outer",) if outer else ()))
            got = Counter(_read(ctx, P.materialize(ctx, A, [("rowid",), m, ("fetch", B, m, "pay")]), 3))
            want = Counter()
            for r, k in enumerate(pk):
                ms = model.matches(k)
                for b in ms:
                    want[(r, b, int(bcols["pay"][b]))] += 1
                if outer and not ms:
                    want[(r, None, None)] += 1
            assert sum(want.values()) > 10 * na
            assert got == want
    finally:
        runtime.state_destroy(ctx, kt)
        A.clear()
        B.clear()


def test_correlated_partsupp_pairs_at_sf1_size(gpu_ctx):
    """(ps_partkey, ps_suppkey) of TPC-H SF1: 800 000 pairs whose suppliers follow the part key.  Every pair finds its own row, every
    pair shifted by one supplier misses.  The placement hash keeps their probe runs short: in the table's 2^21 slots no entry lies more
    than 32 slots from its home and no run of occupied slots passes 128 (7 and 30 with the mix64 tuple hash; the reference's XOR combine
    of per-key hashes gives 281 and 1 230 on these pairs)."""
    ctx = gpu_ctx
    P_, S = 200_000, 10_000
    p = np.repeat(np.arange(1, P_ + 1, dtype=np.int64), 4)
    i = np.tile(np.arange(4, dtype=np.int64), P_)
    s = (p + i * (S // 4 + (p - 1) // S)) % S + 1
    displacement, cluster = _probe_runs(_tuple_hash([p, s]), 1 << 21)
    assert displacement <= 32 and cluster <= 128, (displacement, cluster)
    T = _table(ctx, "ps", {"p": p, "s": s}, {}, (300_000, 600_000))
    kt = runtime.join_table_keys(ctx, 2, len(p))
    P.build_join(ctx, T, kt, [col("p"), col("s")], payload=("rowid",))
    try:
        assert runtime.join_count(ctx, kt) == len(p)
        own = ("probe", kt, col("p"), col("s"))
        shifted = ("probe", kt, col("p"), ("add", col("s"), const(S)))
        st = P.group_by(ctx, T, [], [("count", own), ("sum", ("case", ("cmp", "=", own, ("rowid",)), const(1), const(0))), ("count", shifted)])
        got = P.decode_groups(P.read_groups(ctx, st, 4), 0, 3)[()]
        runtime.state_destroy(ctx, st)
        assert got == [len(p), len(p), 0]
    finally:
        runtime.state_destroy(ctx, kt)
        T.clear()


def test_keys_and_payloads_outside_int64(gpu_ctx):
    """a build key or payload past int64 fails the build (LDB_ERR_UNSUPPORTED); a probe key past int64 never matches"""
    ctx = gpu_ctx
    n = 1000
    k = np.arange(n, dtype=np.int64) - 500
    T = _table(ctx, "t", {"k": k, "v": k * 3}, {}, (333,))
    big = ("mul", col("k"), const(1 << 62))  # |k| >= 2 leaves int64
    for keys, pay in (([col("k"), big], col("v")), ([col("k"), col("v")], big)):
        kt = runtime.join_table_keys(ctx, 2, n)
        with pytest.raises(capi.LdbRuntimeError) as ei:
            P.build_join(ctx, T, kt, keys, payload=pay)
        assert ei.value.code == capi.LDB_ERR_UNSUPPORTED and "int64" in str(ei.value)
        runtime.state_destroy(ctx, kt)
    kt = runtime.join_table_keys(ctx, 2, n)
    P.build_join(ctx, T, kt, [col("k"), col("v")], payload=col("v"))
    # (k, v + 2^64) wraps to (k, v) in 64 bits: it must still miss
    st = P.group_by(ctx, T, [], [("count", ("probe", kt, col("k"), col("v"))), ("count", ("probe", kt, col("k"), ("add", col("v"), const(1 << 64)))),
                                 ("count", ("probe", kt, big, col("v")))])
    # (k * 2^62, 3k) is a present tuple only for k = 0; the rows whose first key leaves int64 (k >= 2, k <= -3) never match
    assert P.decode_groups(P.read_groups(ctx, st, 4), 0, 3)[()] == [n, 0, 1]
    runtime.state_destroy(ctx, st)
    runtime.state_destroy(ctx, kt)
    T.clear()


def test_full_directory_fails_with_capacity(gpu_ctx):
    ctx = gpu_ctx
    k = np.arange(40, dtype=np.int64)
    T = _table(ctx, "t", {"k": k, "z": np.zeros(40, dtype=np.int64)}, {}, (13,))
    for unique, keys in ((True, [col("k"), col("z")]), (False, [col("z"), col("z")])):  # 40 distinct tuples / 40 duplicates of one
        kt = runtime.join_table_keys(ctx, 2, 8, unique=unique)  # 16 slots
        with pytest.raises(capi.LdbRuntimeError) as ei:
            P.build_join(ctx, T, kt, keys)
        assert ei.value.code == capi.LDB_ERR_CAPACITY and "full" in str(ei.value)
        runtime.state_destroy(ctx, kt)
    T.clear()


def test_overfull_builds_fail_fast(gpu_ctx):
    """An insert walks at most 65 536 slots: 3 x 2^20 distinct tuples into a table of 2^20 slots, and 70 000 duplicates of one tuple in
    a multimap, fail with LDB_ERR_CAPACITY in well under a second instead of walking the whole directory for every row."""
    ctx = gpu_ctx
    n = 3 << 20
    k = np.arange(n, dtype=np.int64)
    T = _table(ctx, "t", {"a": k, "b": k * 7}, {}, (n // 3, 2 * n // 3))
    D = _table(ctx, "d", {"a": np.full(70_000, 3, dtype=np.int64), "b": np.full(70_000, 4, dtype=np.int64)}, {}, ())
    for src, expected, unique in ((T, 1 << 19, True), (D, 1 << 18, False)):
        kt = runtime.join_table_keys(ctx, 2, expected, unique=unique)  # 2^20 / 2^19 slots
        t0 = time.perf_counter()
        with pytest.raises(capi.LdbRuntimeError) as ei:
            P.build_join(ctx, src, kt, [col("a"), col("b")])
        took = time.perf_counter() - t0
        assert ei.value.code == capi.LDB_ERR_CAPACITY and "duplicates" in str(ei.value)
        assert took < 5, took
        runtime.state_destroy(ctx, kt)
    T.clear()
    D.clear()


def test_probe_run_at_the_bound_fails_rather_than_truncate(gpu_ctx):
    """20 000 duplicates of one tuple form one probe run longer than the interpreter's 16 384-slot bound: PROBE_EACH of that tuple, and
    PROBE of absent tuples whose home slots lie inside the run, fail with LDB_ERR_CAPACITY — no truncated match list, no false miss.
    PROBE of the tuple itself stops at its first match and succeeds."""
    ctx = gpu_ctx
    n = 20_000
    T = _table(ctx, "t", {"a": np.full(n, 5, dtype=np.int64), "b": np.full(n, -7, dtype=np.int64)}, {}, (7_000,))
    rng = np.random.default_rng(3)
    Q = _table(ctx, "q", {"a": rng.integers(-(1 << 40), 1 << 40, 4000), "b": rng.integers(-(1 << 40), 1 << 40, 4000)}, {}, (1000,))
    kt = runtime.join_table_keys(ctx, 2, 40_000, unique=False, bloom=False)
    P.build_join(ctx, T, kt, [col("a"), col("b")], payload=("rowid",))
    try:
        assert runtime.join_count(ctx, kt) == n
        st = P.group_by(ctx, T, [], [("count", ("probe", kt, col("a"), col("b")))])
        assert P.decode_groups(P.read_groups(ctx, st, 4), 0, 1)[()] == [n]
        runtime.state_destroy(ctx, st)
        with pytest.raises(capi.LdbRuntimeError) as ei:
            P.group_by(ctx, T, [], [("count", ("probe_each", kt, col("a"), col("b")))])
        assert ei.value.code == capi.LDB_ERR_CAPACITY and "16384" in str(ei.value)
    finally:
        runtime.state_destroy(ctx, kt)
    kt = runtime.join_table_keys(ctx, 2, 40_000, unique=False, bloom=False)  # the error word stays set: a fresh table for PROBE
    P.build_join(ctx, T, kt, [col("a"), col("b")])
    try:
        with pytest.raises(capi.LdbRuntimeError) as ei:
            P.group_by(ctx, Q, [], [("count", ("probe", kt, col("a"), col("b")))])
        assert ei.value.code == capi.LDB_ERR_CAPACITY
    finally:
        runtime.state_destroy(ctx, kt)
        T.clear()
        Q.clear()


def _raw(ctx, table, instr, tables, sink_kind=P.SINK_MATERIALIZE, sink=None, n_keys=0, key_regs=(), build_key_reg=-1, columns=("k0", "k1")):
    """ldb_gpu_run_program on a hand-written instruction list; returns (code, message)"""
    b = P.Builder()
    b.columns, b.instr, b.tables = list(columns), list(instr), list(tables)
    d, keep = P._desc(ctx, table, b, -1)
    d.sink_kind, d.sink = sink_kind, sink
    d.n_keys = n_keys
    for i, r in enumerate(key_regs):
        d.key_regs[i] = r
    d.build_key_reg, d.build_payload_reg = build_key_reg, -1
    out = C.c_void_p()
    if sink_kind == P.SINK_MATERIALIZE:
        d.n_out, d.out_regs[0], d.out_table = 1, instr[-1][1], C.pointer(out)
    e = capi.Error()
    rc = ctx.L.ldb_gpu_run_program(ctx.h, C.byref(d), C.byref(e))
    if out.value:
        ctx.L.ldb_gpu_table_destroy(out)
    return rc, e.message.decode()


def test_invalid_programs_and_refusals(gpu_ctx):
    ctx = gpu_ctx
    O = P.OPS
    k = np.arange(100, dtype=np.int64)
    T = _table(ctx, "t", {"k0": k, "k1": -k}, {}, (50,))
    kt = runtime.join_table_keys(ctx, 2, 100)
    P.build_join(ctx, T, kt, [col("k0"), col("k1")], payload=col("k0"))
    load0, load1 = (O["load"], 0, 0, 0, 0), (O["load"], 1, 0, 0, 1)
    INVALID = capi.LDB_ERR_INVALID
    try:
        # a valid hand-written probe first: registers 0, 1 hold the tuple
        assert _raw(ctx, T, [load0, load1, (O["probe"], 2, 0, 0, 0)], [kt])[0] == capi.LDB_OK
        # key registers past register 47 (47, 48) / not yet written (1)
        assert _raw(ctx, T, [(O["load"], 47, 0, 0, 0), (O["probe"], 2, 47, 0, 0)], [kt])[0] == INVALID
        assert _raw(ctx, T, [load0, (O["probe"], 2, 0, 0, 0)], [kt])[0] == INVALID
        assert _raw(ctx, T, [load0, (O["probe_each"], 2, 0, 0, 0)], [kt])[0] == INVALID
        # build: wrong n_keys, build_key_reg != -1, building and probing one table
        dst = runtime.join_table_keys(ctx, 2, 100)
        assert _raw(ctx, T, [load0, load1], [], P.SINK_JOIN_BUILD, dst, 2, (0, 1))[0] == capi.LDB_OK
        assert _raw(ctx, T, [load0, load1], [], P.SINK_JOIN_BUILD, dst, 1, (0,))[0] == INVALID
        assert _raw(ctx, T, [load0, load1], [], P.SINK_JOIN_BUILD, dst, 2, (0, 1), build_key_reg=0)[0] == INVALID
        rc, msg = _raw(ctx, T, [load0, load1, (O["probe"], 2, 0, 0, 0)], [dst], P.SINK_JOIN_BUILD, dst, 2, (0, 1))
        assert rc == INVALID and "probe" in msg
        assert runtime.join_count(ctx, dst) == 100
        runtime.state_destroy(ctx, dst)
        # a table of another context, probed or built
        ctx2 = runtime.Context(0)
        try:
            other = runtime.join_table_keys(ctx2, 2, 100)
            rc, msg = _raw(ctx, T, [load0, load1, (O["probe"], 2, 0, 0, 0)], [other])
            assert rc == INVALID and "context" in msg
            rc, msg = _raw(ctx, T, [load0, load1], [], P.SINK_JOIN_BUILD, other, 2, (0, 1))
            assert rc == INVALID and "context" in msg
        finally:
            ctx2.close()
        # the new kind is refused by a specialised pipeline and by every other join-table entry point
        with pytest.raises(capi.LdbRuntimeError) as ei:
            runtime.run_pipeline(ctx, "scan_build", T, build_key="k0", build_payload="k1", sink=kt)
        assert ei.value.code == INVALID and "state" in str(ei.value)
        e = capi.Error()
        keys = (C.c_int32 * 4)(1, 2, 3, 4)
        assert ctx.L.ldb_gpu_join_table_insert(ctx.h, kt, keys, keys, None, 4, C.byref(e)) == INVALID
        ptr, nbytes = C.c_void_p(), C.c_int64()
        assert ctx.L.ldb_gpu_join_table_bloom(kt, C.byref(ptr), C.byref(nbytes), C.byref(e)) == INVALID
        rows, nr = (capi.TopKRow * 4)(), C.c_int32()
        assert ctx.L.ldb_gpu_join_table_topk(kt, 4, rows, C.byref(nr), C.byref(e)) == INVALID
        (comm,) = parallel.Comm.local_group([ctx])
        try:
            assert ctx.L.ldb_gpu_join_table_insert_received(kt, comm.h, 0, 16, 0, C.byref(e)) == INVALID
        finally:
            comm.close()
        # named like any state, and still whole
        assert ctx.L.ldb_gpu_register_state(ctx.h, b"partsupp_keys", kt, C.byref(e)) == capi.LDB_OK
        assert ctx.L.ldb_gpu_find_state(ctx.h, b"partsupp_keys") == kt.value
        # a serialised step whose sink it is, found by its registered name, is refused like a specialised pipeline
        step = {"kind": "scan_build", "source": "t", "build": {"key": "k0"}, "sink": {"name": "partsupp_keys"}}
        rc = ctx.L.ldb_gpu_run_step(ctx.h, json.dumps(step).encode(), C.byref(e))
        assert rc == INVALID and b"state" in e.message, (rc, e.message)
        assert runtime.join_count(ctx, kt) == 100
    finally:
        runtime.state_destroy(ctx, kt)
        T.clear()
    assert ctx.L.ldb_gpu_find_state(ctx.h, b"partsupp_keys") is None


def test_captured_queries_refuse_key_tuple_tables(gpu_ctx):
    """a program's join build reads the table's error word on the host, which a captured query cannot: creating, building or probing a
    key-tuple table inside a capture fails with LDB_ERR_UNSUPPORTED before anything is recorded"""
    ctx = gpu_ctx
    k = np.arange(100, dtype=np.int64)
    T = _table(ctx, "t", {"k0": k, "k1": -k}, {}, ())
    kt = runtime.join_table_keys(ctx, 2, 100)
    P.build_join(ctx, T, kt, [col("k0"), col("k1")])
    ctx.graph_begin()
    try:
        for fn in (lambda: runtime.join_table_keys(ctx, 2, 100), lambda: P.build_join(ctx, T, kt, [col("k0"), col("k1")]),
                   lambda: P.materialize(ctx, T, [("probe", kt, col("k0"), col("k1"))])):
            with pytest.raises(capi.LdbRuntimeError) as ei:
                fn()
            assert ei.value.code == capi.LDB_ERR_UNSUPPORTED and "captured" in str(ei.value)
    finally:
        ctx.graph_end().destroy()
    assert runtime.join_count(ctx, kt) == 100
    got = _read(ctx, P.materialize(ctx, T, [("probe", kt, col("k0"), col("k1"))]), 1)
    assert sorted(v for (v,) in got) == [0] * 100
    runtime.state_destroy(ctx, kt)
    T.clear()
