"""General hash joins in program pipelines (csrc/program.cu): PROBE_EACH over non-unique build sides (inner and left outer), ROWID
build payloads and side columns read through a row register — against numpy, on ragged multi-batch tables with NULLs on both sides —
and the static validation of ldb_gpu_run_program_ex."""
import ctypes as C

import numpy as np
import pytest

from lingodb_b200 import capi, datagen, dbgen, program as P, runtime

pytestmark = pytest.mark.gpu

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))


def _table(ctx, name, specs, cols, valid, cuts):
    """a TableData cut into ragged batches at `cuts`, with Arrow validity bitmaps for the columns in `valid`"""
    td = datagen.TableData(name, specs)
    n = len(next(iter(cols.values())))
    edges = [0] + list(cuts) + [n]
    for a, b in zip(edges, edges[1:]):
        ch = {k: np.ascontiguousarray(v[a:b]) for k, v in cols.items()}
        for k, v in valid.items():
            ch[k + "$valid"] = np.packbits(v[a:b], bitorder="little")
        td.chunks.append(ch)
        td.chunk_rows.append(b - a)
    return ctx.table_from_host(td)


@pytest.fixture(scope="module")
def nm(gpu_ctx):
    """build side: keys 1..3000 (a fifth absent), 1-40 duplicates each, some NULL keys; probe side: keys 0..3199 (absent ones included),
    some NULL keys.  Both in >= 3 ragged batches."""
    rng = np.random.default_rng(11)
    present = np.flatnonzero(rng.random(3000) < 0.8) + 1
    dup = rng.integers(1, 41, len(present))
    bk = np.repeat(present, dup).astype(np.int32)
    bk = bk[rng.permutation(len(bk))]
    nb = len(bk)
    bv = rng.integers(-10**12, 10**12, nb).astype(np.int64)
    bvalid = rng.random(nb) > 0.03
    na = 30_011
    ak = rng.integers(0, 3200, na).astype(np.int32)
    av = rng.integers(-1000, 1000, na).astype(np.int32)
    avalid = rng.random(na) > 0.05
    B = _table(gpu_ctx, "b", [datagen.ColumnSpec("bk", "int32"), datagen.ColumnSpec("bv", "int64")], {"bk": bk, "bv": bv}, {"bk": bvalid}, (nb // 5, nb // 2, nb - 777))
    A = _table(gpu_ctx, "a", [datagen.ColumnSpec("ak", "int32"), datagen.ColumnSpec("av", "int32")], {"ak": ak, "av": av}, {"ak": avalid}, (4_999, 17_000, 29_000))
    jt = runtime.join_table(gpu_ctx, nb, unique=False)
    P.build_join(gpu_ctx, B, jt, col("bk"), payload=("rowid",))
    assert runtime.join_count(gpu_ctx, jt) == int(bvalid.sum())
    yield dict(B=B, A=A, jt=jt, bk=bk, bv=bv, bvalid=bvalid, ak=ak, av=av, avalid=avalid)
    gpu_ctx.L.ldb_gpu_state_destroy(jt)


def test_inner_many_to_many_count_and_sum(gpu_ctx, nm):
    m = ("probe_each", nm["jt"], col("ak"))
    st = P.group_by(gpu_ctx, nm["A"], [], [("count_star", None), ("sum", ("mul", col("av"), ("fetch", nm["B"], m, "bv"))), ("count", m)])
    got = P.decode_groups(P.read_groups(gpu_ctx, st, 4), 0, 3)[()]
    gpu_ctx.L.ldb_gpu_state_destroy(st)
    ok = nm["bvalid"]
    cnt = np.bincount(nm["bk"][ok], minlength=3201)
    sv = np.zeros(3201, dtype=object)
    for k, v in zip(nm["bk"][ok].tolist(), nm["bv"][ok].tolist()):
        sv[k] += v
    a = nm["avalid"]
    want_n = int(cnt[nm["ak"][a]].sum())
    want_sum = sum(int(x) * sv[k] for k, x in zip(nm["ak"][a].tolist(), nm["av"][a].tolist()))
    assert got == [want_n, want_sum, want_n]


def test_materialize_regrows_to_the_full_join(gpu_ctx, nm):
    """The join has ~15x the probe side's rows: the materialize sink counts past its first capacity, the runtime regrows and runs the
    program again; the rows are the numpy multiset (rows read back grouped by all four columns)."""
    m = ("probe_each", nm["jt"], col("ak"))
    out = P.RawTable(gpu_ctx, P.materialize(gpu_ctx, nm["A"], [col("ak"), col("av"), ("fetch", nm["B"], m, "bv"), m]))
    ok = nm["bvalid"]
    rows_of = {}
    for r in np.flatnonzero(ok).tolist():
        rows_of.setdefault(int(nm["bk"][r]), []).append(r)
    want = {}
    for k, x, v in zip(nm["ak"].tolist(), nm["av"].tolist(), nm["avalid"].tolist()):
        if not v:
            continue
        for r in rows_of.get(k, ()):
            t = (k, x, int(nm["bv"][r]), r)
            want[t] = want.get(t, 0) + 1
    n = sum(want.values())
    assert n > 5 * len(nm["ak"]) and out.num_rows == n
    st = P.group_by(gpu_ctx, out, [col("c0"), col("c1"), col("c2"), col("c3")], [("count_star", None)], expected_groups=n)
    got = {k: v[0] for k, v in P.decode_groups(P.read_groups(gpu_ctx, st, n + 16), 4, 1).items()}
    gpu_ctx.L.ldb_gpu_state_destroy(st)
    out.destroy()
    assert got == want


def test_left_outer_join_counts_customers_without_orders(gpu_ctx):
    """The Q13 shape without its comment filter: count(o_orderkey) per customer over customer LEFT OUTER JOIN orders, then the
    histogram of those counts — dbgen's key mortality leaves a third of the customers with zero orders."""
    t = dbgen.tpch(0.1, chunk_rows=100_003)
    ctx = gpu_ctx
    cu, od = ctx.table_from_host(t["customer"]), ctx.table_from_host(t["orders"])
    jt = runtime.join_table(ctx, t["orders"].num_rows, unique=False)
    P.build_join(ctx, od, jt, col("o_custkey"), payload=("rowid",))
    m = ("probe_each", jt, col("c_custkey"), "outer")
    st = P.group_by(ctx, cu, [col("c_custkey")], [("count", ("fetch", od, m, "o_orderkey"))], expected_groups=t["customer"].num_rows)
    groups = P.groups_table(ctx, st)
    hist = P.group_by(ctx, groups, [col("a0")], [("count_star", None)], expected_groups=256)
    got = {k[0]: v[0] for k, v in P.decode_groups(P.read_groups(ctx, hist, 256), 1, 1).items()}
    ck = np.concatenate([c["o_custkey"] for c in t["orders"].chunks])
    n_c = t["customer"].num_rows
    per = np.bincount(ck, minlength=n_c + 1)[1:]
    assert got == {int(k): int(v) for k, v in zip(*np.unique(per, return_counts=True))}
    assert got[0] == int((per == 0).sum()) > n_c // 4
    groups.destroy()
    for s_ in (st, hist, jt):
        ctx.L.ldb_gpu_state_destroy(s_)


def test_side_column_nulls(gpu_ctx):
    """A nullable side column over three ragged batches: NULL through a NULL row register (absent key) and through the injected
    validity bitmap; utf8 and decimal side columns read at the right batch."""
    rng = np.random.default_rng(3)
    n = 5_000
    keys = (rng.permutation(n) + 1).astype(np.int32)
    v = rng.integers(-2**31, 2**31 - 1, n).astype(np.int32)
    vvalid = rng.random(n) > 0.2
    dec = np.zeros((n, 2), np.int64)
    dec[:, 0] = rng.integers(-10**15, 10**15, n)
    dec[:, 1] = dec[:, 0] >> 63
    words = [b"PROMO BRUSHED TIN", b"ECONOMY PLATED", b"", b"PROMO"]
    widx = rng.integers(0, len(words), n)
    offs = np.zeros(n + 1, np.int32)
    offs[1:] = np.cumsum([len(words[i]) for i in widx])
    sbytes = np.frombuffer(b"".join(words[i] for i in widx), np.uint8).copy()
    S = datagen.TableData("s", [datagen.ColumnSpec("sk", "int32"), datagen.ColumnSpec("v", "int32"), datagen.ColumnSpec("d", "decimal128", 38, 2), datagen.ColumnSpec("s", "utf8")])
    for a, b in ((0, 1_234), (1_234, 1_235), (1_235, n)):
        S.chunks.append({"sk": keys[a:b].copy(), "v": v[a:b].copy(), "v$valid": np.packbits(vvalid[a:b], bitorder="little"), "d": dec[a:b].view(np.uint8).reshape(-1, 16).copy(),
                         "s": ((offs[a:b + 1] - offs[a]).astype(np.int32), sbytes[offs[a]:offs[b]].copy() if offs[b] > offs[a] else np.zeros(1, np.uint8))})
        S.chunk_rows.append(b - a)
    side = gpu_ctx.table_from_host(S)
    m = 700
    probe_keys = rng.integers(-50, n + 50, m).astype(np.int32)
    src = _table(gpu_ctx, "q", [datagen.ColumnSpec("k", "int32")], {"k": probe_keys}, {}, (300,))
    jt = runtime.join_table(gpu_ctx, n, unique=True)
    P.build_join(gpu_ctx, side, jt, col("sk"), payload=("rowid",))
    row = ("probe", jt, col("k"))
    out = P.RawTable(gpu_ctx, P.materialize(gpu_ctx, src, [col("k"), ("fetch", side, row, "v"), ("fetch", side, row, "d"),
                                                          ("like", "prefix", ("fetch", side, row, "s"), "PROMO"), ("isnull", ("fetch", side, row, "v"))]))
    assert out.num_rows == m
    ids = list(range(m))
    got = list(zip(*[out.gather(f"c{i}", ids) for i in range(5)]))
    where = {int(k): i for i, k in enumerate(keys.tolist())}
    full = lambda i: (int(dec[i, 1]) << 64) | (int(dec[i, 0]) & 0xFFFFFFFFFFFFFFFF)  # signed: the high word is a signed int64
    want = []
    for k in probe_keys.tolist():
        i = where.get(k)
        if i is None:
            want.append((k, None, None, None, 1))
        else:
            want.append((k, int(v[i]) if vvalid[i] else None, full(i), int(words[widx[i]].startswith(b"PROMO")), 0 if vvalid[i] else 1))
    assert sorted(got, key=lambda r: (r[0], str(r))) == sorted(want, key=lambda r: (r[0], str(r)))
    assert any(w[1] is None and w[2] is not None for w in want) and any(w[2] is None for w in want)
    out.destroy()
    gpu_ctx.L.ldb_gpu_state_destroy(jt)


def _run_raw(ctx, table, b, out_regs):
    d, keep = P._desc(ctx, table, b, -1)
    d.sink_kind, d.n_out = P.SINK_MATERIALIZE, len(out_regs)
    for i, r in enumerate(out_regs):
        d.out_regs[i] = r
    out = C.c_void_p()
    d.out_table = C.pointer(out)
    P._run(ctx, d, b)
    return out


def test_validation_rejects_malformed_joins(gpu_ctx):
    specs = [datagen.ColumnSpec("k", "int32"), datagen.ColumnSpec("name", "utf8")]
    n = 64
    names = np.frombuffer(b"x" * n, np.uint8).copy()
    td = datagen.TableData("v", specs, [{"k": np.arange(n, dtype=np.int32), "name": (np.arange(n + 1, dtype=np.int32), names)}], [n])
    t = gpu_ctx.table_from_host(td)
    jt = runtime.join_table(gpu_ctx, n, unique=False)
    P.build_join(gpu_ctx, t, jt, col("k"), payload=("rowid",))

    def rejects(code, match, fn):
        with pytest.raises(capi.LdbRuntimeError, match=match) as e:
            fn()
        assert e.value.code == code

    # a side column read before its row register is written
    b = P.Builder()
    r = b.expr(("fetch", t, col("k"), "k"))
    b.side_columns[0] = (0, "k", 40)
    rejects(capi.LDB_ERR_INVALID, "row register of a side column", lambda: _run_raw(gpu_ctx, t, b, [r]))
    # a side table of another context
    other = runtime.Context(0)
    try:
        ot = other.table_from_host(td)
        b = P.Builder()
        r = b.expr(("fetch", ot, col("k"), "k"))
        rejects(capi.LDB_ERR_INVALID, "another context", lambda: _run_raw(gpu_ctx, t, b, [r]))
    finally:
        other.close()
    # a utf8 side column as a value
    b = P.Builder()
    r = b.expr(("fetch", t, col("k"), "name"))
    rejects(capi.LDB_ERR_UNSUPPORTED, "LOAD of a string column", lambda: _run_raw(gpu_ctx, t, b, [r]))
    # a second PROBE_EACH
    b = P.Builder()
    r = b.expr(("probe_each", jt, col("k")))
    b.instr.append((P.OPS["probe_each"], r + 1, r, 0, 0))
    rejects(capi.LDB_ERR_UNSUPPORTED, "at most one PROBE_EACH", lambda: _run_raw(gpu_ctx, t, b, [r]))
    # PROBE_EACH on a pair table
    pair = runtime.join_table_pair(gpu_ctx, 64)
    b = P.Builder()
    r = b.expr(("probe_each", pair, col("k")))
    rejects(capi.LDB_ERR_UNSUPPORTED, "plain single-key or direct-address", lambda: _run_raw(gpu_ctx, t, b, [r]))
    # row ids of a build side with 2^31 rows do not fit the int32 payload (borrowed device column; rejected before any launch)
    import torch
    buf = torch.zeros(16, dtype=torch.int32, device="cuda")
    big = gpu_ctx.table("big", [datagen.ColumnSpec("k", "int32")])
    big._append(1 << 31, {"k": buf.data_ptr()}, capi.MEM_DEVICE, {})
    big._keep.append(buf)
    assert big.num_rows == 1 << 31
    rejects(capi.LDB_ERR_UNSUPPORTED, "2\\^31 rows", lambda: P.build_join(gpu_ctx, big, jt, col("k"), payload=("rowid",)))
    for s_ in (jt, pair):
        gpu_ctx.L.ldb_gpu_state_destroy(s_)
