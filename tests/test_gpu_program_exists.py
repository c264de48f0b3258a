"""Probe-side EXISTS joins in program pipelines (LDB_OP_EXISTS, the reference's anyTuple): semi, anti and mark joins and left outer joins
with a residual predicate over four build sides (a multimap with duplicate and NULL keys, a unique table, a direct-address table and a
2-key key-tuple multimap, all with ROWID payloads), exact against a plain-Python model on seeded data; placement around PROBE_EACH, the
sinks, empty sides, the rejections; Q21 in the reference's probe-side shape against the reference's answers and a Q13-shaped outer join
with a two-sided residual against numpy on the dbgen-faithful SF1 tables."""
import ctypes as C
import json
import os
from collections import Counter

import numpy as np
import pytest

from lingodb_b200 import capi, datagen, dbgen, program as P, runtime

pytestmark = pytest.mark.gpu

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_kats.json")))["tpch_sf1"]
NB, NU, NA = 3000, 2000, 5000
STRS = ["apple", "kiwi", "mango", "zebra", "", "m", "lime", "nut"]


def _table(ctx, name, cols, valid=None, cuts=()):
    """columns {name: int32 array | ("dec", int array) | ("str", [str])} cut into batches at `cuts`, with Arrow validity bitmaps for the
    columns in `valid`"""
    valid = valid or {}
    specs = []
    for k, v in cols.items():
        specs.append(datagen.ColumnSpec(k, "decimal128", 12, 2) if isinstance(v, tuple) and v[0] == "dec" else
                     datagen.ColumnSpec(k, "utf8") if isinstance(v, tuple) else datagen.ColumnSpec(k, "int32"))
    td = datagen.TableData(name, specs)
    n = len(cols[specs[0].name]) if not isinstance(cols[specs[0].name], tuple) else len(cols[specs[0].name][1])
    edges = [0] + list(cuts) + [n]
    for a, b in zip(edges, edges[1:]):
        ch = {}
        for k, v in cols.items():
            if isinstance(v, tuple) and v[0] == "dec":
                ch[k] = dbgen._dec128(np.asarray(v[1][a:b], np.int64))
            elif isinstance(v, tuple):
                ch[k] = datagen.utf8_column(v[1][a:b])
            else:
                ch[k] = np.ascontiguousarray(v[a:b])
        for k, m in valid.items():
            ch[k + "$valid"] = np.packbits(m[a:b], bitorder="little")
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


def _side_cols(rng, n):
    v = rng.integers(0, 4, n).astype(np.int32)
    vvalid = rng.random(n) > 0.15
    d = rng.integers(0, 500, n)
    s = [STRS[j] for j in rng.integers(0, len(STRS), n)]
    svalid = rng.random(n) > 0.15
    model = dict(v=[int(x) if ok else None for x, ok in zip(v, vvalid)], d=d.tolist(), s=[x if ok else None for x, ok in zip(s, svalid)])
    return {"v": v, "d": ("dec", d), "s": ("str", s)}, {"v": vvalid, "s": svalid}, model


@pytest.fixture(scope="module")
def sides(gpu_ctx):
    """the build tables, the probe table and the four join tables with their models (entries: (key tuple, build row))"""
    ctx = gpu_ctx
    rng = np.random.default_rng(4242)
    bk = rng.integers(0, 800, NB).astype(np.int32)  # duplicates
    bk2 = rng.integers(0, 3, NB).astype(np.int32)
    bvalid = rng.random(NB) > 0.1
    bc, bval, bm = _side_cols(rng, NB)
    B = _table(ctx, "b", {"k": bk, "k2": bk2, **bc}, {"k": bvalid, **bval}, (NB // 3,))
    uk = rng.permutation(3000)[:NU].astype(np.int32)  # unique, no NULLs
    uc, uval, um = _side_cols(rng, NU)
    U = _table(ctx, "u", {"k": uk, "rid": np.arange(NU, dtype=np.int32), **uc}, uval)
    ak = rng.integers(0, 1000, NA).astype(np.int32)
    ak2 = rng.integers(0, 3, NA).astype(np.int32)
    av = rng.integers(0, 4, NA).astype(np.int32)
    ac = rng.integers(0, 2, NA).astype(np.int32)
    avalid, cvalid = rng.random(NA) > 0.1, rng.random(NA) > 0.3
    A = _table(ctx, "a", {"pk": ak, "pk2": ak2, "pv": av, "c": ac}, {"pk": avalid, "c": cvalid}, (NA // 7, NA // 2, NA - NA // 5))
    multi = runtime.join_table(ctx, NB, unique=False)
    P.build_join(ctx, B, multi, col("k"), payload=("rowid",))
    uniq = runtime.join_table(ctx, NU)
    P.build_join(ctx, U, uniq, col("k"), payload=("rowid",))
    direct = runtime.join_table_direct(ctx, 0, 2999)
    runtime.run_pipeline(ctx, "scan_build", U, build_key="k", build_payload="rid", sink=direct)
    tup = runtime.join_table_keys(ctx, 2, NB, unique=False)
    P.build_join(ctx, B, tup, [col("k"), col("k2")], payload=("rowid",))
    b_entries = [((int(bk[i]),), i) for i in range(NB) if bvalid[i]]
    u_entries = [((int(uk[i]),), i) for i in range(NU)]
    t_entries = [((int(bk[i]), int(bk2[i])), i) for i in range(NB) if bvalid[i]]
    probe = dict(pk=[int(x) if v else None for x, v in zip(ak, avalid)], pk2=ak2.tolist(), pv=av.tolist(), c=[int(x) if v else None for x, v in zip(ac, cvalid)])
    s = {
        "multi": dict(js=multi, src=B, m=bm, entries=b_entries, keys=[col("pk")], n=1),
        "unique": dict(js=uniq, src=U, m=um, entries=u_entries, keys=[col("pk")], n=1),
        "direct": dict(js=direct, src=U, m=um, entries=u_entries, keys=[col("pk")], n=1),
        "tuple": dict(js=tup, src=B, m=bm, entries=t_entries, keys=[col("pk"), col("pk2")], n=2),
    }
    for sd in s.values():
        sd["by"] = {}
        for k, r in sd["entries"]:
            sd["by"].setdefault(k, []).append(r)
    yield dict(sides=s, A=A, probe=probe, B=B, U=U, bk2=bk2, uk=uk)
    for x in s.values():
        runtime.state_destroy(ctx, x["js"])
    for t in (A, B, U):
        t.clear()


def _or3(a, b):
    if a is True or b is True:
        return True
    return None if a is None or b is None else False


# residuals: (expression over the build side `src` at row `m` and the probe row, its Python model (probe row i, build row r) → True /
# False / None)
def _residual(kind, sd, m, probe):
    bm = sd["m"]
    if kind == "int":  # a nullable build column against a probe column: NULL on some matches
        return (("cmp", "!=", ("fetch", sd["src"], m, "v"), col("pv")),
                lambda i, r: None if bm["v"][r] is None else bm["v"][r] != probe["pv"][i])
    if kind == "dec_str":  # a decimal against a scaled probe value OR a nullable string against a constant
        return (("or", ("cmp", ">", ("fetch", sd["src"], m, "d"), ("mul", col("pv"), const(100))), ("strcmp", "<", ("fetch", sd["src"], m, "s"), "m")),
                lambda i, r: _or3(bm["d"][r] > probe["pv"][i] * 100, None if bm["s"][r] is None else bm["s"][r].encode() < b"m"))
    return None, lambda i, r: True


def _pkey(probe, i, n):
    k = (probe["pk"][i],) if n == 1 else (probe["pk"][i], probe["pk2"][i])
    return None if None in k else k


def _model_exists(sd, probe, cond):
    out = []
    for i in range(NA):
        k = _pkey(probe, i, sd["n"])
        out.append(any(cond(i, r) is True for r in sd["by"].get(k, [])) if k else False)
    return out


SIDES = ["multi", "unique", "direct", "tuple"]


@pytest.mark.parametrize("kind", ["int", "dec_str", None])
@pytest.mark.parametrize("side", SIDES)
def test_semi_anti_and_mark_joins(gpu_ctx, sides, side, kind):
    """mark join (materialize: every row with its verdict), semi join (hash aggregation by c: count and sum of row ids) and anti join
    (materialize of the rows whose verdict is FALSE)"""
    ctx, sd, probe, A = gpu_ctx, sides["sides"][side], sides["probe"], sides["A"]
    cond, fn = _residual(kind, sd, ("match", sd["js"]), probe)
    ex = ("exists", sd["js"], *sd["keys"], cond)
    want = _model_exists(sd, probe, fn)
    assert 0 < sum(want) < NA
    got = _rows(ctx, P.materialize(ctx, A, [("rowid",), ex]), [("c0", 16), ("c1", 16)])
    assert sorted(got) == [(i, int(w)) for i, w in enumerate(want)]
    st = P.group_by(ctx, A, [col("c")], [("count_star", None), ("sum", ("rowid",))], where=ex, expected_groups=8)
    semi = P.decode_groups(P.read_groups(ctx, st, 8), 1, 2)
    runtime.state_destroy(ctx, st)
    exp = {}
    for i in range(NA):
        if want[i]:
            e = exp.setdefault((probe["c"][i],), [0, 0])
            e[0] += 1
            e[1] += i
    assert semi == exp
    anti = _rows(ctx, P.materialize(ctx, A, [("rowid",)], where=("not", ex)), [("c0", 16)])
    assert sorted(r for r, in anti) == [i for i in range(NA) if not want[i]]


@pytest.mark.parametrize("kind", ["int", "dec_str"])
@pytest.mark.parametrize("side", SIDES)
def test_left_outer_join_with_residual(gpu_ctx, sides, side, kind):
    """each match that passes the residual, or exactly one NULL tuple for a row without one — including rows whose key matches but
    whose matches all fail the residual"""
    ctx, sd, probe, A = gpu_ctx, sides["sides"][side], sides["probe"], sides["A"]
    cond, fn = _residual(kind, sd, ("match", sd["js"]), probe)
    m = ("probe_each", sd["js"], *sd["keys"], "outer", ("on", cond))
    got = Counter(_rows(ctx, P.materialize(ctx, A, [("rowid",), m, col("pv")]), [("c0", 16), ("c1", 16), ("c2", 16)]))
    want, all_fail = Counter(), 0
    for i in range(NA):
        k = _pkey(probe, i, sd["n"])
        matches = sd["by"].get(k, []) if k else []
        ok = [r for r in matches if fn(i, r) is True]
        all_fail += bool(matches) and not ok
        for r in ok or [None]:
            want[(i, r, probe["pv"][i])] += 1
    assert all_fail > 0
    assert got == want
    # with a user WHERE on top: ANDed with the residual's condition
    got2 = Counter(_rows(ctx, P.materialize(ctx, A, [("rowid",), m], where=("cmp", "=", col("c"), const(1))), [("c0", 16), ("c1", 16)]))
    assert got2 == Counter({(i, r): n for (i, r, _), n in want.items() if probe["c"][i] == 1})


def test_placement_around_probe_each_and_two_exists(gpu_ctx, sides):
    """an EXISTS before a left-outer PROBE_EACH runs once per row; one after it runs once per match, keyed by the match's build-side v
    on the unique table; two EXISTS share the program"""
    ctx, S, probe, A = gpu_ctx, sides["sides"], sides["probe"], sides["A"]
    mu, mm = S["unique"], S["multi"]
    c_before, f_before = _residual("int", mu, ("match", mu["js"]), probe)
    before = ("exists", mu["js"], col("pk"), c_before)
    each = ("probe_each", mm["js"], col("pk"), "outer")
    after = ("exists", mu["js"], ("fetch", mm["src"], each, "v"), ("cmp", "=", ("fetch", mu["src"], ("match", mu["js"]), "d"), ("fetch", mm["src"], each, "d")))
    after2 = ("exists", S["tuple"]["js"], col("pk"), ("fetch", mm["src"], each, "k2"), None)
    got = Counter(_rows(ctx, P.materialize(ctx, A, [("rowid",), before, each, after, after2]), [(f"c{j}", 16) for j in range(5)]))
    wb = _model_exists(mu, probe, f_before)
    ub, tb, bm, um = mu["by"], S["tuple"]["by"], mm["m"], mu["m"]
    want = Counter()
    for i in range(NA):
        k = probe["pk"][i]
        rs = mm["by"].get((k,), []) if k is not None else []
        if not rs:  # the NULL tuple: both later keys are NULL, so both verdicts are FALSE
            want[(i, int(wb[i]), None, 0, 0)] += 1
        for r in rs:
            v = bm["v"][r]
            a = v is not None and any(um["d"][u] == bm["d"][r] for u in ub.get((v,), []))
            a2 = bool(tb.get((k, int(sides["bk2"][r])), []))
            want[(i, int(wb[i]), r, int(a), int(a2))] += 1
    assert sum(x[3] for x in want.elements()) > 0 and sum(x[4] for x in want.elements()) > 0
    assert got == want


def test_join_build_and_effects_only_sinks(gpu_ctx, sides):
    """a semi join into a JOIN_BUILD sink (the kept row ids, read back through the markers scan) and an EXISTS verdict as the condition of
    a MARK in an LDB_SINK_NONE program"""
    ctx, sd, probe, A = gpu_ctx, sides["sides"]["tuple"], sides["probe"], sides["A"]
    cond, fn = _residual("dec_str", sd, ("match", sd["js"]), probe)
    ex = ("exists", sd["js"], *sd["keys"], cond)
    want = _model_exists(sd, probe, fn)
    kept = runtime.join_table(ctx, NA)
    P.build_join(ctx, A, kept, ("rowid",), payload=col("pv"), where=ex)
    got = _rows(ctx, P.join_marks(ctx, kept, P.ALL), [("key", 8), ("payload", 8)])
    assert sorted(got) == [(i, probe["pv"][i]) for i in range(NA) if want[i]]
    runtime.state_destroy(ctx, kept)
    fresh = runtime.join_table(ctx, NU)
    P.build_join(ctx, sides["U"], fresh, col("k"), payload=("rowid",))
    P.run_effects(ctx, A, [("mark", ("probe", fresh, col("pk")), ex)])
    got = _rows(ctx, P.join_marks(ctx, fresh, P.MARKED), [("key", 8)])
    uk = set(int(x) for x in sides["uk"])
    assert sorted(k for k, in got) == sorted({probe["pk"][i] for i in range(NA) if want[i] and probe["pk"][i] in uk})
    runtime.state_destroy(ctx, fresh)


def test_empty_build_and_probe_sides(gpu_ctx, sides):
    ctx, probe, A = gpu_ctx, sides["probe"], sides["A"]
    empty = runtime.join_table(ctx, 64, unique=False)
    cond = ("cmp", "=", ("fetch", sides["B"], ("match", empty), "v"), col("pv"))
    got = _rows(ctx, P.materialize(ctx, A, [("rowid",), ("exists", empty, col("pk"), cond), ("exists", empty, col("pk"), None)]), [("c0", 16), ("c1", 16), ("c2", 16)])
    assert sorted(got) == [(i, 0, 0) for i in range(NA)]
    got = _rows(ctx, P.materialize(ctx, A, [("rowid",), ("probe_each", empty, col("pk"), "outer", ("on", cond))]), [("c0", 16), ("c1", 16)])
    assert sorted(got) == [(i, None) for i in range(NA)]
    E = _table(ctx, "empty", {"pk": np.zeros(0, np.int32), "pv": np.zeros(0, np.int32)})
    sd = sides["sides"]["multi"]
    cond = ("cmp", "=", ("fetch", sd["src"], ("match", sd["js"]), "v"), col("pv"))
    assert _rows(ctx, P.materialize(ctx, E, [("rowid",), ("exists", sd["js"], col("pk"), cond)]), [("c0", 16), ("c1", 16)]) == []
    assert _rows(ctx, P.materialize(ctx, E, [("probe_each", sd["js"], col("pk"), "outer", ("on", cond))]), [("c0", 16)]) == []
    runtime.state_destroy(ctx, empty)
    E.clear()


def _raises(code, fn, text):
    with pytest.raises(capi.LdbRuntimeError) as ei:
        fn()
    assert ei.value.code == code and text in str(ei.value), str(ei.value)


def _run_raw(ctx, src, b, instr):
    """runs the instruction list `instr` (builder-numbered: side columns negative) with the builder's columns and tables, no sink"""
    b.instr = list(instr)
    b._next = max(i[1] for i in instr) + 1
    d, keep = P._desc(ctx, src, b, -1)
    d.sink_kind = P.SINK_NONE
    P._run(ctx, d, b)


def test_rejections(gpu_ctx, sides):
    ctx, B = gpu_ctx, sides["B"]
    INV, UNS = capi.LDB_ERR_INVALID, capi.LDB_ERR_UNSUPPORTED
    O = P.OPS
    js = sides["sides"]["multi"]["js"]
    b = P.Builder()
    b.expr(("exists", js, col("k"), ("cmp", ">", ("fetch", B, ("match", js), "v"), col("v"))))
    base = list(b.instr)  # load k; exists(b = 3): load side v, load v, cmp
    ex = base[1]
    assert ex[0] == O["exists"] and ex[3] == 3
    last = base[-1]
    # the block runs past the end
    _raises(INV, lambda: _run_raw(ctx, B, b, base[:1] + [ex[:3] + (4, ex[4])] + base[2:]), "runs past the end of the program")
    # nesting, PROBE_EACH, MARK and an inserting STRCODE inside the block
    nested = (O["exists"], 9, 0, 0, 0)
    _raises(INV, lambda: _run_raw(ctx, B, b, base[:1] + [ex[:3] + (4, ex[4])] + base[2:4] + [nested, last]), "EXISTS blocks do not nest")
    for op in (O["probe_each"], O["mark"]):
        _raises(INV, lambda: _run_raw(ctx, B, b, base[:1] + [ex[:3] + (4, ex[4])] + base[2:4] + [(op, 9, 0, 0, 0), last]), "may not contain PROBE_EACH, MARK or an inserting STRCODE")
    dct = P.dict_state(ctx, 64, 1024)
    bs = P.Builder()
    bs.expr(("exists", js, col("k"), ("isnull", ("strcode", dct, "s", "lookup"))))
    sb = list(bs.instr)
    si = next(j for j, i in enumerate(sb) if i[0] == O["strcode"])
    _run_raw(ctx, B, bs, sb)  # a lookup STRCODE is fine
    _raises(INV, lambda: _run_raw(ctx, B, bs, sb[:si] + [sb[si][:3] + (1, sb[si][4])] + sb[si + 1:]), "may not contain PROBE_EACH, MARK or an inserting STRCODE")
    # the block overwrites a register written before the EXISTS (the key), and the EXISTS's own dst
    for r in (base[0][1], ex[1]):
        _raises(INV, lambda: _run_raw(ctx, B, b, base[:-1] + [(last[0], r) + last[2:]]), "overwrites a register written before the EXISTS")
    # after the block: reading a block register, the filter reading one, a side column whose row is the EXISTS's dst
    _raises(INV, lambda: _run_raw(ctx, B, b, base + [(O["isnull"], 20, last[1], 0, 0)]), "written inside an EXISTS block is read after the block")
    _raises(INV, lambda: _run_raw(ctx, B, b, base + [(O["isnull"], 20, base[3][1], 0, 0)]), "written inside an EXISTS block is read after the block")
    side_load = base[2]
    _raises(INV, lambda: _run_raw(ctx, B, b, base + [(O["load"], 20, 0, 0, side_load[4])]), "reads an EXISTS result as its row after the EXISTS block")
    bf = P.Builder()
    bf.expr(("exists", js, col("k"), ("cmp", ">", col("v"), const(1))))
    d, keep = P._desc(ctx, B, bf, bf.instr[-1][1])
    d.sink_kind = P.SINK_NONE
    _raises(INV, lambda: P._run(ctx, d, bf), "written inside an EXISTS block is read after the block (filter)")
    # a MARK of a table probed inside a block (the block also runs for keys without a match)
    mj = sides["sides"]["unique"]["js"]
    _raises(INV, lambda: P.run_effects(ctx, B, [("exists", js, col("k"), ("isnull", ("probe", mj, col("k2")))), ("mark", ("probe", mj, col("k")), const(1))]),
            "MARK: the table it marks is probed inside an EXISTS block")
    # the verdict itself is a value after the block, and a well-formed block runs
    _run_raw(ctx, B, b, base + [(O["not"], 20, ex[1], 0, 0)])
    # table kinds: pair tables and group-join maps as PROBE_EACH splits them, a dictionary
    pair = runtime.join_table_pair(ctx, 64)
    gj = runtime.join_table(ctx, 64, n_side=1)
    for t in (pair, gj):
        _raises(UNS, lambda: P.materialize(ctx, B, [("exists", t, col("k"), None)]), "EXISTS takes a plain single-key, direct-address or key-tuple join table")
    _raises(INV, lambda: P.materialize(ctx, B, [("exists", dct, col("k"), None)]), "EXISTS on a string dictionary")
    # captured queries: refused for every table kind (the probe-run bound is read back after the launch)
    st = P.hashagg_state(ctx, 0, ["count_star"], 1)
    ctx.graph_begin()
    try:
        _raises(UNS, lambda: P.materialize(ctx, B, [("exists", sides["sides"]["tuple"]["js"], col("k"), col("k2"), None)]), "not part of captured queries")
        for side in ("multi", "unique", "direct"):
            _raises(UNS, lambda: P.group_by(ctx, B, [], [("count_star", None)], where=("exists", sides["sides"][side]["js"], col("k"), None), state=st),
                    "programs with EXISTS are not part of captured queries")
    finally:
        ctx.graph_end().destroy()
    assert P.decode_groups(P.read_groups(ctx, st, 4), 0, 1)[()] == [0]  # nothing was recorded into the state
    runtime.state_destroy(ctx, st)
    for t in (pair, gj, dct):
        runtime.state_destroy(ctx, t)


def test_probe_run_bound_fails_the_call(gpu_ctx):
    """20 000 duplicates of one key tuple share one probe run: a walk whose residual never passes reaches the 16384-slot bound"""
    ctx = gpu_ctx
    n = 20000
    D = _table(ctx, "dups", {"a": np.ones(n, np.int32), "b": np.ones(n, np.int32)})
    tup = runtime.join_table_keys(ctx, 2, 2 * n, unique=False)
    P.build_join(ctx, D, tup, [col("a"), col("b")], payload=("rowid",))
    Q = _table(ctx, "q", {"a": np.ones(4, np.int32), "b": np.ones(4, np.int32)})
    with pytest.raises(capi.LdbRuntimeError) as ei:
        P.materialize(ctx, Q, [("exists", tup, col("a"), col("b"), ("cmp", "<", ("match", tup), const(0)))])
    assert ei.value.code == capi.LDB_ERR_CAPACITY and "16384" in str(ei.value)
    runtime.state_destroy(ctx, tup)
    for t in (D, Q):
        t.clear()


def _home(keys, mask):
    """the home slot of int32 keys in a plain join table of mask + 1 slots (hashI32: hash64 of the sign-extended key)"""
    m = keys.astype(np.int64).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C55)
    return (m ^ m.byteswap()) & np.uint64(mask)


def test_plain_table_probe_run_bound_fails_the_call(gpu_ctx):
    """20 000 keys whose home slots are 1 .. 20 000 of a 65 536-slot multimap without a Bloom filter: every insert lands at its home, and
    a key whose home is slot 1 but which is absent walks one run of 20 000 occupied slots, past the interpreter's bound"""
    ctx = gpu_ctx
    cand = np.arange(1, 1 << 22, dtype=np.int64)
    home = _home(cand, 65535)
    slots, first = np.unique(home, return_index=True)
    pick = first[(slots >= 1) & (slots <= 20000)]
    assert len(pick) == 20000
    keys = cand[pick].astype(np.int32)
    absent = int(cand[(home == 1) & ~np.isin(cand, keys)][0])
    js, e = C.c_void_p(), capi.Error()
    capi.check(ctx.L.ldb_gpu_join_table_create(ctx.h, 20000, 2, 0, 0, C.byref(js), C.byref(e)), e)  # multimap, LDB_JOIN_NO_BLOOM
    D = _table(ctx, "run", {"k": keys})
    P.build_join(ctx, D, js, col("k"), payload=("rowid",))
    Q = _table(ctx, "q", {"k": np.array([absent, int(keys[5])], np.int32)})
    with pytest.raises(capi.LdbRuntimeError) as ei:
        P.materialize(ctx, Q, [("exists", js, col("k"), None)])
    assert ei.value.code == capi.LDB_ERR_CAPACITY and "EXISTS: a probe run is longer than the interpreter's bound of 16384 slots" in str(ei.value), str(ei.value)
    runtime.state_destroy(ctx, js)
    for t in (D, Q):
        t.clear()


def test_long_block_rewriting_its_registers(gpu_ctx, sides):
    """a block of 93 instructions (past the 48 registers) built from the raw instruction list: the side-column residual with 90 NEGs that
    rewrite two block registers in between"""
    ctx, sd, probe, A = gpu_ctx, sides["sides"]["multi"], sides["probe"], sides["A"]
    O = P.OPS
    cond, fn = _residual("int", sd, ("match", sd["js"]), probe)
    b = P.Builder()
    b.expr(col("pk"))
    rid = b.expr(("rowid",))
    ex = b.expr(("exists", sd["js"], col("pk"), cond))
    head, blk = b.instr[:3], b.instr[3:]
    assert head[2][0] == O["exists"] and head[2][3] == len(blk) == 3 and b._next == 6
    filler = [(O["neg"], 6 + j % 2, blk[0][1], 0, 0) for j in range(90)]
    block = blk[:2] + filler + blk[2:]
    b.instr = head[:2] + [head[2][:3] + (len(block), head[2][4])] + block
    b._next = 8
    assert len(b.instr) == 96 and b.instr[2][3] == 93
    d, keep = P._desc(ctx, A, b, -1)
    d.sink_kind, d.n_out = P.SINK_MATERIALIZE, 2
    d.out_regs[0], d.out_regs[1] = rid, ex
    out = C.c_void_p()
    d.out_table = C.pointer(out)
    P._run(ctx, d, b)
    got = _rows(ctx, out, [("c0", 16), ("c1", 16)])
    assert sorted(got) == [(i, int(w)) for i, w in enumerate(_model_exists(sd, probe, fn))]


# ---------------------------------------------------------------- Q21 and a Q13-shaped outer join on the SF1 tables
@pytest.fixture(scope="module")
def sf1(gpu_ctx):
    t = dbgen.tpch(1.0, extended=True, attributes=True)
    tabs = {k: gpu_ctx.table_from_host(t[k]) for k in ("lineitem", "orders", "supplier", "customer")}
    cat = lambda n, k: np.concatenate([c[k] for c in t[n].chunks])
    host = {k: cat(n, k) for n, k in (("customer", "c_custkey"), ("customer", "c_nationkey"), ("orders", "o_orderkey"), ("orders", "o_custkey"), ("orders", "o_orderdate"))}
    yield tabs, host
    for x in tabs.values():
        x.clear()


def test_q21_probe_side_exists_and_not_exists(gpu_ctx, sf1):
    """one program over lineitem: a Saudi supplier, a late line, its order F (NOT EXISTS a line whose l_linestatus <> 'F'), EXISTS a line
    of another supplier, NOT EXISTS a late line of another supplier; grouped by l_suppkey"""
    ctx, (t, _) = gpu_ctx, sf1
    li = t["lineitem"]
    names = [n for n, _ in datagen.NATIONS]
    late = ("cmp", ">", col("l_receiptdate"), col("l_commitdate"))
    saudi = runtime.join_table(ctx, 4096)
    P.build_join(ctx, t["supplier"], saudi, col("s_suppkey"), where=("cmp", "=", col("s_nationkey"), const(names.index("SAUDI ARABIA"))))
    lines = runtime.join_table(ctx, 6_100_000, unique=False)
    P.build_join(ctx, li, lines, col("l_orderkey"), payload=("rowid",))
    late_lines = runtime.join_table(ctx, 4_000_000, unique=False)
    P.build_join(ctx, li, late_lines, col("l_orderkey"), payload=("rowid",), where=late)
    open_lines = runtime.join_table(ctx, 3_100_000, unique=False)
    P.build_join(ctx, li, open_lines, col("l_orderkey"), payload=("rowid",), where=("cmp", "!=", col("l_linestatus"), const(ord("F"))))
    other = lambda js: ("cmp", "!=", ("fetch", li, ("match", js), "l_suppkey"), col("l_suppkey"))
    where = ("and", ("and", ("not", ("isnull", ("probe", saudi, col("l_suppkey")))), late),
             ("and", ("and", ("not", ("exists", open_lines, col("l_orderkey"), None)), ("exists", lines, col("l_orderkey"), other(lines))),
                     ("not", ("exists", late_lines, col("l_orderkey"), other(late_lines)))))
    st = P.group_by(ctx, li, [col("l_suppkey")], [("count_star", None)], where=where, expected_groups=4096)
    got = P.decode_groups(P.read_groups(ctx, st, 4096), 1, 1)
    top = sorted((("Supplier#%09d" % k, v[0]) for (k,), v in got.items()), key=lambda kv: (-kv[1], kv[0]))[:100]
    assert [[n, str(v)] for n, v in top] == GOLD["q21_rows"]
    for s_ in (st, saudi, lines, late_lines, open_lines):
        runtime.state_destroy(ctx, s_)


def test_q13_shaped_left_outer_join_with_two_sided_residual(gpu_ctx, sf1):
    """customer ⟕ orders on custkey with o_orderdate < 8400 + 80 * c_nationkey (a bound from the probe side, so it cannot be pushed into
    the build); count(o_orderkey) per customer and the histogram of the counts, against numpy"""
    ctx, (t, h) = gpu_ctx, sf1
    orders = runtime.join_table(ctx, 1_600_000, unique=False)
    P.build_join(ctx, t["orders"], orders, col("o_custkey"), payload=("rowid",))
    cond = ("cmp", "<", ("fetch", t["orders"], ("match", orders), "o_orderdate"), ("add", const(8400), ("mul", const(80), col("c_nationkey"))))
    m = ("probe_each", orders, col("c_custkey"), "outer", ("on", cond))
    st = P.group_by(ctx, t["customer"], [col("c_custkey")], [("count", ("fetch", t["orders"], m, "o_orderkey"))], expected_groups=200_000)
    got = {k: v[0] for (k,), v in P.decode_groups(P.read_groups(ctx, st, 1 << 18), 1, 1).items()}
    runtime.state_destroy(ctx, st)
    runtime.state_destroy(ctx, orders)
    ck, cn = h["c_custkey"].astype(np.int64), h["c_nationkey"].astype(np.int64)
    nation = np.zeros(int(ck.max()) + 1, np.int64)
    nation[ck] = cn
    oc = h["o_custkey"].astype(np.int64)
    keep = h["o_orderdate"].astype(np.int64) < 8400 + 80 * nation[oc]
    counts = np.bincount(oc[keep], minlength=len(nation))
    want = {int(k): int(counts[k]) for k in ck}
    assert 0 < sum(1 for v in want.values() if v == 0) < len(want)
    assert got == want
    assert Counter(got.values()) == Counter(want.values())
