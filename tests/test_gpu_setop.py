"""Set operations on the device (ldb_gpu_table_setop, RawTable.setop / distinct) against the exact model in tests/_setopref.py:

1. the reference's answers: the six queries of setops.test and the select4.test compound queries of tests/golden/setops.json, operands
   filtered on the host and staged, each chain run as device calls with every result table the next call's left side, compared as
   multisets to the reference's answers and cell for cell, in order, to the model;
2. seeded tables, every kind, cell for cell in order: 0, 1, 37 and 2^20 + 7 rows, 1, 7, n/3 and n distinct rows, the ten physical types
   with NULLs and garbage under the NULL cells, utf8 with long shared prefixes, decimals whose 64-bit halves carry, 1, 4 and 16 columns,
   ragged multi-batch HOST tables, bitmaps at bit offsets, validity bytes of result tables, a narrowed decimal against a 16-byte one and
   the same table on both sides;
3. contention: 2^24 equal rows, and INTERSECT ALL / EXCEPT ALL with counts in the millions, against numpy;
4. sharded composition: rows exchanged by key hash on fixed-width columns of the row over 2 and 3 in-process ranks, then a local set
   operation per rank; the union of the ranks' results equals the model as a multiset;
5. every documented error, the capture refusal included, with nothing launched."""
import ctypes as C
import random
import struct
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import _progref as R
import _setopref as S
from lingodb_b200 import capi
from test_gpu_window import WIDTH, read_fixed

# the ten physical types, and six more columns to reach 16; on the right side "dn" is a 16-byte decimal128(38, 2)
COLUMNS = [("i8", "int8", 0, 0), ("i16", "int16", 0, 0), ("i32", "int32", 0, 0), ("i64", "int64", 0, 0), ("dt", "date32", 0, 0),
           ("fs", "fsb4", 0, 0), ("dn", "decimal128", 18, 2), ("dw", "decimal128", 38, 2), ("f4", "float32", 0, 0), ("f8", "float64", 0, 0),
           ("s", "utf8", 0, 0), ("s2", "utf8", 0, 0), ("j64", "int64", 0, 0), ("j32", "int32", 0, 0), ("e8", "float64", 0, 0), ("k16", "int16", 0, 0)]
RIGHT_COLUMNS = [(n, p, 38 if n == "dn" else q, s) for n, p, q, s in COLUMNS]
PHYS = {n: p for n, p, _, _ in COLUMNS}
NAMES = [n for n, *_ in COLUMNS]
SELECTIONS = [["s"], ["dn", "f8", "s2", "i8"], NAMES]
CARRY = [(1 << 64) - 1, 1 << 64, -(1 << 64), (1 << 63), -(1 << 63) - 1, (1 << 100) + 12345, -(1 << 100)]


# ---------------------------------------------------------------------------------------------------- data
def f32(x: float) -> float:
    return struct.unpack("<f", struct.pack("<f", x))[0]


def cell(name: str, g: int, rng: random.Random):
    """column `name` of a row of group g: equal groups give equal rows (floats may differ in the sign of a zero or a NaN's bits)"""
    h = (g * 2654435761 + sum(map(ord, name)) * 97) & 0xFFFFFFFF
    if h % 11 == 3:
        return None
    p = PHYS[name]
    if p == "int8":
        return g % 256 - 128
    if p == "int16":
        return (g * 7) % 65536 - 32768
    if p in ("int32", "date32"):
        return g * 3 - 1000000 if p == "int32" else g % 40000 - 20000
    if p == "fsb4":
        return 32 + g % 95
    if p == "int64":
        return g * (1 << 40) - (1 << 62)
    if name == "dn":
        return g * 1000003 - 5 * 10 ** 16
    if name == "dw":
        return CARRY[g % len(CARRY)] + g // len(CARRY)
    if p.startswith("float"):
        k = g % 13
        if k == 0:
            return rng.choice([0.0, -0.0])
        if k == 1:
            return struct.unpack("<d", struct.pack("<Q", rng.choice([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF8000000000123])))[0]
        v = g * 0.37 - 1e4
        return f32(v) if p == "float32" else v
    return b"a long shared prefix of every string in this column/" * (1 + g % 3) + str(g % 1000003).encode()  # utf8


def gen_rows(n: int, groups, seed: int, names=NAMES) -> dict:
    rng = random.Random(seed)
    gs = [groups(rng) for _ in range(n)]
    return {c: [cell(c, g, rng) for g in gs] for c in names}


def garbage_under_nulls(td, seed: int):
    """random bytes under every NULL cell of a staged TableData (utf8: a NULL cell with a non-empty string)"""
    rng = np.random.default_rng(seed)
    for ch in td.chunks:
        for c in [c for c in NAMES if c in ch]:
            bm = ch.get(c + "$valid")
            if bm is None:
                continue
            n = len(ch[c][0]) - 1 if PHYS[c] == "utf8" else len(ch[c])
            null = ~np.unpackbits(bm, bitorder="little")[:n].astype(bool)
            if PHYS[c] == "utf8":
                offs, data = ch[c]
                lens = np.diff(offs)
                lens[null] = 5
                junk = rng.integers(0, 256, (n, 5), dtype=np.uint8)
                pieces = [bytes(data[offs[i]:offs[i + 1]]) if not null[i] else junk[i].tobytes() for i in range(n)]
                no = np.zeros(n + 1, np.int32)
                no[1:] = np.cumsum(lens)
                ch[c] = (no, np.frombuffer(b"".join(pieces) + b"\0", np.uint8).copy())
            else:
                buf = ch[c].view(np.uint8).reshape(n, -1)
                buf[null] = rng.integers(0, 256, (int(null.sum()), buf.shape[1]), dtype=np.uint8)
    return td


def stage(ctx, values: dict, columns, layout: str, seed: int):
    """a table in one of the layouts: "ragged" (HOST batches of uneven sizes), "offset" (HOST batches whose rows and bitmaps start at
    bit 3 of their buffers), "single" (one HOST batch)"""
    from lingodb_b200 import program as P
    columns = [c for c in columns if c[0] in values]
    n = len(next(iter(values.values())))
    rng = random.Random(seed)
    if layout == "offset":
        t = ctx.table(f"t{seed}", R.specs_of(columns))
        edges = [0] + sorted(rng.sample(range(1, n), min(3, n - 1))) + [n] if n > 1 else [0, n]
        for a, b in zip(edges, edges[1:]):
            ch = {}
            for c, p, _, _ in columns:
                buf, bm = R.column_buffers(p, values[c][a:b], 3)
                ch[c] = buf
                if bm is not None:
                    ch[c + "$valid"] = bm
            t.append_host(ch, b - a, offset=3)
        return P.RawTable(ctx, t.h)
    cuts = sorted(rng.sample(range(1, n), min(6, n - 1))) if layout == "ragged" and n > 1 else []
    td = R.to_table_data(f"t{seed}", values, columns, cuts)
    return P.RawTable(ctx, ctx.table_from_host(garbage_under_nulls(td, seed)).h)


# ---------------------------------------------------------------------------------------------------- reading results
def raw(phys: str, v):
    """a cell as the gather returns it: floats by their bits"""
    if v is None:
        return None
    if phys == "float32":
        return int(np.array([v], np.float32).view(np.int32)[0])
    if phys == "float64":
        return int(np.array([v], np.float64).view(np.int64)[0])
    return v


def read_rows(t, names: list, phys: list) -> list:
    cols = [t.gather_strings(c, list(range(t.num_rows)), decode=False) if p == "utf8" else read_fixed(t, c, WIDTH[p]) for c, p in zip(names, phys)]
    return list(zip(*cols)) if cols else []


def check_against_model(out, names: list, phys: list, want: list, what):
    assert out.num_rows == len(want), (what, out.num_rows, len(want))
    got = read_rows(out, names, phys)
    exp = [tuple(raw(p, v) for p, v in zip(phys, r)) for r in want]
    if got != exp:
        i = next(i for i, (a, b) in enumerate(zip(got, exp)) if a != b)
        raise AssertionError((what, i, got[i], exp[i]))


# ---------------------------------------------------------------------------------------------------- 1. the reference's answers
@pytest.mark.gpu
def test_reference_answers_on_the_device():
    from lingodb_b200 import runtime
    from lingodb_b200 import program as P
    from test_setop_model import chain, golden, operand_rows, split_compound, valuesort_answer, values_rows
    g = golden()
    tables = {k: [tuple(r) for r in v] for k, v in g["select4"]["tables"].items()}
    cases = [(q["sql"], [values_rows(o) for o in split_compound(q["sql"])[0]], split_compound(q["sql"])[1], sorted(q["rows"])) for q in g["setops_test"]]
    for q in g["select4"]["queries"]:
        operands, ops = split_compound(q["sql"])
        cases.append((q, [operand_rows(o, tables) for o in operands], ops, None))
    with runtime.Context(0) as ctx:
        for k, (q, operands, ops, rows) in enumerate(cases):
            staged = [P.RawTable(ctx, ctx.table_from_host(R.to_table_data(f"o{k}_{j}", {"v": [r[0] for r in rs]}, [("v", "int64", 0, 0)], [])).h)
                      for j, rs in enumerate(operands)]
            acc, made = staged[0], []
            for op, right in zip(ops, staged[1:]):
                acc = acc.setop(right, op)
                made.append(acc)
            got = read_fixed(acc, "v", 8)
            want = chain(operands, ops)
            assert got == [r[0] for r in want], q
            if rows is not None:  # setops.test: the answer rows
                assert sorted(str(v) for v in got) == rows, q
            else:
                vals, n, md5 = valuesort_answer([(v,) for v in got])
                assert ((n, md5) == (q["n_values"], q["md5"])) if "md5" in q else vals == sorted(q["values"]), q["line"]
            for t in made:
                t.destroy()


# ---------------------------------------------------------------------------------------------------- 2. seeded tables
def group_fn(card, offset=0):
    return lambda rng: offset + rng.randrange(card)


def cards(n: int) -> list:
    out = []
    for c in [1, 7, n // 3, n]:
        if c > 0 and c not in out:
            out.append(c)
    return out


# 2^20 + 7 rows: two of the cardinalities and the 1- and 4-column selections (the 16-column one runs at the smaller sizes), so that the
# Python side stays within seconds
BIG_CARDS = lambda n: [7, n]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 37, (1 << 20) + 7])
def test_device_equals_the_model(n):
    from lingodb_b200 import runtime
    big = n > 1000
    sels = SELECTIONS[:2] if big else SELECTIONS
    need = sorted({c for sel in sels for c in sel}, key=NAMES.index)
    with runtime.Context(0) as ctx:
        case = 0
        for ci, card in enumerate((BIG_CARDS(n) if big else cards(n)) or [1]):
            left = gen_rows(n, group_fn(card), 10 * n + ci, need)
            # the right side: about half as many rows, half of its groups shared with the left's
            nr = n // 2 + (ci % 3)
            right = gen_rows(nr, group_fn(card, card // 2), 10 * n + ci + 5, need)
            L = stage(ctx, left, COLUMNS, ["ragged", "single", "offset"][ci % 3], 2 * ci)
            Rt = stage(ctx, right, RIGHT_COLUMNS, ["offset", "ragged", "single"][ci % 3], 2 * ci + 1)
            copy = L.setop(Rt, "union_all", need, need, name="copy") if ci % 2 else None  # a result table: validity bytes, 16-byte decimals
            for kind in S.KINDS:
                names = sels[(case + ci) % len(sels)]
                phys = [PHYS[c] for c in names]
                lrows = list(zip(*[left[c] for c in names])) if n else []
                rrows = list(zip(*[right[c] for c in names])) if nr else []
                what = (n, card, kind, len(names), case)
                if kind == "distinct":
                    src, rows = (copy, lrows + rrows) if copy is not None else (L, lrows)
                    out = src.distinct(names)
                    check_against_model(out, names, phys, S.setop("distinct", rows), what)
                elif case % 4 == 3:  # the same table on both sides
                    out = L.setop(L, kind, names, names)
                    check_against_model(out, names, phys, S.setop(kind, lrows, lrows), what)
                elif copy is not None and case % 2:  # a result table on the left, a staged table on the right
                    out = copy.setop(Rt, kind, names, names)
                    check_against_model(out, names, phys, S.setop(kind, lrows + rrows, rrows), what)
                else:
                    out = L.setop(Rt, kind, names, names)
                    check_against_model(out, names, phys, S.setop(kind, lrows, rrows), what)
                out.destroy()
                case += 1
            if copy is not None:
                copy.destroy()


@pytest.mark.gpu
def test_results_chain():
    """a result table feeds the next set operation and the window operator; a narrowed decimal on the left meets 16-byte cells"""
    from lingodb_b200 import runtime
    n = 500
    left = gen_rows(n, group_fn(50), 1)
    right = gen_rows(n, group_fn(50, 25), 2)
    lrows, rrows = list(zip(left["dn"], left["i64"])), list(zip(right["dn"], right["i64"]))
    with runtime.Context(0) as ctx:
        L = stage(ctx, left, COLUMNS, "ragged", 1)
        Rt = stage(ctx, right, RIGHT_COLUMNS, "offset", 2)
        u = L.setop(Rt, "union", ["dn", "i64"], ["dn", "i64"], name="u")
        want = S.setop("union", lrows, rrows)
        check_against_model(u, ["dn", "i64"], ["decimal128", "int64"], want, "union")
        ex = u.setop(L, "except_all", ["dn", "i64"], ["dn", "i64"])
        check_against_model(ex, ["dn", "i64"], ["decimal128", "int64"], S.setop("except_all", want, lrows), "chained except all")
        w = ex.window(funcs=[("count_star", None, "c")], columns=["i64"])
        assert w.num_rows == ex.num_rows
        for t in (w, ex, u):
            t.destroy()


# ---------------------------------------------------------------------------------------------------- 3. contention
def first_order_counts(a: np.ndarray):
    vals, first, counts = np.unique(a, return_index=True, return_counts=True)
    o = np.argsort(first)
    return vals[o], counts[o]


@pytest.mark.gpu
def test_contention_equal_rows():
    from lingodb_b200 import datagen, runtime
    from lingodb_b200 import program as P
    n = 1 << 24
    rng = np.random.default_rng(3)
    a = np.full(n, 5, np.int64)
    sprinkle = rng.choice(n, 4096, replace=False)
    a[sprinkle] = rng.integers(0, 1000, 4096)  # a few other rows, some repeated more than the scan writes itself
    b = np.full(3_000_000, 5, np.int64)
    b[rng.choice(len(b), 2048, replace=False)] = rng.integers(500, 1500, 2048)
    spec = [datagen.ColumnSpec("k", "int64")]
    with runtime.Context(0) as ctx:
        L = P.RawTable(ctx, ctx.table_from_host(datagen.TableData("a", spec, [{"k": a}], [n])).h)
        Rt = P.RawTable(ctx, ctx.table_from_host(datagen.TableData("b", spec, [{"k": b}], [len(b)])).h)
        same = P.RawTable(ctx, ctx.table_from_host(datagen.TableData("s", spec, [{"k": np.full(n, -7, np.int64)}], [n])).h)
        d = same.distinct()
        assert read_fixed(d, "k", 8) == [-7]
        d.destroy()
        va, ca = first_order_counts(a)
        vb = dict(zip(*first_order_counts(b)))
        for kind in ("intersect_all", "except_all", "intersect", "except", "union", "distinct"):
            out = L.distinct() if kind == "distinct" else L.setop(Rt, kind)
            got = np.array(read_fixed(out, "k", 8), np.int64)
            if kind in ("union", "distinct"):
                u = np.concatenate([a, b]) if kind == "union" else a
                want = first_order_counts(u)[0]
            else:
                c_r = np.array([vb.get(v, 0) for v in va.tolist()], np.int64)
                times = {"intersect_all": np.minimum(ca, c_r), "except_all": np.maximum(ca - c_r, 0), "intersect": ((c_r > 0)).astype(np.int64),
                         "except": (c_r == 0).astype(np.int64)}[kind]
                want = np.repeat(va, times)
            assert np.array_equal(got, want), (kind, len(got), len(want))
            out.destroy()
        # the counts in the millions: 2^24 - 4096 copies of 5 on the left, about 3 M on the right
        assert (a == 5).sum() > 16_000_000 and (b == 5).sum() > 2_990_000


# ---------------------------------------------------------------------------------------------------- 4. sharded composition
@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_composition(world):
    """rows exchanged by key hash on fixed-width columns of the row, then a local set operation per rank: equal rows share those key
    values, so they meet on one owner, and the ranks' results together are the model's as a multiset"""
    from test_gpu_exchange import ranks
    from lingodb_b200 import program as P
    names = ["i64", "dn", "s", "f8", "i8"]
    keys = ["i64", "dn", "i8"]
    phys = [PHYS[c] for c in names]
    n = 20000
    left = gen_rows(n, group_fn(3000), 11)
    right = gen_rows(n // 2, group_fn(3000, 1500), 12)
    lrows, rrows = list(zip(*[left[c] for c in names])), list(zip(*[right[c] for c in names]))
    cols = [c for c in COLUMNS if c[0] in names]
    with ranks(world, user_bytes=64 << 20) as (ctxs, comms):
        # shard r holds every world-th batch-sized slice of each side
        def shard(values, r, m):
            idx = [i for i in range(m) if (i // 1000) % world == r]
            return {c: [values[c][i] for i in idx] for c in names}
        Ls = [P.RawTable(c, c.table_from_host(R.to_table_data("l", shard(left, r, n), cols, [])).h) for r, c in enumerate(ctxs)]
        Rs = [P.RawTable(c, c.table_from_host(R.to_table_data("r", shard(right, r, n // 2), cols, [])).h) for r, c in enumerate(ctxs)]
        half = 32 << 20

        def run(r):
            lx = comms[r].table_exchange_varlen(Ls[r], keys, names, name="lx", recv_offset=0, recv_bytes=half)
            rx = comms[r].table_exchange_varlen(Rs[r], keys, names, name="rx", recv_offset=half, recv_bytes=half)
            return [(kind, read_rows(lx.setop(rx, kind, names, names) if kind != "distinct" else lx.distinct(names), names, phys)) for kind in S.KINDS]
        with ThreadPoolExecutor(world) as ex:
            res = list(ex.map(run, range(world)))
        for k, kind in enumerate(S.KINDS):
            got = sorted((r for rank in res for r in rank[k][1]), key=repr)
            want = S.setop(kind, lrows, None if kind == "distinct" else rrows)
            exp = sorted((tuple(raw(p, v) for p, v in zip(phys, r)) for r in want), key=repr)
            if kind in ("union_all",):
                assert got == exp, kind
            else:  # equal rows may differ in the bits of a float zero or NaN: compare the canonical rows
                canon = lambda rows: sorted((tuple(S.canon_cell(struct.unpack("<d", struct.pack("<q", v))[0]) if p == "float64" and v is not None else v
                                                   for p, v in zip(phys, r)) for r in rows), key=repr)
                assert canon(got) == canon(exp), kind


# ---------------------------------------------------------------------------------------------------- 5. errors
@pytest.mark.gpu
def test_documented_errors():
    from lingodb_b200 import runtime
    from lingodb_b200 import program as P
    vals = gen_rows(40, group_fn(5), 9)
    with runtime.Context(0) as ctx, runtime.Context(0) as other:
        L = stage(ctx, vals, COLUMNS, "ragged", 1)
        Rt = stage(ctx, vals, RIGHT_COLUMNS, "single", 2)
        X = stage(other, vals, COLUMNS, "single", 3)
        scale = P.RawTable(ctx, ctx.table_from_host(R.to_table_data("sc", {"dn": vals["dn"]}, [("dn", "decimal128", 18, 3)], [])).h)
        before = ctx.launch_count()
        L_ = ctx.L
        out, e = C.c_void_p(), capi.Error()
        enc = lambda xs: (C.c_char_p * len(xs))(*[x.encode() for x in xs])

        def rc(left, right, kind, n, lc, rc_, name=None):
            return L_.ldb_gpu_table_setop(left, right, kind, n, lc, rc_, name, C.byref(out), C.byref(e))
        two = enc(["i64", "s"])
        inv, uns = capi.LDB_ERR_INVALID, capi.LDB_ERR_UNSUPPORTED
        assert rc(None, Rt.h, 3, 2, two, two) == inv  # null arguments
        assert L_.ldb_gpu_table_setop(L.h, Rt.h, 3, 2, two, two, None, None, C.byref(e)) == inv
        assert rc(L.h, Rt.h, 1, 2, two, two) == inv  # right given for DISTINCT
        assert rc(L.h, None, 1, 2, two, None) == capi.LDB_OK and out.value  # (the valid DISTINCT)
        L_.ldb_gpu_table_destroy(out)
        before = ctx.launch_count()
        assert rc(L.h, None, 3, 2, two, two) == inv  # right missing
        for k in (0, 8, -1):
            assert rc(L.h, Rt.h, k, 2, two, two) == inv, k  # unknown kind
        assert rc(L.h, Rt.h, 3, 2, enc(["i64", "nope"]), two) == inv and "nope" in e.message.decode()
        assert rc(L.h, Rt.h, 3, 2, two, enc(["nope", "s"])) == inv
        assert rc(L.h, Rt.h, 3, 0, two, two) == inv  # 0 columns
        assert rc(L.h, Rt.h, 3, 17, enc(NAMES + ["i8"]), enc(NAMES + ["i8"])) == inv  # 17 columns
        assert rc(L.h, Rt.h, 3, 2, two, None) == inv  # 2 against every column of right (16)
        wide = P.RawTable(ctx, ctx.table_from_host(R.to_table_data("w", {f"c{i}": list(range(3)) for i in range(17)}, [(f"c{i}", "int32", 0, 0) for i in range(17)], [])).h)
        assert rc(wide.h, wide.h, 3, 0, None, None) == inv  # every column: 17
        assert rc(L.h, X.h, 3, 2, two, two) == inv  # different contexts
        assert rc(L.h, Rt.h, 3, 2, two, enc(["i32", "s"])) == uns and "i64" in e.message.decode() and "i32" in e.message.decode()
        assert rc(L.h, scale.h, 3, 1, enc(["dn"]), enc(["dn"])) == uns and "scale" in e.message.decode()
        assert ctx.launch_count() == before
        # inside a captured query: refused before anything is enqueued
        ctx.graph_begin()
        try:
            code = rc(L.h, Rt.h, 3, 2, two, two)
            msg = e.message.decode()
        finally:
            ctx.graph_end().destroy()
        assert code == uns and "captured" in msg
        assert ctx.launch_count() == before
        # 2^32 rows: sixteen borrowed DEVICE batches over one buffer of 2^28 rows
        import torch
        from lingodb_b200 import datagen
        buf = torch.zeros(1 << 28, dtype=torch.int8, device="cuda:0")
        huge = ctx.table("huge", [datagen.ColumnSpec("i8", "int8")])
        for _ in range(16):
            huge.append_device({"i8": buf}, 1 << 28)
        before = ctx.launch_count()
        assert rc(huge.h, None, 1, 0, None, None) == uns and "2^32" in e.message.decode()
        assert rc(huge.h, L.h, 2, 1, enc(["i8"]), enc(["i8"])) == uns
        assert ctx.launch_count() == before
        huge.clear()
        del buf
        # and the tables still work afterwards
        u = L.setop(Rt, "union", ["i64", "s"], ["i64", "s"])
        assert u.num_rows == len(S.setop("union", list(zip(vals["i64"], vals["s"])), list(zip(vals["i64"], vals["s"]))))
