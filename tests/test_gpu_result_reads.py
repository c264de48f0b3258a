"""The result side, where every answer leaves the device: ORDER BY (ldb_gpu_table_order_by / _order_by_keys), the cell reads
(ldb_gpu_table_gather / _gather_strings) and the dictionary export (ldb_gpu_dict_to_table), on every kind of single-batch table —
DEVICE batches with Arrow bitmaps at bit offsets 0, 3 and 7 and utf8 offsets that do not start at 0, HOST batches under each
staging mode, exported group tables, materialised rows, join-marker tables and string dictionaries.  Orders are checked row id for
row id against tests/_progref.py's reference_order (NULLs last ascending, first descending, tied; the library's sort is stable, so
no tolerance applies) and cells, validity included, against the values the test wrote."""
import random
import struct

import numpy as np
import pytest
import torch

import _progref as R
from lingodb_b200 import program as P, runtime
from test_gpu_program_ops import ORDER_WIDE, _wide_words

pytestmark = pytest.mark.gpu

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))
M64 = (1 << 64) - 1

BASE_COLUMNS = [("i32", "int32", 0, 0), ("dt", "date32", 0, 0), ("f4", "fsb4", 0, 0), ("i64", "int64", 0, 0), ("dn", "decimal128", 18, 2),
                ("dw", "decimal128", 38, 0), ("s", "utf8", 0, 0)]
CELL = {"int32": 4, "date32": 4, "fsb4": 4, "int64": 8, "decimal128": 16, "float64": 16}
BASE_KEYS = [[("i32", False), ("s", True)], [("s", False), ("i64", True), ("dt", False)], [("dn", True), ("s", False), ("dw", False), ("f4", True)],
             [("f4", False), ("i32", False)], [("dw", True), ("i32", True)]]
PAD = b"#offset#"  # utf8 bytes before the first string: a batch's first offset is not 0
EDGE_STRINGS = [b"", b"\0", b"\0\0", b"a", b"a\0", b"a\0\0", b"a\x7f", b"a\x80", b"\x80", b"\xff", b"\xff\xff", b"PREFIX08", b"PREFIX08\0",
                b"PREFIX08PREFIX16", b"PREFIX08PREFIX16z", b"PREFIX08Z", b"PREFIX08\xff", b"x" * 64, b"x" * 63 + b"\xff", b"x" * 70, b"x" * 69 + b"\0"]


# ---------------------------------------------------------------------------------------------------- values
def _one_digit(rng, n, base, digits):
    """base with one random 8-bit digit (of `digits`) replaced: between two such values exactly one radix pass decides"""
    d = rng.integers(0, digits, n).astype(np.uint64)
    b = rng.integers(0, 256, n).astype(np.uint64)
    shift = d * np.uint64(8)
    return (np.uint64(base) & ~(np.uint64(255) << shift)) | (b << shift)


def _ints(rng, n, bits):
    """n signed `bits`-bit values (as uint64 words): a third differ from one base value in a single digit, a quarter are small
    (heavy ties), some are the type's edges, the rest uniform"""
    kind = rng.integers(0, 12, n)
    v = rng.integers(0, 1 << 63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
    v = np.where(kind < 4, _one_digit(rng, n, int(rng.integers(0, 1 << 63)) * 2 + 1, bits // 8), v)
    v = np.where((kind >= 4) & (kind < 7), rng.integers(-3, 4, n).astype(np.int64).view(np.uint64), v)
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    edges = np.array([x & M64 for x in (0, 1, -1, lo, hi, lo + 1, hi - 1)], np.uint64)
    v = np.where(kind == 7, edges[rng.integers(0, len(edges), n)], v)
    if bits == 32:
        return v.astype(np.uint32).view(np.int32)
    return v.view(np.int64)


def _wide(rng, n):
    """decimal128 cells over the whole i128 range: _wide_words' ties and ORDER_WIDE rows, and a third that differ from one base
    value in a single digit of either word (every one of the 16 passes decides somewhere).  (n, 2) uint64 [low, high]."""
    hi, lo = _wide_words(rng, n)
    hi = hi.view(np.uint64).copy()
    word = rng.integers(0, 2, n).astype(bool)
    base_lo, base_hi = int(rng.integers(0, 1 << 63)) * 2 + 1, int(rng.integers(0, 1 << 63))
    pick = (rng.integers(0, 3, n) == 0) & (np.arange(n) >= len(ORDER_WIDE))
    lo = np.where(pick, np.where(word, np.uint64(base_lo), _one_digit(rng, n, base_lo, 8)), lo)
    hi = np.where(pick, np.where(word, _one_digit(rng, n, base_hi, 8), np.uint64(base_hi)), hi)
    return np.stack([lo, hi], axis=1)


def _strings(rng, n):
    """bytes values: the edge strings, strings that share 8- and 16-byte prefixes, and lengths 0..70 (nine 8-byte chunks) over an
    alphabet with 0x00, 0x7f, 0x80 and 0xff; drawn from a pool, so there are ties"""
    r = random.Random(int(rng.integers(0, 1 << 30)))
    alphabet = b"\0\x01AB\x7f\x80\xfe\xff"
    pool = list(EDGE_STRINGS)
    for _ in range(4000):
        s = bytes(r.choice(alphabet) for _ in range(r.randrange(0, 71)))
        pool.append(r.choice([b"", b"PREFIX08", b"PREFIX08PREFIX16"]) + s[:r.randrange(0, 71)] if r.random() < 0.4 else s)
    return [pool[i] for i in rng.integers(0, len(pool), n)]


def base_values(seed, n, null_share=0.2):
    """{column: (physical cells, NULL mask)} for BASE_COLUMNS: int arrays, (n, 2) uint64 decimal cells, or a list of bytes.  A NULL
    row keeps the random cell under it, so an order that reads it shows.  Row 0 is NULL in i32 and valid elsewhere (a one-row
    batch has a NULL too)."""
    rng = np.random.default_rng(seed)
    out = {}
    for name, phys, _, _ in BASE_COLUMNS:
        null = rng.random(n) < null_share
        if n:
            null[0] = name == "i32"
        if phys in ("int32", "date32", "fsb4"):
            raw = _ints(rng, n, 32)
        elif phys == "int64":
            raw = _ints(rng, n, 64)
        elif name == "dn":
            v = _ints(rng, n, 64)
            raw = np.stack([v.view(np.uint64), (v >> 63).view(np.uint64)], axis=1)
        elif phys == "decimal128":
            raw = _wide(rng, n)
        else:
            raw = _strings(rng, n)
        out[name] = (raw, null)
    return out


def cells_of(phys, raw, null):
    """the reference cells: int (a decimal's full i128) or bytes, None for NULL"""
    if phys == "utf8":
        vals = raw
    elif phys == "decimal128":
        vals = [R.wrap128((int(h) << 64) | int(lo)) for lo, h in raw.tolist()]
    else:
        vals = raw.tolist()
    return [None if z else v for v, z in zip(vals, null.tolist())]


def arrow(phys, raw, null, offset):
    """Arrow buffers with `offset` filler rows in front: values or (offsets, bytes), and the validity bitmap (LSB first)"""
    valid = np.concatenate([np.zeros(offset, bool), ~null])
    bitmap = np.packbits(valid, bitorder="little")
    if phys == "utf8":
        strs = [b"filler"] * offset + list(raw)
        offs = np.zeros(len(strs) + 1, np.int64)
        offs[1:] = np.cumsum([len(s) for s in strs])
        return (offs.astype(np.int32) + len(PAD), np.frombuffer(PAD + b"".join(strs) + b"\0", np.uint8).copy()), bitmap
    if phys == "decimal128":
        return np.concatenate([np.zeros((offset, 2), np.uint64), raw]).view(np.uint8).reshape(-1, 16), bitmap
    return np.concatenate([np.zeros(offset, raw.dtype), raw]), bitmap


def host_table(ctx, name, data, n, offset=0):
    t = runtime.Table(ctx, name, R.specs_of(BASE_COLUMNS))
    chunk = {}
    for c, phys, _, _ in BASE_COLUMNS:
        chunk[c], chunk[c + "$valid"] = arrow(phys, *data[c], offset)
    t.append_host(chunk, n, offset=offset)
    return t


def device_table(ctx, name, data, n, offset):
    t = runtime.Table(ctx, name, R.specs_of(BASE_COLUMNS))
    dev = lambda a: torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).cuda()
    tensors = {}
    for c, phys, _, _ in BASE_COLUMNS:
        buf, bitmap = arrow(phys, *data[c], offset)
        tensors[c] = (dev(buf[0]), dev(buf[1])) if phys == "utf8" else dev(buf)
        tensors[c + "$valid"] = dev(bitmap)
    t.append_device(tensors, n, offset=offset)
    return t


# ---------------------------------------------------------------------------------------------------- the checks
def f64_of(v):
    return None if v is None else struct.unpack("<d", struct.pack("<Q", v & M64))[0]


def read(raw, c, phys, ids):
    if phys == "utf8":
        return raw.gather_strings(c, ids, decode=False)
    got = raw.gather(c, ids, cell_bytes=CELL[phys])
    return [f64_of(v) for v in got] if phys == "float64" else got


def id_runs(n, seed):
    """row-id lists: consecutive runs, scattered ids and repeated ids (each at most a few thousand long)"""
    if n == 0:
        return [[]]
    r = random.Random(seed)
    runs = list(range(min(n, 3000))) + list(range(max(0, n - 700), n))
    scattered = [r.randrange(n) for _ in range(min(2000, 2 * n))]
    repeated = [r.randrange(n)] * 5 + [0, 0, n - 1, n - 1] + [x for i in r.sample(range(n), min(n, 100)) for x in (i, i + 1 if i + 1 < n else i, i)]
    return [runs, scattered, repeated]


def check_reads(raw, cols: dict, keysets=(), seed=0):
    """cols: {column: (phys, cells)}, the table in row order.  Every column reads back its cells and validity at consecutive,
    scattered and repeated row ids; every orderable column orders as reference_order, ASC and DESC, at limits 0, 1, 17, n and n + 5;
    each key list of `keysets` orders as reference_order."""
    n = raw.num_rows
    wrong = []  # every mismatch, not just the first: a failure names all the reads it broke, once each
    for c, (phys, cells) in cols.items():
        assert len(cells) == n, c
        for ids in id_runs(n, seed):
            if read(raw, c, phys, ids) != [cells[i] for i in ids]:
                wrong.append(("gather", c))
        if phys == "float64":
            continue  # ORDER BY refuses doubles
        for desc in (False, True):
            want = R.reference_order([cells], [(0, desc)])
            for limit in sorted({0, 1, 17, n, n + 5}):
                got = raw.order_by_keys([(c, desc)], limit=limit) if phys == "utf8" else raw.order_by(c, descending=desc, limit=limit)
                if got != want[:limit]:
                    wrong.append(("order", c, "desc" if desc else "asc"))
    by_name = {c: cells for c, (_, cells) in cols.items()}
    for keys in keysets:
        want = R.reference_order(by_name, keys)
        if raw.order_by_keys(keys) != want or raw.order_by_keys(keys, limit=17) != want[:17]:
            wrong.append(("order", tuple(keys)))
    assert not wrong, list(dict.fromkeys(wrong))


def check_base(ctx, t, data, seed):
    cols = {c: (phys, cells_of(phys, *data[c])) for c, phys, _, _ in BASE_COLUMNS}
    check_reads(P.RawTable(ctx, t.h), cols, BASE_KEYS, seed)


# ---------------------------------------------------------------------------------------------------- base batches
@pytest.mark.parametrize("offset", [0, 3, 7])
@pytest.mark.parametrize("n", [1, 4095, 4096, 4097, 65536, 65537])
def test_device_batches(gpu_ctx, n, offset):
    data = base_values(n * 8 + offset, n)
    t = device_table(gpu_ctx, f"dev{n}_{offset}", data, n, offset)
    check_base(gpu_ctx, t, data, n)
    t.clear()


def test_device_batch_of_a_million_rows(gpu_ctx):
    n = 1_000_003
    data = base_values(5, n)
    t = device_table(gpu_ctx, "dev1m", data, n, 3)
    check_base(gpu_ctx, t, data, n)
    t.clear()


STAGING = {"packed+narrow": ("1", "1"), "packed": ("1", "0"), "narrow": ("0", "1"), "plain": ("0", "0")}


@pytest.fixture(scope="module", params=list(STAGING))
def staged_ctx(request):
    """a context created under one HOST staging mode (the context reads LDB_PACKED_STAGING / LDB_NARROW_STAGING when it is made):
    below 65 536 rows a batch is copied (decimals narrowed to 8 bytes unless narrowing is off), from 65 536 rows on it is packed
    (unless packing is off)"""
    packed, narrow = STAGING[request.param]
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("LDB_PACKED_STAGING", packed)
        mp.setenv("LDB_NARROW_STAGING", narrow)
        ctx = runtime.Context(0)
    yield ctx
    ctx.close()


@pytest.mark.parametrize("offset", [0, 3])
@pytest.mark.parametrize("n", [0, 1, 4095, 4096, 4097, 65535, 65536, 65537])
def test_host_batches(staged_ctx, n, offset):
    data = base_values(n * 8 + offset + 1, n)
    t = host_table(staged_ctx, f"host{n}_{offset}", data, n, offset)
    check_base(staged_ctx, t, data, n)
    t.clear()


def test_host_batch_of_a_million_rows(gpu_ctx):
    n = 1_000_003
    data = base_values(6, n)
    t = host_table(gpu_ctx, "host1m", data, n)
    check_base(gpu_ctx, t, data, n)
    t.clear()


def test_all_keys_equal_and_desc_over_heavy_ties(gpu_ctx):
    n = 70_000
    rng = np.random.default_rng(3)
    data = base_values(4, n, null_share=0.0)
    data["i32"] = (np.full(n, -7, np.int32), np.zeros(n, bool))                    # one value
    data["i64"] = (rng.integers(-1, 2, n).astype(np.int64), rng.random(n) < 0.3)   # three values and NULLs
    data["dt"] = (np.zeros(n, np.int32), np.ones(n, bool))                         # NULL everywhere
    data["s"] = ([b"same"] * n, rng.random(n) < 0.5)
    t = host_table(gpu_ctx, "ties", data, n)
    check_base(gpu_ctx, t, data, 4)
    t.clear()


# ---------------------------------------------------------------------------------------------------- library-made tables
def test_exported_group_tables(gpu_ctx):
    """NULL keys (two keys, so the NULLs of k0 are ordered by k1), and SUM / MIN / MAX and the f64 MIN / MAX over groups whose
    inputs are all NULL: the cells under those NULLs are 0, an identity value or NaN bits"""
    n = 30_000
    rng = np.random.default_rng(11)
    g = rng.integers(-40, 40, n).astype(np.int32)
    h = rng.integers(0, 6, n).astype(np.int32)
    v = _ints(rng, n, 64) >> 2
    w = _wide(rng, n)
    gnull, hnull = rng.random(n) < 0.1, rng.random(n) < 0.1
    vnull = (np.abs(g) % 7 == 0) | (rng.random(n) < 0.2)  # every group of g = 0, ±7, ±14 … has no v
    wnull = (np.abs(g) % 5 == 0) | (rng.random(n) < 0.2)
    spec = [("g", "int32", 0, 0), ("h", "int32", 0, 0), ("v", "int64", 0, 0), ("w", "decimal128", 38, 0)]
    raw = {"g": (g, gnull), "h": (h, hnull), "v": (v, vnull), "w": (w, wnull)}
    t = runtime.Table(gpu_ctx, "gsrc", R.specs_of(spec))
    chunk = {}
    for c, phys, _, _ in spec:
        chunk[c], chunk[c + "$valid"] = arrow(phys, *raw[c], 0)
    t.append_host(chunk, n)
    cells = {c: cells_of(phys, *raw[c]) for c, phys, _, _ in spec}
    fv = [None if x is None else float(x) for x in cells["v"]]
    aggs = [("sum", col("v"), cells["v"]), ("min", col("v"), cells["v"]), ("max", col("v"), cells["v"]), ("count", col("v"), cells["v"]),
            ("min_f64", ("i2f", col("v")), fv), ("max_f64", ("i2f", col("v")), fv), ("sum", col("w"), cells["w"]), ("max", col("w"), cells["w"])]
    st = P.group_by(gpu_ctx, t, [col("g"), col("h")], [(k, e) for k, e, _ in aggs], expected_groups=4096)
    want = R.group_by(n, [cells["g"], cells["h"]], [(k, vals) for k, _, vals in aggs])
    gt = P.groups_table(gpu_ctx, st)
    m = gt.num_rows
    phys = {"k0": "int64", "k1": "int64"}
    phys.update({f"a{i}": "float64" if k.endswith("_f64") else "decimal128" for i, (k, _, _) in enumerate(aggs)})
    got = {c: read(gt, c, p, list(range(m))) for c, p in phys.items()}
    assert {(k0, k1): [got[f"a{i}"][r] for i in range(len(aggs))] for r, (k0, k1) in enumerate(zip(got["k0"], got["k1"]))} == want
    assert any(x is None for x in got["k0"]) and all(any(x is None for x in got[f"a{i}"]) for i in (0, 1, 2, 4, 5, 6, 7))
    check_reads(gt, {c: (p, got[c]) for c, p in phys.items()},
                [[("k0", False), ("k1", True)], [("k0", True), ("a0", False)], [("a1", False), ("a7", True), ("k1", False), ("k0", False)],
                 [("a3", True), ("a2", True), ("k0", False), ("k1", False)]], seed=11)
    gt.destroy()
    runtime.state_destroy(gpu_ctx, st)
    t.clear()


def test_materialized_rows_with_null_outputs(gpu_ctx):
    """a left outer probe_each's side column (NULL without a match, and where the build column is NULL), a NULL-propagating sum and a
    CASE whose chosen branch is NULL"""
    rng = np.random.default_rng(12)
    nb, n = 3000, 40_000
    bk = (rng.permutation(nb) * 2).astype(np.int32)  # even keys only: odd probe keys miss
    bv, bnull = _ints(rng, nb, 64), rng.random(nb) < 0.2
    bt = runtime.Table(gpu_ctx, "mbuild", R.specs_of([("bk", "int32", 0, 0), ("bv", "int64", 0, 0)]))
    bt.append_host({"bk": bk, "bv": bv, "bv$valid": arrow("int64", bv, bnull, 0)[1]}, nb)
    k = rng.integers(0, 2 * nb, n).astype(np.int32)
    x, xnull = _ints(rng, n, 64) >> 1, rng.random(n) < 0.2
    y, ynull = _ints(rng, n, 32), rng.random(n) < 0.2
    z = _wide(rng, n)
    znull = rng.random(n) < 0.3
    spec = [("k", "int32", 0, 0), ("x", "int64", 0, 0), ("y", "int32", 0, 0), ("z", "decimal128", 38, 0)]
    raw = {"k": (k, np.zeros(n, bool)), "x": (x, xnull), "y": (y, ynull), "z": (z, znull)}
    pt = runtime.Table(gpu_ctx, "mprobe", R.specs_of(spec))
    chunk = {}
    for c, phys, _, _ in spec:
        chunk[c], chunk[c + "$valid"] = arrow(phys, *raw[c], 0)
    pt.append_host(chunk, n)
    jt = runtime.join_table(gpu_ctx, nb)
    P.build_join(gpu_ctx, bt, jt, col("bk"), payload=("rowid",))
    m = ("probe_each", jt, col("k"), "outer")
    outs = [("rowid",), ("fetch", bt, m, "bv"), ("add", col("x"), col("y")), ("case", ("cmp", ">", col("y"), const(0)), col("x"), col("z"))]
    mt = P.RawTable(gpu_ctx, P.materialize(gpu_ctx, pt, outs))
    c = {f: cells_of(p, *raw[f]) for f, p, _, _ in spec}
    row_of = {int(key): i for i, key in enumerate(bk)}
    bcells = cells_of("int64", bv, bnull)
    want = {i: [bcells[row_of[c["k"][i]]] if c["k"][i] in row_of else None,
                None if c["x"][i] is None or c["y"][i] is None else c["x"][i] + c["y"][i],
                c["x"][i] if c["y"][i] is not None and c["y"][i] > 0 else c["z"][i]] for i in range(n)}
    rows = mt.num_rows
    got = {f"c{j}": mt.gather(f"c{j}", list(range(rows))) for j in range(4)}
    assert {r: [got["c1"][q], got["c2"][q], got["c3"][q]] for q, r in enumerate(got["c0"])} == want
    assert all(None in got[f"c{j}"] for j in (1, 2, 3))
    check_reads(mt, {f: ("decimal128", v) for f, v in got.items()},
                [[("c1", False), ("c2", True), ("c0", False)], [("c3", True), ("c1", False), ("c2", False)], [("c2", False), ("c0", True)]], seed=12)
    mt.destroy()
    runtime.state_destroy(gpu_ctx, jt)
    for tab in (bt, pt):
        tab.clear()


def test_join_marker_tables(gpu_ctx):
    rng = np.random.default_rng(13)
    nb = 20_000
    bk = rng.choice(np.arange(-50_000, 50_000), nb, replace=False).astype(np.int32)
    bt = runtime.Table(gpu_ctx, "kbuild", R.specs_of([("bk", "int32", 0, 0)]))
    bt.append_host({"bk": bk}, nb)
    pk = rng.integers(-50_000, 50_000, 30_000).astype(np.int32)
    pt = runtime.Table(gpu_ctx, "kprobe", R.specs_of([("pk", "int32", 0, 0)]))
    pt.append_host({"pk": pk}, len(pk))
    jt = runtime.join_table(gpu_ctx, nb)
    P.build_join(gpu_ctx, bt, jt, col("bk"), payload=("rowid",))
    P.run_effects(gpu_ctx, pt, [("mark", ("probe", jt, col("pk")), ("cmp", ">", col("pk"), const(-20_000)))])
    mt = P.join_marks(gpu_ctx, jt, P.ALL)
    m = mt.num_rows
    phys = {"key": "int64", "payload": "int64", "marked": "int32"}
    got = {c: read(mt, c, p, list(range(m))) for c, p in phys.items()}
    hit = {int(x) for x in pk if x > -20_000}
    assert sorted(zip(got["key"], got["payload"], got["marked"])) == sorted((int(x), i, int(int(x) in hit)) for i, x in enumerate(bk))
    check_reads(mt, {c: (p, got[c]) for c, p in phys.items()}, [[("marked", True), ("key", False)], [("marked", False), ("payload", True)]], seed=13)
    mt.destroy()
    runtime.state_destroy(gpu_ctx, jt)
    for tab in (bt, pt):
        tab.clear()


def test_dictionary_ranks_are_the_reference_order(gpu_ctx):
    rng = np.random.default_rng(14)
    n = 50_000
    s = _strings(rng, n)
    null = rng.random(n) < 0.1
    t = runtime.Table(gpu_ctx, "dsrc", R.specs_of([("s", "utf8", 0, 0)]))
    buf, bitmap = arrow("utf8", s, null, 0)
    t.append_host({"s": buf, "s$valid": bitmap}, n)
    d = P.dict_state(gpu_ctx, 8192, 1 << 20)
    P.run_effects(gpu_ctx, t, [("strcode", d, "s")])
    dt = P.dict_table(gpu_ctx, d)
    m = dt.num_rows
    strs = dt.gather_strings("str", list(range(m)), decode=False)
    assert sorted(strs) == sorted({v for v, z in zip(s, null) if not z})
    ranks = dt.gather("rank", list(range(m)), cell_bytes=4)
    order = R.reference_order([strs], [(0, False)])
    assert [ranks[i] for i in order] == list(range(m))
    check_reads(dt, {"str": ("utf8", strs), "rank": ("int32", ranks)}, [[("rank", True)], [("str", True), ("rank", False)]], seed=14)
    dt.destroy()
    runtime.state_destroy(gpu_ctx, d)
    t.clear()
