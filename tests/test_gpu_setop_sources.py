"""Set operations (ldb_gpu_table_setop) where their device map is most likely to be wrong, cell for cell and in order against the exact
model in tests/_setopref.py (numpy for the large tables, as tests/test_gpu_setop.py's contention test does):

1. full collisions: thousands of distinct rows with one 64-bit row hash (so one home slot and one tag: every probe is a tag match and
   only the row compare decides), built with tests/_keyhash.py's solvers: one-column decimal and utf8 rows, multi-column rows whose
   last cell compensates, rows that differ only in a decimal's high half or in one byte of a string, and NULL against the value whose
   word is the NULL word in int64, float64, decimal128 and utf8 columns; true duplicates in the same chain, colliding rows on both sides;
2. chains that start at the directory's last slot and wrap to slot 0, with equal tags and with distinct tags;
3. 63 to 66 copies on each side (the scan's store writes up to 64 itself), and more rows of 65-300 copies than setBigKernel has CTAs;
4. sources: HOST batches under each staging mode at 65 535 / 65 536 rows and bit offsets 0 and 3 with garbage under NULL cells,
   DEVICE batches at bit offsets 0, 3 and 7 with utf8 offsets past 0, exported groups (float64 in 16-byte cells), join-marker and
   dictionary tables, set-operation and window results, narrowed decimals on either side, batches with and without a bitmap, empty
   batches, hundreds of one-row batches, swapped column lists over one table, NULL ("every column") against an explicit list;
5. emitting-row counts on and next to the scan's 2 048-row tiles and 524 288-row chunks, and 2^20;
6. errors: a repeated left column name refused before any launch, and the 2^31 - 1 byte limit of a utf8 result."""
import ctypes as C
import random
import struct

import numpy as np
import pytest

import _keyhash as K
import _progref as R
import _setopref as S
from lingodb_b200 import capi
from test_gpu_result_reads import BASE_COLUMNS, STAGING, _strings, arrow, base_values, cells_of, device_table, host_table, read
from test_gpu_setop import COLUMNS, PHYS, RIGHT_COLUMNS, check_against_model, first_order_counts, gen_rows, group_fn, stage
from test_gpu_window import read_column, read_fixed

pytestmark = pytest.mark.gpu


def spec_of(names, phys):
    return [(n, p, 38 if p == "decimal128" else 0, 2 if p == "decimal128" else 0) for n, p in zip(names, phys)]


_STAGED = []  # every table host() and int_table() staged on the session's context, cleared when this module ends


@pytest.fixture(scope="module", autouse=True)
def _clear_staged():
    yield
    for t in _STAGED:
        t.clear()
    _STAGED.clear()


def host(ctx, name, names, phys, rows, cuts=()):
    from lingodb_b200 import program as P
    values = {c: [r[j] for r in rows] for j, c in enumerate(names)}
    _STAGED.append(ctx.table_from_host(R.to_table_data(name, values, spec_of(names, phys), cuts)))
    return P.RawTable(ctx, _STAGED[-1].h)


def every_kind(ctx, L, Rt, names, phys, lrows, rrows, what, kinds=S.KINDS):
    for kind in kinds:
        if kind == "distinct":
            out, want = L.distinct(names), S.setop("distinct", lrows)
        else:
            out, want = L.setop(Rt, kind, names, names), S.setop(kind, lrows, rrows)
        check_against_model(out, names, phys, want, (what, kind))
        out.destroy()


def sides(pool, rng, dup=3):
    """left and right rows over a pool of distinct rows: each pool row 0..dup times per side, shuffled, some rows on one side only"""
    left, right = [], []
    for i, r in enumerate(pool):
        left += [r] * (rng.randrange(dup + 1) if i % 5 else 0)
        right += [r] * (rng.randrange(dup + 1) if i % 7 else 0)
    rng.shuffle(left)
    rng.shuffle(right)
    return left, right


# ---------------------------------------------------------------------------------------------------- 1. full collisions
def collision_pool(kind: str, target: int, n: int, rng):
    """(names, phys, n distinct rows, each with row hash `target`)"""
    w0 = K.last_word([], target)
    if kind == "decimal":  # one column; rows differ in the high half (and so the low)
        return ["d"], ["decimal128"], [(K.decimal_for(w0, rng.getrandbits(64) if i % 2 else i),) for i in range(n)]
    if kind == "utf8":  # one column; 16- and 24-byte strings, one chunk solved
        rows = []
        for i in range(n):
            tail = i.to_bytes(8, "little")
            rows.append((K.utf8_for(w0, b"\0" * 8 + tail) if i % 3 else K.utf8_for(w0, b"prefix!!" + b"\0" * 8 + tail, 1),))
        return ["s"], ["utf8"], rows
    if kind == "high_half":  # two decimals whose low halves are fixed: the rows differ only in high halves
        lo1, lo2 = rng.getrandbits(64), rng.getrandbits(64)
        rows = []
        for i in range(n):
            d1 = R.wrap128(((i + 1) << 64) | lo1)
            w2 = K.last_word([K.int_word(d1)], target)
            rows.append((d1, R.wrap128((K.unmix64(w2 ^ lo2) << 64) | lo2)))
        return ["d1", "d2"], ["decimal128", "decimal128"], rows
    if kind == "one_byte":  # two 16-byte strings: the first differs from a base in one byte, the second compensates
        base = bytearray(b"one byte differs")
        rows = []
        for i in range(n):
            s1 = bytearray(base)
            s1[i % 16] = (base[i % 16] + 1 + i // 16) % 256
            s1 = bytes(s1)
            rows.append((s1, K.utf8_for(K.last_word([K.str_hash(s1)], target), b"\0" * 16)))
        return ["s1", "s2"], ["utf8", "utf8"], list(dict.fromkeys(rows))
    # multi-column rows whose early columns differ, the last one of type `kind` compensating (int64 and float64 always / nearly always)
    last = {"multi_decimal": "decimal128", "multi_utf8": "utf8", "multi_f64": "float64", "multi_i64": "int64"}[kind]
    names, phys = ["a", "b", "c", "z"], ["int64", "utf8", "float64", last]
    rows = []
    while len(rows) < n:
        a = rng.choice([None, rng.randrange(-50, 50), rng.getrandbits(63)])
        b = rng.choice([None, b"", b"x" * rng.randrange(0, 20), bytes(rng.randrange(256) for _ in range(9))])
        c = rng.choice([None, 0.0, -0.0, float("nan"), rng.random() * 100])
        z = K.cell_for(last, K.last_word([K.cell_word(p, v) for p, v in zip(phys, (a, b, c))], target), rng.getrandbits(64))
        if z is not None:
            rows.append((a, b, c, z))
    rows = list({S.canon(r): r for r in rows}.values())  # distinct under the set operations' equality
    return names, phys, rows


def null_word_pool(n: int, rng):
    """rows (i, NULL, z) and (i, W, z), W the value of the middle column's type whose word is the NULL word, z solving every row to one
    hash; and the one-column pairs NULL / W of each type"""
    target = rng.getrandbits(64)
    pools = []
    for p in ("int64", "float64", "decimal128", "utf8"):
        w = K.cell_for(p, K.NULL_WORD, b"\0" * 8 if p == "utf8" else 7)
        assert w is not None and K.cell_word(p, w) == K.NULL_WORD
        rows = []
        for i in range(n):
            for mid in (None, w):
                z = K.decimal_for(K.last_word([K.int_word(i), K.cell_word(p, mid)], target), i % 3)
                rows.append((i, mid, z))
        pools.append((["i", "m", "z"], ["int64", p, "decimal128"], rows))
        pools.append((["m"], [p], [(None,), (w,)]))
    return pools


@pytest.mark.parametrize("kind", ["decimal", "utf8", "high_half", "one_byte", "multi_decimal", "multi_utf8", "multi_f64", "multi_i64"])
def test_full_collisions(gpu_ctx, kind):
    rng = random.Random(sum(map(ord, kind)))
    n = 16000 if kind == "decimal" else 3000
    target = rng.getrandbits(64)
    names, phys, pool = collision_pool(kind, target, n, rng)
    assert len(pool) > n // 2 and all(K.row_hash_of(phys, r) == target for r in pool)
    assert len({S.canon(r) for r in pool}) == len(pool)
    left, right = sides(pool, rng)
    L, Rt = host(gpu_ctx, "cl", names, phys, left, [len(left) // 3]), host(gpu_ctx, "cr", names, phys, right)
    every_kind(gpu_ctx, L, Rt, names, phys, left, right, kind)


def test_null_against_the_null_word(gpu_ctx):
    rng = random.Random(17)
    for names, phys, pool in null_word_pool(1500, rng):
        if len(pool) > 2:
            assert len({K.row_hash_of(phys, r) for r in pool}) == 1
        else:
            assert K.row_hash_of(phys, pool[0]) == K.row_hash_of(phys, pool[1])
        left, right = sides(pool * (40 if len(pool) == 2 else 1), rng, 2)
        left, right = left + list(pool), right + [pool[0]]  # every row on the left, NULL on the right
        L, Rt = host(gpu_ctx, "nl", names, phys, left), host(gpu_ctx, "nr", names, phys, right)
        every_kind(gpu_ctx, L, Rt, names, phys, left, right, ("null word", phys))


# ---------------------------------------------------------------------------------------------------- 2. wrap-around
def test_chains_wrap_from_the_last_slot(gpu_ctx):
    """row hashes whose low 32 bits are all ones: every chain's home is the last slot of any directory"""
    rng = random.Random(23)
    tag = rng.getrandbits(32)
    equal = collision_pool("decimal", (tag << 32) | 0xFFFFFFFF, 3000, rng)[2]
    distinct = [(K.decimal_for(K.last_word([], (t << 32) | 0xFFFFFFFF), 5),) for t in rng.sample(range(1 << 32), 3000)]
    for pool in (equal, distinct, equal[:1500] + distinct[:1500]):
        left, right = sides(pool, rng)
        for n in (len(left), 1, 3, 700):  # small left sides: small directories, the chain wraps many times
            lrows = left[:n]
            L, Rt = host(gpu_ctx, "wl", ["d"], ["decimal128"], lrows), host(gpu_ctx, "wr", ["d"], ["decimal128"], right)
            every_kind(gpu_ctx, L, Rt, ["d"], ["decimal128"], lrows, right, ("wrap", n))


# ---------------------------------------------------------------------------------------------------- 3. many copies
def int_table(ctx, name, a):
    from lingodb_b200 import datagen
    from lingodb_b200 import program as P
    _STAGED.append(ctx.table_from_host(datagen.TableData(name, [datagen.ColumnSpec("k", "int64")], [{"k": np.asarray(a, np.int64)}], [len(a)])))
    return P.RawTable(ctx, _STAGED[-1].h)


def read_k(t):
    return np.array(read_fixed(t, "k", 8), np.int64)


def test_copies_around_the_direct_limit(gpu_ctx):
    counts = [0, 1, 63, 64, 65, 66, 130]
    rng = random.Random(29)
    left, right = [], []
    for i, (cl, cr) in enumerate((a, b) for a in counts for b in counts):
        left += [(i,)] * cl
        right += [(i,)] * cr
    rng.shuffle(left)
    rng.shuffle(right)
    L, Rt = host(gpu_ctx, "ml", ["k"], ["int64"], left), host(gpu_ctx, "mr", ["k"], ["int64"], right)
    every_kind(gpu_ctx, L, Rt, ["k"], ["int64"], left, right, "copies", kinds=("intersect_all", "except_all", "union", "distinct"))


def test_more_rows_of_many_copies_than_big_ctas(gpu_ctx):
    """3 000 values of 65-300 copies (setBigKernel runs smCount x 4 CTAs, 528 on an H100 SXM) among direct rows"""
    rng = np.random.default_rng(31)
    nbig = 3000
    cl = rng.integers(65, 301, nbig)
    a = np.concatenate([np.repeat(np.arange(nbig), cl), rng.integers(10_000, 30_000, 50_000)])
    cr = np.where(rng.random(nbig) < 0.5, rng.integers(0, 301, nbig), 0)
    b = np.concatenate([np.repeat(np.arange(nbig), cr), rng.integers(20_000, 40_000, 20_000)])
    a, b = rng.permutation(a), rng.permutation(b)
    L, Rt = int_table(gpu_ctx, "bl", a), int_table(gpu_ctx, "br", b)
    va, ca = first_order_counts(a)
    vb = dict(zip(*first_order_counts(b)))
    c_r = np.array([vb.get(v, 0) for v in va.tolist()], np.int64)
    for kind, times in (("intersect_all", np.minimum(ca, c_r)), ("except_all", np.maximum(ca - c_r, 0))):
        assert (times > 64).sum() > 4 * 132, kind
        out = L.setop(Rt, kind)
        assert np.array_equal(read_k(out), np.repeat(va, times)), kind
        out.destroy()


# ---------------------------------------------------------------------------------------------------- 4. sources
BASE_NAMES = [c for c, *_ in BASE_COLUMNS]


def base_rows(data):
    return list(zip(*[cells_of(p, *data[c]) for c, p, _, _ in BASE_COLUMNS]))


def base_check(ctx, L, lrows, Rt, rrows, what, kinds=("distinct", "union", "intersect_all", "except")):
    names = [c for c, *_ in BASE_COLUMNS]
    phys = [p for _, p, _, _ in BASE_COLUMNS]
    every_kind(ctx, L, Rt, names, phys, lrows, rrows, what, kinds)


@pytest.fixture(scope="module", params=["packed+narrow", "packed", "narrow", "plain"])
def staged_ctx(request):
    from lingodb_b200 import runtime
    packed, narrow = STAGING[request.param]
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("LDB_PACKED_STAGING", packed)
        mp.setenv("LDB_NARROW_STAGING", narrow)
        ctx = runtime.Context(0)
    yield ctx
    ctx.close()


def _pooled(seed, n):
    """base_values whose rows repeat: every column drawn from the same 3 000 source rows, so whole rows tie"""
    pool = base_values(seed, 3000)
    idx = np.random.default_rng(seed).integers(0, 3000, n)
    return {c: ([raw[i] for i in idx] if isinstance(raw, list) else raw[idx], null[idx]) for c, (raw, null) in pool.items()}


@pytest.mark.parametrize("offset", [0, 3])
@pytest.mark.parametrize("n", [65535, 65536])
def test_host_batches_under_each_staging_mode(staged_ctx, n, offset):
    from lingodb_b200 import program as P
    data, other = _pooled(n + offset, n), _pooled(n + offset, 5000)  # the same pool: the right side shares rows
    t, u = host_table(staged_ctx, "hl", data, n, offset), host_table(staged_ctx, "hr", other, 5000, offset)
    base_check(staged_ctx, P.RawTable(staged_ctx, t.h), base_rows(data), P.RawTable(staged_ctx, u.h), base_rows(other), ("host", n, offset))
    t.clear()
    u.clear()


@pytest.mark.parametrize("offset", [0, 3, 7])
def test_device_batches_at_bit_offsets(gpu_ctx, offset):
    from lingodb_b200 import program as P
    data, other = _pooled(40 + offset, 9000), _pooled(40 + offset, 4000)
    t, u = device_table(gpu_ctx, "dl", data, 9000, offset), host_table(gpu_ctx, "dr", other, 4000, 0)
    base_check(gpu_ctx, P.RawTable(gpu_ctx, t.h), base_rows(data), P.RawTable(gpu_ctx, u.h), base_rows(other), ("device", offset),
               kinds=S.KINDS)
    t.clear()
    u.clear()


def test_exported_groups_against_staged_floats(gpu_ctx):
    """a group table's int64 keys (8-byte cells) and float64 aggregate (16-byte cells) against a staged (int64, float64) table"""
    from lingodb_b200 import program as P, runtime
    col = lambda x: ("col", x)
    rng = np.random.default_rng(37)
    n = 20000
    g = rng.integers(-40, 40, n).astype(np.int64)
    v = rng.integers(-5, 5, n).astype(np.int64)
    t = runtime.Table(gpu_ctx, "gsrc", R.specs_of([("g", "int64", 0, 0), ("v", "int64", 0, 0)]))
    t.append_host({"g": g, "v": v, "v$valid": np.packbits(rng.random(n) > 0.05, bitorder="little")}, n)
    st = P.group_by(gpu_ctx, t, [col("g")], [("min_f64", ("i2f", col("v")))], expected_groups=256)
    gt = P.groups_table(gpu_ctx, st)
    m = gt.num_rows
    ids = list(range(m))
    grows = list(zip(read(gt, "k0", "int64", ids), read(gt, "a0", "float64", ids)))
    right = grows[::2] + [(k, None if x is None else x + 1.0) for k, x in grows[1::3]] + [(None, -0.0), (3, 0.0)]
    Rt = host(gpu_ctx, "gr", ["k0", "a0"], ["int64", "float64"], right)
    every_kind(gpu_ctx, gt, Rt, ["k0", "a0"], ["int64", "float64"], grows, right, "groups")
    gt.destroy()
    runtime.state_destroy(gpu_ctx, st)
    t.clear()


def test_join_marker_and_dictionary_tables(gpu_ctx):
    from lingodb_b200 import program as P, runtime
    col, const = (lambda x: ("col", x)), (lambda v: ("const", v))
    rng = np.random.default_rng(41)
    nb = 5000
    bk = rng.choice(np.arange(-20_000, 20_000), nb, replace=False).astype(np.int32)
    bt = runtime.Table(gpu_ctx, "kb", R.specs_of([("bk", "int32", 0, 0)]))
    bt.append_host({"bk": bk}, nb)
    pk = rng.integers(-20_000, 20_000, 8000).astype(np.int32)
    pt = runtime.Table(gpu_ctx, "kp", R.specs_of([("pk", "int32", 0, 0)]))
    pt.append_host({"pk": pk}, len(pk))
    jt = runtime.join_table(gpu_ctx, nb)
    P.build_join(gpu_ctx, bt, jt, col("bk"), payload=("rowid",))
    P.run_effects(gpu_ctx, pt, [("mark", ("probe", jt, col("pk")), ("cmp", ">", col("pk"), const(-5000)))])
    mt = P.join_marks(gpu_ctx, jt, P.ALL)
    ids = list(range(mt.num_rows))
    mrows = list(zip(read(mt, "key", "int64", ids), read(mt, "marked", "int32", ids)))
    right = [(k % 7, mk) for k, mk in mrows[:3000]] + mrows[::3]
    Rt = host(gpu_ctx, "mr", ["key", "marked"], ["int64", "int32"], right)
    every_kind(gpu_ctx, mt, Rt, ["key", "marked"], ["int64", "int32"], mrows, right, "marks")
    d1 = mt.distinct(["marked"])
    check_against_model(d1, ["marked"], ["int32"], S.setop("distinct", [(mk,) for _, mk in mrows]), "marks distinct")
    d1.destroy()
    n = 20000
    s = _strings(rng, n)
    t = runtime.Table(gpu_ctx, "dsrc", R.specs_of([("s", "utf8", 0, 0)]))
    buf, bitmap = arrow("utf8", s, rng.random(n) < 0.1, 0)
    t.append_host({"s": buf, "s$valid": bitmap}, n)
    d = P.dict_state(gpu_ctx, 8192, 1 << 20)
    P.run_effects(gpu_ctx, t, [("strcode", d, "s")])
    dt = P.dict_table(gpu_ctx, d)
    m = dt.num_rows
    drows = list(zip(dt.gather_strings("str", list(range(m)), decode=False), dt.gather("rank", list(range(m)), cell_bytes=4)))
    right = drows[::2] + [(x, r + 1) for x, r in drows[1::5]] + [(None, 0)]
    Rt2 = host(gpu_ctx, "dr", ["str", "rank"], ["utf8", "int32"], right)
    every_kind(gpu_ctx, dt, Rt2, ["str", "rank"], ["utf8", "int32"], drows, right, "dictionary")
    dt.destroy()
    mt.destroy()
    runtime.state_destroy(gpu_ctx, d)
    runtime.state_destroy(gpu_ctx, jt)
    for tab in (bt, pt, t):
        tab.clear()


def test_setop_and_window_results(gpu_ctx):
    """a DISTINCT result (validity bytes, 16-byte decimals) and a window result (one batch in window order) as sources"""
    n = 3000
    values = gen_rows(n, group_fn(400), 43)
    t = stage(gpu_ctx, values, COLUMNS, "single", 43)
    names = ["i8", "dn", "s", "f8", "dw"]
    phys = [PHYS[c] for c in names]
    rows = list(zip(*[values[c] for c in names]))
    d = t.distinct(names)
    drows = S.setop("distinct", rows)
    every_kind(gpu_ctx, d, t, names, phys, drows, rows, "distinct result")
    w = t.window(partition_by=["i32"], order_by=[], frame=(None, None), funcs=[("row_number", None, "rn")], columns=names)
    wrows = list(zip(*[read_column(w, c, p) for c, p in zip(names, phys)]))
    wrows = [tuple(x if p != "float64" or x is None else struct.unpack("<d", struct.pack("<q", x))[0] for x, p in zip(r, phys)) for r in wrows]
    every_kind(gpu_ctx, w, d, names, phys, wrows, drows, "window result")
    w.destroy()
    d.destroy()


def test_narrowed_decimals_on_either_side(gpu_ctx):
    n = 4000
    left, right = gen_rows(n, group_fn(900), 47), gen_rows(n // 2, group_fn(900, 300), 48)
    names = ["dn", "i64", "s"]
    phys = [PHYS[c] for c in names]
    lrows, rrows = list(zip(*[left[c] for c in names])), list(zip(*[right[c] for c in names]))
    narrow, wide = stage(gpu_ctx, left, COLUMNS, "single", 47), stage(gpu_ctx, right, RIGHT_COLUMNS, "ragged", 48)
    every_kind(gpu_ctx, narrow, wide, names, phys, lrows, rrows, "narrow left")
    wide_l, narrow_r = stage(gpu_ctx, left, RIGHT_COLUMNS, "offset", 49), stage(gpu_ctx, right, COLUMNS, "single", 50)
    every_kind(gpu_ctx, wide_l, narrow_r, names, phys, lrows, rrows, "narrow right")


def batches_table(ctx, name, names, phys, rows, sizes):
    """a HOST table cut into batches of `sizes` rows (0 = an empty batch); a batch whose cells hold no NULL has no bitmap"""
    from lingodb_b200 import runtime
    spec = spec_of(names, phys)
    t = runtime.Table(ctx, name, R.specs_of(spec))
    at = 0
    for k in sizes:
        ch = {}
        for j, (c, p, _, _) in enumerate(spec):
            buf, bm = R.column_buffers(p, [r[j] for r in rows[at:at + k]])
            ch[c] = buf
            if bm is not None:
                ch[c + "$valid"] = bm
        t.append_host(ch, k)
        at += k
    assert at == len(rows)
    return t


def test_batch_layouts(gpu_ctx):
    """empty batches first, between and last; batches with and without a bitmap on one side; 400 one-row batches"""
    from lingodb_b200 import program as P
    rng = random.Random(53)
    names, phys = ["i64", "s", "dw"], ["int64", "utf8", "decimal128"]
    pool = [(rng.randrange(50), rng.choice([b"a", b"bb", b"", None]), rng.choice([None, 1 << 70, -3, 5])) for _ in range(300)]
    clean = [(a, b or b"z", c or 1) for a, b, c in pool]  # no NULL cells: those batches carry no bitmap
    lrows = [rng.choice(pool) for _ in range(2000)] + [rng.choice(clean) for _ in range(1000)] + [rng.choice(pool) for _ in range(500)]
    rrows = [rng.choice(clean + pool) for _ in range(400)]
    lt = batches_table(gpu_ctx, "bl", names, phys, lrows, [0, 0, 2000, 0, 1000, 500, 0])
    rt = batches_table(gpu_ctx, "br", names, phys, rrows, [1] * 400)
    L, Rt = P.RawTable(gpu_ctx, lt.h), P.RawTable(gpu_ctx, rt.h)
    every_kind(gpu_ctx, L, Rt, names, phys, lrows, rrows, "batches")
    every_kind(gpu_ctx, Rt, L, names, phys, rrows, lrows, "batches swapped")
    lt.clear()
    rt.clear()


def test_swapped_lists_and_every_column(gpu_ctx):
    n = 3000
    values = gen_rows(n, group_fn(40), 59)
    t = stage(gpu_ctx, values, COLUMNS, "ragged", 59)
    for a, b in (("i64", "j64"), ("s", "s2"), ("f8", "e8")):
        p = [PHYS[a], PHYS[b]]
        ab, ba = list(zip(values[a], values[b])), list(zip(values[b], values[a]))
        for kind in S.KINDS[1:]:
            out = t.setop(t, kind, [a, b], [b, a])
            check_against_model(out, [a, b], p, S.setop(kind, ab, ba), ("swapped", a, kind))
            out.destroy()
    # NULL ("every column") on one side, an explicit list on the other
    names = ["i32", "dn", "s"]  # in COLUMNS order: the staged table's own order
    small = stage(gpu_ctx, {c: values[c] for c in names}, COLUMNS, "single", 60)
    rows = list(zip(*[values[c] for c in names]))
    phys = [PHYS[c] for c in names]
    for kind in S.KINDS[1:]:
        out = small.setop(t, kind, None, names)
        check_against_model(out, names, phys, S.setop(kind, rows, rows), ("left all", kind))
        out.destroy()
        out = t.setop(small, kind, names, None)
        check_against_model(out, names, phys, S.setop(kind, rows, rows), ("right all", kind))
        out.destroy()
    out = small.distinct()
    check_against_model(out, names, phys, S.setop("distinct", rows), "distinct all")
    out.destroy()


# ---------------------------------------------------------------------------------------------------- 5. scan edges
EDGES = [2047, 2048, 2049, 524287, 524288, 524289, 1 << 20]


@pytest.mark.parametrize("edge", EDGES)
def test_emitting_rows_at_the_scan_edges(gpu_ctx, edge):
    rng = np.random.default_rng(edge)
    a = rng.integers(0, max(2, edge // 3), edge)
    # DISTINCT: `edge` emitting rows
    L = int_table(gpu_ctx, "el", a)
    out = L.distinct()
    assert np.array_equal(read_k(out), first_order_counts(a)[0]), ("distinct", edge)
    out.destroy()
    # UNION: nL + nR on the edge, nL not
    nl = edge // 3 + 1
    u1, u2 = int_table(gpu_ctx, "u1", a[:nl]), int_table(gpu_ctx, "u2", a[nl:] + 7)
    out = u1.setop(u2, "union")
    assert np.array_equal(read_k(out), first_order_counts(np.concatenate([a[:nl], a[nl:] + 7]))[0]), ("union", edge)
    out.destroy()
    # EXCEPT ALL: nL on the edge
    b = rng.integers(0, max(2, edge // 3), edge // 2)
    Rt = int_table(gpu_ctx, "er", b)
    out = L.setop(Rt, "except_all")
    va, ca = first_order_counts(a)
    vb = dict(zip(*first_order_counts(b)))
    c_r = np.array([vb.get(v, 0) for v in va.tolist()], np.int64)
    assert np.array_equal(read_k(out), np.repeat(va, np.maximum(ca - c_r, 0))), ("except all", edge)
    out.destroy()


# ---------------------------------------------------------------------------------------------------- 6. errors
def test_repeated_left_names_are_refused_before_any_launch(gpu_ctx):
    from lingodb_b200 import datagen
    from lingodb_b200 import program as P
    ctx = gpu_ctx
    vals = gen_rows(40, group_fn(5), 61)
    L = stage(ctx, vals, COLUMNS, "single", 61)
    Rt = stage(ctx, vals, RIGHT_COLUMNS, "ragged", 62)
    dup = P.RawTable(ctx, ctx.table("dup", [datagen.ColumnSpec("x", "int64"), datagen.ColumnSpec("x", "int64")]).h)
    out, e = C.c_void_p(), capi.Error()
    enc = lambda xs: (C.c_char_p * len(xs))(*[x.encode() for x in xs])
    rc = lambda l, r, kind, n, lc, rc_: ctx.L.ldb_gpu_table_setop(l, r, kind, n, lc, rc_, None, C.byref(out), C.byref(e))
    before = ctx.launch_count()
    cases = [(L.h, None, capi.SETOP["distinct"], 2, enc(["i64", "i64"]), None, "i64"),
             (L.h, Rt.h, capi.SETOP["union"], 3, enc(["s", "i8", "s"]), enc(["s", "i8", "s2"]), "s"),
             (L.h, Rt.h, capi.SETOP["except_all"], 2, enc(["dn", "dn"]), enc(["dn", "dn"]), "dn"),
             (dup.h, None, capi.SETOP["distinct"], 0, None, None, "x"),
             (dup.h, dup.h, capi.SETOP["intersect"], 0, None, None, "x")]
    for l, r, kind, n, lc, rc_, clash in cases:
        assert rc(l, r, kind, n, lc, rc_) == capi.LDB_ERR_INVALID, clash
        assert clash in e.message.decode() and "two columns" in e.message.decode(), e.message
    assert ctx.launch_count() == before
    # a repeated right name is legal: right columns are positional
    out_t = L.setop(Rt, "union", ["i64", "j64"], ["i64", "i64"])
    want = S.setop("union", list(zip(vals["i64"], vals["j64"])), list(zip(vals["i64"], vals["i64"])))
    check_against_model(out_t, ["i64", "j64"], ["int64", "int64"], want, "repeated right name")
    out_t.destroy()


def test_utf8_result_byte_limit(gpu_ctx):
    """UNION ALL of borrowed DEVICE tables of 1 MiB strings: 2^31 - 1 bytes in the result is made, 2^31 refused naming the column"""
    import torch
    from lingodb_b200 import program as P, runtime
    ctx = gpu_ctx
    mib, rows = 1 << 20, 1024
    # byte i is i % 251, made from one 251-byte period so the test holds no more than the 1 GiB of strings and the 2 GiB result
    data = torch.arange(251, dtype=torch.uint8, device="cuda:0").repeat((rows * mib + 16) // 251 + 1)[:rows * mib + 16]
    full = torch.arange(rows + 1, dtype=torch.int32, device="cuda:0") * mib
    short = full.clone()
    short[-1] -= 1  # the last string one byte shorter

    def table(name, offs):
        t = runtime.Table(ctx, name, R.specs_of([("s", "utf8", 0, 0)]))
        t.append_device({"s": (offs, data)}, rows)
        return t
    a, b = table("a", full), table("b", short)
    A, B = P.RawTable(ctx, a.h), P.RawTable(ctx, b.h)
    out = A.setop(B, "union_all")
    assert out.num_rows == 2 * rows
    pattern = lambda start, n: bytes((np.arange(start, start + n, dtype=np.int64) % 251).astype(np.uint8))
    for i in (0, 1, 777, rows - 1, rows, rows + 1, 2 * rows - 2, 2 * rows - 1):
        s = out.gather_strings("s", [i], decode=False)[0]
        r = i % rows
        n = mib - 1 if i == 2 * rows - 1 else mib
        assert len(s) == n and s[:64] == pattern(r * mib, 64) and s[-64:] == pattern(r * mib + n - 64, 64), i
    out.destroy()
    with pytest.raises(capi.LdbRuntimeError) as ei:
        A.setop(A, "union_all")
    assert ei.value.code == capi.LDB_ERR_UNSUPPORTED
    msg = str(ei.value)
    assert "set operation" in msg and "utf8 column s" in msg and str(1 << 31) in msg, msg
    a.clear()
    b.clear()
    del data, full, short
    torch.cuda.empty_cache()  # hand the strings back to the device for the tests after this one
    # the context still works
    vals = gen_rows(50, group_fn(7), 67)
    t = stage(ctx, vals, COLUMNS, "single", 67)
    u = t.setop(t, "union", ["s", "i64"], ["s", "i64"])
    check_against_model(u, ["s", "i64"], ["utf8", "int64"], S.setop("union", list(zip(vals["s"], vals["i64"])), list(zip(vals["s"], vals["i64"]))), "after")
    u.destroy()
