"""The multi-GPU exchange layer against the exact reference of tests/_exchref.py, bit for bit: K6 partitioning, the fused partition-send
pipelines K10 / K11 read back sub-region by sub-region, the receive side (publish_counts, insert_received, probe_received_groupby and
_groupby2), the K7 merges (merge_rows, merge_exported, the peer all-merge) with their lane-width rules, and the peer collectives
(barrier, allgather_small, or_reduce) — including a collective issued after a captured one, and every documented error.

Ranks are contexts of this process on device 0 wired by parallel.Comm.local_group: the same kernels, flags and mailboxes as the
multi-process NVLink path.  Every rank issues every collective in the same order, and every comm and context is closed in `finally`."""
import contextlib
import ctypes as C
import os
import random
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest

import _exchref as X
import _piperef as P
from test_gpu_pipelines import SCHEMA, build_table, capi, expect_error, gpu_payloads, new_table, read_groups, rt, table, values

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SENTINEL = 0x5A5A5A5A
# user-heap layout of the pipeline tests
CURSORS, COUNTS, RECV = 0, 256, 1024


# ---------------------------------------------------------------------------------------------------- helpers
def par():
    from lingodb_b200 import parallel
    return parallel


@contextlib.contextmanager
def ranks(world: int, user_bytes: int = 1 << 20):
    """`world` contexts on device 0 and their comms; closed in `finally` (comms first)"""
    ctxs, comms = [], []
    try:
        ctxs = [rt().Context(0) for _ in range(world)]
        comms = par().Comm.local_group(ctxs, user_bytes=user_bytes)
        yield ctxs, comms
        for cm in comms:
            cm.check()
    finally:
        for cm in comms:
            cm.close()
        for c in ctxs:
            c.close()


def call(fn, *args):
    e = capi().Error()
    capi().check(fn(*args, C.byref(e)), e)


def heap_read(cm, off: int, n: int) -> bytes:
    buf = (C.c_uint8 * n)()
    call(cm.L.ldb_gpu_comm_heap_read, cm.h, off, n, buf)
    return bytes(buf)


def heap_words(cm, off: int, n_words: int) -> list:
    return np.frombuffer(heap_read(cm, off, 8 * n_words), dtype=np.uint64).tolist()


def dev_view(ptr: int, n_bytes: int):
    """int32 torch view (no copy) of device memory the library owns"""
    import torch
    return par()._device_view(ptr, n_bytes // 4, torch.device("cuda", 0))


def heap_fill(cm, off: int, n: int, value: int = SENTINEL):
    import torch
    cm.ctx.synchronize()
    base, _ = cm.heap()
    dev_view(base + off, n).fill_(value)
    torch.cuda.synchronize()


def dev_bytes(ptr: int, n: int) -> bytes:
    return dev_view(ptr, n).cpu().numpy().tobytes()


def tuples_of(raw: bytes, words: int) -> list:
    a = np.frombuffer(raw, dtype=np.uint64).reshape(-1, words)
    return [tuple(int(x) for x in row) for row in a]


def groups_of(ctx, s, n_aggs):
    return read_groups(ctx, s, n_aggs)


def simple_read(ctx, s, n_aggs):
    out = (capi().I128 * 8)()
    call(ctx.L.ldb_gpu_simple_state_read, s, out)
    return {(): [out[i].value() for i in range(n_aggs)]}


def simple_state(ctx, n_aggs):
    s = C.c_void_p()
    call(ctx.L.ldb_gpu_simple_state_create, ctx.h, n_aggs, C.byref(s))
    return s


def wide_keys(vals, seed: int, extremes=True):
    """many distinct partition keys (and int32 extremes) in column k"""
    rng = random.Random(seed)
    n = len(vals["k"])
    ks = [rng.randrange(-(1 << 31), 1 << 31) for _ in range(n)]
    if extremes:
        for i, k in enumerate([P.I32_MIN, P.I32_MAX, -1, 0, 1]):
            if i < n:
                ks[i] = k
    vals["k"] = ks
    return vals


def run_send(ctxs, comms, srcs, capacity, words, send, zero=True):
    """K10 / K11 on every rank (`send(r)` runs rank r's pipeline), counts published, barrier: the receive sub-regions of every rank, the
    cursors each rank kept and the counts it received"""
    world = len(ctxs)
    if zero:
        for cm in comms:
            call(cm.L.ldb_gpu_comm_heap_zero, cm.h, CURSORS, 512)
    for r in range(world):
        send(r)
    for cm in comms:
        call(cm.L.ldb_gpu_comm_publish_counts, cm.h, CURSORS, COUNTS)
    for cm in comms:
        cm.barrier()
    regions, cursors, counts = [], [], []
    for cm in comms:
        raw = heap_read(cm, RECV, world * capacity * words * 8)
        sub = len(raw) // world
        regions.append([tuples_of(raw[s * sub:(s + 1) * sub], words) for s in range(world)])
        cursors.append(heap_words(cm, CURSORS, 16))
        counts.append(heap_words(cm, COUNTS, 8)[:world])
    return regions, cursors, counts


def check_exchange(regions, cursors, counts, want, capacity):
    """want[s][d]: the tuples source s ships to d (reference).  Cursors count every tuple; the stored tuples are exactly the
    reference's multiset when nothing overflowed, a sub-multiset of it when something did"""
    world = len(want)
    for s in range(world):
        overflow = False
        for d in range(world):
            n, over, kept = X.stored(want[s][d], capacity)
            assert cursors[s][d] == n, (s, d)
            assert counts[d][s] == n, (s, d)  # publish_counts: the transpose of the cursors
            got = Counter(regions[d][s][:kept])
            if over:
                overflow = True
                assert not got - Counter(want[s][d]), (s, d)
            else:
                assert got == Counter(want[s][d]), (s, d)
        assert (cursors[s][8] != 0) == overflow, s


# ---------------------------------------------------------------------------------------------------- K6
@pytest.mark.parametrize("n_rows", [0, 1, 31, 33, 4097, 200003])
def test_partition_tuples(gpu_ctx, n_rows):
    import torch
    rng = np.random.default_rng(n_rows)
    dev = torch.device("cuda", 0)
    patterns = {
        "random": rng.integers(-(1 << 31), 1 << 31, n_rows, dtype=np.int64),
        "equal": np.full(n_rows, 77, np.int64),
        "extremes": np.resize(np.array([P.I32_MIN, P.I32_MAX, -1, 0, 1], np.int64), n_rows),
        "colliding": np.resize(np.array(P.colliding_keys(16, 4093, 64), np.int64), n_rows),
    }
    width_sets = [[], [4], [8, 16], [16, 4, 8], [4, 8, 16, 4]]
    for pi, (pat, keys) in enumerate(patterns.items()):
        keys = keys.astype(np.int32)
        parts_by_key = {}
        for ni, n_parts in enumerate((1, 2, 3, 7, 8, 64)):
            widths = width_sets[(pi + ni) % len(width_sets)]
            cols = []
            for c, w in enumerate(widths):  # payload of row i identifies the row: i * (c + 2) in every width
                v = np.arange(n_rows, dtype=np.int64) * (c + 2) - n_rows
                if w == 4:
                    cols.append(v.astype(np.int32))
                elif w == 8:
                    cols.append(v)
                else:
                    a = np.zeros((n_rows, 2), np.int64)
                    a[:, 0], a[:, 1] = v, ~v
                    cols.append(a)
            d_keys = torch.from_numpy(np.ascontiguousarray(keys) if n_rows else np.zeros(1, np.int32)).to(dev)
            d_in = [torch.from_numpy(np.ascontiguousarray(c) if n_rows else np.zeros(4, np.int32)).to(dev) for c in cols]
            d_out_k = torch.zeros(max(n_rows, 1), dtype=torch.int32, device=dev)
            d_out = [torch.zeros_like(t) for t in d_in]
            offs = (C.c_int64 * (n_parts + 1))()
            pin = (C.c_void_p * 4)(*[t.data_ptr() for t in d_in])
            pout = (C.c_void_p * 4)(*[t.data_ptr() for t in d_out])
            wid = (C.c_int32 * 4)(*widths)
            torch.cuda.synchronize()
            call(gpu_ctx.L.ldb_gpu_partition_tuples, gpu_ctx.h, d_keys.data_ptr(), pin, wid, len(widths), n_rows, n_parts, d_out_k.data_ptr(), pout, offs)
            got_offs = list(offs)
            ok = d_out_k.cpu().numpy()[:n_rows]
            outs = [t.cpu().numpy()[:n_rows] for t in d_out]
            # reference: the offsets, then per partition the multiset of (key, payload…) rows (compared as sorted row matrices)
            dest = X.parts_of(keys, n_parts) if n_rows else np.zeros(0, np.int64)
            want_offs = [0] + np.cumsum(np.bincount(dest, minlength=n_parts)).tolist()
            assert got_offs == want_offs, (pat, n_parts)
            for p in range(n_parts):
                lo, hi = got_offs[p], got_offs[p + 1]
                got = _rows(ok[lo:hi], [o[lo:hi] for o in outs])
                want = _rows(keys[dest == p], [c[dest == p] for c in cols])
                assert np.array_equal(got, want), (pat, n_parts, p)
            parts_by_key[n_parts] = want_offs
        if pat == "equal" and n_rows:  # one partition takes everything
            assert all(sum(1 for a, b in zip(o, o[1:]) if b > a) == 1 for o in parts_by_key.values())


def _rows(keys, cols):
    """(key, payload words…) rows of a partition, sorted: equal arrays = equal multisets"""
    m = np.column_stack([keys.astype(np.int64)] + [c.astype(np.int64).reshape(len(keys), -1) for c in cols]) if len(keys) else np.zeros((0, 1))
    return m[np.lexsort(m.T[::-1])] if len(keys) else m


# ---------------------------------------------------------------------------------------------------- K10
K10_CASES = [  # (name, out columns, year?, probe: None | "unique" | "multi" | "bloom", filters)
    ("plain2", ["k", "i"], False, None, []),
    ("year", ["k", "dt"], True, None, [("i", ">", -(1 << 30))]),
    ("dec4", ["k", "i", "a", "b"], False, None, [("k2", ">=", -(1 << 19)), ("k2", "<=", 1 << 19)]),
    ("payload3", ["k", "$payload", "c"], False, "unique", []),
    ("semi", ["k", "i", "a"], False, "multi", [("dt", ">", "1950-01-01")]),
    ("bloom", ["k", "k2", "a", "d"], False, "bloom", []),
]


def _probe_tables(ctxs, comms, kind, seed):
    """the probe side of every rank: reference tables and states.  'bloom': each rank builds its hash partition of one key set into a
    shared-Bloom table, and the filters are OR-reduced; the reference filter is the model's filter of the whole key set"""
    world = len(ctxs)
    rng = random.Random(seed)
    keys = rng.sample(range(-3000, 3000), 1500)
    refs, states, bloom = [], [], None
    if kind == "bloom":
        words = X.shared_bloom_words(4000)
        boff = RECV + (8 << 20)
        before = []
        for r, (c, cm) in enumerate(zip(ctxs, comms)):
            mine = [k for k in keys if X.part_of(k, world) == r]
            src = table(c, "bk", {"k": mine, "i": [k & 0xFFFF for k in mine]}, columns=[("k", "int32", 0, 0), ("i", "int32", 0, 0)])
            s, nb = C.c_void_p(), C.c_int64()
            call(c.L.ldb_gpu_join_table_create_shared_bloom, c.h, 4000, 1, cm.h, boff, C.byref(nb), C.byref(s))
            assert nb.value == words * 4
            rt().run_pipeline(c, "scan_build", src, build_key="k", build_payload="i", sink=s)
            states.append(s)
        for cm in comms:
            cm.barrier()
        for cm in comms:
            before.append(np.frombuffer(heap_read(cm, boff, words * 4), dtype=np.uint32))
        for cm in comms:
            call(cm.L.ldb_gpu_comm_or_reduce, cm.h, boff, words * 4)
        for cm in comms:
            cm.barrier()
        union = np.bitwise_or.reduce(before)
        assert [int(x) for x in union] == X.bloom_filter(keys, words)  # every rank's filter is exactly the model's
        for cm in comms:
            assert np.array_equal(np.frombuffer(heap_read(cm, boff, words * 4), dtype=np.uint32), union)
        bloom = [int(x) for x in union]
        return [None] * world, states, bloom
    for c in ctxs:
        ref = new_table(expected_rows=4096, unique=kind == "unique")
        ks = keys if kind == "unique" else keys[:700] * 2 + keys[700:900]
        pays = [rng.randrange(-(1 << 31), 1 << 31) for _ in ks]
        src = table(c, "pk", {"k": ks, "i": pays}, columns=[("k", "int32", 0, 0), ("i", "int32", 0, 0)])
        s = build_table(c, ref)
        rt().run_pipeline(c, "scan_build", src, build_key="k", build_payload="i", sink=s)
        P.scan_build({"k": ks, "i": pays}, {"k": ("int32", 0, 0), "i": ("int32", 0, 0)}, [], ref, "k", payload="i")
        refs.append(ref)
        states.append(s)
    return refs, states, None


def _k10_round(ctxs, comms, case, vals_of, capacity, cuts_of=lambda r: (), device_of=lambda r: ()):
    name, outs, year, probe, filters = case
    world = len(ctxs)
    refs, states, bloom = _probe_tables(ctxs, comms, probe, 5) if probe else ([None] * world, [None] * world, None)
    srcs = []
    for r, c in enumerate(ctxs):
        v = vals_of(r)
        if probe:  # probe keys: half of them in the key set
            v["k2"] = [x % 6000 - 3000 for x in v["k2"]]
        srcs.append((v, table(c, "src", v, cuts=cuts_of(r), device=device_of(r))))
    words = 1 + len(outs) - 2
    pkey = "k2"

    def send(r):
        kw = {}
        if probe:
            kw = {"probes": [(states[r], pkey)], "bloom_only": probe == "bloom"}
        rt().run_pipeline(ctxs[r], "scan_partition_send", srcs[r][1], filters=filters, out_columns=outs, build_payload_expr="year" if year else "column",
                          comm=comms[r], send_offset=RECV, send_capacity=capacity, send_cursors_offset=CURSORS, **kw)
    want = []
    for r in range(world):
        pr = None
        if probe:
            pr = (refs[r] if probe != "bloom" else P.JoinTable("hash", 64), pkey)
        want.append(X.partition_send(srcs[r][0], SCHEMA, filters, outs, world, probe=pr, bloom_only=probe == "bloom", bloom=bloom, year=year))
    return run_send(ctxs, comms, srcs, capacity, words, send), want, words


@pytest.mark.parametrize("world", [1, 2, 3])
def test_partition_send_every_shape_and_probe(world):
    with ranks(world, user_bytes=16 << 20) as (ctxs, comms):
        for ci, case in enumerate(K10_CASES):
            def vals_of(r, ci=ci):
                v = wide_keys(values(100 * ci + r, 3000 + 517 * r, "wide"), 7 * ci + r)
                rng = random.Random(ci * 31 + r)
                v["k2"] = [rng.randrange(-(1 << 20), 1 << 20) for _ in v["k2"]]
                return v
            cuts = lambda r: (1, 31, 64, 64, 2000)  # ragged batches and an empty one
            (regions, cursors, counts), want, _ = _k10_round(ctxs, comms, case, vals_of, 8192, cuts_of=cuts, device_of=lambda r: (1, 4) if r % 2 else ())
            assert sum(len(x) for w in want for x in w) > 100, case[0]
            check_exchange(regions, cursors, counts, want, 8192)


def test_partition_send_non_unique_probe_ships_one_tuple_per_row():
    """a probe key with several matches ships ONE tuple (the full probe is a semi-join); "$payload" over such a table is refused"""
    with ranks(2) as (ctxs, comms):
        c = ctxs[0]
        ref = new_table(expected_rows=64, unique=False)
        s = build_table(c, ref)
        kv = {"k": [4, 4, 4, 9], "i": [1, 2, 3, 4]}
        rt().run_pipeline(c, "scan_build", table(c, "pk", kv, columns=[("k", "int32", 0, 0), ("i", "int32", 0, 0)]), build_key="k", build_payload="i", sink=s)
        src = table(c, "src", {"k": [4, 5, 9, 4], "i": [10, 20, 30, 40]}, columns=[("k", "int32", 0, 0), ("i", "int32", 0, 0)])
        expect_error(capi().LDB_ERR_UNSUPPORTED, rt().run_pipeline, c, "scan_partition_send", src, out_columns=["k", "$payload"], probes=[(s, "k")],
                     comm=comms[0], send_offset=RECV, send_capacity=16, send_cursors_offset=CURSORS)
        for cm in comms:
            call(cm.L.ldb_gpu_comm_heap_zero, cm.h, CURSORS, 512)
        rt().run_pipeline(c, "scan_partition_send", src, out_columns=["k", "i"], probes=[(s, "k")], comm=comms[0], send_offset=RECV, send_capacity=16,
                          send_cursors_offset=CURSORS)
        cur = heap_words(comms[0], CURSORS, 16)
        assert cur[0] + cur[1] == 3  # rows 4, 9, 4 — not one per match
        for cm in comms:
            cm.barrier()


def test_partition_send_overflow_keeps_the_heap_outside_the_claimed_ranges():
    world, cap = 3, 40
    with ranks(world) as (ctxs, comms):
        region = world * cap * 24
        for cm in comms:
            heap_fill(cm, RECV, region + 4096)
        srcs = [values(50 + r, 400, "negative") for r in range(world)]

        def vals_of(r):
            return wide_keys(srcs[r], r)
        (regions, cursors, counts), want, words = _k10_round(ctxs, comms, ("over", ["k", "i", "a", "b"], False, None, []), vals_of, cap)
        assert any(len(want[s][d]) > cap for s in range(world) for d in range(world))
        check_exchange(regions, cursors, counts, want, cap)
        for d, cm in enumerate(comms):  # every byte outside the claimed ranges still holds the sentinel
            raw = np.frombuffer(heap_read(cm, RECV, region + 4096), dtype=np.uint32).copy()
            sub = cap * words * 2  # uint32 words per source sub-region
            for s in range(world):
                kept = min(cursors[s][d], cap) * words * 2
                raw[s * sub: s * sub + kept] = SENTINEL
            assert (raw == SENTINEL).all(), d


def test_partition_send_large_host_batch():
    """a HOST batch of >= 65 536 rows goes through compressed staging (and narrowed decimals); a child process repeats it with
    LDB_NARROW_STAGING=0"""
    world = 2
    with ranks(world, user_bytes=32 << 20) as (ctxs, comms):
        def vals_of(r):
            return wide_keys(values(900 + r, 70_001, "negative", key_domain=1000), r)
        (regions, cursors, counts), want, _ = _k10_round(ctxs, comms, ("big", ["k", "i", "a", "d"], False, None, [("k2", "!=", 1)]), vals_of, 70_001)
        check_exchange(regions, cursors, counts, want, 70_001)


def test_partition_send_large_host_batch_wide_staging():
    if os.environ.get("LDB_NARROW_STAGING") == "0":
        pytest.skip("already inside the child process")
    env = dict(os.environ, LDB_NARROW_STAGING="0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu", os.path.join(HERE, "test_gpu_exchange.py") + "::test_partition_send_large_host_batch"],
                       env=env, cwd=os.path.dirname(HERE), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "1 passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------- K11 + groupby2
def _star_side(c, seed, s_kind, unique_p):
    """pair table P (k, k2) → a (int64), foreign-key table S (i → g0) of one rank, with their references"""
    rng = random.Random(seed)
    pk = [(rng.randrange(-50, 50), rng.randrange(-3, 3)) for _ in range(300)]
    if unique_p:
        pk = list(dict.fromkeys(pk))
    pv = {"k": [a for a, _ in pk], "k2": [b for _, b in pk], "a": [rng.randrange(-10**12, 10**12) for _ in pk]}
    pcols = [("k", "int32", 0, 0), ("k2", "int32", 0, 0), ("a", "decimal128", 18, 2)]
    pref = new_table("pair", expected_rows=1024, unique=unique_p)
    ps = build_table(c, pref)
    rt().run_pipeline(c, "scan_build", table(c, "p", pv, columns=pcols), build_key="k", build_key2="k2", build_payload="a", sink=ps)
    P.scan_build(pv, P.schema_of(pcols), [], pref, "k", payload="a", key2="k2")
    skeys = list(range(-20, 20)) if s_kind != "multi" else list(range(-20, 20)) * 2
    sv = {"i": skeys, "g": [rng.randrange(-5, 3) for _ in skeys]}
    scols = [("i", "int32", 0, 0), ("g", "int32", 0, 0)]
    sref = new_table("direct", key_min=-20, key_max=19) if s_kind == "direct" else new_table(expected_rows=256, unique=s_kind == "unique")
    ss = build_table(c, sref)
    rt().run_pipeline(c, "scan_build", table(c, "s", sv, columns=scols), build_key="i", build_payload="g", sink=ss)
    P.scan_build(sv, P.schema_of(scols), [], sref, "i", payload="g")
    return pref, ps, sref, ss


@pytest.mark.parametrize("world", [1, 2, 3])
def test_star_probe_send_and_groupby2(world):
    cap = 60_000
    with ranks(world, user_bytes=8 << 20) as (ctxs, comms):
        for s_kind, unique_p in (("unique", True), ("multi", False), ("direct", True)):
            sides = [_star_side(c, 10 * r + len(s_kind), s_kind, unique_p) for r, c in enumerate(ctxs)]
            srcs = []
            for r, c in enumerate(ctxs):
                v = values(70 + r, 2500, "wide" if r % 2 else "negative")
                rng = random.Random(r)
                v["k"] = [rng.randrange(-50, 50) for _ in v["k"]]
                v["i"] = [rng.randrange(-22, 22) for _ in v["i"]]
                v["dt"] = [rng.randrange(-40, 40) for _ in v["dt"]]  # the partition key: order keys
                srcs.append((v, table(c, "li", v, cuts=(1000,), device=(1,) if r == 0 else ())))

            def send(r):
                rt().run_pipeline(ctxs[r], "scan_star_probe_send", srcs[r][1], probes=[(sides[r][1], "k", "k2"), (sides[r][3], "i")],
                                  aggs=[("mul_1minus_minus_paymul", ["a", "b", "d"])], out_columns=["dt"], comm=comms[r], send_offset=RECV,
                                  send_capacity=cap, send_cursors_offset=CURSORS)
            regions, cursors, counts = run_send(ctxs, comms, srcs, cap, 3, send)
            want = [X.star_probe_send(srcs[r][0], SCHEMA, [], sides[r][0], ("k", "k2"), sides[r][2], "i", "dt", ("a", "b", "d"), world) for r in range(world)]
            assert sum(len(x) for w in want for x in w) > 500
            check_exchange(regions, cursors, counts, want, cap)
            # receive side: the orders partition of every rank (order key → year-like payload g1), probed by the received tuples
            states, refs = [], []
            for d, (c, cm) in enumerate(zip(ctxs, comms)):
                okeys = [k for k in range(-40, 40) if X.part_of(k, world) == d]
                oref = new_table(expected_rows=1024, unique=s_kind != "multi")
                opay = [k * 3 + 1 for k in okeys]
                if s_kind == "multi":  # a non-unique partition: two payloads for every other key, the second one -1 (a negative group)
                    okeys, opay = okeys + okeys[::2], opay + [-1 if k != -1 else -4 for k in okeys[::2]]
                ov = {"k": okeys, "i": opay}
                ocols = [("k", "int32", 0, 0), ("i", "int32", 0, 0)]
                os_ = build_table(c, oref)
                rt().run_pipeline(c, "scan_build", table(c, "o", ov, columns=ocols), build_key="k", build_payload="i", sink=os_)
                P.scan_build(ov, P.schema_of(ocols), [], oref, "k", payload="i")
                g = rt().groupby_state(c, 2, 1, 1024)
                call(c.L.ldb_gpu_probe_received_groupby2, os_, g, cm.h, RECV, cap, COUNTS)
                got = groups_of(c, g, 1)
                tuples = X.received([want[s][d] for s in range(world)], counts[d], cap)
                ref = X.probe_received_groupby2(oref, tuples)
                assert got == ref, (s_kind, d)
                if s_kind == "multi":
                    assert any(k[1] == -1 for k in ref)
                states.append(g)
                refs.append(ref)
            # _groupby2 fixed its lane as 128-bit, so its states merge (a merge refuses a state with an unbound lane)
            for cm, g in zip(comms, states):
                cm.allmerge(g)
            want_all = X.merge(refs, [False], capacity=1024)
            for c, g in zip(ctxs, states):
                assert groups_of(c, g, 1) == want_all, s_kind


def test_star_probe_groupby_states_merge_at_128_bits():
    """K9 fixes its lane as 128-bit, so the per-rank Q9-shaped states of a sharded star join all-merge and read back whole.  (No
    pipeline writes a 64-bit sum into a 2-key, 1-aggregate state, so the width K9 binds shows only through such merges.)"""
    world = 2
    with ranks(world) as (ctxs, comms):
        states, refs = [], []
        for r, c in enumerate(ctxs):
            pref, ps, sref, ss = _star_side(c, 60 + r, "unique", True)
            ov = {"k": list(range(-40, 40)), "i": [k % 7 - (1 if k == 0 else 0) for k in range(-40, 40)]}
            ocols = [("k", "int32", 0, 0), ("i", "int32", 0, 0)]
            oref = new_table(expected_rows=256)
            os_ = build_table(c, oref)
            rt().run_pipeline(c, "scan_build", table(c, "o", ov, columns=ocols), build_key="k", build_payload="i", sink=os_)
            P.scan_build(ov, P.schema_of(ocols), [], oref, "k", payload="i")
            v = values(80 + r, 3000, "wide" if r else "negative")
            rng = random.Random(r)
            v["k"] = [rng.randrange(-50, 50) for _ in v["k"]]
            v["i"] = [rng.randrange(-22, 22) for _ in v["i"]]
            v["dt"] = [rng.randrange(-42, 42) for _ in v["dt"]]
            g = rt().groupby_state(c, 2, 1, 1024)
            rt().run_pipeline(c, "scan_star_probe_groupby", table(c, "li", v, cuts=(1000,)), aggs=[("mul_1minus_minus_paymul", ["a", "b", "d"])],
                              probes=[(ps, "k", "k2"), (ss, "i"), (os_, "dt")], sink=g)
            ref = P.star_probe_groupby(v, SCHEMA, [], pref, ("k", "k2"), sref, "i", oref, "dt", ("a", "b", "d"))
            assert groups_of(c, g, 1) == ref and len(ref) > 20
            states.append(g)
            refs.append(ref)
        for cm, g in zip(comms, states):
            cm.allmerge(g)
        want = X.merge(refs, [False], capacity=1024)
        for r, (c, g) in enumerate(zip(ctxs, states)):
            assert groups_of(c, g, 1) == want, r


def test_groupby2_group_minus_one_and_many_groups():
    """more than 256 groups (the CTA-local table overflows into the state) and the group (-1, -1): tuples written by K10 with a
    decimal pair standing in for K11's {lo, hi}"""
    world, cap = 2, 4096
    with ranks(world) as (ctxs, comms):
        vals = []
        for r, c in enumerate(ctxs):
            rng = random.Random(r)
            n = 1500
            v = values(r, n, "wide")
            v["k"] = [rng.randrange(0, 400) for _ in range(n)]
            v["i"] = [rng.randrange(-1, 300) for _ in range(n)]  # g0, -1 included
            v["k"][:20], v["i"][:20] = [0] * 20, [-1] * 20  # the group (-1, -1): key 0 has payload -1
            vals.append(v)
        srcs = [(v, table(c, "t", v)) for v, c in zip(vals, ctxs)]

        def send(r):
            rt().run_pipeline(ctxs[r], "scan_partition_send", srcs[r][1], out_columns=["k", "i", "a", "b"], comm=comms[r], send_offset=RECV, send_capacity=cap,
                              send_cursors_offset=CURSORS)
        regions, cursors, counts = run_send(ctxs, comms, srcs, cap, 3, send)
        want = [X.partition_send(vals[r], SCHEMA, [], ["k", "i", "a", "b"], world) for r in range(world)]
        check_exchange(regions, cursors, counts, want, cap)
        for d, c in enumerate(ctxs):
            okeys = list(range(0, 400))
            ov = {"k": okeys, "i": [-1 if k % 7 == 0 else k % 5 for k in okeys]}
            oref = new_table(expected_rows=1024)
            ocols = [("k", "int32", 0, 0), ("i", "int32", 0, 0)]
            os_ = build_table(c, oref)
            rt().run_pipeline(c, "scan_build", table(c, "o", ov, columns=ocols), build_key="k", build_payload="i", sink=os_)
            P.scan_build(ov, P.schema_of(ocols), [], oref, "k", payload="i")
            g = rt().groupby_state(c, 2, 1, 2048)
            call(c.L.ldb_gpu_probe_received_groupby2, os_, g, comms[d].h, RECV, cap, COUNTS)
            ref = X.probe_received_groupby2(oref, X.received([want[s][d] for s in range(world)], counts[d], cap), capacity=2048)
            assert len(ref) > 256 and ((-1, -1) in ref) == (d == X.part_of(0, world))
            assert groups_of(c, g, 1) == ref, d


# ---------------------------------------------------------------------------------------------------- receive side
def test_insert_received_and_duplicates_across_sources():
    world, cap = 3, 2048
    with ranks(world) as (ctxs, comms):
        vals = []
        for r in range(world):
            rng = random.Random(40 + r)
            v = values(40 + r, 900, "tpch")
            v["k"] = rng.sample(range(-2000, 2000), 900)  # unique within a source, repeated across sources
            v["i"] = [rng.randrange(-(1 << 31), 1 << 31) for _ in v["i"]]
            vals.append(v)
        srcs = [(v, table(c, "t", v)) for v, c in zip(vals, ctxs)]

        def send(r):
            rt().run_pipeline(ctxs[r], "scan_partition_send", srcs[r][1], out_columns=["k", "i"], comm=comms[r], send_offset=RECV, send_capacity=cap,
                              send_cursors_offset=CURSORS)
        regions, cursors, counts = run_send(ctxs, comms, srcs, cap, 1, send)
        want = [X.partition_send(vals[r], SCHEMA, [], ["k", "i"], world) for r in range(world)]
        check_exchange(regions, cursors, counts, want, cap)
        for d, c in enumerate(ctxs):
            ref = new_table(expected_rows=4096, unique=False)
            s = build_table(c, ref)
            call(c.L.ldb_gpu_join_table_insert_received, s, comms[d].h, RECV, cap, COUNTS)
            X.insert_received(ref, X.received([want[q][d] for q in range(world)], counts[d], cap))
            assert rt().join_count(c, s) == ref.count()
            keys = sorted({k for k, _ in ((e[0], e[1]) for e in ref.entries)}) + [5000]
            assert gpu_payloads(c, s, keys) == sorted((k, e[1]) for k in keys for e in ref.index().get(k, []))
            # a unique table: a key that arrives from two sources fails the count
            sources_of = {}
            for q in range(world):
                got_q = [X.unpack(t[0])[0] for t in want[q][d][: min(counts[d][q], cap)]]
                assert len(set(got_q)) == len(got_q)  # no key repeats within one source
                for k in got_q:
                    sources_of.setdefault(k, set()).add(q)
            assert any(len(qs) > 1 for qs in sources_of.values()), d
            u = rt().join_table(c, 4096, True)
            call(c.L.ldb_gpu_join_table_insert_received, u, comms[d].h, RECV, cap, COUNTS)
            expect_error(capi().LDB_ERR_INVALID, rt().join_count, c, u)


@pytest.mark.parametrize("scale", [0, 2, 18])
def test_probe_received_groupby(scale):
    world, cap = 2, 4096
    with ranks(world) as (ctxs, comms):
        vals = []
        for r in range(world):
            rng = random.Random(scale * 10 + r)
            v = values(scale + r, 2000, "wide" if scale == 18 else "negative")
            v["k"] = [rng.randrange(0, 500) for _ in v["k"]]
            v["i"] = [rng.randrange(0, 50) for _ in v["i"]]
            vals.append(v)
        srcs = [(v, table(c, "t", v)) for v, c in zip(vals, ctxs)]

        def send(r):
            rt().run_pipeline(ctxs[r], "scan_partition_send", srcs[r][1], out_columns=["k", "i", "a", "b"], comm=comms[r], send_offset=RECV, send_capacity=cap,
                              send_cursors_offset=CURSORS)
        regions, cursors, counts = run_send(ctxs, comms, srcs, cap, 3, send)
        want = [X.partition_send(vals[r], SCHEMA, [], ["k", "i", "a", "b"], world) for r in range(world)]
        check_exchange(regions, cursors, counts, want, cap)
        cols2 = [("k", "int32", 0, 0), ("i", "int32", 0, 0)]
        for d, c in enumerate(ctxs):
            # A: order key → nation (k % 25), B: supplier key → nation ((i * 7) % 25): about 1 in 25 rows agrees
            av = {"k": list(range(500)), "i": [k % 25 for k in range(500)]}
            bv = {"k": list(range(50)), "i": [(i * 7) % 25 for i in range(50)]}
            refs, sts = [], []
            for v in (av, bv):
                ref = new_table(expected_rows=1024)
                s = build_table(c, ref)
                rt().run_pipeline(c, "scan_build", table(c, "x", v, columns=cols2), build_key="k", build_payload="i", sink=s)
                P.scan_build(v, P.schema_of(cols2), [], ref, "k", payload="i")
                refs.append(ref)
                sts.append(s)
            g = rt().groupby_state(c, 1, 1, 64)
            call(c.L.ldb_gpu_probe_received_groupby, sts[0], sts[1], g, comms[d].h, RECV, cap, COUNTS, scale)
            tuples = X.received([want[s][d] for s in range(world)], counts[d], cap)
            ref = X.probe_received_groupby(refs[0], refs[1], tuples, scale)
            assert len(ref) > 3
            assert groups_of(c, g, 1) == ref, d


def test_receive_sinks_bind_their_lane_as_128_bit():
    """probe_received_groupby's sums are 128-bit: a sink whose lane a 64-bit pipeline fixed first is refused, and the other order too"""
    world = 1
    with ranks(world) as (ctxs, comms):
        c, cm = ctxs[0], comms[0]
        cols2 = [("k", "int32", 0, 0), ("i", "int32", 0, 0)]
        a = rt().join_table(c, 64)
        rt().run_pipeline(c, "scan_build", table(c, "x", {"k": [1, 2], "i": [7, 7]}, columns=cols2), build_key="k", build_payload="i", sink=a)
        v = values(3, 50, "negative")
        v["k"], v["k2"] = [1] * 50, [2] * 50
        src = table(c, "p", v)
        for cm_ in comms:
            call(cm_.L.ldb_gpu_comm_heap_zero, cm_.h, 0, 4096)
        g = rt().groupby_state(c, 1, 1, 64)
        rt().run_pipeline(c, "scan_probe2_groupby", src, aggs=[("col", ["a"])], probes=[(a, "k"), (a, "k2")], sink=g)
        expect_error(capi().LDB_ERR_UNSUPPORTED, call, c.L.ldb_gpu_probe_received_groupby, a, a, g, cm.h, RECV, 16, COUNTS, 2)
        g2 = rt().groupby_state(c, 1, 1, 64)
        call(c.L.ldb_gpu_probe_received_groupby, a, a, g2, cm.h, RECV, 16, COUNTS, 2)
        expect_error(capi().LDB_ERR_UNSUPPORTED, rt().run_pipeline, c, "scan_probe2_groupby", src, aggs=[("col", ["a"])], probes=[(a, "k"), (a, "k2")], sink=g2)
        rt().run_pipeline(c, "scan_probe2_groupby", src, aggs=[("mul_1minus", ["a", "b"])], probes=[(a, "k"), (a, "k2")], sink=g2)  # 128-bit: fine
        want = {(7, 0): [sum(x * (100 - y) for x, y in zip(v["a"], v["b"]))]}
        assert groups_of(c, g2, 1) == want


# ---------------------------------------------------------------------------------------------------- K7
Q1_SIG = P.SIGNATURES[0]  # 2 keys; 64-bit (col, one) and 128-bit lanes
ONE_KEY = P.SIGNATURES[7]  # 1 key; col, one


def _shard(c, seed, sig, cap, keys_of_rank, mix, keyless=False, empty=False):
    """a group state of one rank from a K1 / K2 pipeline and its raw cells"""
    from test_gpu_pipelines import sig_aggs
    keys, aggs = sig_aggs(sig)
    v = values(seed, 3000, mix)
    rng = random.Random(seed)
    ks = keys_of_rank(rng)
    v["k"] = [ks[rng.randrange(len(ks))] for _ in v["k"]]
    filters = [("k2", ">", 100)] if empty else []
    src = table(c, "t", v)
    if keyless:
        s = simple_state(c, len(aggs))
        rt().run_pipeline(c, "scan_reduce", src, filters=filters, aggs=aggs, sink=s)
        ref = P.scan_groupby(v, SCHEMA, filters, [], aggs)
    else:
        s = rt().groupby_state(c, len(keys), len(aggs), cap)
        rt().run_pipeline(c, "scan_groupby", src, filters=filters, keys=keys, aggs=aggs, sink=s)
        ref = P.scan_groupby(v, SCHEMA, filters, keys, aggs, capacity=max(cap, 4096))
    return s, ref, [e in P.IS64 for e, _ in aggs]


def _read(c, s, n_aggs, keyless):
    return simple_read(c, s, n_aggs) if keyless else groups_of(c, s, n_aggs)


# At most six lanes: no pipeline sums into lanes 6 and 7, and a merge into a state with an unbound lane is refused (see
# test_merges_past_the_capacity_and_lane_widths), so lanes 6-7 of the merge and image kernels cannot be reached through the C-ABI.
K7_CASES = [  # (signature, capacity, keyless, key pattern, mix)
    (Q1_SIG, 16, False, "shared", "negative"),
    (Q1_SIG, 64, False, "own", "wide"),
    (ONE_KEY, 1024, False, "colliding", "negative"),
    (ONE_KEY, 256, False, "own", "mixed"),
    (P.SIGNATURES[2], 1, True, None, "wide"),
    (P.SIGNATURES[4], 1, True, "empty", "negative"),
]


def _keys_for(pattern, r, cap):
    if pattern == "shared":
        return lambda rng: [-1, 0, 1, 2]
    if pattern == "own":  # groups present on only one rank next to shared ones
        return lambda rng: [0, 1] + [1000 * (r + 1) + i for i in range(cap // 16)]
    if pattern == "colliding":  # one directory slot near the end of the table: runs that wrap around
        ks = P.colliding_keys(10, 1021, 300)
        return lambda rng: ks[r * 60: r * 60 + 150]
    return lambda rng: [0]


@pytest.mark.parametrize("world", [2, 3])
def test_allmerge_merge_exported_and_merge_rows(world):
    import torch
    with ranks(world) as (ctxs, comms):
        for ci, (sig, cap, keyless, pat, mix) in enumerate(K7_CASES):
            for rep in range(2):  # twice in a row: both mailbox parities
                shards = [_shard(c, 100 * ci + 10 * rep + r, sig, cap, _keys_for(pat, r, cap), mix, keyless, empty=pat == "empty" and r == 1)
                          for r, c in enumerate(ctxs)]
                n_aggs = len(sig[1])
                raw = [sh[1] for sh in shards]
                want = X.merge(raw, shards[0][2], capacity=cap, keyless=keyless)
                # merge_exported into rank 0 (what a rank does after an NCCL all-gather), merge_rows into rank 1 from reads of the others
                c0 = ctxs[0]
                nbytes = int(c0.L.ldb_gpu_groupby_export_bytes(shards[0][0]))
                buf = torch.zeros(world * nbytes, dtype=torch.uint8, device="cuda")
                torch.cuda.synchronize()
                for r, c in enumerate(ctxs):
                    call(c.L.ldb_gpu_groupby_export, shards[r][0], C.c_void_p(buf.data_ptr() + r * nbytes))
                    c.synchronize()
                if not keyless:
                    rows = []
                    for r in (0, 2) if world == 3 else (0,):
                        rs = (capi().GroupRow * 4096)()
                        n = C.c_int32()
                        call(ctxs[r].L.ldb_gpu_groupby_read, shards[r][0], rs, 4096, C.byref(n))
                        rows.extend(rs[: n.value])
                    arr = (capi().GroupRow * max(1, len(rows)))(*rows)
                    call(ctxs[1].L.ldb_gpu_groupby_merge_rows, shards[1][0], arr, len(rows))
                    assert _read(ctxs[1], shards[1][0], n_aggs, False) == want, ("rows", ci, rep)
                call(c0.L.ldb_gpu_groupby_merge_exported, shards[0][0], C.c_void_p(buf.data_ptr()), world, 0)
                assert _read(c0, shards[0][0], n_aggs, keyless) == want, ("exported", ci, rep)
                # the peer all-merge over fresh copies of the shards
                fresh = [_shard(c, 100 * ci + 10 * rep + r, sig, cap, _keys_for(pat, r, cap), mix, keyless, empty=pat == "empty" and r == 1)[0]
                         for r, c in enumerate(ctxs)]
                for cm, s in zip(comms, fresh):
                    cm.allmerge(s)
                for r, c in enumerate(ctxs):
                    assert _read(c, fresh[r], n_aggs, keyless) == want, ("allmerge", ci, rep, r)
                for r, c in enumerate(ctxs):
                    for s in (shards[r][0], fresh[r]):
                        rt().state_destroy(c, s)


def test_merges_past_the_capacity_and_lane_widths():
    world = 2
    with ranks(world) as (ctxs, comms):
        c0 = ctxs[0]
        # more distinct groups across the ranks than a 16-group table holds: LDB_ERR_CAPACITY on read
        shards = [_shard(c, 7 + r, ONE_KEY, 16, lambda rng, r=r: [100 * r + i for i in range(12)], "negative") for r, c in enumerate(ctxs)]
        for cm, sh in zip(comms, shards):
            cm.allmerge(sh[0])
        for r, c in enumerate(ctxs):
            expect_error(capi().LDB_ERR_CAPACITY, groups_of, c, shards[r][0], 2)
        # a 2048-group table does not fit a mailbox slot
        big = [rt().groupby_state(c, 1, 2, 2048) for c in ctxs]
        for c, s in zip(ctxs, big):
            rt().run_pipeline(c, "scan_groupby", table(c, "t", values(1, 10, "tpch")), keys=["k"], aggs=[("col", ["a"]), ("one", [])], sink=s)
        for cm, s in zip(comms, big):
            expect_error(capi().LDB_ERR_UNSUPPORTED, cm.allmerge, s)
        # a target whose lanes no pipeline bound: every merge is refused (a 64-bit lane's -5 would read back as 2^64 - 5)
        src, ref, _ = _shard(c0, 3, ONE_KEY, 64, lambda rng: [1, 2], "negative")
        fresh = [rt().groupby_state(c, 1, 2, 64) for c in ctxs]
        for cm, s in zip(comms, fresh):
            expect_error(capi().LDB_ERR_UNSUPPORTED, cm.allmerge, s)
        rows = (capi().GroupRow * 4)()
        n = C.c_int32()
        call(c0.L.ldb_gpu_groupby_read, src, rows, 4, C.byref(n))
        expect_error(capi().LDB_ERR_UNSUPPORTED, call, c0.L.ldb_gpu_groupby_merge_rows, fresh[0], rows, n.value)
        import torch
        img = torch.zeros(int(c0.L.ldb_gpu_groupby_export_bytes(src)), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        call(c0.L.ldb_gpu_groupby_export, src, C.c_void_p(img.data_ptr()))
        c0.synchronize()
        expect_error(capi().LDB_ERR_UNSUPPORTED, call, c0.L.ldb_gpu_groupby_merge_exported, fresh[0], C.c_void_p(img.data_ptr()), 1, 0)
        # a bound target reads the merged 64-bit lane sign-extended
        tgt, tref, w64 = _shard(c0, 4, ONE_KEY, 64, lambda rng: [1, 2], "negative")
        call(c0.L.ldb_gpu_groupby_merge_rows, tgt, rows, n.value)
        assert groups_of(c0, tgt, 2) == X.merge([ref, tref], w64)
        for c, s in zip(ctxs, fresh):
            rt().state_destroy(c, s)


# ---------------------------------------------------------------------------------------------------- collectives
def _blocks(world, nbytes, tag):
    return [bytes(((tag * 131 + r * 17 + i) & 0xFF) for i in range(nbytes)) for r in range(world)]


def _gather(ctxs, comms, blocks):
    """allgather_small on every rank; returns (result addresses, source tensors kept alive)"""
    import torch
    srcs = [torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() for b in blocks]
    torch.cuda.synchronize()
    res = []
    for cm, s in zip(comms, srcs):
        p = C.c_void_p()
        call(cm.L.ldb_gpu_comm_allgather_small, cm.h, C.c_void_p(s.data_ptr()), len(blocks[0]), C.byref(p))
        res.append(p.value)
    for c in ctxs:
        c.synchronize()
    return res, srcs


def _check_gather(res, blocks):
    slot = X.SLOT_BYTES
    want = X.allgather_small(blocks)
    for r, p in enumerate(res):
        for q, b in enumerate(want):
            assert dev_bytes(p + q * slot, len(b)) == b, (r, q)


@pytest.mark.parametrize("world", [1, 2, 5, 8])
def test_allgather_small_sizes_and_lifetime(world):
    with ranks(world, user_bytes=4096) as (ctxs, comms):
        for nbytes in (16, 4096, X.SLOT_BYTES):
            b1, b2, b3 = (_blocks(world, nbytes, t) for t in (1, 2, 3))
            r1, k1 = _gather(ctxs, comms, b1)
            _check_gather(r1, b1)
            r2, k2 = _gather(ctxs, comms, b2)
            _check_gather(r1, b1)  # the first result is still valid before the third gather
            _check_gather(r2, b2)
            r3, k3 = _gather(ctxs, comms, b3)
            _check_gather(r3, b3)
        for cm in comms:
            cm.barrier()


def test_gathers_interleaved_with_allmerges_and_after_a_captured_one():
    world = 2
    with ranks(world) as (ctxs, comms):
        shards = [_shard(c, 20 + r, Q1_SIG, 16, _keys_for("own", r, 16), "negative") for r, c in enumerate(ctxs)]
        want = X.merge([sh[1] for sh in shards], shards[0][2], capacity=16)
        b = _blocks(world, 4096, 9)
        r1, _ = _gather(ctxs, comms, b)
        _check_gather(r1, b)
        for cm, sh in zip(comms, shards):
            cm.allmerge(sh[0])
        b = _blocks(world, 512, 10)
        r2, _ = _gather(ctxs, comms, b)
        _check_gather(r2, b)
        for r, c in enumerate(ctxs):
            assert groups_of(c, shards[r][0], 6) == want
        # a captured all-merge, replayed twice, then eager gathers: their results must be the blocks just gathered
        fresh = [_shard(c, 20 + r, Q1_SIG, 16, _keys_for("own", r, 16), "negative")[0] for r, c in enumerate(ctxs)]
        graphs = []
        for c, cm, s in zip(ctxs, comms, fresh):
            c.graph_begin()
            cm.allmerge(s)
            graphs.append(c.graph_end())
        try:
            for g in graphs:
                g.launch()
            for c in ctxs:
                c.synchronize()
            for r, c in enumerate(ctxs):
                assert groups_of(c, fresh[r], 6) == want
            for t in (11, 12, 13):
                b = _blocks(world, 1024, t)
                res, _ = _gather(ctxs, comms, b)
                _check_gather(res, b)
            for g in graphs:
                g.launch()
            b = _blocks(world, 2048, 14)
            res, _ = _gather(ctxs, comms, b)
            _check_gather(res, b)
            for cm in comms:
                cm.barrier()
        finally:
            for g in graphs:
                g.destroy()


@pytest.mark.parametrize("world", [2, 3, 8])
def test_or_reduce_is_the_or_of_the_filters(world):
    nbytes, off = 64 << 10, 4096
    with ranks(world, user_bytes=1 << 20) as (ctxs, comms):
        before = []
        for r, cm in enumerate(comms):
            rng = np.random.default_rng(r)
            words = (rng.integers(0, 1 << 32, nbytes // 4, dtype=np.uint64) & rng.integers(0, 1 << 32, nbytes // 4, dtype=np.uint64)).astype(np.uint32)
            base, _ = cm.heap()
            import torch
            dev_view(base + off, nbytes).copy_(torch.from_numpy(words.view(np.int32)).cuda())
            torch.cuda.synchronize()
            before.append(words)
        for cm in comms:
            cm.barrier()
        for cm in comms:
            call(cm.L.ldb_gpu_comm_or_reduce, cm.h, off, nbytes)
        for cm in comms:
            cm.barrier()
        want = np.bitwise_or.reduce(before)
        for r, cm in enumerate(comms):
            assert np.array_equal(np.frombuffer(heap_read(cm, off, nbytes), dtype=np.uint32), want), r


# ---------------------------------------------------------------------------------------------------- documented errors
def test_documented_errors():
    cc = capi()
    INV, UNS, CAPY = cc.LDB_ERR_INVALID, cc.LDB_ERR_UNSUPPORTED, cc.LDB_ERR_CAPACITY
    c0 = rt().Context(0)
    try:
        h, e = C.c_void_p(), cc.Error()
        handle = (C.c_uint8 * 64)()
        for rank, world in ((0, 9), (2, 2), (-1, 1), (0, 0)):
            assert c0.L.ldb_gpu_comm_create(c0.h, rank, world, 0, C.byref(h), handle, C.byref(e)) == INV, (rank, world)
        assert c0.L.ldb_gpu_comm_create(c0.h, 0, 1, -1, C.byref(h), handle, C.byref(e)) == INV
    finally:
        c0.close()
    with ranks(2, user_bytes=1 << 16) as (ctxs, comms):
        c, cm = ctxs[0], comms[0]
        L = c.L
        buf = rt().join_table(c, 64)
        pair = rt().join_table_pair(c, 64)
        direct = rt().join_table_direct(c, 0, 10)
        g1 = rt().groupby_state(c, 1, 1, 64)
        g2 = rt().groupby_state(c, 2, 1, 64)
        g12 = rt().groupby_state(c, 1, 2, 64)
        user = 1 << 16
        ptr = C.c_void_p(cm.heap()[0])
        cases = [
            (INV, L.ldb_gpu_comm_allgather_small, cm.h, ptr, 0, None),
            (INV, L.ldb_gpu_comm_allgather_small, cm.h, ptr, 8, None),
            (INV, L.ldb_gpu_comm_allgather_small, cm.h, ptr, X.SLOT_BYTES + 16, None),
            (INV, L.ldb_gpu_comm_or_reduce, cm.h, 8, 16),
            (INV, L.ldb_gpu_comm_or_reduce, cm.h, 0, 24),
            (INV, L.ldb_gpu_comm_or_reduce, cm.h, user - 16, 32),
            (INV, L.ldb_gpu_comm_heap_zero, cm.h, user - 8, 16),
            (INV, L.ldb_gpu_comm_heap_zero, cm.h, -1, 1),
            (CAPY, L.ldb_gpu_comm_publish_counts, cm.h, user - 64, 0),
            (CAPY, L.ldb_gpu_comm_publish_counts, cm.h, 8, 256),
            (CAPY, L.ldb_gpu_comm_publish_counts, cm.h, 0, user - 32),
            (INV, L.ldb_gpu_join_table_insert_received, pair, cm.h, RECV, 16, COUNTS),
            (INV, L.ldb_gpu_join_table_insert_received, direct, cm.h, RECV, 16, COUNTS),
            (INV, L.ldb_gpu_join_table_insert_received, g1, cm.h, RECV, 16, COUNTS),
            (CAPY, L.ldb_gpu_join_table_insert_received, buf, cm.h, RECV, user, COUNTS),
            (CAPY, L.ldb_gpu_join_table_insert_received, buf, cm.h, 8, 16, COUNTS),
            (INV, L.ldb_gpu_probe_received_groupby, buf, pair, g1, cm.h, RECV, 16, COUNTS, 2),
            (INV, L.ldb_gpu_probe_received_groupby, buf, buf, g2, cm.h, RECV, 16, COUNTS, 2),
            (INV, L.ldb_gpu_probe_received_groupby, buf, buf, g12, cm.h, RECV, 16, COUNTS, 2),
            (INV, L.ldb_gpu_probe_received_groupby, buf, buf, g1, cm.h, RECV, 16, COUNTS, 19),
            (INV, L.ldb_gpu_probe_received_groupby, buf, buf, g1, cm.h, RECV, 16, COUNTS, -1),
            (CAPY, L.ldb_gpu_probe_received_groupby, buf, buf, g1, cm.h, RECV, user, COUNTS, 2),
            (INV, L.ldb_gpu_probe_received_groupby2, direct, g2, cm.h, RECV, 16, COUNTS),
            (INV, L.ldb_gpu_probe_received_groupby2, buf, g1, cm.h, RECV, 16, COUNTS),
            (CAPY, L.ldb_gpu_probe_received_groupby2, buf, g2, cm.h, RECV, user, COUNTS),
            (INV, L.ldb_gpu_groupby_allmerge, buf, cm.h),
            (INV, L.ldb_gpu_groupby_allmerge, g1, comms[1].h),  # a state of another context
        ]
        for code, fn, *args in cases:
            e = cc.Error()
            assert fn(*args, C.byref(e)) == code, (fn.__name__, args, e.message)
        # K10 / K11 descriptors
        v = values(1, 64, "tpch")
        src = table(c, "e", v)
        run = rt().run_pipeline
        send = dict(comm=cm, send_offset=RECV, send_capacity=16, send_cursors_offset=CURSORS)
        multi = rt().join_table(c, 64, False)
        k10 = [
            (INV, dict(out_columns=["k"])),
            (INV, dict(out_columns=["k", "$payload"])),
            (INV, dict(out_columns=["k", "$payload"], probes=[(buf, "k")], bloom_only=True)),
            (UNS, dict(out_columns=["k", "$payload"], probes=[(multi, "k")])),
            (INV, dict(out_columns=["k", "$payload"], probes=[(buf, "k")], build_payload_expr="year")),
            (UNS, dict(out_columns=["k", "i"], probes=[(pair, "k")])),
            (UNS, dict(out_columns=["k", "i", "k2"])),
            (INV, dict(out_columns=["nope", "i"])),
            (UNS, dict(out_columns=["k", "i"], probes=[(buf, "k"), (buf, "k")])),
            (CAPY, dict(out_columns=["k", "i"], send_capacity=0)),
            (CAPY, dict(out_columns=["k", "i"], send_offset=8)),
            (CAPY, dict(out_columns=["k", "i"], send_capacity=user)),
            (CAPY, dict(out_columns=["k", "i"], send_cursors_offset=user - 64)),
            (INV, dict(out_columns=["k", "i"], comm=comms[1])),
            (INV, dict(out_columns=["k", "i"], comm=None)),
        ]
        for code, kw in k10:
            expect_error(code, run, c, "scan_partition_send", src, **dict(send, **kw))
        star = dict(probes=[(pair, "k", "k2"), (buf, "i")], aggs=[("mul_1minus_minus_paymul", ["a", "b", "d"])], out_columns=["k"])
        k11 = [
            (INV, dict(probes=[(pair, "k", "k2")])),
            (UNS, dict(aggs=[("mul_1minus", ["a", "b"])])),
            (INV, dict(out_columns=["k", "i"])),
            (INV, dict(probes=[(buf, "k"), (buf, "i")])),
            (INV, dict(probes=[(pair, "k", "k2"), (pair, "i", "k")])),
            (CAPY, dict(send_capacity=user)),
            (UNS, dict(aggs=[("mul_1minus_minus_paymul", ["a", "b", "i"])])),
            (INV, dict(comm=comms[1])),
        ]
        for code, kw in k11:
            expect_error(code, run, c, "scan_star_probe_send", src, **dict(send, **dict(star, **kw)))
