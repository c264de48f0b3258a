"""Multi-GPU plumbing (one process per GPU, torch.distributed): how relations are split across ranks
and how small partial aggregates are merged.  The reference has no counterpart (single process;
SURVEY §2 "Parallelism strategies"): scans shard by row range with no data-path collective, only
the 4-group partial tables (≈9 KB) are all-gathered and folded by a merge kernel (K7).

The table image exchanged is exactly what ldb_gpu_groupby_export writes:
    int32 state[cap] | int32 keys[cap][2] | uint64 acc[cap][8][2]      (cap = table capacity)
"""
import ctypes as C
from typing import List, Tuple

import numpy as np

from . import datagen

MAX_KEYS, MAX_AGGS = 2, 8


def order_range(s: datagen.GenScale, rank: int, world: int) -> Tuple[int, int, int, int]:
    """Orders [o_lo, o_hi) and their lineitem rows [r_lo, r_hi) owned by `rank` (contiguous, exhaustive, disjoint)."""
    o_lo, o_hi = s.n_orders * rank // world, s.n_orders * (rank + 1) // world
    L = datagen.lib()
    return o_lo, o_hi, int(L.ldbgen_order_first_line(C.byref(s), o_lo)), int(L.ldbgen_order_first_line(C.byref(s), o_hi))


def row_range(n_rows: int, rank: int, world: int) -> Tuple[int, int]:
    return n_rows * rank // world, n_rows * (rank + 1) // world


def image_bytes(cap: int) -> int:
    return cap * 4 + cap * MAX_KEYS * 4 + cap * MAX_AGGS * 2 * 8


def pack_image(cap: int, groups: List[Tuple[Tuple[int, int], List[int]]]) -> np.ndarray:
    """groups: [((k0, k1), [agg0, agg1, … as python ints (128-bit two's complement)])] → image bytes."""
    state = np.zeros(cap, np.int32)
    keys = np.zeros((cap, MAX_KEYS), np.int32)
    acc = np.zeros((cap, MAX_AGGS, 2), np.uint64)
    for i, ((k0, k1), aggs) in enumerate(groups):
        state[i] = 2
        keys[i] = (k0, k1)
        for a, v in enumerate(aggs):
            v &= (1 << 128) - 1
            acc[i, a, 0] = v & 0xFFFFFFFFFFFFFFFF
            acc[i, a, 1] = v >> 64
    return np.concatenate([state.view(np.uint8), keys.reshape(-1).view(np.uint8), acc.reshape(-1).view(np.uint8)])


def unpack_image(img: np.ndarray, cap: int):
    img = np.ascontiguousarray(img, dtype=np.uint8)
    state = img[: cap * 4].view(np.int32)
    keys = img[cap * 4: cap * 4 + cap * MAX_KEYS * 4].view(np.int32).reshape(cap, MAX_KEYS)
    acc = img[cap * 4 + cap * MAX_KEYS * 4:].view(np.uint64).reshape(cap, MAX_AGGS, 2)
    out = []
    for i in range(cap):
        if state[i] == 2:
            out.append(((int(keys[i, 0]), int(keys[i, 1])), [(int(acc[i, a, 1]) << 64) | int(acc[i, a, 0]) for a in range(MAX_AGGS)]))
    return out


def merge_images_host(images: List[np.ndarray], cap: int):
    """Reference semantics of the K7 merge (groupMergeImagesKernel): sums mod 2^128 per key."""
    total = {}
    for img in images:
        for key, aggs in unpack_image(img, cap):
            cur = total.setdefault(key, [0] * MAX_AGGS)
            for a in range(MAX_AGGS):
                cur[a] = (cur[a] + aggs[a]) & ((1 << 128) - 1)
    return total


def _signed(v: int, bits: int) -> int:
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def q1_rows_from_groups(total) -> list:
    """Host finish of Q1 from merged groups (mirror of ldb_tpch_q1_finish): avg = (sum * 10^19) sdiv count."""
    rows = []
    for (k0, k1), a in sorted(total.items()):
        sum_qty, sum_base, sum_disc, cnt = _signed(a[0], 64), _signed(a[1], 64), _signed(a[4], 64), _signed(a[5], 64)

        def avg(x):
            q = abs(x * 10**19) // cnt
            return q if x >= 0 else -q

        rows.append({"l_returnflag": k0, "l_linestatus": k1, "sum_qty": sum_qty, "sum_base_price": sum_base, "sum_disc_price": _signed(a[2], 128),
                     "sum_charge": _signed(a[3], 128), "avg_qty": avg(sum_qty), "avg_price": avg(sum_base), "avg_disc": avg(sum_disc), "count_order": cnt})
    return rows


class Comm:
    """Peer-mapped exchange over NVLink (include/ldb_gpu.h "multi-GPU", csrc/peer.cu): every rank's symmetric heap is mapped
    into its peers through CUDA IPC; collectives are kernels that store into peer HBM and publish a flag.  torch.distributed
    only carries the 64-byte handles at start-up (`exchange` may be any callable bytes → [bytes per rank])."""

    def __init__(self, ctx, rank: int, world: int, user_bytes: int = 0, exchange=None, connect: bool = True):
        from . import capi
        self.ctx, self.rank, self.world, self.L = ctx, rank, world, ctx.L
        self._local = None  # local_group: what the ranks of this process share (host barrier, per-rank counts)
        self.h = C.c_void_p()
        handle = (C.c_uint8 * 64)()
        e = capi.Error()
        capi.check(self.L.ldb_gpu_comm_create(ctx.h, rank, world, int(user_bytes), C.byref(self.h), handle, C.byref(e)), e)
        if world > 1 and connect:
            if exchange is None:
                import torch.distributed as dist

                def exchange(b):
                    out = [None] * world
                    dist.all_gather_object(out, b)
                    return out
            handles = exchange(bytes(handle))
            blob = (C.c_uint8 * (64 * world)).from_buffer_copy(b"".join(handles))
            capi.check(self.L.ldb_gpu_comm_connect(self.h, blob, C.byref(e)), e)

    @classmethod
    def local_group(cls, ctxs, user_bytes: int = 0):
        """All ranks inside ONE process (tests; contexts may share a device): peers are wired by pointer, no IPC."""
        from . import capi
        comms = [cls(c, r, len(ctxs), user_bytes, connect=False) for r, c in enumerate(ctxs)]
        arr = (C.c_void_p * len(comms))(*[c.h for c in comms])
        e = capi.Error()
        capi.check(comms[0].L.ldb_gpu_comm_connect_local(arr, len(comms), C.byref(e)), e)
        import threading
        import types
        shared = types.SimpleNamespace(barrier=threading.Barrier(len(comms)), counts=[0] * len(comms))
        for c in comms:
            c._local = shared
        return comms

    def close(self):
        if self.h:
            self.L.ldb_gpu_comm_destroy(self.h)
            self.h = C.c_void_p()

    def barrier(self):
        from . import capi
        e = capi.Error()
        capi.check(self.L.ldb_gpu_comm_barrier(self.h, C.byref(e)), e)

    def allmerge(self, state):
        """K7 over NVLink: afterwards every rank's group state holds the merged groups of all ranks."""
        from . import capi
        e = capi.Error()
        capi.check(self.L.ldb_gpu_groupby_allmerge(state, self.h, C.byref(e)), e)

    def hashagg_exchange(self, local, owned, capacity: int = None, recv_offset: int = 0):
        """Partitioned merge of program hash aggregations (ldb_gpu_hashagg_exchange): every group of `local` is folded into `owned` on
        the rank that owns its key hash, so the ranks' `owned` states hold disjoint groups whose union is the whole aggregation; a
        keyless state is merged on every rank.  Collective, and it waits for the peers on the host: the ranks of one process call it
        from one thread each.  The receive region starts at user-heap offset `recv_offset`; without a `capacity` it holds the largest
        group count of any rank's `local` per source (found by a host barrier in one process, a small all-gather across processes)."""
        from . import capi
        e = capi.Error()
        if capacity is None:
            n = C.c_int64()
            capi.check(self.L.ldb_gpu_hashagg_count(local, C.byref(n), C.byref(e)), e)
            capacity = max(self._gather_counts(int(n.value)))
        capi.check(self.L.ldb_gpu_hashagg_exchange(local, owned, self.h, int(recv_offset), int(capacity), C.byref(e)), e)

    def table_exchange(self, table, keys, columns=None, name: str = "received", recv_offset: int = 0, recv_bytes: int = None):
        """Repartition of a table's rows (ldb_gpu_table_exchange): with 1..4 `keys` every row goes to the rank that owns its key tuple
        (the rank hashagg_exchange gives the group with those keys); with no keys every row goes to every rank.  `table` is a runtime
        table, a program.RawTable or a table handle; `columns` the columns to ship (None: all).  Returns this rank's received rows as a
        program.RawTable, source rank 0's rows first, each source's in its row order.  Collective, and it waits for the peers on the
        host: the ranks of one process call it from one thread each.  The receive region starts at user-heap offset `recv_offset` and
        spans `recv_bytes` (None: the rest of the user heap); rows that do not fit fail with LDB_ERR_CAPACITY on every rank.  The
        received table is named `name` ("received" when None)."""
        return self._exchange(self.L.ldb_gpu_table_exchange, table, keys, columns, name, recv_offset, recv_bytes)

    def table_exchange_varlen(self, table, keys, columns=None, name: str = "received", recv_offset: int = 0, recv_bytes: int = None):
        """table_exchange whose shipped columns may also be utf8 (ldb_gpu_table_exchange_varlen): string columns travel with their rows,
        without a dictionary, and arrive as ordinary utf8 columns (offsets from 0, the bytes, validity bytes).  Keys, owners, order and
        errors are those of table_exchange, and without utf8 columns the received table is the same.  The receive region also holds the
        received strings' bytes; a receiver whose bytes of one utf8 column pass 2^31 - 1 fails with LDB_ERR_UNSUPPORTED on every rank, rows
        and bytes that do not fit `recv_bytes` with LDB_ERR_CAPACITY on every rank."""
        return self._exchange(self.L.ldb_gpu_table_exchange_varlen, table, keys, columns, name, recv_offset, recv_bytes)

    def sort_exchange(self, table, keys, columns=None, limit=None, name: str = "sorted", recv_offset: int = 0, recv_bytes: int = None):
        """ORDER BY (… LIMIT) across ranks (ldb_gpu_table_sort_exchange): `keys` are 1..4 (column, descending) pairs (a bare column name
        is ascending), in the order of order_by_keys, with ties broken by (source rank, source row).  Without a `limit` every rank gets one
        range of the global order, cut by splitters sampled from every rank; with one, rank 0 gets the first `limit` rows and the other
        ranks empty tables.  `columns` are the columns to ship (None: all, utf8 included); keys need not be among them.  Returns
        (program.RawTable, first_row, total_rows): this rank's rows already in order, the result rows on lower ranks and on all ranks.
        Collective, and it waits for the peers on the host: the ranks of one process call it from one thread each.  The receive region
        starts at user-heap offset `recv_offset` and spans `recv_bytes` (None: the rest of the user heap); rows that do not fit fail with
        LDB_ERR_CAPACITY on every rank."""
        from . import capi
        from .program import RawTable, _handle
        keys = [(k, False) if isinstance(k, str) else (k[0], bool(k[1])) for k in keys or []]
        kn = [k.encode() for k, _ in keys]
        karr = (C.c_char_p * max(1, len(kn)))(*kn)
        darr = (C.c_int32 * max(1, len(kn)))(*[int(d) for _, d in keys])
        cn = [c.encode() for c in columns] if columns is not None else []
        carr = (C.c_char_p * max(1, len(cn)))(*cn) if columns is not None else None
        if recv_bytes is None:
            recv_bytes = self.heap()[1] - int(recv_offset)
        out, first, total, e = C.c_void_p(), C.c_int64(), C.c_int64(), capi.Error()
        capi.check(self.L.ldb_gpu_table_sort_exchange(C.c_void_p(_handle(table)), len(kn), karr, darr, len(cn), carr, -1 if limit is None else int(limit), self.h,
                                                      int(recv_offset), int(recv_bytes), name.encode() if name is not None else None, C.byref(out),
                                                      C.byref(first), C.byref(total), C.byref(e)), e)
        return RawTable(self.ctx, out), int(first.value), int(total.value)

    def _exchange(self, entry, table, keys, columns, name, recv_offset, recv_bytes):
        from . import capi
        from .program import RawTable, _handle
        keys = list(keys or [])
        kn = [k.encode() for k in keys]
        karr = (C.c_char_p * max(1, len(kn)))(*kn)
        cn = [c.encode() for c in columns] if columns is not None else []
        carr = (C.c_char_p * max(1, len(cn)))(*cn) if columns is not None else None
        if recv_bytes is None:
            recv_bytes = self.heap()[1] - int(recv_offset)
        out, e = C.c_void_p(), capi.Error()
        capi.check(entry(C.c_void_p(_handle(table)), len(kn), karr, len(cn), carr, self.h, int(recv_offset), int(recv_bytes),
                         name.encode() if name is not None else None, C.byref(out), C.byref(e)), e)
        return RawTable(self.ctx, out)

    def dict_unify(self, local, recv_offset: int = 0, recv_bytes: int = None):
        """Union of every rank's string dictionary (ldb_gpu_dict_unify): returns a new dictionary state, the same on every rank, whose
        codes are the strings' positions in bytewise order, so ("strcode", unified, column, "lookup") gives codes that agree across ranks
        and order like the strings.  Programs may only look strings up in it.  Collective, and it waits for the peers on the host: the
        ranks of one process call it from one thread each.  The receive region starts at user-heap offset `recv_offset` and spans
        `recv_bytes` (None: the rest of the user heap); strings that do not fit fail with LDB_ERR_CAPACITY on every rank."""
        from . import capi
        if recv_bytes is None:
            recv_bytes = self.heap()[1] - int(recv_offset)
        out, e = C.c_void_p(), capi.Error()
        capi.check(self.L.ldb_gpu_dict_unify(local, self.h, int(recv_offset), int(recv_bytes), C.byref(out), C.byref(e)), e)
        return out

    def _gather_counts(self, n: int) -> List[int]:
        """every rank's `n`, in rank order"""
        if self.world == 1:
            return [n]
        if self._local is not None:
            self._local.counts[self.rank] = n
            self._local.barrier.wait()
            out = list(self._local.counts)
            self._local.barrier.wait()  # nobody overwrites its count before every rank has read them all
            return out
        import torch

        from . import capi
        # no device-wide synchronisation and no pageable copy here: the all-gather kernel waits for the peers, and a device-wide wait
        # would also wait for that kernel.  The block is pinned host memory the kernel reads through unified addressing; the result
        # comes back into pinned memory on a stream of its own.
        dev = torch.device("cuda", self.ctx.device)
        block = torch.tensor([n, 0], dtype=torch.int64).pin_memory()
        res, e = C.c_void_p(), capi.Error()
        capi.check(self.L.ldb_gpu_comm_allgather_small(self.h, C.c_void_p(block.data_ptr()), 16, C.byref(res), C.byref(e)), e)
        self.ctx.synchronize()
        slot = int(self.L.ldb_gpu_comm_slot_bytes())
        out = torch.empty(2 * self.world, dtype=torch.int64).pin_memory()
        side = torch.cuda.Stream(dev)
        with torch.cuda.stream(side):
            for r in range(self.world):
                out[2 * r: 2 * r + 2].view(torch.int32).copy_(_device_view(res.value + r * slot, 4, dev), non_blocking=True)
        side.synchronize()
        return [int(out[2 * r]) for r in range(self.world)]

    def check(self):
        from . import capi
        e = capi.Error()
        capi.check(self.L.ldb_gpu_comm_check(self.h, C.byref(e)), e)

    def heap(self):
        n = C.c_int64()
        p = self.L.ldb_gpu_comm_heap(self.h, C.byref(n))
        return int(p or 0), int(n.value)


def allgather_merge_state(ctx, state, world: int, rank: int, bufs: dict):
    """NCCL path (kept as the comparison arm of bench.py --merge nccl): export → all_gather_into_tensor → merge kernel."""
    import torch
    import torch.distributed as dist

    from . import capi
    L = ctx.L
    nbytes = int(L.ldb_gpu_groupby_export_bytes(state))
    if "send" not in bufs or bufs["send"].numel() != nbytes:
        dev = torch.device("cuda", ctx.device)
        bufs["send"] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        bufs["recv"] = torch.empty(nbytes * world, dtype=torch.uint8, device=dev)
    if "stream" not in bufs:
        bufs["stream"] = torch.cuda.ExternalStream(int(L.ldb_gpu_context_stream(ctx.h)), device=torch.device("cuda", ctx.device))
    e = capi.Error()
    capi.check(L.ldb_gpu_groupby_export(state, C.c_void_p(bufs["send"].data_ptr()), C.byref(e)), e)
    # torch sees the context's compute stream as its current stream: NCCL orders itself after the export and the merge
    # kernel after NCCL with stream events only — no host synchronisation inside the step
    with torch.cuda.stream(bufs["stream"]):
        dist.all_gather_into_tensor(bufs["recv"], bufs["send"])
    capi.check(L.ldb_gpu_groupby_merge_exported(state, C.c_void_p(bufs["recv"].data_ptr()), world, rank, C.byref(e)), e)


def q9_sharded(ctx, tpch, world: int, rank: int, bufs: dict, name_contains: str = "green", comm: "Comm" = None):
    """Q9 with lineitem ⋈ orders co-partitioned by order range (each rank's `tpch` holds its lineitem/orders shard and
    replicas of part, partsupp, supplier, nation): per-rank pipelines → merge of the group tables across ranks (peer-mapped
    all-merge kernel when a Comm is given, else NCCL all-gather + K7)."""
    from . import runtime
    st = tpch.q9_partial(name_contains)
    if world > 1:
        if comm is not None:
            comm.allmerge(st)
        else:
            allgather_merge_state(ctx, st, world, rank, bufs)
    rows = tpch.q9_finish(st)
    runtime.state_destroy(ctx, st)
    return rows


# ------------------------------------------------------------------------------------------------ repartitioned joins (C++ drivers)
# (round 1 orchestrated this plan from Python with NCCL all-to-alls and host synchronisations between the phases; it is now
#  csrc/tpch_plans.cpp + csrc/peer.cu: fused partition → NVLink peer stores, device-side barriers, no host round trip)
def q5_heap_bytes(ctx, n_orders_total: int, n_lineitem_total: int, world: int) -> int:
    return int(ctx.L.ldb_tpch_q5_repartitioned_heap_bytes(int(n_orders_total), int(n_lineitem_total), world))


def q5_repartitioned_peer(ctx, tpch, comm: "Comm", n_orders_total: int, n_lineitem_total: int, region_name="ASIA", date_ge="1994-01-01", date_lt="1995-01-01"):
    """The C++ driver (include/ldb_tpch.h ldb_tpch_q5_repartitioned): fused partition + NVLink peer stores, device-side barriers,
    Bloom OR through peer loads, peer all-merge — no NCCL, no host synchronisation inside the data path.  Returns (rows, stats)."""
    from . import capi
    rows, n, st, e = (capi.Q5Row * 25)(), C.c_int32(), capi.Q5ShuffleStats(), capi.Error()
    capi.check(ctx.L.ldb_tpch_q5_repartitioned(ctx.h, C.byref(tpch.t), comm.h, region_name.encode(), date_ge.encode(), date_lt.encode(), int(n_orders_total), int(n_lineitem_total),
                                               rows, C.byref(n), C.byref(st), C.byref(e)), e)
    out = [{"n_name": tpch.nation_names[r.n_nationkey], "revenue": r.revenue.value()} for r in rows[: n.value]]
    out.sort(key=lambda r: (-r["revenue"], r["n_name"]))
    return out, {k: int(getattr(st, k)) for k, _ in capi.Q5ShuffleStats._fields_}


def q9_heap_bytes(ctx, n_orders_total: int, n_lineitem_total: int, world: int) -> int:
    return int(ctx.L.ldb_tpch_q9_repartitioned_heap_bytes(int(n_orders_total), int(n_lineitem_total), world))


def q9_repartitioned_peer(ctx, tpch, comm: "Comm", n_orders_total: int, n_lineitem_total: int, name_contains: str = "green"):
    """ldb_tpch_q9_repartitioned: orders hash-partitioned across the ranks, lineitem contributions shipped to the owner of their order
    (K10 + K11 peer stores, device barriers, peer all-merge).  Returns (rows, stats)."""
    from . import capi
    rows, n, st, e = (capi.Q9Row * 1024)(), C.c_int32(), capi.Q5ShuffleStats(), capi.Error()
    capi.check(ctx.L.ldb_tpch_q9_repartitioned(ctx.h, C.byref(tpch.t), comm.h, name_contains.encode(), int(n_orders_total), int(n_lineitem_total), rows, 1024, C.byref(n),
                                               C.byref(st), C.byref(e)), e)
    return tpch._q9_rows(rows, n.value), {k: int(getattr(st, k)) for k, _ in capi.Q5ShuffleStats._fields_}


def _materialize(ctx, table, out_columns, widths, capacity, dev, **kw):
    """Run a K8 (scan → filters → [probe] → compacted columns) pipeline into fresh device buffers; regrow if the estimate was too small."""
    import torch

    from . import runtime
    while True:
        bufs = [torch.empty((capacity, 16), dtype=torch.uint8, device=dev) if w == 16 else torch.empty(capacity, dtype=torch.int32, device=dev) for w in widths]
        count = torch.zeros(1, dtype=torch.int64, device=dev)
        torch.cuda.synchronize(dev)
        runtime.run_pipeline(ctx, "scan_materialize", table, out_columns=out_columns, out_buffers=[t.data_ptr() for t in bufs], out_capacity=capacity,
                             out_count=count.data_ptr(), **kw)
        ctx.synchronize()
        n = int(count.item())
        if n <= capacity:
            return bufs, n
        capacity = int(n * 1.1) + 1024


class _CudaArray:
    def __init__(self, ptr: int, n: int):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 2}


def _device_view(ptr: int, n_int32: int, dev):
    """torch view (no copy) of device memory owned by libldb_gpu.so, so NCCL can work on it in place."""
    import torch
    return torch.as_tensor(_CudaArray(ptr, n_int32), device=dev)
