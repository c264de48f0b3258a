"""Python face of the GPU operator runtime: contexts, Arrow-layout tables in HBM, TPC-H drivers.

Thin plumbing over the C-ABI (capi.py): numpy/torch only hold buffers; every data-parallel step is
a hand-written sm_90a kernel inside libldb_gpu.so.  Results come back as exact python ints in the
same dict shapes the CPU oracle uses, so the parity tests compare with `==`.
"""
import ctypes as C
from typing import Dict, List, Optional

import numpy as np

from . import capi, datagen
from .capi import Error, check


class Context:
    """One per device (ExecutionContext + scheduler hand-off of the reference)."""

    def __init__(self, device: int = 0):
        self.L = capi.lib()
        self.h = C.c_void_p()
        e = Error()
        check(self.L.ldb_gpu_context_create(device, C.byref(self.h), C.byref(e)), e)
        self.device = device
        self._tables = []

    def close(self):
        if self.h:
            self.L.ldb_gpu_context_destroy(self.h)
            self.h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def info(self) -> dict:
        d, e = capi.DeviceInfo(), Error()
        check(self.L.ldb_gpu_device_info(self.h, C.byref(d), C.byref(e)), e)
        return {"device": d.device, "sm_count": d.sm_count, "cc": (d.cc_major, d.cc_minor), "total_mem": d.total_mem,
                "free_mem": d.free_mem, "l2_bytes": d.l2_bytes, "name": d.name.decode()}

    def synchronize(self):
        e = Error()
        check(self.L.ldb_gpu_synchronize(self.h, C.byref(e)), e)

    def launch_count(self) -> int:
        return int(self.L.ldb_gpu_launch_count(self.h))

    def timer_start(self):
        e = Error()
        check(self.L.ldb_gpu_timer_start(self.h, C.byref(e)), e)

    def timer_stop(self) -> float:
        ms, e = C.c_float(), Error()
        check(self.L.ldb_gpu_timer_stop(self.h, C.byref(ms), C.byref(e)), e)
        return ms.value

    def kernel_time_reset(self, enable: bool = True):
        e = Error()
        check(self.L.ldb_gpu_kernel_time_reset(self.h, int(enable), C.byref(e)), e)

    def kernel_time(self, family: str):
        ms, n, e = C.c_float(), C.c_int64(), Error()
        check(self.L.ldb_gpu_kernel_time(self.h, family.encode(), C.byref(ms), C.byref(n), C.byref(e)), e)
        return ms.value, n.value

    # ------------------------------------------------------------------ captured queries (CUDA graphs)
    def graph_begin(self):
        e = Error()
        check(self.L.ldb_gpu_graph_begin(self.h, C.byref(e)), e)

    def graph_end(self) -> "Graph":
        g, e = C.c_void_p(), Error()
        check(self.L.ldb_gpu_graph_end(self.h, C.byref(g), C.byref(e)), e)
        return Graph(self, g)

    # ------------------------------------------------------------------ tables
    def table(self, name: str, columns: List[datagen.ColumnSpec]) -> "Table":
        return Table(self, name, columns)

    def table_from_host(self, t: datagen.TableData) -> "Table":
        """Stage a host TableData (numpy Arrow buffers) to HBM, batch by batch."""
        tab = Table(self, t.name, t.columns)
        for chunk, n in zip(t.chunks, t.chunk_rows):
            tab.append_host(chunk, n)
        return tab

    def hash_i64(self, a: np.ndarray, b: Optional[np.ndarray] = None) -> np.ndarray:
        a = np.ascontiguousarray(a, dtype=np.int64)
        out = np.zeros(a.shape[0], dtype=np.uint64)
        bp = None
        if b is not None:
            b = np.ascontiguousarray(b, dtype=np.int64)
            bp = b.ctypes.data
        e = Error()
        check(self.L.ldb_gpu_hash_i64(self.h, a.ctypes.data, bp, a.shape[0], out.ctypes.data, C.byref(e)), e)
        return out


class Graph:
    """A captured query: launch() replays every kernel / memset / peer collective recorded between graph_begin and graph_end."""

    def __init__(self, ctx: Context, h):
        self.ctx, self.h = ctx, h

    def launch(self):
        e = Error()
        check(self.ctx.L.ldb_gpu_graph_launch(self.h, C.byref(e)), e)

    def destroy(self):
        if self.h:
            self.ctx.L.ldb_gpu_graph_destroy(self.h)
            self.h = C.c_void_p()


class Table:
    def __init__(self, ctx: Context, name: str, columns: List[datagen.ColumnSpec]):
        self.ctx, self.name, self.columns = ctx, name, list(columns)
        self._names = [c.name.encode() for c in columns]
        schema = (capi.ColumnSchema * len(columns))()
        for i, c in enumerate(columns):
            schema[i] = capi.ColumnSchema(self._names[i], capi.PHYS[c.phys], c.precision, c.scale)
        self.h = C.c_void_p()
        e = Error()
        check(ctx.L.ldb_gpu_table_create(ctx.h, name.encode(), len(columns), schema, C.byref(self.h), C.byref(e)), e)
        self._keep = []
        ctx._tables.append(self)

    def _append(self, n_rows: int, bufs: Dict[str, object], location: int, utf8_sizes: Dict[str, int], valids: Optional[Dict[str, int]] = None,
                offset: int = 0):
        """bufs: column → address (int) or (offsets_addr, bytes_addr) for utf8; valids: column → address of an Arrow validity bitmap.
        offset: the batch's first row is row `offset` of every buffer (Arrow's ArrayView.offset, bitmaps included)."""
        nc = len(self.columns)
        views = (capi.ArrayView * nc)()
        sizes = (C.c_int64 * nc)()
        keep = []
        for i, c in enumerate(self.columns):
            arr = (C.c_void_p * 3)()
            v = bufs[c.name]
            if c.phys == "utf8":
                arr[1], arr[2] = v[0], v[1]
                sizes[i] = utf8_sizes[c.name]
            else:
                arr[1] = v
            nulls = 0
            if valids and valids.get(c.name):
                arr[0] = valids[c.name]
                nulls = -1  # "unknown, look at the bitmap" (Arrow's convention)
            keep.append(arr)
            views[i] = capi.ArrayView(n_rows, nulls, offset, 3 if c.phys == "utf8" else 2, 0, C.cast(arr, C.POINTER(C.c_void_p)), None)
        e = Error()
        check(self.ctx.L.ldb_gpu_table_append_batch(self.h, n_rows, views, sizes, location, C.byref(e)), e)
        self._keep.append((keep, views))

    def append_host(self, chunk: Dict[str, object], n_rows: int, offset: int = 0):
        """chunk: column → numpy buffer ((offsets, bytes) for utf8); an optional entry "<column>$valid" holds the column's Arrow
        validity bitmap (numpy uint8, LSB first, bit i = row i is NOT NULL).  With `offset`, the batch is rows offset .. offset +
        n_rows - 1 of every buffer and bitmap (an Arrow slice)."""
        bufs, sizes, valids = {}, {}, {}
        for c in self.columns:
            v = chunk[c.name]
            if c.name + "$valid" in chunk:
                valids[c.name] = chunk[c.name + "$valid"].ctypes.data
            if c.phys == "utf8":
                offs, data = v
                bufs[c.name] = (offs.ctypes.data, data.ctypes.data)
                sizes[c.name] = int(offs[offset + n_rows])
            else:
                bufs[c.name] = v.ctypes.data
        self._keep.append(chunk)
        self._append(n_rows, bufs, capi.MEM_HOST, sizes, valids, offset)

    def append_device(self, tensors: Dict[str, object], n_rows: int, offset: int = 0):
        """tensors: column → torch CUDA tensor (or (offsets, bytes) pair for utf8), and optionally "<column>$valid" → the column's
        Arrow validity bitmap as a uint8 CUDA tensor; borrowed.  `offset` as in append_host."""
        bufs, sizes, valids = {}, {}, {}
        for c in self.columns:
            v = tensors[c.name]
            if c.name + "$valid" in tensors:
                valids[c.name] = tensors[c.name + "$valid"].data_ptr()
            if c.phys == "utf8":
                bufs[c.name] = (v[0].data_ptr(), v[1].data_ptr())
                sizes[c.name] = int(v[1].numel())
            else:
                bufs[c.name] = v.data_ptr()
        self._keep.append(tensors)
        self._append(n_rows, bufs, capi.MEM_DEVICE, sizes, valids, offset)

    def clear(self):
        e = Error()
        check(self.ctx.L.ldb_gpu_table_clear(self.h, C.byref(e)), e)
        self._keep.clear()

    @property
    def num_rows(self) -> int:
        return int(self.ctx.L.ldb_gpu_table_num_rows(self.h))


# ---------------------------------------------------------------------- TPC-H drivers (include/ldb_tpch.h)
class Tpch:
    """Holds the six table handles and runs the C++ query drivers."""

    def __init__(self, ctx: Context, tables: Dict[str, Table], nation_names: Optional[List[str]] = None):
        self.ctx, self.tables = ctx, tables
        self.t = capi.TpchTables(**{k: (tables[k].h if k in tables else None) for k in ("lineitem", "orders", "customer", "supplier", "nation", "region", "part", "partsupp")})
        self.nation_names = nation_names or [n for n, _ in datagen.NATIONS]

    def q6(self, date_ge="1994-01-01", date_lt="1995-01-01", disc_ge="0.05", disc_le="0.07", qty_lt=24):
        rev, e = capi.I128(), Error()
        check(self.ctx.L.ldb_tpch_q6(self.ctx.h, C.byref(self.t), date_ge.encode(), date_lt.encode(), disc_ge.encode(), disc_le.encode(), qty_lt,
                                     C.byref(rev), C.byref(e)), e)
        return {"revenue": rev.value()}

    @staticmethod
    def _q1_rows(rows, n):
        return [{"l_returnflag": r.l_returnflag, "l_linestatus": r.l_linestatus, "sum_qty": r.sum_qty, "sum_base_price": r.sum_base_price,
                 "sum_disc_price": r.sum_disc_price.value(), "sum_charge": r.sum_charge.value(), "avg_qty": r.avg_qty.value(),
                 "avg_price": r.avg_price.value(), "avg_disc": r.avg_disc.value(), "count_order": r.count_order} for r in rows[:n]]

    def q1(self, date_le="1998-09-02"):
        rows, n, e = (capi.Q1Row * 64)(), C.c_int32(), Error()
        check(self.ctx.L.ldb_tpch_q1(self.ctx.h, C.byref(self.t), date_le.encode(), rows, 64, C.byref(n), C.byref(e)), e)
        return self._q1_rows(rows, n.value)

    def q1_partial(self, date_le="1998-09-02") -> C.c_void_p:
        s, e = C.c_void_p(), Error()
        check(self.ctx.L.ldb_tpch_q1_partial(self.ctx.h, C.byref(self.t), date_le.encode(), C.byref(s), C.byref(e)), e)
        return s

    def q1_finish(self, state, lazy: bool = False):
        """Result rows of a Q1 group state.  lazy=True returns the C rows (host memory, `LazyQ1Rows`) and converts them to python
        dicts only when they are looked at — a benchmark loop then does not spend the GPU's idle time between two queries on
        building dictionaries."""
        ring = getattr(self, "_q1_ring", None)
        if ring is None:  # two reusable result buffers: a lazy result stays valid until the call after the next one
            ring = self._q1_ring = [((capi.Q1Row * 64)(), C.c_int32(), Error()) for _ in range(2)]
            self._q1_next = 0
        rows, n, e = ring[self._q1_next]
        self._q1_next ^= 1
        check(self.ctx.L.ldb_tpch_q1_finish(state, rows, 64, C.byref(n), C.byref(e)), e)
        if lazy:
            return LazyQ1Rows(rows, n.value)
        return self._q1_rows(rows, n.value)

    def q3(self, segment="BUILDING", date="1995-03-15"):
        rows, n, e = (capi.Q3Row * 10)(), C.c_int32(), Error()
        check(self.ctx.L.ldb_tpch_q3(self.ctx.h, C.byref(self.t), segment.encode(), date.encode(), rows, C.byref(n), C.byref(e)), e)
        return [{"l_orderkey": r.l_orderkey, "revenue": r.revenue.value(), "o_orderdate": r.o_orderdate, "o_shippriority": r.o_shippriority}
                for r in rows[: n.value]]

    def _q9_rows(self, rows, n):
        out = [{"nation": self.nation_names[r.n_nationkey], "o_year": r.o_year, "sum_profit": r.sum_profit.value()} for r in rows[:n]]
        return sorted(out, key=lambda r: (r["nation"], -r["o_year"]))  # order by nation, o_year desc

    def q9(self, name_contains="green"):
        rows, n, e = (capi.Q9Row * 1024)(), C.c_int32(), Error()
        check(self.ctx.L.ldb_tpch_q9(self.ctx.h, C.byref(self.t), name_contains.encode(), rows, 1024, C.byref(n), C.byref(e)), e)
        return self._q9_rows(rows, n.value)

    def q9_partial(self, name_contains="green") -> C.c_void_p:
        s, e = C.c_void_p(), Error()
        check(self.ctx.L.ldb_tpch_q9_partial(self.ctx.h, C.byref(self.t), name_contains.encode(), C.byref(s), C.byref(e)), e)
        return s

    def q9_finish(self, state):
        rows, n, e = (capi.Q9Row * 1024)(), C.c_int32(), Error()
        check(self.ctx.L.ldb_tpch_q9_finish(state, rows, 1024, C.byref(n), C.byref(e)), e)
        return self._q9_rows(rows, n.value)

    def q5(self, region_name="ASIA", date_ge="1994-01-01", date_lt="1995-01-01"):
        rows, n, e = (capi.Q5Row * 25)(), C.c_int32(), Error()
        check(self.ctx.L.ldb_tpch_q5(self.ctx.h, C.byref(self.t), region_name.encode(), date_ge.encode(), date_lt.encode(), rows, C.byref(n), C.byref(e)), e)
        # n_name is resolved at materialisation from the (host) nation table
        out = [{"n_name": self.nation_names[r.n_nationkey], "revenue": r.revenue.value()} for r in rows[: n.value]]
        out.sort(key=lambda r: (-r["revenue"], r["n_name"]))
        return out


class LazyQ1Rows:
    """Q1 result rows as the C structs ldb_tpch_q1_finish filled (host memory); materialised as python dicts on first use."""

    def __init__(self, rows, n):
        self._rows, self._n, self._list = rows, n, None

    def materialize(self) -> list:
        if self._list is None:
            self._list = Tpch._q1_rows(self._rows, self._n)
        return self._list

    def __len__(self):
        return self._n

    def __eq__(self, other):
        return self.materialize() == (other.materialize() if isinstance(other, LazyQ1Rows) else other)

    def __iter__(self):
        return iter(self.materialize())

    def __getitem__(self, i):
        return self.materialize()[i]


def groupby_read(ctx: Context, state) -> list:
    rows, n, e = (capi.GroupRow * 1024)(), C.c_int32(), Error()
    check(ctx.L.ldb_gpu_groupby_read(state, rows, 1024, C.byref(n), C.byref(e)), e)
    return rows, n.value


def state_destroy(ctx: Context, state):
    ctx.L.ldb_gpu_state_destroy(state)


# ---------------------------------------------------------------------- generic pipeline call
def run_pipeline(ctx: Context, kind: str, source: Table, filters=(), keys=(), aggs=(), probes=(), build_key=None, build_payload=None,
                 side=(), sink=None, out_columns=(), out_buffers=(), out_capacity=0, out_count=None, bloom_only=False,
                 build_key2=None, build_payload_expr="column", comm=None, send_offset=0, send_capacity=0, send_cursors_offset=0):
    """ldb_gpu_run_pipeline from keyword arguments.  filters: (column, op, value) with value str or int;
    aggs: (expr, [columns]); probes: (state, key_column).  comm (a parallel.Comm or its handle) and send_*: the receive regions and
    cursors of the partition-send pipelines (K10, K11)."""
    keep = []

    def b(s):
        if s is None:
            return None
        v = s.encode()
        keep.append(v)
        return v

    d = capi.PipelineDesc()
    d.kind = capi.PIPE[kind]
    d.source = source.h
    fl = (capi.FilterDesc * max(1, len(filters)))()
    for i, (col, op, val) in enumerate(filters):
        if op == "in":  # list of ints or of strings
            fd = capi.FilterDesc(b(col), capi.OPS[op], int(isinstance(val[0], int)), None, 0)
            fd.n_values = len(val)
            for k, v in enumerate(val):
                if isinstance(v, int):
                    fd.int_values[k] = v
                else:
                    fd.str_values[k] = b(v)
            fl[i] = fd
        elif isinstance(val, int):
            fl[i] = capi.FilterDesc(b(col), capi.OPS[op], 1, None, val)
        else:
            fl[i] = capi.FilterDesc(b(col), capi.OPS[op], 0, b(val), 0)
    d.n_filters, d.filters = len(filters), fl
    d.n_keys = len(keys)
    for i, k in enumerate(keys):
        d.key_columns[i] = b(k)
    d.n_aggs = len(aggs)
    for i, (expr, cols) in enumerate(aggs):
        d.aggs[i].expr = capi.EXPR[expr]
        for j, c in enumerate(cols):
            d.aggs[i].columns[j] = b(c)
    d.n_probes = len(probes)
    for i, pr in enumerate(probes):  # (state, key column[, second key column])
        d.probe_states[i] = pr[0]
        d.probe_key_columns[i] = b(pr[1])
        d.probe_key2_columns[i] = b(pr[2]) if len(pr) > 2 else None
    d.build_key_column, d.build_payload_column = b(build_key), b(build_payload)
    d.build_key2_column = b(build_key2)
    d.build_payload_expr = capi.PAYLOAD_EXPR[build_payload_expr]
    d.n_side = len(side)
    for i, c in enumerate(side):
        d.side_columns[i] = b(c)
    d.sink = sink
    d.n_out_cols = len(out_columns)
    for i, c in enumerate(out_columns):  # (the partition-send pipelines name columns without buffers)
        d.out_columns[i] = b(c)
    for i, buf in enumerate(out_buffers):
        d.out_buffers[i] = buf
    d.out_capacity = out_capacity
    d.out_count = out_count
    d.probe_bloom_only = int(bloom_only)
    d.comm = getattr(comm, "h", comm)
    d.send_offset, d.send_capacity, d.send_cursors_offset = send_offset, send_capacity, send_cursors_offset
    e = Error()
    check(ctx.L.ldb_gpu_run_pipeline(ctx.h, C.byref(d), C.byref(e)), e)


def join_table(ctx: Context, expected_rows: int, unique: bool = True, n_side: int = 0, n_aggs: int = 0) -> C.c_void_p:
    s, e = C.c_void_p(), Error()
    check(ctx.L.ldb_gpu_join_table_create(ctx.h, int(expected_rows), int(unique), n_side, n_aggs, C.byref(s), C.byref(e)), e)
    return s


def join_table_pair(ctx: Context, expected_rows: int, unique: bool = True) -> C.c_void_p:
    s, e = C.c_void_p(), Error()
    check(ctx.L.ldb_gpu_join_table_create_pair(ctx.h, int(expected_rows), int(unique), C.byref(s), C.byref(e)), e)
    return s


def join_table_keys(ctx: Context, n_keys: int, expected_rows: int, unique: bool = True, bloom: bool = True) -> C.c_void_p:
    """A key-tuple join table for program pipelines: 1..4 int64 keys → int64 payload (unique: duplicate tuples are dropped)."""
    s, e = C.c_void_p(), Error()
    flags = (1 if unique else 0) | (0 if bloom else 2)
    check(ctx.L.ldb_gpu_join_table_create_keys(ctx.h, int(n_keys), int(expected_rows), flags, C.byref(s), C.byref(e)), e)
    return s


def join_table_direct(ctx: Context, key_min: int, key_max: int) -> C.c_void_p:
    s, e = C.c_void_p(), Error()
    check(ctx.L.ldb_gpu_join_table_create_direct(ctx.h, int(key_min), int(key_max), C.byref(s), C.byref(e)), e)
    return s


def column_range(ctx: Context, table: Table, column: str):
    lo, hi, e = C.c_int32(), C.c_int32(), Error()
    check(ctx.L.ldb_gpu_table_column_range(table.h, column.encode(), C.byref(lo), C.byref(hi), C.byref(e)), e)
    return lo.value, hi.value


def join_count(ctx: Context, state) -> int:
    n, e = C.c_int64(), Error()
    check(ctx.L.ldb_gpu_join_table_count(state, C.byref(n), C.byref(e)), e)
    return n.value


def groupby_state(ctx: Context, n_keys: int, n_aggs: int, capacity: int = 64) -> C.c_void_p:
    s, e = C.c_void_p(), Error()
    check(ctx.L.ldb_gpu_groupby_create(ctx.h, n_keys, n_aggs, capacity, C.byref(s), C.byref(e)), e)
    return s
