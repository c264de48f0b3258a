"""ctypes binding of the C-ABI (include/ldb_gpu.h, include/ldb_tpch.h) — libldb_gpu.so.

Loading the library works without a GPU (the -m "not gpu" tests check the exported symbols); every
compute entry point then fails with LDB_ERR_NO_DEVICE: there is no CPU fallback on this path.
"""
import ctypes as C
import os

from . import build as _build
from .datagen import CustomerCols, GenScale, LineitemCols, OrdersCols, PartCols, PartsuppCols, SupplierCols

LDB_OK, LDB_ERR_CUDA, LDB_ERR_UNSUPPORTED, LDB_ERR_INVALID, LDB_ERR_CAPACITY, LDB_ERR_NO_DEVICE = range(6)
PHYS = {"int32": 0, "int64": 1, "date32": 2, "decimal128": 3, "fsb4": 4, "utf8": 5, "int8": 6, "int16": 7, "float32": 8, "float64": 9}
MEM_HOST, MEM_DEVICE = 0, 1
OPS = {"=": 0, "!=": 1, "<": 2, "<=": 3, ">": 4, ">=": 5, "notnull": 6, "in": 7, "contains": 8}
EXPR = {"col": 0, "mul": 1, "mul_1minus": 2, "mul_1minus_1plus": 3, "one": 4, "mul_1minus_minus_paymul": 5}
PIPE = {"scan_reduce": 1, "scan_groupby": 2, "scan_build": 3, "scan_probe_agg": 4, "scan_probe2_groupby": 5, "scan_materialize": 6,
        "scan_star_probe_groupby": 7, "scan_partition_send": 8, "scan_star_probe_send": 9}
PAYLOAD_EXPR = {"column": 0, "year": 1}
MAX_AGGS, MAX_KEYS, MAX_SIDE = 8, 2, 2


class LdbRuntimeError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(f"[ldb_gpu error {code}] {message}")
        self.code = code


class Error(C.Structure):
    _fields_ = [("code", C.c_int32), ("message", C.c_char * 252)]


class DeviceInfo(C.Structure):
    _fields_ = [("device", C.c_int32), ("sm_count", C.c_int32), ("cc_major", C.c_int32), ("cc_minor", C.c_int32),
                ("total_mem", C.c_int64), ("free_mem", C.c_int64), ("l2_bytes", C.c_int64), ("name", C.c_char * 64)]


class ArrayView(C.Structure):
    pass


ArrayView._fields_ = [("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64),
                      ("n_children", C.c_int64), ("buffers", C.POINTER(C.c_void_p)), ("children", C.c_void_p)]


class ColumnSchema(C.Structure):
    _fields_ = [("name", C.c_char_p), ("type", C.c_int32), ("precision", C.c_int32), ("scale", C.c_int32)]


class I128(C.Structure):
    _fields_ = [("lo", C.c_uint64), ("hi", C.c_int64)]

    def value(self) -> int:
        return (int(self.hi) << 64) | int(self.lo)


class GroupRow(C.Structure):
    _fields_ = [("keys", C.c_int32 * MAX_KEYS), ("aggs", I128 * MAX_AGGS)]


class TopKRow(C.Structure):
    _fields_ = [("key", C.c_int32), ("side", C.c_int32 * MAX_SIDE), ("pad", C.c_int32), ("agg", I128)]


class FilterDesc(C.Structure):
    _fields_ = [("column", C.c_char_p), ("op", C.c_int32), ("value_is_int", C.c_int32), ("str_value", C.c_char_p), ("int_value", C.c_int64),
                ("n_values", C.c_int32), ("str_values", C.c_char_p * 8), ("int_values", C.c_int64 * 8)]


class AggDesc(C.Structure):
    _fields_ = [("expr", C.c_int32), ("columns", C.c_char_p * 3)]


class PipelineDesc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("source", C.c_void_p), ("n_filters", C.c_int32), ("filters", C.POINTER(FilterDesc)),
                ("n_keys", C.c_int32), ("key_columns", C.c_char_p * MAX_KEYS), ("n_aggs", C.c_int32), ("aggs", AggDesc * MAX_AGGS),
                ("n_probes", C.c_int32), ("probe_states", C.c_void_p * 3), ("probe_key_columns", C.c_char_p * 3),
                ("probe_key2_columns", C.c_char_p * 3),
                ("build_key_column", C.c_char_p), ("build_key2_column", C.c_char_p), ("build_payload_column", C.c_char_p),
                ("build_payload_expr", C.c_int32), ("n_side", C.c_int32),
                ("side_columns", C.c_char_p * MAX_SIDE), ("sink", C.c_void_p),
                ("n_out_cols", C.c_int32), ("out_columns", C.c_char_p * 4), ("out_buffers", C.c_void_p * 4), ("out_capacity", C.c_int64),
                ("out_count", C.c_void_p), ("probe_bloom_only", C.c_int32),
                ("comm", C.c_void_p), ("send_offset", C.c_int64), ("send_capacity", C.c_int64), ("send_cursors_offset", C.c_int64)]


class TpchTables(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("lineitem", "orders", "customer", "supplier", "nation", "region", "part", "partsupp")]


class Q1Row(C.Structure):
    _fields_ = [("l_returnflag", C.c_int32), ("l_linestatus", C.c_int32), ("sum_qty", C.c_int64), ("sum_base_price", C.c_int64),
                ("sum_disc_price", I128), ("sum_charge", I128), ("avg_qty", I128), ("avg_price", I128), ("avg_disc", I128),
                ("count_order", C.c_int64)]


class Q3Row(C.Structure):
    _fields_ = [("l_orderkey", C.c_int32), ("o_orderdate", C.c_int32), ("o_shippriority", C.c_int32), ("pad", C.c_int32), ("revenue", I128)]


class Q5Row(C.Structure):
    _fields_ = [("n_nationkey", C.c_int32), ("pad", C.c_int32), ("revenue", I128)]


class Instr(C.Structure):
    _fields_ = [("op", C.c_uint8), ("dst", C.c_uint8), ("a", C.c_uint8), ("b", C.c_uint8), ("arg", C.c_int32)]


class ProgAgg(C.Structure):
    _fields_ = [("kind", C.c_int32), ("reg", C.c_int32)]


class ProgramDesc(C.Structure):
    _fields_ = [("source", C.c_void_p), ("n_columns", C.c_int32), ("columns", C.POINTER(C.c_char_p)), ("n_instr", C.c_int32), ("instr", C.POINTER(Instr)),
                ("n_consts", C.c_int32), ("consts", C.POINTER(I128)), ("n_strings", C.c_int32), ("strings", C.POINTER(C.c_char_p)),
                ("n_tables", C.c_int32), ("tables", C.POINTER(C.c_void_p)), ("filter_reg", C.c_int32), ("sink_kind", C.c_int32), ("sink", C.c_void_p),
                ("n_keys", C.c_int32), ("key_regs", C.c_int32 * 4), ("n_aggs", C.c_int32), ("aggs", ProgAgg * MAX_AGGS),
                ("build_key_reg", C.c_int32), ("build_payload_reg", C.c_int32), ("n_out", C.c_int32), ("out_regs", C.c_int32 * MAX_AGGS),
                ("out_table", C.POINTER(C.c_void_p))]


class SideColumn(C.Structure):
    _fields_ = [("table", C.c_int32), ("column", C.c_char_p), ("row_reg", C.c_int32)]


class ProgramJoins(C.Structure):
    _fields_ = [("n_side_tables", C.c_int32), ("side_tables", C.POINTER(C.c_void_p)), ("n_side_columns", C.c_int32), ("side_columns", C.POINTER(SideColumn))]


class HashAggRow(C.Structure):
    _fields_ = [("keys", C.c_int64 * 4), ("key_null_mask", C.c_uint32), ("agg_valid_mask", C.c_uint32), ("aggs", I128 * MAX_AGGS)]


# LdbWindowKind; "rank" is the reference's RankWindowFunc, which is ROW_NUMBER; "sql_rank" is SQL's RANK (ties share a rank).  Kinds
# from "sql_rank" on are ldb_gpu_table_window_ex's only
WIN = {"row_number": 1, "rank": 1, "count_star": 2, "count": 3, "sum": 4, "min": 5, "max": 6, "sql_rank": 7, "dense_rank": 8, "percent_rank": 9,
       "cume_dist": 10, "ntile": 11, "lag": 12, "lead": 13, "first_value": 14, "last_value": 15, "nth_value": 16}
# LdbWindowFrameMode
FRAME = {"rows": 0, "range": 1}


class WindowFunc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("column", C.c_char_p), ("name", C.c_char_p)]


class WindowFrame(C.Structure):
    _fields_ = [("mode", C.c_int32), ("pad", C.c_int32), ("from_", C.c_int64), ("to", C.c_int64)]


class WindowFuncEx(C.Structure):
    _fields_ = [("kind", C.c_int32), ("has_default", C.c_int32), ("column", C.c_char_p), ("name", C.c_char_p), ("n", C.c_int64), ("value", I128),
                ("fvalue", C.c_double)]


# LdbSetOpKind
SETOP = {"distinct": 1, "union_all": 2, "union": 3, "intersect": 4, "intersect_all": 5, "except": 6, "except_all": 7}

# LdbNlJoinKind
NLJOIN = {"inner": 1, "left": 2, "right": 3, "full": 4, "semi": 5, "anti": 6, "mark": 7, "count": 8}


class JoinCond(C.Structure):
    _fields_ = [("left", C.c_char_p), ("op", C.c_int32), ("right", C.c_char_p), ("value", I128), ("fvalue", C.c_double)]


class Q5ShuffleStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("orders_tuples_sent", "orders_tuples_received", "lineitem_tuples_sent", "lineitem_tuples_received", "shuffle_bytes_out", "heap_bytes")]


class Q9Row(C.Structure):
    _fields_ = [("n_nationkey", C.c_int32), ("o_year", C.c_int32), ("sum_profit", I128)]


# every symbol include/ldb_gpu.h and include/ldb_tpch.h declare: (restype, argtypes)
_P = C.c_void_p
_E = C.POINTER(Error)
SIGNATURES = {
    "ldb_gpu_context_create": (C.c_int, [C.c_int, C.POINTER(_P), _E]),
    "ldb_gpu_context_destroy": (None, [_P]),
    "ldb_gpu_device_info": (C.c_int, [_P, C.POINTER(DeviceInfo), _E]),
    "ldb_gpu_synchronize": (C.c_int, [_P, _E]),
    "ldb_gpu_context_stream": (C.c_void_p, [_P]),
    "ldb_gpu_context_h2d_bytes": (C.c_int64, [_P]),
    "ldb_gpu_context_raw_staged_rows": (C.c_int64, [_P]),
    "ldb_gpu_effective_cpus": (C.c_int32, []),
    "ldb_gpu_set_tuning": (None, [C.c_int32] * 5),
    "ldb_gpu_set_filter_specialisation": (None, [C.c_int32]),
    "ldb_gpu_set_encoded_scan": (None, [C.c_int32]),
    "ldb_gpu_context_encoded_bytes": (C.c_int64, [_P]),
    "ldb_gpu_set_poll_pause": (None, [C.c_int32, C.c_int32]),
    "ldb_gpu_launch_count": (C.c_int64, [_P]),
    "ldb_gpu_timer_start": (C.c_int, [_P, _E]),
    "ldb_gpu_timer_stop": (C.c_int, [_P, C.POINTER(C.c_float), _E]),
    "ldb_gpu_kernel_time": (C.c_int, [_P, C.c_char_p, C.POINTER(C.c_float), C.POINTER(C.c_int64), _E]),
    "ldb_gpu_kernel_time_reset": (C.c_int, [_P, C.c_int, _E]),
    "ldb_gpu_graph_begin": (C.c_int, [_P, _E]),
    "ldb_gpu_graph_end": (C.c_int, [_P, C.POINTER(_P), _E]),
    "ldb_gpu_graph_launch": (C.c_int, [_P, _E]),
    "ldb_gpu_graph_destroy": (None, [_P]),
    "ldb_gpu_table_create": (C.c_int, [_P, C.c_char_p, C.c_int32, C.POINTER(ColumnSchema), C.POINTER(_P), _E]),
    "ldb_gpu_table_append_batch": (C.c_int, [_P, C.c_int64, C.POINTER(ArrayView), C.POINTER(C.c_int64), C.c_int32, _E]),
    "ldb_gpu_table_clear": (C.c_int, [_P, _E]),
    "ldb_gpu_table_num_rows": (C.c_int64, [_P]),
    "ldb_gpu_table_destroy": (None, [_P]),
    "ldb_gpu_state_destroy": (None, [_P]),
    "ldb_gpu_simple_state_create": (C.c_int, [_P, C.c_int32, C.POINTER(_P), _E]),
    "ldb_gpu_simple_state_read": (C.c_int, [_P, C.POINTER(I128), _E]),
    "ldb_gpu_groupby_create": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P), _E]),
    "ldb_gpu_groupby_read": (C.c_int, [_P, C.POINTER(GroupRow), C.c_int32, C.POINTER(C.c_int32), _E]),
    "ldb_gpu_groupby_merge_rows": (C.c_int, [_P, C.POINTER(GroupRow), C.c_int32, _E]),
    "ldb_gpu_groupby_export_bytes": (C.c_int64, [_P]),
    "ldb_gpu_groupby_export": (C.c_int, [_P, _P, _E]),
    "ldb_gpu_groupby_merge_exported": (C.c_int, [_P, _P, C.c_int32, C.c_int32, _E]),
    "ldb_gpu_join_table_create": (C.c_int, [_P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P), _E]),
    "ldb_gpu_join_table_create_pair": (C.c_int, [_P, C.c_int64, C.c_int32, C.POINTER(_P), _E]),
    "ldb_gpu_join_table_create_direct": (C.c_int, [_P, C.c_int32, C.c_int32, C.POINTER(_P), _E]),
    "ldb_gpu_table_column_range": (C.c_int, [_P, C.c_char_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), _E]),
    "ldb_gpu_join_table_create_keys": (C.c_int, [_P, C.c_int32, C.c_int64, C.c_int32, C.POINTER(_P), _E]),
    "ldb_gpu_join_table_count": (C.c_int, [_P, C.POINTER(C.c_int64), _E]),
    "ldb_gpu_join_table_marks": (C.c_int, [_P, C.c_int32, C.c_char_p, C.POINTER(_P), _E]),
    "ldb_gpu_join_table_clear_marks": (C.c_int, [_P, _E]),
    "ldb_gpu_join_table_bloom": (C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_int64), _E]),
    "ldb_gpu_join_table_topk": (C.c_int, [_P, C.c_int32, C.POINTER(TopKRow), C.POINTER(C.c_int32), _E]),
    "ldb_gpu_run_pipeline": (C.c_int, [_P, C.POINTER(PipelineDesc), _E]),
    "ldb_gpu_step_validate": (C.c_int, [C.c_char_p, _E]),
    "ldb_gpu_run_step": (C.c_int, [_P, C.c_char_p, _E]),
    "ldb_gpu_run_step_hex": (C.c_int, [_P, C.c_char_p, _E]),
    "ldb_gpu_register_state": (C.c_int, [_P, C.c_char_p, _P, _E]),
    "ldb_gpu_find_state": (C.c_void_p, [_P, C.c_char_p]),
    "ldb_gpu_run_program": (C.c_int, [_P, C.POINTER(ProgramDesc), _E]),
    "ldb_gpu_run_program_ex": (C.c_int, [_P, C.POINTER(ProgramDesc), C.POINTER(ProgramJoins), _E]),
    "ldb_gpu_hashagg_create": (C.c_int, [_P, C.c_int32, C.c_int32, C.POINTER(ProgAgg), C.c_int64, C.POINTER(_P), _E]),
    "ldb_gpu_hashagg_count": (C.c_int, [_P, C.POINTER(C.c_int64), _E]),
    "ldb_gpu_hashagg_read": (C.c_int, [_P, C.POINTER(HashAggRow), C.c_int64, C.POINTER(C.c_int64), _E]),
    "ldb_gpu_hashagg_to_table": (C.c_int, [_P, C.c_char_p, C.POINTER(_P), _E]),
    "ldb_gpu_table_order_by": (C.c_int, [_P, C.c_char_p, C.c_int32, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64), _E]),
    "ldb_gpu_table_gather": (C.c_int, [_P, C.c_char_p, C.POINTER(C.c_int64), C.c_int64, _P, _P, _E]),
    "ldb_gpu_table_order_by_keys": (C.c_int, [_P, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_int32), C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64), _E]),
    "ldb_gpu_table_gather_strings": (C.c_int, [_P, C.c_char_p, C.POINTER(C.c_int64), C.c_int64, C.POINTER(C.c_int64), _P, C.c_int64, C.POINTER(C.c_int64), _P, _E]),
    "ldb_gpu_table_window": (C.c_int, [_P, C.c_int32, C.POINTER(C.c_char_p), C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_int32), C.c_int64, C.c_int64,
                                       C.c_int32, C.POINTER(WindowFunc), C.c_int32, C.POINTER(C.c_char_p), C.c_char_p, C.POINTER(_P), _E]),
    "ldb_gpu_table_window_ex": (C.c_int, [_P, C.c_int32, C.POINTER(C.c_char_p), C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_int32), C.POINTER(WindowFrame),
                                          C.c_int32, C.POINTER(WindowFuncEx), C.c_int32, C.POINTER(C.c_char_p), C.c_char_p, C.POINTER(_P), _E]),
    "ldb_gpu_table_setop": (C.c_int, [_P, _P, C.c_int32, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.c_char_p, C.POINTER(_P), _E]),
    "ldb_gpu_table_nl_join": (C.c_int, [_P, _P, C.c_int32, C.c_int32, C.POINTER(JoinCond), C.c_int32, C.POINTER(C.c_char_p), C.c_int32, C.POINTER(C.c_char_p),
                                        C.POINTER(C.c_char_p), C.c_char_p, C.c_char_p, C.POINTER(_P), _E]),
    "ldb_gpu_dict_create": (C.c_int, [_P, C.c_int64, C.c_int64, C.POINTER(_P), _E]),
    "ldb_gpu_dict_count": (C.c_int, [_P, C.POINTER(C.c_int64), _E]),
    "ldb_gpu_dict_to_table": (C.c_int, [_P, C.c_char_p, C.POINTER(_P), _E]),
    "ldb_gpu_partition_tuples": (C.c_int, [_P, _P, C.POINTER(_P), C.POINTER(C.c_int32), C.c_int32, C.c_int64, C.c_int32, _P, C.POINTER(_P), C.POINTER(C.c_int64), _E]),
    "ldb_gpu_join_table_insert": (C.c_int, [_P, _P, _P, _P, C.POINTER(_P), C.c_int64, _E]),
    "ldb_gpu_comm_create": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_int64, C.POINTER(_P), _P, _E]),
    "ldb_gpu_comm_connect": (C.c_int, [_P, _P, _E]),
    "ldb_gpu_comm_connect_local": (C.c_int, [C.POINTER(_P), C.c_int32, _E]),
    "ldb_gpu_comm_destroy": (None, [_P]),
    "ldb_gpu_comm_rank": (C.c_int32, [_P]),
    "ldb_gpu_comm_world": (C.c_int32, [_P]),
    "ldb_gpu_comm_reserved_bytes": (C.c_int64, []),
    "ldb_gpu_comm_slot_bytes": (C.c_int64, []),
    "ldb_gpu_comm_heap": (C.c_void_p, [_P, C.POINTER(C.c_int64)]),
    "ldb_gpu_comm_barrier": (C.c_int, [_P, _E]),
    "ldb_gpu_comm_allgather_small": (C.c_int, [_P, _P, C.c_int64, C.POINTER(_P), _E]),
    "ldb_gpu_groupby_allmerge": (C.c_int, [_P, _P, _E]),
    "ldb_gpu_hashagg_exchange": (C.c_int, [_P, _P, _P, C.c_int64, C.c_int64, _E]),
    "ldb_gpu_table_exchange": (C.c_int, [_P, C.c_int32, C.POINTER(C.c_char_p), C.c_int32, C.POINTER(C.c_char_p), _P, C.c_int64, C.c_int64, C.c_char_p, C.POINTER(_P), _E]),
    "ldb_gpu_table_exchange_varlen": (C.c_int, [_P, C.c_int32, C.POINTER(C.c_char_p), C.c_int32, C.POINTER(C.c_char_p), _P, C.c_int64, C.c_int64, C.c_char_p, C.POINTER(_P), _E]),
    "ldb_gpu_table_sort_exchange": (C.c_int, [_P, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_char_p), C.c_int64, _P, C.c_int64,
                                              C.c_int64, C.c_char_p, C.POINTER(_P), C.POINTER(C.c_int64), C.POINTER(C.c_int64), _E]),
    "ldb_gpu_dict_unify": (C.c_int, [_P, _P, C.c_int64, C.c_int64, C.POINTER(_P), _E]),
    "ldb_gpu_comm_heap_zero": (C.c_int, [_P, C.c_int64, C.c_int64, _E]),
    "ldb_gpu_comm_heap_read": (C.c_int, [_P, C.c_int64, C.c_int64, _P, _E]),
    "ldb_gpu_comm_publish_counts": (C.c_int, [_P, C.c_int64, C.c_int64, _E]),
    "ldb_gpu_join_table_insert_received": (C.c_int, [_P, _P, C.c_int64, C.c_int64, C.c_int64, _E]),
    "ldb_gpu_probe_received_groupby": (C.c_int, [_P, _P, _P, _P, C.c_int64, C.c_int64, C.c_int64, C.c_int32, _E]),
    "ldb_gpu_probe_received_groupby2": (C.c_int, [_P, _P, _P, C.c_int64, C.c_int64, C.c_int64, _E]),
    "ldb_gpu_join_table_create_shared_bloom": (C.c_int, [_P, C.c_int64, C.c_int32, _P, C.c_int64, C.POINTER(C.c_int64), C.POINTER(_P), _E]),
    "ldb_gpu_comm_or_reduce": (C.c_int, [_P, C.c_int64, C.c_int64, _E]),
    "ldb_gpu_comm_check": (C.c_int, [_P, _E]),
    "ldb_gpu_hash_i64": (C.c_int, [_P, _P, _P, C.c_int64, _P, _E]),
    "ldb_gpu_datagen_lineitem": (C.c_int, [_P, C.POINTER(GenScale), C.c_int64, C.c_int64, C.POINTER(LineitemCols), _E]),
    "ldb_gpu_datagen_orders": (C.c_int, [_P, C.POINTER(GenScale), C.c_int64, C.c_int64, C.POINTER(OrdersCols), _E]),
    "ldb_gpu_datagen_customer_fixed": (C.c_int, [_P, C.POINTER(GenScale), C.c_int64, C.c_int64, C.POINTER(CustomerCols), _P, _E]),
    "ldb_gpu_datagen_customer_bytes": (C.c_int, [_P, C.POINTER(GenScale), C.c_int64, C.c_int64, _P, _P, _E]),
    "ldb_gpu_datagen_supplier": (C.c_int, [_P, C.POINTER(GenScale), C.c_int64, C.c_int64, C.POINTER(SupplierCols), _E]),
    "ldb_gpu_datagen_part_fixed": (C.c_int, [_P, C.POINTER(GenScale), C.c_int64, C.c_int64, C.POINTER(PartCols), _P, _E]),
    "ldb_gpu_datagen_part_bytes": (C.c_int, [_P, C.POINTER(GenScale), C.c_int64, C.c_int64, _P, _P, _E]),
    "ldb_gpu_datagen_partsupp": (C.c_int, [_P, C.POINTER(GenScale), C.c_int64, C.c_int64, C.POINTER(PartsuppCols), _E]),
    "ldb_gpu_dbgen_line_counts": (C.c_int, [_P, C.POINTER(GenScale), C.c_int64, C.c_int64, _P, _E]),
    "ldb_gpu_dbgen_lineitem": (C.c_int, [_P, C.POINTER(GenScale), C.c_int64, C.c_int64, _P, C.POINTER(LineitemCols), _E]),
    "ldb_gpu_dbgen_orders": (C.c_int, [_P, C.POINTER(GenScale), C.c_int64, C.c_int64, C.POINTER(OrdersCols), _E]),
    "ldb_gpu_dbgen_small_fixed": (C.c_int, [_P, C.POINTER(GenScale), C.c_int32, C.c_int64, C.c_int64, _P, _P, _P, _P, _E]),
    "ldb_gpu_dbgen_bytes": (C.c_int, [_P, C.POINTER(GenScale), C.c_int32, C.c_int64, C.c_int64, _P, _P, _E]),
    "ldb_tpch_q6": (C.c_int, [_P, C.POINTER(TpchTables), C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int64, C.POINTER(I128), _E]),
    "ldb_tpch_q6_partial": (C.c_int, [_P, C.POINTER(TpchTables), C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int64, C.POINTER(_P), _E]),
    "ldb_tpch_q1": (C.c_int, [_P, C.POINTER(TpchTables), C.c_char_p, C.POINTER(Q1Row), C.c_int32, C.POINTER(C.c_int32), _E]),
    "ldb_tpch_q1_partial": (C.c_int, [_P, C.POINTER(TpchTables), C.c_char_p, C.POINTER(_P), _E]),
    "ldb_tpch_q1_finish": (C.c_int, [_P, C.POINTER(Q1Row), C.c_int32, C.POINTER(C.c_int32), _E]),
    "ldb_tpch_q3": (C.c_int, [_P, C.POINTER(TpchTables), C.c_char_p, C.c_char_p, C.POINTER(Q3Row), C.POINTER(C.c_int32), _E]),
    "ldb_tpch_q5": (C.c_int, [_P, C.POINTER(TpchTables), C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(Q5Row), C.POINTER(C.c_int32), _E]),
    "ldb_tpch_q5_repartitioned_heap_bytes": (C.c_int64, [C.c_int64, C.c_int64, C.c_int32]),
    "ldb_tpch_q5_repartitioned": (C.c_int, [_P, C.POINTER(TpchTables), _P, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int64, C.c_int64, C.POINTER(Q5Row), C.POINTER(C.c_int32),
                                            C.POINTER(Q5ShuffleStats), _E]),
    "ldb_tpch_q9_repartitioned_heap_bytes": (C.c_int64, [C.c_int64, C.c_int64, C.c_int32]),
    "ldb_tpch_q9_repartitioned": (C.c_int, [_P, C.POINTER(TpchTables), _P, C.c_char_p, C.c_int64, C.c_int64, C.POINTER(Q9Row), C.c_int32, C.POINTER(C.c_int32),
                                            C.POINTER(Q5ShuffleStats), _E]),
    "ldb_tpch_q9_partial": (C.c_int, [_P, C.POINTER(TpchTables), C.c_char_p, C.POINTER(_P), _E]),
    "ldb_tpch_q9_finish": (C.c_int, [_P, C.POINTER(Q9Row), C.c_int32, C.POINTER(C.c_int32), _E]),
    "ldb_tpch_q9": (C.c_int, [_P, C.POINTER(TpchTables), C.c_char_p, C.POINTER(Q9Row), C.c_int32, C.POINTER(C.c_int32), _E]),
}

_lib = None


def lib_path() -> str:
    return _build.GPU_LIB


def lib():
    """Load libldb_gpu.so (building it in-tree if the sources changed)."""
    global _lib
    if _lib is None:
        path = _build.build_gpu()
        if not os.path.exists(path):
            raise FileNotFoundError(f"{path} is missing: the GPU operator runtime has no fallback; run lingodb_b200.build.build_gpu()")
        L = C.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError here = header/library mismatch
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc: int, err: Error):
    if rc != LDB_OK:
        raise LdbRuntimeError(rc, err.message.decode(errors="replace"))
