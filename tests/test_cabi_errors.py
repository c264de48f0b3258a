"""Error codes and messages of C-ABI entry points that reject their arguments before they touch a device, one or more per
translation unit that reports errors through the shared guard (runtime, program pipelines, peer exchange, serialised steps) —
without a GPU.  The device generator's entry points (datagen) have no such check: each one starts on the context's device.

Every call is made twice: with an LdbError, whose code and message are pinned, and with err = NULL, which must return the
same code and write nothing."""
import ctypes as C

import pytest

from lingodb_b200 import capi

INVALID = capi.LDB_ERR_INVALID
_P = C.c_void_p
_NULL = None


def _calls():
    i64, i32, p = C.c_int64(), C.c_int32(), _P()
    i32b = C.c_int32()
    return [
        # runtime.cpp
        ("ldb_gpu_graph_begin", (_NULL,), INVALID, "null context"),
        ("ldb_gpu_graph_end", (_NULL, C.byref(p)), INVALID, "no capture in progress"),
        ("ldb_gpu_graph_launch", (_NULL,), INVALID, "null graph"),
        ("ldb_gpu_table_column_range", (_NULL, b"x", C.byref(i32), C.byref(i32b)), INVALID, "null argument"),
        ("ldb_gpu_groupby_merge_rows", (_NULL, _NULL, 0), INVALID, "not a group state"),
        ("ldb_gpu_join_table_count", (_NULL, C.byref(i64)), INVALID, "not a join table"),
        ("ldb_gpu_join_table_topk", (_NULL, 1, _NULL, C.byref(i32)), INVALID, "not a group-join table"),
        ("ldb_gpu_join_table_create", (_NULL, 100, 0, 0, 0, C.byref(p)), INVALID, "null argument"),
        ("ldb_gpu_join_table_create_direct", (_NULL, 0, 10, C.byref(p)), INVALID, "null argument"),
        ("ldb_gpu_partition_tuples", (_NULL, _NULL, _NULL, _NULL, 0, 0, 0, _NULL, _NULL, _NULL), INVALID, "n_parts must be in [1, 64]"),
        # program_rt.cpp
        ("ldb_gpu_run_program", (_NULL, _NULL), INVALID, "null argument"),
        ("ldb_gpu_run_program_ex", (_NULL, _NULL, _NULL), INVALID, "null argument"),
        ("ldb_gpu_hashagg_create", (_NULL, 1, 0, _NULL, 16, C.byref(p)), INVALID, "null argument"),
        ("ldb_gpu_hashagg_count", (_NULL, C.byref(i64)), INVALID, "not a hash aggregation state"),
        ("ldb_gpu_hashagg_read", (_NULL, _NULL, 0, C.byref(i64)), INVALID, "not a hash aggregation state"),
        ("ldb_gpu_hashagg_to_table", (_NULL, b"g", C.byref(p)), INVALID, "not a hash aggregation state"),
        ("ldb_gpu_dict_create", (_NULL, 16, 16, C.byref(p)), INVALID, "null argument"),
        ("ldb_gpu_dict_count", (_NULL, C.byref(i64)), INVALID, "not a string dictionary"),
        ("ldb_gpu_dict_to_table", (_NULL, b"d", C.byref(p)), INVALID, "not a string dictionary"),
        ("ldb_gpu_table_order_by", (_NULL, b"x", 0, -1, _NULL, _NULL), INVALID, "null argument"),
        ("ldb_gpu_table_order_by_keys", (_NULL, 1, _NULL, _NULL, -1, _NULL, _NULL), INVALID, "null argument"),
        ("ldb_gpu_table_gather", (_NULL, b"x", _NULL, 0, _NULL, _NULL), INVALID, "null argument"),
        ("ldb_gpu_table_gather_strings", (_NULL, b"x", _NULL, 0, _NULL, _NULL, 0, _NULL, _NULL), INVALID, "null argument"),
        # peer.cu
        ("ldb_gpu_comm_create", (_NULL, 0, 1, 0, C.byref(p), _NULL), INVALID, "null argument"),
        ("ldb_gpu_comm_connect", (_NULL, _NULL), INVALID, "null argument"),
        ("ldb_gpu_comm_connect_local", (_NULL, 1), INVALID, "bad comm list"),
        ("ldb_gpu_comm_barrier", (_NULL,), INVALID, "null comm"),
        ("ldb_gpu_comm_check", (_NULL,), INVALID, "null comm"),
        ("ldb_gpu_comm_heap_zero", (_NULL, 0, 8), INVALID, "range outside the comm's user heap"),
        ("ldb_gpu_groupby_allmerge", (_NULL, _NULL), INVALID, "not a group state"),
        # step_json.cpp
        ("ldb_gpu_step_validate", (_NULL,), INVALID, "null argument"),
        ("ldb_gpu_register_state", (_NULL, b"s", _NULL), INVALID, "null argument"),
        ("ldb_gpu_run_step", (_NULL, b"{}"), INVALID, "null argument"),
        ("ldb_gpu_run_step_hex", (_NULL, _NULL), INVALID, "null argument"),
        ("ldb_gpu_run_step_hex", (_NULL, b"abc"), INVALID, "step description: odd number of hex digits"),
    ]


_CASES = _calls()


@pytest.mark.parametrize("i", range(len(_CASES)), ids=[f"{c[0]}-{k}" for k, c in enumerate(_CASES)])
def test_rejected_before_the_device(i):
    name, args, code, message = _calls()[i]
    fn = getattr(capi.lib(), name)
    e = capi.Error()
    e.code, e.message = -1, b"stale"
    assert fn(*args, C.byref(e)) == code
    assert e.code == code
    assert e.message.decode() == message
    assert fn(*args, None) == code
