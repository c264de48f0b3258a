"""Error codes and messages of the join-table marker entry points (ldb_gpu_join_table_marks, ldb_gpu_join_table_clear_marks) for
arguments they reject before they touch a device — without a GPU.  Every call is made twice: with an LdbError, whose code and message
are pinned, and with err = NULL, which must return the same code."""
import ctypes as C

import pytest

from lingodb_b200 import capi

INVALID = capi.LDB_ERR_INVALID
_NULL = None


def _calls():
    p = C.c_void_p()
    return [
        ("ldb_gpu_join_table_marks", (_NULL, 1, b"m", C.byref(p)), INVALID, "null argument"),
        ("ldb_gpu_join_table_marks", (_NULL, 0, _NULL, C.byref(p)), INVALID, "null argument"),
        ("ldb_gpu_join_table_marks", (_NULL, -1, b"m", _NULL), INVALID, "null argument"),
        ("ldb_gpu_join_table_marks", (_NULL, 7, b"m", C.byref(p)), INVALID, "null argument"),
        ("ldb_gpu_join_table_clear_marks", (_NULL,), INVALID, "null argument"),
    ]


_CASES = _calls()


@pytest.mark.parametrize("i", range(len(_CASES)), ids=[f"{c[0]}-{k}" for k, c in enumerate(_CASES)])
def test_marks_rejected_before_the_device(i):
    name, args, code, message = _calls()[i]
    fn = getattr(capi.lib(), name)
    e = capi.Error()
    e.code, e.message = -1, b"stale"
    assert fn(*args, C.byref(e)) == code
    assert e.code == code
    assert e.message.decode() == message
    assert fn(*args, None) == code
