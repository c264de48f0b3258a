"""Builder side of key-tuple join tables in program pipelines (lingodb_b200/program.py): key placement in consecutive registers, the
moves the builder emits, PROBE_EACH with a key tuple, JOIN_BUILD descriptors, and the C-ABI surface — without a GPU."""
import ctypes as C
import os

import pytest

from lingodb_b200 import capi, program as P, runtime

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))
SELECT = P.OPS["select"]


def test_keys_already_consecutive_need_no_moves():
    b = P.Builder()
    t = C.c_void_p(61)
    r = b.expr(("probe", t, col("ps_partkey"), col("ps_suppkey")))
    ins = b.instructions()
    assert [i[0] for i in ins] == [P.OPS["load"], P.OPS["load"], P.OPS["probe"]]
    # (op, dst, a = first key register, b, arg = table index)
    assert ins[-1] == (P.OPS["probe"], r, ins[0][1], 0, 0) and ins[1][1] == ins[0][1] + 1
    assert b.tables == [t]


def test_scattered_keys_are_moved_to_consecutive_registers():
    b = P.Builder()
    t = C.c_void_p(62)
    x = b.expr(col("a"))
    b.expr(col("b"))
    y = b.expr(col("c"))
    r = b.expr(("probe", t, col("c"), col("a"), ("add", col("a"), const(1)), col("c")))
    ins = b.instructions()
    probe = ins[-1]
    assert probe[0] == P.OPS["probe"] and probe[1] == r
    first = probe[2]
    moves = [i for i in ins if i[0] == SELECT]
    assert len(moves) == 4
    # each move is SELECT dst, x, x, x (condition, then and else the same register), into dst = first, first + 1, …
    assert [m[1] for m in moves] == [first + k for k in range(4)]
    add = next(i for i in ins if i[0] == P.OPS["add"])
    assert [m[2] for m in moves] == [y, x, add[1], y]
    assert all(m[2] == m[3] == m[4] for m in moves)
    # a single key is used in place, whatever register it lives in
    one = P.Builder()
    one.expr(col("z"))
    k = one.expr(col("k"))
    one.expr(("probe", t, col("k")))
    assert one.instr[-1][2] == k and not [i for i in one.instr if i[0] == SELECT]


def test_probe_each_takes_a_key_tuple_and_outer():
    t = C.c_void_p(63)
    inner = P.Builder()
    inner.expr(col("x"))
    m = inner.expr(("probe_each", t, col("p"), col("x"), col("q")))
    each = inner.instr[-1]
    assert each[0] == P.OPS["probe_each"] and each[1] == m and each[3] == 0 and each[4] == 0
    moves = [i for i in inner.instr if i[0] == SELECT]
    assert [mv[1] for mv in moves] == [each[2], each[2] + 1, each[2] + 2]
    outer = P.Builder()
    outer.expr(("probe_each", t, col("p"), col("q"), "outer"))
    each = outer.instr[-1]
    assert each[3] == 1 and not [i for i in outer.instr if i[0] == SELECT]  # loaded consecutively: no moves
    loads = [i for i in outer.instr if i[0] == P.OPS["load"]]
    assert [i[1] for i in loads] == [each[2], each[2] + 1]
    # nothing written after PROBE_EACH overwrites a register written before it (the moves are fresh registers)
    written = set()
    for op, dst, a, bb, arg in inner.instructions():
        assert dst not in written
        written.add(dst)


class _Ctx:
    """Stands in for a context: records the descriptor ldb_gpu_run_program receives."""

    def __init__(self):
        self.h = C.c_void_p(1)
        self.L = self
        self.seen = None

    def ldb_gpu_run_program(self, h, dref, eref):
        d = dref._obj  # the ProgramDesc behind C.byref
        self.seen = dict(sink_kind=d.sink_kind, n_keys=d.n_keys, key_regs=list(d.key_regs), build_key_reg=d.build_key_reg,
                         build_payload_reg=d.build_payload_reg, instr=[(d.instr[i].op, d.instr[i].dst, d.instr[i].a, d.instr[i].b, d.instr[i].arg)
                                                                      for i in range(d.n_instr)])
        return capi.LDB_OK


class _Table:
    h = C.c_void_p(2)


def test_build_descriptor_of_a_key_tuple_table():
    ctx = _Ctx()
    P.build_join(ctx, _Table(), C.c_void_p(64), [col("l_partkey"), ("add", col("l_suppkey"), const(1)), col("l_partkey")], payload=("rowid",),
                 where=("cmp", ">", col("l_quantity"), const(0)))
    d = ctx.seen
    assert d["sink_kind"] == P.SINK_JOIN_BUILD and d["n_keys"] == 3 and d["build_key_reg"] == -1
    dst = {i[1]: i for i in d["instr"]}
    k0, k1, k2 = d["key_regs"][:3]
    assert k0 == k2 and dst[k0][0] == P.OPS["load"] and dst[k1][0] == P.OPS["add"]
    assert dst[d["build_payload_reg"]][0] == P.OPS["rowid"]
    # a single key expression keeps the plain-table descriptor
    P.build_join(ctx, _Table(), C.c_void_p(65), col("o_orderkey"))
    d = ctx.seen
    assert d["n_keys"] == 0 and d["build_key_reg"] >= 0 and d["build_payload_reg"] == -1


def test_capi_declares_the_key_tuple_table():
    S = capi.SIGNATURES
    P_, E = C.c_void_p, C.POINTER(capi.Error)
    assert S["ldb_gpu_join_table_create_keys"] == (C.c_int, [P_, C.c_int32, C.c_int64, C.c_int32, C.POINTER(P_), E])
    assert hasattr(capi.lib(), "ldb_gpu_join_table_create_keys")
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "ldb_gpu.h")).read()
    assert "LDB_STATE_KEY_JOIN = 6" in hdr
    # the program descriptor keeps its layout: a build takes its keys from the existing n_keys / key_regs
    names = [f for f, _ in capi.ProgramDesc._fields_]
    assert names[14:16] == ["n_keys", "key_regs"] and names[18:20] == ["build_key_reg", "build_payload_reg"]


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_no_device_from_the_new_entry_point():
    L = capi.lib()
    s, e = C.c_void_p(), capi.Error()
    assert L.ldb_gpu_join_table_create_keys(None, 2, 1000, 1, C.byref(s), C.byref(e)) == capi.LDB_ERR_NO_DEVICE
    assert b"no CPU fallback" in e.message and not s.value
    class NoContext:
        h, L = None, capi.lib()

    with pytest.raises(capi.LdbRuntimeError) as ei:
        runtime.join_table_keys(NoContext(), 2, 1000)
    assert ei.value.code == capi.LDB_ERR_NO_DEVICE
