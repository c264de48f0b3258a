"""Builder side of string dictionaries in program pipelines (lingodb_b200/program.py): STRCODE in insert and lookup mode, over source
and side columns, and the C-ABI surface of dictionaries, multi-key ORDER BY and string gathers — without a GPU."""
import ctypes as C

import pytest

from lingodb_b200 import capi, program as P

col = lambda n: ("col", n)


def test_strcode_insert_and_lookup_modes():
    b = P.Builder()
    brands, types = C.c_void_p(41), C.c_void_p(42)
    ins = b.expr(("strcode", brands, "p_brand"))
    look = b.expr(("strcode", brands, "p_brand", "lookup"))
    other = b.expr(("strcode", types, "p_type"))
    assert b.expr(("strcode", brands, "p_brand")) == ins  # the same expression is emitted once
    assert b.tables == [brands, types]
    assert b.columns == ["p_brand", "p_type"]
    codes = [i for i in b.instructions() if i[0] == P.OPS["strcode"]]
    assert P.OPS["strcode"] == 27
    # (op, dst, a = column, b = 1 insert / 0 lookup, arg = table index)
    assert codes == [(27, ins, 0, 1, 0), (27, look, 0, 0, 0), (27, other, 1, 1, 1)]
    with pytest.raises(ValueError, match="lookup"):
        P.Builder().expr(("strcode", brands, "p_brand", "insert"))
    with pytest.raises(ValueError, match="not a column"):
        P.Builder().expr(("strcode", brands, ("col", "p_brand")))


def test_strcode_over_side_columns_is_renumbered_after_the_source_columns():
    b = P.Builder()
    part, brands = C.c_void_p(51), C.c_void_p(52)
    join = C.c_void_p(53)
    row = ("probe", join, col("ps_partkey"))
    code = b.expr(("strcode", brands, ("fetch", part, row, "p_brand")))
    b.expr(("strcode", brands, "s_name", "lookup"))
    b.expr(("strkey8", ("fetch", part, row, "p_type")))
    ins = b.instructions()
    n_src = len(b.columns)
    assert b.columns == ["ps_partkey", "s_name"]
    assert [c for _, c, _ in b.side_columns] == ["p_brand", "p_type"]
    assert sorted(t.value for t in b.tables) == [52, 53]  # the probe's join table and the dictionary share the tables list
    d = b.tables.index(brands)
    strcodes = [i for i in ins if i[0] == P.OPS["strcode"]]
    assert [(i[2], i[3], i[4]) for i in strcodes] == [(n_src + 0, 1, d), (1, 0, d)]
    assert [i for i in ins if i[0] == P.OPS["probe"]][0][4] == b.tables.index(join)
    assert [i for i in ins if i[0] == P.OPS["strkey8"]][0][2] == n_src + 1
    probe_at = next(k for k, i in enumerate(ins) if i[0] == P.OPS["probe"])
    code_at = next(k for k, i in enumerate(ins) if i[1] == code)
    assert probe_at < code_at  # the side column's row register is written before STRCODE reads it
    (_, _, reg), = {sc for sc in b.side_columns if sc[1] == "p_brand"}
    assert ins[probe_at][1] == reg


def test_capi_covers_dictionaries_order_by_keys_and_string_gathers():
    S = capi.SIGNATURES
    P_, E = C.c_void_p, C.POINTER(capi.Error)
    assert S["ldb_gpu_dict_create"] == (C.c_int, [P_, C.c_int64, C.c_int64, C.POINTER(P_), E])
    assert S["ldb_gpu_dict_count"] == (C.c_int, [P_, C.POINTER(C.c_int64), E])
    assert S["ldb_gpu_dict_to_table"] == (C.c_int, [P_, C.c_char_p, C.POINTER(P_), E])
    assert S["ldb_gpu_table_order_by_keys"][1][1:4] == [C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_int32)]
    assert S["ldb_gpu_table_gather_strings"][1][4] == C.POINTER(C.c_int64) and S["ldb_gpu_table_gather_strings"][1][6] == C.c_int64
    L = capi.lib()
    for name in ("ldb_gpu_dict_create", "ldb_gpu_dict_count", "ldb_gpu_dict_to_table", "ldb_gpu_table_order_by_keys", "ldb_gpu_table_gather_strings"):
        assert hasattr(L, name)
    # the program descriptor keeps its layout: dictionaries travel in the existing tables list
    assert [f for f, _ in capi.ProgramDesc._fields_][9:11] == ["n_tables", "tables"]
