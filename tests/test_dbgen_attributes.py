"""dbgen.tpch(..., attributes=True): the part / partsupp / supplier / lineitem attribute columns decode back to the generator's
streams (part_attributes, balances_and_quantities, extra_columns) element for element, and the default tables do not change."""
import numpy as np

from lingodb_b200 import dbgen

SF = 0.01


def _strings(t, name):
    out = []
    for ch in t.chunks:
        offs, data = ch[name]
        out += [bytes(data[offs[i]:offs[i + 1]]).decode() for i in range(len(offs) - 1)]
    return out


def _cat(t, name):
    return np.concatenate([ch[name] for ch in t.chunks])


def test_attribute_columns_decode_to_the_generator_streams():
    t = dbgen.tpch(SF, chunk_rows=777, attributes=True)
    pa, bq = dbgen.part_attributes(SF), dbgen.balances_and_quantities(SF)
    assert [c.name for c in t["part"].columns][-5:] == ["p_mfgr", "p_brand", "p_type", "p_size", "p_container"]
    assert _strings(t["part"], "p_mfgr") == ["Manufacturer#%d" % (b // 10) for b in pa["p_brand"].tolist()]
    assert _strings(t["part"], "p_brand") == ["Brand#%d" % b for b in pa["p_brand"].tolist()]
    assert _strings(t["part"], "p_type") == [dbgen.type_name(i) for i in pa["p_type"].tolist()]
    assert _strings(t["part"], "p_container") == [f"{dbgen.CONTAINER_SYLLABLES[0][i // 8]} {dbgen.CONTAINER_SYLLABLES[1][i % 8]}" for i in pa["p_container"].tolist()]
    assert [dbgen.container_index(s) for s in _strings(t["part"], "p_container")] == pa["p_container"].tolist()
    size = _cat(t["part"], "p_size")
    assert size.dtype == np.int32 and (size == pa["p_size"]).all()
    avail = _cat(t["partsupp"], "ps_availqty")
    assert avail.dtype == np.int32 and (avail == bq["ps_availqty"]).all()
    bal = _cat(t["supplier"], "s_acctbal")
    assert bal.shape == (len(bq["s_acctbal"]), 16)
    lo, hi = bal[:, :8].copy().view(np.int64).reshape(-1), bal[:, 8:].copy().view(np.int64).reshape(-1)
    assert (lo == bq["s_acctbal"]).all() and (hi == (lo >> 63)).all()  # sign-extended decimal(12,2) cents
    assert [c for c in t["supplier"].columns if c.name == "s_acctbal"][0].precision == 12
    lkey = _cat(t["lineitem"], "l_orderkey")
    counts = np.diff(np.r_[0, np.flatnonzero(np.r_[np.diff(lkey) != 0, True]) + 1])
    x = dbgen.extra_columns(SF, counts)
    assert _strings(t["lineitem"], "l_shipinstruct") == [dbgen.SHIP_INSTRUCTIONS[i] for i in x["l_shipinstruct"].tolist()]


def test_default_tables_are_unchanged():
    plain, ext, attr = dbgen.tpch(SF), dbgen.tpch(SF, extended=True), dbgen.tpch(SF, extended=True, attributes=True)
    for name, t in plain.items():
        want = [c.name for c in ext[name].columns]
        got = [c.name for c in attr[name].columns]
        assert got[:len(want)] == want, name  # attributes only append
        for a, b in zip(plain[name].chunks, ext[name].chunks):
            for c in plain[name].columns:
                va, vb = a[c.name], b[c.name]
                if isinstance(va, tuple):
                    assert all((x == y).all() for x, y in zip(va, vb))
                else:
                    assert (va == vb).all()
    for name, t in attr.items():  # every column the default tables have is bit-identical in the attribute tables
        for a, b in zip(ext[name].chunks, t.chunks):
            for c in ext[name].columns:
                va, vb = a[c.name], b[c.name]
                if isinstance(va, tuple):
                    assert all((x == y).all() for x, y in zip(va, vb)), (name, c.name)
                else:
                    assert (va == vb).all(), (name, c.name)
    assert [c.name for c in plain["part"].columns] == ["p_partkey", "p_name"]
