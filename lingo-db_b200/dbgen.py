"""dbgen-faithful TPC-H tables (host, numpy) for the columns Q1/Q3/Q5/Q6/Q9 reference.

The reference obtains its test data by downloading and running the TPC's `dbgen` (tools/generate/tpch.sh) — impossible here
(no network), and dbgen is not under /root/reference.  This module RESTATES dbgen's published data-generation algorithm
(TPC-H tools 2.x/3.x, the same algorithm the widely used re-implementations follow) for exactly the columns the five
queries read, so that the reference's OWN expected answers (test/sqlite-datasets/tpchSf1.test) become an external pin for
the oracle and for the GPU path:

  * RNG: one Park-Miller stream per column, seed' = seed * 16807 mod (2^31 - 1), with the per-column start seeds of dbgen's
    seed table; UnifInt(lo, hi) = lo + (int) ((double) seed' / 2147483647.0 * (hi - lo + 1)).
  * Every stream is advanced by a fixed number of draws per ROW ("seeds per row"): 1 for orders/customer/supplier columns,
    7 (O_LCNT_MAX) for lineitem columns (unused draws of an order with fewer lines are skipped), 4 for partsupp, 92 for p_name.
    The k-th draw of row r is therefore stream element r * perRow + k — which is what makes the generator vectorisable.
  * o_orderkey sparse (keep 3 low bits, insert 2 zero bits); o_custkey skips multiples of 3 (+1, clamp, -1 …);
    l_suppkey / ps_suppkey by the PS_SUPPKEY formula; p_retailprice formula; l_returnflag drawn ('R','A') only for lines
    received by 1995-06-17, else 'N'; l_linestatus 'F' iff shipped by 1995-06-17; p_name = first 5 of a fresh Fisher-Yates
    pass over the 92 colours (swap position i with UnifInt(i, 91)).

Pinned by tests/test_reference_answers_sf1.py: at SF1 the oracle reproduces tpchSf1.test's Q1, Q3, Q5, Q6 and Q9 answers digit for
digit from these tables (6 001 215 lineitem rows, part 1 = "goldenrod lavender spring chocolate lace").
Plain numpy: meant for SF <= ~3 in tests, not for the SF100 bench (csrc/tpch_gen.h is the counter-based device generator).
"""
from typing import Dict

import numpy as np

from .datagen import (CUSTOMER_SCHEMA, LINEITEM_SCHEMA, ORDERS_SCHEMA, PART_SCHEMA, PARTSUPP_SCHEMA, SUPPLIER_SCHEMA, TableData, nation, region)

MODULUS, MULTIPLIER = 2147483647, 16807
EPOCH_OFFSET = 83966      # dbgen's day counter: 92001 = 1992-01-01 = epoch day 8035
MIN_DATE = 92001
CURRENT_EPOCH_DAY = 9298  # 1995-06-17
SEGMENTS = ["AUTOMOBILE", "BUILDING", "FURNITURE", "HOUSEHOLD", "MACHINERY"]
COLORS = ("almond antique aquamarine azure beige bisque black blanched blue blush brown burlywood burnished chartreuse chiffon chocolate coral "
          "cornflower cornsilk cream cyan dark deep dim dodger drab firebrick floral forest frosted gainsboro ghost goldenrod green grey honeydew "
          "hot indian ivory khaki lace lavender lawn lemon light lime linen magenta maroon medium metallic midnight mint misty moccasin navajo navy "
          "olive orange orchid pale papaya peach peru pink plum powder puff purple red rose rosy royal saddle salmon sandy seashell sienna sky slate "
          "smoke snow spring steel tan thistle tomato turquoise violet wheat white yellow").split()
# start seeds of the dbgen streams used here
SEED = {"o_orderdate": 1066728069, "o_custkey": 851767375, "o_linecount": 1434868289, "l_quantity": 209208115, "l_discount": 554590007,
        "l_tax": 721958466, "l_partkey": 1808217256, "l_suppnum": 2095021727, "l_shipdate": 1769349045, "l_commitdate": 904914315,
        "l_receiptdate": 373135028, "l_returnflag": 717419739, "c_mktsegment": 1140279430, "c_nationkey": 1489529863, "s_nationkey": 110356601,
        "p_name": 709314158, "ps_supplycost": 1051288424}

# further streams, verified against tpchSf1.test's Q4 / Q12 answers (tests/test_reference_answers_sf1.py); not yet columns of the tables
SEED.update({"o_orderpriority": 591449447, "l_shipmode": 675466456})
ORDER_PRIORITIES = ["1-URGENT", "2-HIGH", "3-MEDIUM", "4-NOT SPECIFIED", "5-LOW"]
SHIP_MODES = ["REG AIR", "AIR", "RAIL", "TRUCK", "MAIL", "FOB", "SHIP"]  # positions of MAIL and SHIP are pinned by Q12; the rest follows dists.dss

_POW = None


def stream(seed: int, n: int) -> np.ndarray:
    """The first n elements of a Park-Miller stream (element k = seed after k+1 steps), block-vectorised."""
    global _POW
    block = 1 << 16
    if _POW is None:
        p, cur = np.empty(block, dtype=np.uint64), 1
        for k in range(block):
            cur = cur * MULTIPLIER % MODULUS
            p[k] = cur
        _POW = p
    out, s = np.empty(n, dtype=np.uint64), seed
    for b in range(0, n, block):
        m = min(block, n - b)
        out[b:b + m] = (np.uint64(s) * _POW[:m]) % np.uint64(MODULUS)  # < 2^31 * 2^31: exact in uint64
        s = int(out[b + m - 1])
    return out


def unif(seeds: np.ndarray, lo: int, hi: int) -> np.ndarray:
    return lo + ((seeds.astype(np.float64) / 2147483647.0) * float(hi - lo + 1)).astype(np.int64)


def _dec128(v: np.ndarray) -> np.ndarray:
    out = np.zeros((v.shape[0], 16), dtype=np.uint8)
    out[:, :8] = np.ascontiguousarray(v.astype(np.int64)).view(np.uint8).reshape(-1, 8)
    out[:, 8:] = np.where(v < 0, 255, 0).astype(np.uint8)[:, None]
    return out


def _chunked(name, schema, cols: Dict[str, object], n: int, chunk_rows: int) -> TableData:
    t = TableData(name, schema)
    for b in range(0, n, chunk_rows):
        m = min(chunk_rows, n - b)
        chunk = {}
        for c in schema:
            v = cols[c.name]
            if c.phys == "utf8":
                offs, data = v
                chunk[c.name] = (np.ascontiguousarray(offs[b:b + m + 1] - offs[b]).astype(np.int32), np.ascontiguousarray(data[offs[b]:offs[b + m]]) if offs[b + m] > offs[b] else np.zeros(1, np.uint8))
            else:
                chunk[c.name] = np.ascontiguousarray(v[b:b + m])
        t.chunks.append(chunk)
        t.chunk_rows.append(m)
    return t


def _utf8(strings):
    data = "".join(strings).encode()
    offs = np.zeros(len(strings) + 1, dtype=np.int64)
    np.cumsum([len(s) for s in strings], out=offs[1:])
    return offs, np.frombuffer(data, dtype=np.uint8).copy()


def part_supplier(partkey: np.ndarray, j: np.ndarray, n_supp: int) -> np.ndarray:
    return (partkey + j * (n_supp // 4 + (partkey - 1) // n_supp)) % n_supp + 1


def _categorical_utf8(idx: np.ndarray, names):
    enc = [n.encode() for n in names]
    lens = np.array([len(e) for e in enc], dtype=np.int64)[idx]
    offs = np.zeros(len(idx) + 1, dtype=np.int64)
    np.cumsum(lens, out=offs[1:])
    return offs, np.frombuffer(b"".join(enc[i] for i in idx.tolist()), dtype=np.uint8).copy()


def tpch(sf: float = 1.0, chunk_rows: int = 1 << 20, extended: bool = False, attributes: bool = False) -> Dict[str, TableData]:
    """extended=True adds orders.o_orderpriority, orders.o_totalprice, lineitem.l_shipmode and customer.c_name — the columns the
    Q4 / Q12 / Q18 twins of the oracle read.  attributes=True adds part.p_mfgr / p_brand / p_type / p_container (utf8) and p_size,
    partsupp.ps_availqty, supplier.s_acctbal (decimal(12,2)) and lineitem.l_shipinstruct (utf8), from part_attributes,
    balances_and_quantities and extra_columns — the columns Q2, Q8, Q11, Q14, Q17, Q19 and Q20 read."""
    n_o, n_c, n_s, n_p = int(1500000 * sf), int(150000 * sf), int(10000 * sf), int(200000 * sf)
    # ---- orders
    idx = np.arange(1, n_o + 1, dtype=np.int64)
    okey = ((idx >> 3) << 5) | (idx & 7)
    odate = MIN_DATE + unif(stream(SEED["o_orderdate"], n_o), 0, 2557 - 151 - 1)
    ck = unif(stream(SEED["o_custkey"], n_o), 1, n_c)
    delta = np.ones(n_o, dtype=np.int64)
    while True:  # customer "mortality": keys that are multiples of 3 never order
        bad = ck % 3 == 0
        if not bad.any():
            break
        ck = np.where(bad, np.minimum(ck + delta, n_c), ck)
        delta = np.where(bad, -delta, delta)
    lcnt = unif(stream(SEED["o_linecount"], n_o), 1, 7)
    orders = {"o_orderkey": okey.astype(np.int32), "o_custkey": ck.astype(np.int32), "o_orderdate": (odate - EPOCH_OFFSET).astype(np.int32),
              "o_shippriority": np.zeros(n_o, np.int32)}
    # ---- lineitem: element (order r, line k) of a 7-per-row stream
    valid = np.arange(7)[None, :] < lcnt[:, None]

    def draws(col, lo, hi):
        return unif(stream(SEED[col], 7 * n_o), lo, hi).reshape(n_o, 7)[valid]

    def per_line(a):
        return np.repeat(a, 7).reshape(n_o, 7)[valid]

    qty, disc, tax = draws("l_quantity", 1, 50), draws("l_discount", 0, 10), draws("l_tax", 0, 8)
    pkey, snum = draws("l_partkey", 1, n_p), draws("l_suppnum", 0, 3)
    l_od = per_line(odate)
    ship = l_od + draws("l_shipdate", 1, 121)
    commit = l_od + draws("l_commitdate", 30, 90)
    receipt = ship + draws("l_receiptdate", 1, 30)
    received = np.zeros((n_o, 7), dtype=bool)
    received[valid] = receipt - EPOCH_OFFSET <= CURRENT_EPOCH_DAY
    # the flag stream is drawn only for received lines: the k-th received line of an order takes the order's k-th element
    rank = np.clip(np.cumsum(received, axis=1) - 1, 0, 6)
    flag_seed = np.take_along_axis(stream(SEED["l_returnflag"], 7 * n_o).reshape(n_o, 7), rank, axis=1)[valid]
    flag = np.where(received[valid], np.where(unif(flag_seed, 0, 1) == 0, ord("R"), ord("A")), ord("N"))
    status = np.where(ship - EPOCH_OFFSET <= CURRENT_EPOCH_DAY, ord("F"), ord("O"))
    price = 90000 + (pkey // 10) % 20001 + 100 * (pkey % 1000)
    n_l = int(valid.sum())
    lineitem = {"l_orderkey": per_line(okey).astype(np.int32), "l_partkey": pkey.astype(np.int32), "l_suppkey": part_supplier(pkey, snum, n_s).astype(np.int32),
                "l_quantity": _dec128(qty * 100), "l_extendedprice": _dec128(qty * price), "l_discount": _dec128(disc), "l_tax": _dec128(tax),
                "l_returnflag": flag.astype(np.int32), "l_linestatus": status.astype(np.int32), "l_shipdate": (ship - EPOCH_OFFSET).astype(np.int32),
                "l_commitdate": (commit - EPOCH_OFFSET).astype(np.int32), "l_receiptdate": (receipt - EPOCH_OFFSET).astype(np.int32)}
    # ---- customer / supplier
    seg = unif(stream(SEED["c_mktsegment"], n_c), 0, 4)
    customer = {"c_custkey": np.arange(1, n_c + 1, dtype=np.int32), "c_nationkey": unif(stream(SEED["c_nationkey"], n_c), 0, 24).astype(np.int32),
                "c_mktsegment": _utf8([SEGMENTS[i] for i in seg.tolist()])}
    supplier = {"s_suppkey": np.arange(1, n_s + 1, dtype=np.int32), "s_nationkey": unif(stream(SEED["s_nationkey"], n_s), 0, 24).astype(np.int32)}
    # ---- part (92 seeds per row, 5 used) / partsupp (4 per part)
    ps = stream(SEED["p_name"], 92 * n_p).reshape(n_p, 92)[:, :5].astype(np.float64) / 2147483647.0
    names = []
    for row in ps.tolist():
        words = list(range(92))  # dbgen permutes a fresh identity every row
        for pos in range(5):
            sw = pos + int(row[pos] * float(92 - pos))
            words[pos], words[sw] = words[sw], words[pos]
        names.append(" ".join(COLORS[w] for w in words[:5]))
    part = {"p_partkey": np.arange(1, n_p + 1, dtype=np.int32), "p_name": _utf8(names)}
    pp = np.repeat(np.arange(1, n_p + 1, dtype=np.int64), 4)
    jj = np.tile(np.arange(4, dtype=np.int64), n_p)
    partsupp = {"ps_partkey": pp.astype(np.int32), "ps_suppkey": part_supplier(pp, jj, n_s).astype(np.int32),
                "ps_supplycost": _dec128(unif(stream(SEED["ps_supplycost"], 4 * n_p), 100, 100000))}
    li_schema, od_schema, cu_schema = list(LINEITEM_SCHEMA), list(ORDERS_SCHEMA), list(CUSTOMER_SCHEMA)
    su_schema, pa_schema, ps_schema = list(SUPPLIER_SCHEMA), list(PART_SCHEMA), list(PARTSUPP_SCHEMA)
    if extended:
        from .datagen import ColumnSpec
        x = extra_columns(sf, lcnt)
        orders["o_orderpriority"] = _categorical_utf8(x["o_orderpriority"], ORDER_PRIORITIES)
        lineitem["l_shipmode"] = _categorical_utf8(x["l_shipmode"], SHIP_MODES)
        od_schema.append(ColumnSpec("o_orderpriority", "utf8"))
        li_schema.append(ColumnSpec("l_shipmode", "utf8"))
        # o_totalprice = sum over the order's lines of ((eprice * (100 - disc)) / 100) * (100 + tax) / 100, integer cents (dbgen mk_order);
        # pinned by Q18's answer rows
        line_total = ((qty * price) * (100 - disc) // 100) * (100 + tax) // 100
        total = np.zeros(n_o, dtype=np.int64)
        np.add.at(total, np.repeat(np.arange(n_o), lcnt), line_total)
        orders["o_totalprice"] = _dec128(total)
        od_schema.append(ColumnSpec("o_totalprice", "decimal128", 12, 2))
        customer["c_name"] = _utf8(["Customer#%09d" % k for k in range(1, n_c + 1)])
        cu_schema.append(ColumnSpec("c_name", "utf8"))
    if attributes:
        from .datagen import ColumnSpec
        pa, bq = part_attributes(sf), balances_and_quantities(sf)
        part["p_mfgr"] = _utf8(["Manufacturer#%d" % (b // 10) for b in pa["p_brand"].tolist()])
        part["p_brand"] = _utf8(["Brand#%d" % b for b in pa["p_brand"].tolist()])
        part["p_type"] = _categorical_utf8(pa["p_type"], [type_name(i) for i in range(150)])
        part["p_size"] = pa["p_size"]
        part["p_container"] = _categorical_utf8(pa["p_container"], [f"{a} {b}" for a in CONTAINER_SYLLABLES[0] for b in CONTAINER_SYLLABLES[1]])
        pa_schema += [ColumnSpec("p_mfgr", "utf8"), ColumnSpec("p_brand", "utf8"), ColumnSpec("p_type", "utf8"), ColumnSpec("p_size", "int32"), ColumnSpec("p_container", "utf8")]
        partsupp["ps_availqty"] = bq["ps_availqty"].astype(np.int32)
        ps_schema.append(ColumnSpec("ps_availqty", "int32"))
        supplier["s_acctbal"] = _dec128(bq["s_acctbal"])
        su_schema.append(ColumnSpec("s_acctbal", "decimal128", 12, 2))
        lineitem["l_shipinstruct"] = _categorical_utf8(extra_columns(sf, lcnt)["l_shipinstruct"], SHIP_INSTRUCTIONS)
        li_schema.append(ColumnSpec("l_shipinstruct", "utf8"))
    return {"lineitem": _chunked("lineitem", li_schema, lineitem, n_l, chunk_rows), "orders": _chunked("orders", od_schema, orders, n_o, chunk_rows),
            "customer": _chunked("customer", cu_schema, customer, n_c, chunk_rows), "supplier": _chunked("supplier", su_schema, supplier, n_s, chunk_rows),
            "part": _chunked("part", pa_schema, part, n_p, chunk_rows), "partsupp": _chunked("partsupp", ps_schema, partsupp, 4 * n_p, chunk_rows),
            "nation": nation(), "region": region()}


def extra_columns(sf: float, line_counts: np.ndarray) -> Dict[str, np.ndarray]:
    """o_orderpriority (index into ORDER_PRIORITIES, per order) and l_shipmode (index into SHIP_MODES, per lineitem row) —
    the next columns a widening to Q4 / Q12 needs.  line_counts = lines per order (e.g. from the compiled twin)."""
    n_o = int(1500000 * sf)
    valid = np.arange(7)[None, :] < line_counts[:, None]
    return {"o_orderpriority": unif(stream(SEED["o_orderpriority"], n_o), 0, 4).astype(np.int32),
            "l_shipmode": unif(stream(SEED["l_shipmode"], 7 * n_o), 0, 6).reshape(n_o, 7)[valid].astype(np.int32),
            "l_shipinstruct": unif(stream(SEED["l_shipinstruct"], 7 * n_o), 0, 3).reshape(n_o, 7)[valid].astype(np.int32)}


# part attributes and l_shipinstruct: the streams and distributions behind Q14 / Q17 / Q19 (pinned by tpchSf1.test's answers to those queries,
# tests/test_reference_answers_sf1.py); one draw per part row each, pick_str index = UnifInt(1, count) - 1 over dists.dss' lists
SEED.update({"p_mfgr": 1, "p_brand": 46831694, "p_type": 1841581359, "p_size": 1193163244, "p_container": 727633698, "l_shipinstruct": 1371272478})
TYPE_SYLLABLES = (["STANDARD", "SMALL", "MEDIUM", "LARGE", "ECONOMY", "PROMO"], ["ANODIZED", "BURNISHED", "PLATED", "POLISHED", "BRUSHED"], ["TIN", "NICKEL", "BRASS", "STEEL", "COPPER"])
CONTAINER_SYLLABLES = (["SM", "LG", "MED", "JUMBO", "WRAP"], ["CASE", "BOX", "BAG", "JAR", "PKG", "PACK", "CAN", "DRUM"])
SHIP_INSTRUCTIONS = ["DELIVER IN PERSON", "COLLECT COD", "NONE", "TAKE BACK RETURN"]  # position of DELIVER IN PERSON pinned by Q19


def part_attributes(sf: float) -> Dict[str, np.ndarray]:
    """Per part (row p_partkey - 1): p_brand as the two-digit number of 'Brand#MN', p_type as an index into the 150 three-syllable types
    (first syllable = index // 25 — the level Q14's LIKE 'PROMO%' pins; the order of the inner syllables follows the TPC-H specification's
    lists), p_size, p_container as index // 8 = first and index % 8 = second syllable of CONTAINER_SYLLABLES."""
    n_p = int(200000 * sf)
    mfgr = unif(stream(SEED["p_mfgr"], n_p), 1, 5)
    return {"p_brand": (mfgr * 10 + unif(stream(SEED["p_brand"], n_p), 1, 5)).astype(np.int32), "p_type": (unif(stream(SEED["p_type"], n_p), 1, 150) - 1).astype(np.int32),
            "p_size": unif(stream(SEED["p_size"], n_p), 1, 50).astype(np.int32), "p_container": (unif(stream(SEED["p_container"], n_p), 1, 40) - 1).astype(np.int32)}


# account balances and available quantities (UnifInt in cents / units, one draw per row; 4 per part for partsupp): pinned by Q2 / Q11 / Q20 / Q22.
# The country code of c_phone is 10 + c_nationkey (dbgen gen_phone), so Q22's substring(c_phone, 1, 2) needs no further stream.
SEED.update({"ps_availqty": 1671059989, "c_acctbal": 298370230, "s_acctbal": 962338209})


def balances_and_quantities(sf: float) -> Dict[str, np.ndarray]:
    n_c, n_s, n_p = int(150000 * sf), int(10000 * sf), int(200000 * sf)
    return {"c_acctbal": unif(stream(SEED["c_acctbal"], n_c), -99999, 999999), "s_acctbal": unif(stream(SEED["s_acctbal"], n_s), -99999, 999999),
            "ps_availqty": unif(stream(SEED["ps_availqty"], 4 * n_p), 1, 9999)}


# suppliers whose comment carries "Customer … Complaints" (dbgen mk_supp: one supplier in a thousand gets a Better-Business-Bureau remark,
# half of them complaints): drawn from two streams of their own, so Q16's NOT IN needs no generated text
SEED.update({"s_bbb_comment": 202794285, "s_bbb_type": 753643799})


def complaint_suppliers(sf: float) -> np.ndarray:
    n_s = int(10000 * sf)
    bad_press, kind = unif(stream(SEED["s_bbb_comment"], n_s), 1, 10000), unif(stream(SEED["s_bbb_type"], n_s), 0, 100)
    return (np.flatnonzero((bad_press <= 10) & (kind < 50)) + 1).astype(np.int32)


def type_name(index: int) -> str:
    a, b, c = TYPE_SYLLABLES
    return f"{a[index // 25]} {b[index // 5 % 5]} {c[index % 5]}"


def container_index(name: str) -> int:
    a, b = name.split()
    return CONTAINER_SYLLABLES[0].index(a) * 8 + CONTAINER_SYLLABLES[1].index(b)


# ---------------------------------------------------------------------------------------------------------------------
# compiled twin (csrc/dbgen_gen.h through libldb_datagen_host.so): same tables, random access, multi-threaded — and the
# code the device generator shares.  tests/test_datagen.py checks it against the numpy version above.
def scale_compiled(sf: float, count_lines: bool = True):
    import ctypes as C

    from . import datagen
    L = datagen.lib()
    L.ldbgen_dbgen_scale.argtypes = [C.c_double, C.c_int32, C.POINTER(datagen.GenScale)]
    s = datagen.GenScale()
    L.ldbgen_dbgen_scale(float(sf), int(count_lines), C.byref(s))
    return s


def tpch_compiled(sf: float = 1.0, chunk_rows: int = 1 << 20) -> Dict[str, TableData]:
    import ctypes as C

    from . import datagen
    L = datagen.lib()
    G = C.POINTER(datagen.GenScale)
    L.ldbgen_dbgen_line_counts_host.argtypes = [G, C.c_int64, C.c_int64, C.c_void_p]
    L.ldbgen_dbgen_lineitem_host.argtypes = [G, C.c_int64, C.c_int64, C.c_void_p, C.POINTER(datagen.LineitemCols)]
    L.ldbgen_dbgen_orders_host.argtypes = [G, C.c_int64, C.c_int64, C.POINTER(datagen.OrdersCols)]
    L.ldbgen_dbgen_customer_host.restype = C.c_int64
    L.ldbgen_dbgen_customer_host.argtypes = [G, C.c_int64, C.c_int64, C.POINTER(datagen.CustomerCols)]
    L.ldbgen_dbgen_supplier_host.argtypes = [G, C.c_int64, C.c_int64, C.POINTER(datagen.SupplierCols)]
    L.ldbgen_dbgen_part_host.restype = C.c_int64
    L.ldbgen_dbgen_part_host.argtypes = [G, C.c_int64, C.c_int64, C.POINTER(datagen.PartCols)]
    L.ldbgen_dbgen_partsupp_host.argtypes = [G, C.c_int64, C.c_int64, C.POINTER(datagen.PartsuppCols)]
    s = scale_compiled(sf)
    ptr = datagen._ptr
    n_o = s.n_orders
    counts = np.zeros(n_o, np.int32)
    L.ldbgen_dbgen_line_counts_host(C.byref(s), 0, n_o, ptr(counts))
    first = np.zeros(n_o + 1, np.int64)
    np.cumsum(counts, out=first[1:])
    n_l = int(first[-1])
    assert n_l == s.n_lineitem
    li = {c.name: datagen._alloc(c, n_l) for c in LINEITEM_SCHEMA}
    L.ldbgen_dbgen_lineitem_host(C.byref(s), 0, n_o, ptr(first), C.byref(datagen.LineitemCols(**{k: ptr(v) for k, v in li.items()})))
    od = {c.name: datagen._alloc(c, n_o) for c in ORDERS_SCHEMA}
    L.ldbgen_dbgen_orders_host(C.byref(s), 0, n_o, C.byref(datagen.OrdersCols(**{k: ptr(v) for k, v in od.items()})))

    def utf8(fn, cols_cls, n, fixed):
        offs = np.zeros(n + 1, np.int32)
        nbytes = fn(C.byref(s), 0, n, C.byref(cols_cls(*[ptr(a) for a in fixed], ptr(offs), None)))
        data = np.zeros(max(1, nbytes), np.uint8)
        fn(C.byref(s), 0, n, C.byref(cols_cls(*[None for _ in fixed], None, ptr(data))))
        return offs.astype(np.int64), data

    ck, cn = np.zeros(s.n_customer, np.int32), np.zeros(s.n_customer, np.int32)
    cu = {"c_custkey": ck, "c_nationkey": cn, "c_mktsegment": utf8(L.ldbgen_dbgen_customer_host, datagen.CustomerCols, s.n_customer, [ck, cn])}
    su = {c.name: datagen._alloc(c, s.n_supplier) for c in SUPPLIER_SCHEMA}
    L.ldbgen_dbgen_supplier_host(C.byref(s), 0, s.n_supplier, C.byref(datagen.SupplierCols(**{k: ptr(v) for k, v in su.items()})))
    pk = np.zeros(s.n_part, np.int32)
    pa = {"p_partkey": pk, "p_name": utf8(L.ldbgen_dbgen_part_host, datagen.PartCols, s.n_part, [pk])}
    ps = {c.name: datagen._alloc(c, 4 * s.n_part) for c in PARTSUPP_SCHEMA}
    L.ldbgen_dbgen_partsupp_host(C.byref(s), 0, 4 * s.n_part, C.byref(datagen.PartsuppCols(**{k: ptr(v) for k, v in ps.items()})))
    return {"lineitem": _chunked("lineitem", LINEITEM_SCHEMA, li, n_l, chunk_rows), "orders": _chunked("orders", ORDERS_SCHEMA, od, n_o, chunk_rows),
            "customer": _chunked("customer", CUSTOMER_SCHEMA, cu, s.n_customer, chunk_rows), "supplier": _chunked("supplier", SUPPLIER_SCHEMA, su, s.n_supplier, chunk_rows),
            "part": _chunked("part", PART_SCHEMA, pa, s.n_part, chunk_rows), "partsupp": _chunked("partsupp", PARTSUPP_SCHEMA, ps, 4 * s.n_part, chunk_rows),
            "nation": nation(), "region": region()}
