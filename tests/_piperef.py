"""Exact reference for the specialised scan pipelines (LdbPipelineDesc, include/ldb_gpu.h: K1/K2 scan → reduce / group-by, K3 join
build, K4 probe-probe-group, K5 probe into a group-join map + top-k, K8 materialize, K9 star probe) — plain Python, no GPU.

Written from the header's contract, restated:
  - filters are a conjunction.  int32, date32 and fsb4 compare as int32 (an fsb4 constant is its bytes read little-endian, a date
    constant "YYYY-MM-DD" is days since 1970-01-01); a decimal(p<19) compares its low 64 bits, signed, with the constant at the
    column's scale (an integer constant is multiplied by 10^scale; a constant beyond 64 bits is LDB_ERR_UNSUPPORTED); utf8 = / <>
    compare bytewise and CONTAINS is a substring test (an empty needle matches every string); IN holds 1..8 values; NOTNULL is
    always true.  At most 4 filter entries, where a second compare on a column joins the first one as its range bound;
  - aggregates (`one` = 100, the 10^scale of decimal(12,2)): COL and ONE wrap at 64 bits and are read back sign-extended; MUL,
    MUL_1MINUS, MUL_1MINUS_1PLUS and MUL_1MINUS_MINUS_PAYMUL are computed exactly, then wrapped at 128 bits;
  - join tables are multimaps (a unique table rejects a duplicate key; a direct table rejects keys outside its range and duplicates);
    the pair (key -1, payload -1) cannot be stored (a direct table: the payload 0x80808080), nor can a negative payload in a table
    with side or aggregate lanes ("wide").  A hash or pair table is full when it holds as many entries as its directory has slots
    (modelled for directories of at most 16 384 slots).  Probes of a wide table ignore bit 31 of the payload, the group-join marker.
    A group-join map's aggregate lane keeps the width (64 / 128 bits) of its first probe-aggregate;
  - K4 keeps a row only when the two payloads agree; K5's top-k orders (agg desc, side0 asc, key asc) over the entries that were
    probed at least once; K9 groups (payload 1, payload 2) and sums a * (1 - b) - $payload0 * c.
Errors raise PipeError with the LdbStatus the C-ABI reports."""
import datetime
from typing import Dict, List, Optional, Sequence

import numpy as np

import _progref as R
from _progref import I32_MAX, I32_MIN, I64_MAX, I64_MIN, wrap128

LDB_ERR_UNSUPPORTED, LDB_ERR_INVALID, LDB_ERR_CAPACITY = 2, 3, 4
ONE = 100
M64 = (1 << 64) - 1
DIRECT_EMPTY = -0x7F7F7F80  # 0x80808080 as int32
MAX_SLOTS = 16384  # the largest hash / pair table whose overflow the reference models (JoinTable)


class PipeError(Exception):
    def __init__(self, code: int, what: str):
        super().__init__(f"[{code}] {what}")
        self.code = code


def wrap64(v: int) -> int:
    v &= M64
    return v - (1 << 64) if v >> 63 else v


# ---------------------------------------------------------------------------------------------------- reference hash
def h64(keys) -> np.ndarray:
    """util.hash_64 of int32 keys (sign-extended to 64 bits): m = k * 0x9E3779B97F4A7C55, m ^ bswap(m) — vectorised"""
    k = np.asarray(keys, dtype=np.int64).astype(np.uint64)
    with np.errstate(over="ignore"):
        m = k * np.uint64(0x9E3779B97F4A7C55)
    return m ^ m.byteswap()


def colliding_keys(low_bits: int, target: int, count: int, start: int = -(1 << 31), step: int = 1 << 22) -> List[int]:
    """`count` int32 keys whose h64 has `target` in its low `low_bits` bits (they share a directory slot in any table of at most
    2^low_bits slots), searched block by block from `start`"""
    out: List[int] = []
    lo = start
    mask = np.uint64((1 << low_bits) - 1)
    while len(out) < count and lo <= I32_MAX:
        hi = min(lo + step, I32_MAX + 1)
        ks = np.arange(lo, hi, dtype=np.int64)
        hit = ks[(h64(ks) & mask) == np.uint64(target)]
        out.extend(int(x) for x in hit[: count - len(out)])
        lo = hi
    return out


def table_slots(expected_rows: int) -> int:
    """directory slots of ldb_gpu_join_table_create / _create_pair: nextPow2(2 * max(expected, 8))"""
    n = max(expected_rows, 8) * 2
    return 1 << (n - 1).bit_length()


def group_slots(capacity: int) -> int:
    """groups a ldb_gpu_groupby_create state holds: nextPow2(max(capacity, 16))"""
    n = max(capacity, 16)
    return 1 << (n - 1).bit_length()


# ---------------------------------------------------------------------------------------------------- tables
# (name, phys, precision, scale): the types the specialised pipelines accept
PIPE_COLUMNS = [("k", "int32", 0, 0), ("i", "int32", 0, 0), ("dt", "date32", 0, 0), ("fs", "fsb4", 0, 0), ("a", "decimal128", 18, 2),
                ("b", "decimal128", 18, 2), ("c", "decimal128", 18, 2), ("s", "utf8", 0, 0)]


def gen_table(seed: int, n: int, columns=PIPE_COLUMNS, key_domain: int = 16) -> Dict[str, list]:
    """seeded values without NULLs (the generator of _progref); decimals are kept inside their declared precision"""
    vals = R.gen_values(seed, n, columns, null_rate=0.0, key_domain=key_domain)
    for name, phys, prec, _ in columns:
        zero = b"" if phys == "utf8" else 0
        vals[name] = [zero if v is None else v for v in vals[name]]  # the generator's one NULL per column
        if phys == "decimal128":
            lim = 10**prec - 1
            vals[name] = [v if -lim <= v <= lim else (v % lim if v > 0 else -(-v % lim)) for v in vals[name]]
    return vals


def schema_of(columns=PIPE_COLUMNS) -> Dict[str, tuple]:
    return {n: (p, pr, sc) for n, p, pr, sc in columns}


# ---------------------------------------------------------------------------------------------------- filters
_OPS = {"=": lambda x, c: x == c, "!=": lambda x, c: x != c, "<": lambda x, c: x < c, "<=": lambda x, c: x <= c,
        ">": lambda x, c: x > c, ">=": lambda x, c: x >= c}


def date32(s: str) -> int:
    return (datetime.date.fromisoformat(s) - datetime.date(1970, 1, 1)).days


def decimal_const(s: str, scale: int) -> int:
    neg = s.startswith("-")
    t = s.lstrip("+-")
    whole, _, frac = t.partition(".")
    if len(frac) > scale and int(frac[scale:] or 0):
        raise PipeError(LDB_ERR_INVALID, "decimal rescale would lose data")
    v = int((whole or "0") + (frac[:scale] if len(frac) >= scale else frac.ljust(scale, "0")))
    if v > I64_MAX:
        raise PipeError(LDB_ERR_UNSUPPORTED, "decimal constant beyond 64 bits")
    return -v if neg else v


def constant(schema: Dict[str, tuple], col: str, value):
    """a filter constant typed by the column (str or int as LdbFilterDesc carries it)"""
    phys, prec, scale = schema[col]
    if phys == "int32":
        if not isinstance(value, int):
            raise PipeError(LDB_ERR_INVALID, "integer column needs an integer constant")
        return value
    if phys == "date32":
        if not isinstance(value, str):
            raise PipeError(LDB_ERR_INVALID, "could not parse date")
        return date32(value)
    if phys == "fsb4":
        if not isinstance(value, str) or len(value.encode()) > 4:
            raise PipeError(LDB_ERR_INVALID, "char(1) constant too long")
        return int.from_bytes(value.encode().ljust(4, b"\0"), "little", signed=True)
    if phys == "decimal128":
        if prec >= 19:
            raise PipeError(LDB_ERR_UNSUPPORTED, "decimal precision >= 19")
        if isinstance(value, str):
            return decimal_const(value, scale)
        v = value * 10**scale
        if not I64_MIN <= v <= I64_MAX:
            raise PipeError(LDB_ERR_UNSUPPORTED, "decimal constant beyond 64 bits")
        return v
    raise PipeError(LDB_ERR_UNSUPPORTED, "unsupported type in filter")


def filter_rows(cols: Dict[str, list], schema: Dict[str, tuple], filters: Sequence[tuple]) -> List[bool]:
    """filters: (column, op, value) as runtime.run_pipeline takes them; op in = != < <= > >= notnull in contains"""
    n = len(next(iter(cols.values())))
    keep = [True] * n
    entries: List[tuple] = []  # (column, merged-range?) as the host plans them: at most 4
    for col, op, val in filters:
        if col not in schema:
            raise PipeError(LDB_ERR_INVALID, "unknown column in filter")
        phys = schema[col][0]
        if op == "notnull":
            continue
        vs = cols[col]
        if phys == "decimal128":
            vs = [wrap64(v) for v in vs]  # the low 64 bits, signed
        if op == "in":
            if phys == "utf8":
                raise PipeError(LDB_ERR_UNSUPPORTED, "IN over strings")
            if not 1 <= len(val) <= 8:
                raise PipeError(LDB_ERR_UNSUPPORTED, "IN lists hold 1..8 values")
            if len(entries) == 4:
                raise PipeError(LDB_ERR_UNSUPPORTED, "more than 4 filter columns")
            cs = {constant(schema, col, x) for x in val}
            entries.append((col, "in"))
            pred = lambda x, cs=cs: x in cs
        elif phys == "utf8":
            if op not in ("=", "!=", "contains"):
                raise PipeError(LDB_ERR_UNSUPPORTED, "unsupported filter op for string")
            if not isinstance(val, str) or len(val.encode()) > 24:
                raise PipeError(LDB_ERR_UNSUPPORTED, "string constant longer than 24 bytes")
            if len(entries) == 4:
                raise PipeError(LDB_ERR_UNSUPPORTED, "more than 4 filter columns")
            entries.append((col, "str"))
            needle = val.encode()
            pred = (lambda s, p=needle: p in s) if op == "contains" else (lambda s, p=needle, f=_OPS[op]: f(s, p))
        else:
            if op == "contains":
                raise PipeError(LDB_ERR_UNSUPPORTED, "LIKE-contains needs a utf8 column")
            if op not in _OPS:
                raise PipeError(LDB_ERR_UNSUPPORTED, "unsupported filter op")
            c = constant(schema, col, val)
            if (col, "open") in entries:
                entries[entries.index((col, "open"))] = (col, "range")
            else:
                if len(entries) == 4:
                    raise PipeError(LDB_ERR_UNSUPPORTED, "more than 4 filter columns")
                entries.append((col, "open"))
            pred = lambda x, c=c, f=_OPS[op]: f(x, c)
        keep = [k and pred(v) for k, v in zip(keep, vs)]
    return keep


# ---------------------------------------------------------------------------------------------------- aggregates
EXPR_COLS = {"col": 1, "mul": 2, "mul_1minus": 2, "mul_1minus_1plus": 3, "one": 0}
IS64 = ("col", "one")

# the signatures launchScanGroupBy compiles: (number of keys, aggregate list with operand positions over the value columns)
SIGNATURES = [
    (2, [("col", [0]), ("col", [1]), ("mul_1minus", [1, 2]), ("mul_1minus_1plus", [1, 2, 3]), ("col", [2]), ("one", [])]),  # Q1
    (1, [("col", [0]), ("col", [1]), ("mul_1minus", [1, 2]), ("mul_1minus_1plus", [1, 2, 3]), ("col", [2]), ("one", [])]),
    (0, [("mul", [0, 1])]),  # Q6
    (0, [("mul_1minus", [0, 1])]),
    (0, [("col", [0]), ("one", [])]),
    (1, [("mul_1minus", [0, 1])]),
    (2, [("mul_1minus", [0, 1])]),
    (1, [("col", [0]), ("one", [])]),
    (2, [("col", [0]), ("one", [])]),
]


def agg_term(expr: str, a: int = 0, b: int = 0, c: int = 0, pay: int = 0, d: int = 0) -> int:
    """one row's contribution, exact (operands are the low 64 bits of decimal(p<19, 2) cells)"""
    if expr == "col":
        return a
    if expr == "one":
        return 1
    if expr == "mul":
        return a * b
    if expr == "mul_1minus":
        return a * (ONE - b)
    if expr == "mul_1minus_1plus":
        return a * (ONE - b) * (ONE + c)
    if expr == "mul_1minus_minus_paymul":
        return a * (ONE - b) - pay * d
    raise PipeError(LDB_ERR_UNSUPPORTED, "unknown aggregate expression kind")


def finish_sum(expr: str, total: int) -> int:
    return wrap64(total) if expr in IS64 else wrap128(total)


def _agg_operands(cols, schema, aggs):
    for expr, names in aggs:
        if expr not in EXPR_COLS:
            raise PipeError(LDB_ERR_UNSUPPORTED, "unknown aggregate expression kind")
        for name in names[: EXPR_COLS[expr]]:
            if name not in schema or schema[name][0] != "decimal128":
                raise PipeError(LDB_ERR_UNSUPPORTED if name in schema else LDB_ERR_INVALID, "aggregate operand")
            if schema[name][1] >= 19 or schema[name][2] != 2:
                raise PipeError(LDB_ERR_UNSUPPORTED, "aggregate operands must be decimal(p<19, 2)")


def signature_of(n_keys: int, aggs) -> tuple:
    """(n_keys, aggregates with operand positions in first-appearance order): what launchScanGroupBy dispatches on"""
    order: List[str] = []
    out = []
    for expr, names in aggs:
        pos = []
        for name in names[: EXPR_COLS[expr]]:
            if name not in order:
                order.append(name)
            pos.append(order.index(name))
        out.append((expr, pos))
    return n_keys, out


def _row_terms(cols, i, aggs):
    return [agg_term(expr, *[wrap64(cols[c][i]) for c in names[: EXPR_COLS[expr]]]) for expr, names in aggs]


def scan_groupby(cols, schema, filters, keys: Sequence[str], aggs, capacity: int = 64) -> Dict[tuple, list]:
    """K1 (no keys: the one group () over zero or more rows) and K2: {(k0, k1): [sums]} (a single key pads k1 = 0)"""
    keep = filter_rows(cols, schema, filters)
    _agg_operands(cols, schema, aggs)
    for k in keys:
        if k not in schema:
            raise PipeError(LDB_ERR_INVALID, "unknown column for group key")
        if schema[k][0] not in ("int32", "date32", "fsb4"):
            raise PipeError(LDB_ERR_UNSUPPORTED, "group key type")
    sig = signature_of(len(keys), aggs)
    if sig not in [(nk, [(e, list(p)) for e, p in a]) for nk, a in SIGNATURES]:
        raise PipeError(LDB_ERR_UNSUPPORTED, "no compiled group-by pipeline for this aggregate signature")
    sums: Dict[tuple, list] = {} if keys else {(): [0] * len(aggs)}
    for i, ok in enumerate(keep):
        if not ok:
            continue
        g = tuple(cols[k][i] for k in keys)
        acc = sums.setdefault(g, [0] * len(aggs))
        for j, t in enumerate(_row_terms(cols, i, aggs)):
            acc[j] += t
    if keys and len(sums) > group_slots(capacity):
        raise PipeError(LDB_ERR_CAPACITY, "group-by table overflow")
    out = {}
    for g, acc in sums.items():
        key = (g + (0,) * 2)[:2] if keys else ()
        out[key] = [finish_sum(expr, v) for (expr, _), v in zip(aggs, acc)]
    return out


# ---------------------------------------------------------------------------------------------------- join tables
class JoinTable:
    """A join table as a multimap in insertion order.  kind: "hash" (ldb_gpu_join_table_create), "pair" (composite key → int64
    payload) or "direct" (dense unique keys in [key_min, key_max]).  Entries: [key, payload, side0, side1, agg, marked]; a pair
    table's key is the tuple (k0, k1).  `error` holds the first failure of a build (the C-ABI raises it at the next read)."""

    def __init__(self, kind="hash", expected_rows=1024, unique=True, n_side=0, n_aggs=0, key_min=0, key_max=0):
        self.kind, self.unique, self.n_side, self.n_aggs = kind, unique or kind == "direct", n_side, n_aggs
        self.key_min, self.key_max = key_min, key_max
        self.slots = table_slots(expected_rows) if kind != "direct" else key_max - key_min + 1
        if kind != "direct" and self.slots > MAX_SLOTS:
            # a table is full when it holds as many entries as slots; in a larger directory an insert fails earlier, once its probe
            # run passes 16 384 slots, and where that happens depends on the order of the concurrent inserts: not modelled
            raise ValueError("the reference models hash tables of at most 16384 slots")
        self.entries: List[list] = []
        self._keys: set = set()
        self.error: Optional[PipeError] = None
        self.agg64: Optional[bool] = None  # the width of the aggregate lane, fixed by the first probe-aggregate

    @property
    def wide(self) -> bool:
        return self.n_side > 0 or self.n_aggs > 0

    def _fail(self, code, what):
        if self.error is None:
            self.error = PipeError(code, what)

    def insert(self, key, payload: int, side0: int = 0, side1: int = 0):
        if self.kind == "direct":
            if not self.key_min <= key <= self.key_max:
                return self._fail(LDB_ERR_INVALID, "key outside the declared range of a direct-address table")
            if payload == DIRECT_EMPTY:
                return self._fail(LDB_ERR_UNSUPPORTED, "the direct-address empty marker cannot be stored")
        elif self.kind == "pair":
            if key == (-1, -1):
                return self._fail(LDB_ERR_UNSUPPORTED, "the pair (-1, -1) cannot be stored")
        else:
            if key == -1 and payload == -1:
                return self._fail(LDB_ERR_UNSUPPORTED, "the pair (key=-1, payload=-1) cannot be stored")
            if self.wide and payload < 0:
                return self._fail(LDB_ERR_UNSUPPORTED, "tables with side/aggregate lanes need non-negative payloads")
        if self.unique and key in self._keys:
            return self._fail(LDB_ERR_INVALID, "duplicate key in a unique join table")
        if self.kind != "direct" and len(self.entries) >= self.slots:
            return self._fail(LDB_ERR_CAPACITY, "join table full")
        self._keys.add(key)
        self.entries.append([key, payload, side0, side1, 0, False])

    def index(self) -> Dict[object, List[list]]:
        d: Dict[object, List[list]] = {}
        for e in self.entries:
            d.setdefault(e[0], []).append(e)
        if self.unique:
            d = {k: v[:1] for k, v in d.items()}
        return d

    def count(self) -> int:
        if self.error is not None:
            raise self.error
        return len(self.entries)

    def multimap(self) -> Dict[object, List[int]]:
        """{key: sorted payloads}: what a $payload materialize of every key reads back"""
        d: Dict[object, List[int]] = {}
        for e in self.entries:
            d.setdefault(e[0], []).append(e[1])
        return {k: sorted(v) for k, v in d.items()}


def _key_col(schema, name, role):
    if name not in schema:
        raise PipeError(LDB_ERR_INVALID, f"unknown column for {role}")
    if schema[name][0] not in ("int32", "date32", "fsb4"):
        raise PipeError(LDB_ERR_UNSUPPORTED, f"unsupported type for {role}")


def scan_build(cols, schema, filters, sink: JoinTable, key: str, payload: Optional[str] = None, payload_expr: str = "column",
               side: Sequence[str] = (), probe: Optional[tuple] = None, key2: Optional[str] = None):
    """K3: every row that passes the filters (and, with probe = (table, key column), once per match of its probe key) inserts
    {key, payload, side...}.  payload: the column's value, its year (payload_expr "year", a date32 column), else the probe's
    payload (bit 31 cleared for a wide probe table), else 0."""
    keep = filter_rows(cols, schema, filters)
    _key_col(schema, key, "build key")
    if len(side) != sink.n_side:
        raise PipeError(LDB_ERR_INVALID, "side column count differs from the table's")
    if (sink.kind == "pair") != (key2 is not None):
        raise PipeError(LDB_ERR_INVALID, "a second build key goes with a composite-key table")
    if payload_expr == "year" and (sink.kind == "pair" or payload is None or schema[payload][0] != "date32"):
        raise PipeError(LDB_ERR_UNSUPPORTED, "year payloads come from a date32 column of a single-key build")
    pidx = probe[0].index() if probe else None
    for i, ok in enumerate(keep):
        if not ok:
            continue
        k = (cols[key][i], cols[key2][i]) if key2 else cols[key][i]
        s = [cols[c][i] for c in side] + [0, 0]
        if payload is not None:
            own = cols[payload][i]
            if sink.kind == "pair" and schema[payload][0] == "decimal128":
                own = wrap64(own)
            elif payload_expr == "year":
                own = R.year_of_days(own)
        if probe is None:
            sink.insert(k, own if payload is not None else 0, s[0], s[1])
            continue
        for e in pidx.get(cols[probe[1]][i], []):
            p = own if payload is not None else (e[1] & 0x7FFFFFFF if probe[0].wide else e[1])
            sink.insert(k, p, s[0], s[1])


def probe_agg(cols, schema, filters, table: JoinTable, key: str, agg: tuple):
    """K5: every row that passes the filters adds its aggregate term into each entry its key visits and marks it"""
    if not table.n_aggs:
        raise PipeError(LDB_ERR_INVALID, "join table was created without aggregate lanes")
    keep = filter_rows(cols, schema, filters)
    _agg_operands(cols, schema, [agg])
    expr, names = agg
    if table.agg64 is not None and table.agg64 != (expr in IS64):
        raise PipeError(LDB_ERR_UNSUPPORTED, "64-bit and 128-bit sums cannot share an aggregate lane")
    table.agg64 = expr in IS64
    idx = table.index()
    for i, ok in enumerate(keep):
        if not ok:
            continue
        hits = idx.get(cols[key][i], [])
        if hits:
            t = _row_terms(cols, i, [agg])[0]
            for e in hits:
                e[4] += t
                e[5] = True


def topk(table: JoinTable, k: int) -> List[tuple]:
    """ldb_gpu_join_table_topk: (key, side0, side1, agg) of the marked entries by (agg desc, side0 asc, key asc), first k"""
    if table.error is not None:
        raise table.error
    if not 1 <= k <= 64:
        raise PipeError(LDB_ERR_INVALID, "k must be in [1, 64]")
    rows = [(e[0], e[2], e[3], wrap64(e[4]) if table.agg64 else wrap128(e[4])) for e in table.entries if e[5]]
    rows.sort(key=lambda r: (-r[3], r[1], r[0]))
    return rows[:k]


def probe2_groupby(cols, schema, filters, table_a: JoinTable, key_a: str, table_b: JoinTable, key_b: str, agg: tuple,
                   capacity: int = 64) -> Dict[tuple, list]:
    """K4: each (match in A, match in B) pair whose payloads agree adds the row's term to the group of that payload"""
    keep = filter_rows(cols, schema, filters)
    _agg_operands(cols, schema, [agg])
    ia, ib = table_a.index(), table_b.index()
    sums: Dict[tuple, int] = {}
    for i, ok in enumerate(keep):
        if not ok:
            continue
        for ea in ia.get(cols[key_a][i], []):
            for eb in ib.get(cols[key_b][i], []):
                pa = ea[1] & 0x7FFFFFFF if table_a.wide else ea[1]
                pb = eb[1] & 0x7FFFFFFF if table_b.wide else eb[1]
                if pa != pb:
                    continue
                g = (pb, 0)
                sums[g] = sums.get(g, 0) + _row_terms(cols, i, [agg])[0]
    if len(sums) > group_slots(capacity):
        raise PipeError(LDB_ERR_CAPACITY, "group-by table overflow")
    return {g: [finish_sum(agg[0], v)] for g, v in sums.items()}


def materialize(cols, schema, filters, out_columns: Sequence[str], probe: Optional[tuple] = None) -> List[tuple]:
    """K8: one tuple per row that passes the filters (per match of its probe key with a probe); "$payload" = the match's payload
    (bit 31 cleared for a wide table), a decimal column = its full cell.  The order of the tuples is not specified."""
    keep = filter_rows(cols, schema, filters)
    out = []
    idx = probe[0].index() if probe else None
    for i, ok in enumerate(keep):
        if not ok:
            continue
        pays = [None]
        if probe is not None:
            pays = [e[1] & 0x7FFFFFFF if probe[0].wide else e[1] for e in idx.get(cols[probe[1]][i], [])]
        for p in pays:
            out.append(tuple(p if c == "$payload" else cols[c][i] for c in out_columns))
    return out


def star_probe_groupby(cols, schema, filters, table_p: JoinTable, keys_p: tuple, table_s: JoinTable, key_s: str, table_o: JoinTable,
                       key_o: str, values: tuple, capacity: int = 1024) -> Dict[tuple, list]:
    """K9: per match c of P on (k0, k1), g0 of S on key_s and g1 of O on key_o: group (g0, g1) += a * (1 - b) - c * d"""
    if table_p.kind != "pair":
        raise PipeError(LDB_ERR_INVALID, "probe 0 of a star-probe pipeline is a composite-key table")
    if table_s.kind == "pair" or table_o.kind == "pair":
        raise PipeError(LDB_ERR_INVALID, "probes 1 and 2 of a star-probe pipeline are single-key tables")
    keep = filter_rows(cols, schema, filters)
    _agg_operands(cols, schema, [("mul_1minus_1plus", list(values))])
    ip, is_, io = table_p.index(), table_s.index(), table_o.index()
    sums: Dict[tuple, int] = {}
    a, b, d = values
    for i, ok in enumerate(keep):
        if not ok:
            continue
        for ep in ip.get((cols[keys_p[0]][i], cols[keys_p[1]][i]), []):
            for es in is_.get(cols[key_s][i], []):
                for eo in io.get(cols[key_o][i], []):
                    g0 = es[1] & 0x7FFFFFFF if table_s.wide else es[1]
                    g1 = eo[1] & 0x7FFFFFFF if table_o.wide else eo[1]
                    t = agg_term("mul_1minus_minus_paymul", wrap64(cols[a][i]), wrap64(cols[b][i]), pay=ep[1], d=wrap64(cols[d][i]))
                    sums[(g0, g1)] = sums.get((g0, g1), 0) + t
    if len(sums) > group_slots(capacity):
        raise PipeError(LDB_ERR_CAPACITY, "group-by table overflow")
    return {g: [wrap128(v)] for g, v in sums.items()}
