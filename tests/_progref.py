"""Exact reference evaluator for register programs, plus seeded table and program generators (no GPU).

The evaluator takes the expression tuples `program.py` accepts and evaluates them over host columns in plain Python.  Its semantics
are the op comments of include/ldb_gpu.h ("program pipelines"), restated:
  - integers, decimals, dates and booleans are signed 128-bit values; ADD / SUB / MUL / NEG wrap at 128 bits;
  - DIV truncates toward zero and x / 0 is NULL (INT128_MIN / -1 is undefined and never generated);
  - every operator but ISNULL, the connectives and CASE is NULL when an operand is NULL;
  - AND / OR / NOT use SQL three-valued logic; CASE with a NULL condition takes the else branch;
  - doubles are IEEE binary64, one rounding per operation (x / 0.0 is ±inf or NaN, never an error); I2F is `float(int)`;
  - YEAR is the proleptic Gregorian year of `date32` days since 1970-01-01 (`datetime` where it reaches, the 400-year cycle beyond);
  - strings compare bytewise (shorter first on a common prefix); STRKEY8 is the first 8 bytes, zero padded, read big-endian as a
    signed int64;
  - a join table (Join) is its kind and a multimap from key tuple to payloads.  A plain table takes one int32 key (outside int32:
    no match), a direct-address table one key in [min, max], a key-tuple table n int64 keys (a NULL component, or one outside
    int64, never matches); a NULL key never matches;
  - PROBE is the payload of the key's match (NULL when absent).  On a multimap key with several matches it is any one of them: a
    OneOf value, which compares equal to each of its members and takes part in no arithmetic;  PROBE_EACH yields one tuple per match
    ("outer": a row without a match yields one tuple with a NULL payload; "outer" + ("on", cond): each match whose cond is TRUE, or
    exactly one NULL tuple when none is);
  - EXISTS (t, keys…, cond) is TRUE when some match of the keys has a TRUE cond (("match", t) = that match's payload; NULL is not
    TRUE; cond None: any match), else FALSE, never NULL;
  - MARK (probe, cond) is TRUE exactly when cond is TRUE and the probe matched, else FALSE.  Its effect is recorded in the table's
    Join.marks (MarkModel): through PROBE_EACH every walked match with a TRUE cond (with ("on", c) the walk reaches every match of a
    key that has one passing c, the rejected ones too: WHERE drops their tuples, not the MARK), through PROBE on a key with one entry that entry,
    through PROBE on a multimap key at least one of the key's entries;
  - STRCODE is the string's code in a dictionary whose string → code map is read back after the run (`dicts`): codes are
    unspecified, so the map is an input; lookups of absent strings are NULL; inserting STRCODEs record their non-NULL strings in
    `inserted` (their key set must be the dictionary's);
  - ROWID is the row's number in its table; FETCH reads a side table's column at a row number, and a NULL or out-of-range row
    reads NULL;
  - ORDER BY (order_rows) is a stable sort over the full i128 cell.
Values: int for integer-typed results, float for doubles, None for NULL."""
import datetime
import math
import random
import struct
from typing import Dict, List, Optional

import numpy as np

from lingodb_b200 import datagen

M128 = (1 << 128) - 1
I128_MIN, I128_MAX = -(1 << 127), (1 << 127) - 1
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
I16_MIN, I16_MAX = -(1 << 15), (1 << 15) - 1
I8_MIN, I8_MAX = -(1 << 7), (1 << 7) - 1


def wrap128(v: int) -> int:
    v &= M128
    return v - (1 << 128) if v >> 127 else v


def f64(x) -> float:
    """round-trip through an IEEE binary64 (Python floats already are; float32 inputs widen exactly)"""
    return struct.unpack("<d", struct.pack("<d", float(x)))[0]


def f64_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def bits_f64(b: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", b & 0xFFFFFFFFFFFFFFFF))[0]


def fdiv(a: float, b: float) -> float:
    if b != 0.0:
        return a / b
    if math.isnan(a) or a == 0.0:
        return math.nan
    return math.copysign(math.inf, a) * math.copysign(1.0, b)


def _fbin(op, a, b):
    if op == "fadd":
        return a + b
    if op == "fsub":
        return a - b
    if op == "fmul":
        return a * b
    return fdiv(a, b)


def tdiv(a: int, b: int) -> int:
    """signed division truncating toward zero"""
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


_ORD_1970 = 719163  # date(1970, 1, 1).toordinal()
_CYCLE_DAYS, _CYCLE_YEARS = 146097, 400  # one Gregorian cycle


def year_of_days(days: int) -> int:
    o = _ORD_1970 + days
    cycles = 0
    if o < 1:
        cycles = -((1 - o + _CYCLE_DAYS - 1) // _CYCLE_DAYS)
    elif o > datetime.date.max.toordinal():
        cycles = (o - datetime.date.max.toordinal() + _CYCLE_DAYS - 1) // _CYCLE_DAYS
    return datetime.date.fromordinal(o - cycles * _CYCLE_DAYS).year + cycles * _CYCLE_YEARS


def strkey8(s: bytes) -> int:
    return int.from_bytes(s[:8].ljust(8, b"\0"), "big", signed=True)


def _cmp(op, a, b) -> int:
    return int({"=": a == b, "!=": a != b, "<": a < b, "<=": a <= b, ">": a > b, ">=": a >= b}[op])


def _like(kind, s: bytes, p: bytes) -> int:
    return int(s.startswith(p) if kind == "prefix" else s.endswith(p) if kind == "suffix" else p in s)


def _truth(v):
    """three-valued truth of a register: True, False or None"""
    return None if v is None else v != 0


# ---------------------------------------------------------------------------------------------------- host tables
def decode_table(td: datagen.TableData) -> Dict[str, list]:
    """column → list of values over all batches (None for NULL): ints, floats, or bytes for utf8"""
    out = {c.name: [] for c in td.columns}
    for ch, n in zip(td.chunks, td.chunk_rows):
        for c in td.columns:
            v = ch[c.name]
            if c.phys == "utf8":
                offs, data = v
                raw = bytes(np.asarray(data, np.uint8))
                vals = [raw[int(offs[i]):int(offs[i + 1])] for i in range(n)]
            elif c.phys == "decimal128":
                w = np.asarray(v).view(np.uint8).reshape(-1, 16)[:n]
                vals = [int.from_bytes(bytes(w[i]), "little", signed=True) for i in range(n)]
            elif c.phys in ("float32", "float64"):
                vals = [f64(x) for x in np.asarray(v)[:n].tolist()]
            else:
                vals = [int(x) for x in np.asarray(v)[:n].tolist()]
            bm = ch.get(c.name + "$valid")
            if bm is not None:
                ok = np.unpackbits(np.asarray(bm, np.uint8), bitorder="little")[:n]
                vals = [x if ok[i] else None for i, x in enumerate(vals)]
            out[c.name].extend(vals)
    return out


class Side:
    """a side table for FETCH: its decoded columns"""

    def __init__(self, cols: Dict[str, list]):
        self.cols = cols
        self.n = len(next(iter(cols.values()))) if cols else 0


# ---------------------------------------------------------------------------------------------------- joins
class OneOf(frozenset):
    """PROBE of a multimap key with several matches: the payload is one of these, which one is not determined"""


class MarkModel:
    """The markers a join table must end up with: `must` entries marked, for every key in `some` at least one of its entries, and no
    entry outside those two (an entry = its payload, a build row id)."""

    def __init__(self):
        self.must, self.some = set(), set()

    def check(self, join: "Join", marked: set, what=""):
        allowed = set(self.must)
        for k in self.some:
            allowed |= set(join.by.get(k, []))
        assert self.must <= marked, (what, "entries that should be marked are not", sorted(self.must - marked)[:10])
        assert marked <= allowed, (what, "entries marked that no qualifying probe reached", sorted(marked - allowed)[:10], len(marked), len(allowed))
        missing = [k for k in self.some if not marked & set(join.by.get(k, []))]
        assert not missing, (what, "keys probed with a TRUE condition but none of their entries marked", missing[:10])


class Join:
    """A join table's model: kind "plain" (one int32 key), "direct" (one int32 key in [lo, hi]) or "tuple" (n_keys int64 keys), and
    its entries as a multimap {key tuple: [payloads]}; `marks` accumulates MARK effects until cleared."""

    def __init__(self, kind: str, entries, n_keys: int = 1, lo: Optional[int] = None, hi: Optional[int] = None):
        self.kind, self.n_keys, self.lo, self.hi = kind, n_keys, lo, hi
        self.by: Dict[tuple, list] = {}
        for k, p in entries:
            k = k if isinstance(k, tuple) else (k,)
            if None not in k:
                self.by.setdefault(k, []).append(p)
        self.marks = MarkModel()

    def hits(self, keys) -> list:
        if len(keys) != self.n_keys or any(k is None for k in keys):
            return []
        if self.kind == "tuple":
            if not all(I64_MIN <= k <= I64_MAX for k in keys):
                return []
        elif not I32_MIN <= keys[0] <= I32_MAX or (self.kind == "direct" and not self.lo <= keys[0] <= self.hi):
            return []
        return self.by.get(tuple(keys), [])

    def clear_marks(self):
        self.marks = MarkModel()


def as_join(j) -> Join:
    """the older form of a plain table, {key: [payloads]}, as a Join"""
    return j if isinstance(j, Join) else Join("plain", [(k, p) for k, ps in j.items() for p in ps])


def check_dictionary(strings: list, ranks: list, keys: set) -> Dict[bytes, int]:
    """A dictionary read back as rows (row i = code i: its string and rank) against the strings its inserting STRCODEs saw: the codes
    are a bijection onto 0..n-1, the key set is exactly `keys`, and the rank is the bytewise order.  Returns the string → code map."""
    assert None not in strings and len(set(strings)) == len(strings), "two codes for one string"
    assert set(strings) == keys, ("dictionary keys", sorted(set(strings) ^ keys)[:10])
    order = sorted(range(len(strings)), key=lambda i: strings[i])
    assert [ranks[i] for i in order] == list(range(len(strings))), "ranks are not the bytewise order"
    return {s: i for i, s in enumerate(strings)}


def order_rows(values: list, descending: bool = False) -> list:
    """ORDER BY one column of cells (ints: the i128, or a double's bits): the row numbers of a stable sort"""
    return sorted(range(len(values)), key=lambda i: -values[i] if descending else values[i])


# ---------------------------------------------------------------------------------------------------- evaluator
def _split_probe(e):
    """("probe_each", t, keys…[, "outer"[, ("on", cond)]]) → (keys, outer, cond)"""
    keys, on = list(e[2:]), None
    if keys and isinstance(keys[-1], tuple) and len(keys[-1]) == 2 and keys[-1][0] == "on":
        on = keys.pop()[1]
    outer = bool(keys) and keys[-1] == "outer"
    if outer:
        keys.pop()
    return keys, outer, on


class Evaluator:
    """Evaluates expressions column-wise over `cols` (column → list).  `joins` maps a join table's handle value to its Join (or, for a
    plain table, its multimap {key: [payloads]}); `sides` maps a side table's handle value to a Side; `dicts` a dictionary's handle
    value to its string → code map."""

    def __init__(self, cols: Dict[str, list], joins: Optional[dict] = None, sides: Optional[dict] = None, first_row: int = 0,
                 dicts: Optional[dict] = None):
        self.cols, self.sides = cols, sides or {}
        self.joins = {h: as_join(j) for h, j in (joins or {}).items()}
        self.dicts = dicts or {}
        self.inserted: Dict[object, set] = {}
        self.n = len(next(iter(cols.values()))) if cols else 0
        self.first_row = first_row
        self._each_key = None

    @staticmethod
    def _h(t):
        h = getattr(t, "h", t)
        return getattr(h, "value", h)

    def _find_each(self, e):
        if not isinstance(e, tuple):
            return None
        if e and e[0] == "probe_each":
            return e
        for x in e[1:]:
            f = self._find_each(x)
            if f is not None:
                return f
        return None

    def run(self, exprs: list, where=None):
        """the materialize sink's tuples: one list per expression plus the source row of each tuple (PROBE_EACH expands rows);
        with `where`, only the tuples whose predicate is TRUE"""
        each = None
        for e in list(exprs) + ([where] if where is not None else []):
            f = self._find_each(e)
            if f is not None:
                if each is not None and f != each:
                    raise ValueError("at most one probe_each per program")
                each = f
        src = list(range(self.n))
        memo = {}
        self._each_key, self._walked = None, None
        if each is not None:
            kexprs, outer, on = _split_probe(each)
            keys = list(zip(*[self._eval(k, memo, src) for k in kexprs]))
            hits = [self.joins[self._h(each[1])].hits(k) for k in keys]
            if on is not None:  # the walk covers every match of a key with a passing one (WHERE drops the rejected ones' tuples)
                passing = self._passing(each[1], on, memo, src, hits)
                self._walked = [(r, hs) for r, hs, ok in zip(src, hits, passing) if ok]
                hits = passing
            s2, pay = [], []
            for r, hs in zip(src, hits):
                for p in hs or ([None] if outer else []):
                    s2.append(r)
                    pay.append(p)
            src = s2
            self._each_key = repr(each)
            memo = {self._each_key: pay}
        outs = [self._eval(e, memo, src) for e in exprs]
        if where is not None:
            w = self._eval(where, memo, src)
            keep = [i for i, v in enumerate(w) if v is not None and v != 0]
            outs = [[o[i] for i in keep] for o in outs]
            src = [src[i] for i in keep]
        return outs, src

    def eval(self, e) -> list:
        return self.run([e])[0][0]

    def _column(self, name, memo, src):
        if isinstance(name, tuple):  # ("fetch", side, row, column)
            side = self.sides[self._h(name[1])]
            rows = self._eval(name[2], memo, src)
            c = side.cols[name[3]]
            return [c[r] if r is not None and 0 <= r < side.n else None for r in rows]
        c = self.cols[name]
        return [c[r] for r in src]

    def _eval(self, e, memo, src) -> list:
        key = repr(e)
        if key in memo:
            return memo[key]
        r = self._eval1(e, memo, src)
        memo[key] = r
        return r

    def _eval1(self, e, memo, src) -> list:
        k = e[0]
        ev = lambda x: self._eval(x, memo, src)
        n = len(src)
        if k == "col":
            return self._column(e[1], memo, src)
        if k == "fetch":
            return self._column(e, memo, src)
        if k == "const":
            return [wrap128(int(e[1]))] * n
        if k == "f64":
            return [f64(e[1])] * n
        if k == "rowid":
            return [self.first_row + r for r in src]
        if k in ("add", "sub", "mul"):
            f = {"add": lambda x, y: x + y, "sub": lambda x, y: x - y, "mul": lambda x, y: x * y}[k]
            return [None if x is None or y is None else wrap128(f(x, y)) for x, y in zip(ev(e[1]), ev(e[2]))]
        if k == "div":
            return [None if x is None or y is None or y == 0 else wrap128(tdiv(x, y)) for x, y in zip(ev(e[1]), ev(e[2]))]
        if k == "neg":
            return [None if x is None else wrap128(-x) for x in ev(e[1])]
        if k == "cmp":
            return [None if x is None or y is None else _cmp(e[1], x, y) for x, y in zip(ev(e[2]), ev(e[3]))]
        if k == "between":
            return ev(("and", ("cmp", ">=", e[1], e[2]), ("cmp", "<=", e[1], e[3])))
        if k == "and":
            out = []
            for x, y in zip(ev(e[1]), ev(e[2])):
                tx, ty = _truth(x), _truth(y)
                out.append(0 if tx is False or ty is False else None if tx is None or ty is None else 1)
            return out
        if k == "or":
            out = []
            for x, y in zip(ev(e[1]), ev(e[2])):
                tx, ty = _truth(x), _truth(y)
                out.append(1 if tx is True or ty is True else None if tx is None or ty is None else 0)
            return out
        if k == "not":
            return [None if x is None else int(x == 0) for x in ev(e[1])]
        if k == "isnull":
            return [int(x is None) for x in ev(e[1])]
        if k == "case":
            return [a if _truth(c) is True else b for c, a, b in zip(ev(e[1]), ev(e[2]), ev(e[3]))]
        if k == "i2f":
            return [None if x is None else float(x) for x in ev(e[1])]
        if k in ("fadd", "fsub", "fmul", "fdiv"):
            return [None if x is None or y is None else f64(_fbin(k, x, y)) for x, y in zip(ev(e[1]), ev(e[2]))]
        if k == "fcmp":
            return [None if x is None or y is None else _cmp(e[1], x, y) for x, y in zip(ev(e[2]), ev(e[3]))]
        if k == "strcmp":
            p = e[3].encode()
            return [None if s is None else _cmp(e[1], s, p) for s in self._column(e[2], memo, src)]
        if k == "like":
            p = e[3].encode()
            return [None if s is None else _like(e[1], s, p) for s in self._column(e[2], memo, src)]
        if k == "strkey8":
            return [None if s is None else strkey8(s) for s in self._column(e[1], memo, src)]
        if k == "year":
            return [None if x is None else year_of_days(x) for x in ev(e[1])]
        if k == "probe":
            j = self.joins[self._h(e[1])]
            out = []
            for keys in zip(*[ev(x) for x in e[2:]]):
                hits = j.hits(keys)
                out.append(None if not hits else hits[0] if len(hits) == 1 else OneOf(hits))
            return out
        if k == "probe_each":
            raise ValueError("probe_each is expanded by run()")
        if k == "match":
            return memo[f"match:{self._h(e[1])}"]
        if k == "exists":
            j = self.joins[self._h(e[1])]
            hits = [j.hits(keys) for keys in zip(*[ev(x) for x in e[2:-1]])]
            if e[-1] is not None:
                hits = self._passing(e[1], e[-1], memo, src, hits)
            return [int(bool(h)) for h in hits]
        if k == "mark":
            probe = e[1]
            c = ev(e[2])
            j = self.joins[self._h(probe[1])]
            if probe[0] == "probe_each":
                out = [int(_truth(x) is True and p is not None) for x, p in zip(c, ev(probe))]
                if self._walked is None:
                    j.marks.must |= {p for p, v in zip(ev(probe), out) if v}
                    return out
                # with ("on", cond) the walk also reaches the matches cond rejects: MARK runs on their tuples too
                wsrc = [r for r, hs in self._walked for _ in hs]
                wpay = [p for _, hs in self._walked for p in hs]
                wc = self._eval(e[2], {self._each_key: wpay}, wsrc)
                j.marks.must |= {p for p, x in zip(wpay, wc) if _truth(x) is True}
                return out
            out = []
            for keys, x in zip(zip(*[ev(k) for k in probe[2:]]), c):
                hits = j.hits(keys)
                out.append(int(_truth(x) is True and bool(hits)))
                if out[-1] and len(hits) == 1:
                    j.marks.must.add(hits[0])
                elif out[-1]:
                    j.marks.some.add(tuple(keys))
            return out
        if k == "strcode":
            h = self._h(e[1])
            d = self.dicts.get(h, {})
            ss = self._column(e[2], memo, src)
            if len(e) <= 3:
                self.inserted.setdefault(h, set()).update(s for s in ss if s is not None)
            return [None if s is None else d.get(s) for s in ss]
        raise ValueError(f"unknown expression {k}")

    def _passing(self, table, cond, memo, src, hits) -> list:
        """per tuple, the matches in `hits` whose cond is TRUE, cond evaluated once per (tuple, match) with ("match", table) = the match"""
        idx = [i for i, hs in enumerate(hits) for _ in hs]
        sub = {f"match:{self._h(table)}": [p for hs in hits for p in hs]}
        if self._each_key in memo:  # what PROBE_EACH expanded stays in reach of the residual
            sub[self._each_key] = [memo[self._each_key][i] for i in idx]
        c = self._eval(cond, sub, [src[i] for i in idx])
        out = [[] for _ in hits]
        for i, p, v in zip(idx, sub[f"match:{self._h(table)}"], c):
            if _truth(v) is True:
                out[i].append(p)
        return out


def cell(v) -> Optional[int]:
    """a value as the materialize sink stores it: the i128 (signed) or the double's bits (high word 0); None for NULL"""
    if v is None:
        return None
    if isinstance(v, float):
        return f64_bits(v)
    return wrap128(v)


def same_cell(got: Optional[int], want) -> bool:
    """bit-for-bit equality of a materialized cell with a reference value; any NaN equals any NaN"""
    if want is None or got is None:
        return got is None and want is None
    if isinstance(want, OneOf):
        return got in want
    if isinstance(want, float) and math.isnan(want):
        return got >> 64 == 0 and math.isnan(bits_f64(got))
    return got == cell(want)


# ---------------------------------------------------------------------------------------------------- aggregates
def aggregate(kind: str, values: list):
    """one aggregate over a group's inputs (None = NULL input, skipped); None when no input was seen (COUNT: 0)"""
    if kind == "count_star":
        return len(values)
    vs = [v for v in values if v is not None]
    if kind == "count":
        return len(vs)
    if not vs:
        return None
    if kind == "sum":
        return wrap128(sum(vs))
    if kind == "sum_f64":
        return f64(math.fsum(vs))
    if kind in ("min", "min_f64"):
        return min(vs)
    if kind in ("max", "max_f64"):
        return max(vs)
    if kind == "any":
        return set(vs)
    raise ValueError(kind)


def group_by(n: int, keys: List[list], aggs: List[tuple]) -> dict:
    """n tuples; keys: one value list per key expression; aggs: (kind, values | None for count_star) → {key tuple: [aggregate...]}.
    Without keys there is always the one group, also over zero tuples."""
    groups: Dict[tuple, List[int]] = {}
    for i in range(n):
        groups.setdefault(tuple(k[i] for k in keys), []).append(i)
    if not keys:
        groups.setdefault((), [])
    return {g: [aggregate(kind, [None] * len(rows) if vals is None else [vals[i] for i in rows]) for kind, vals in aggs] for g, rows in groups.items()}


# ---------------------------------------------------------------------------------------------------- table generator
INT_EDGES = {
    "int8": [0, 1, -1, I8_MIN, I8_MAX],
    "int16": [0, 1, -1, I8_MIN, I8_MAX, I16_MIN, I16_MAX],
    "int32": [0, 1, -1, I16_MIN, I16_MAX, I32_MIN, I32_MAX],
    "int64": [0, 1, -1, I32_MIN, I32_MAX, I64_MIN, I64_MAX],
    "fsb4": [0, 1, -1, ord("A"), I32_MIN, I32_MAX],
}
WIDE_EDGES = [0, 1, -1, I64_MIN, I64_MAX, I64_MIN - 1, I64_MAX + 1, 1 << 64, -(1 << 64), (7 << 64) + 3, -(5 << 100) - 9, I128_MIN, I128_MAX]
NARROW_DEC_EDGES = [0, 1, -1, 10**18 - 1, -(10**18 - 1), I32_MIN, I32_MAX, I64_MIN, I64_MAX]
FLOAT_EDGES = [0.0, -0.0, 1.0, -1.0, math.inf, -math.inf, math.nan, 5e-324, -5e-324, 2.2250738585072014e-308, 1.7976931348623157e308, 0.1, 2.0**53 + 2]
FLOAT32_EDGES = [0.0, -0.0, 1.0, -1.0, math.inf, -math.inf, math.nan, 1.401298464324817e-45, 3.4028234663852886e38, 0.1]
DATE_EDGES = [0, -1, 1, -719162, -719163, 2932896, 2932897, 10957, 11016, 11017, -25508, -25567, 47482, -10**6, 10**7, I32_MIN, I32_MAX,
              -1 - 146097 * 5000]  # 1970-01-01 ± 1 day, year 1 and 9999 at their edges, 2000-02-29/03-01, 1900-02-28, 1900-01-01, 2100, beyond
PATTERNS = ["a", "ab", "zz", "é", "€x", "abcdefghijklmnopqrstuvwxyz012345", "", "b\x7f"]  # the 32-byte maximum, bytes >= 0x80 (utf-8)
STRINGS = [b"", b"a", b"ab", b"abc", b"ba", b"zz", b"zza", b"\xc3\xa9", b"x\xc3\xa9", b"\xc3\xa9tat", b"\xff\xfe", b"\x80", b"\x7f",
           b"\xe2\x82\xacx", b"abcdefghijklmnopqrstuvwxyz012345", b"abcdefghijklmnopqrstuvwxyz0123456", b"bcdefghijklmnopqrstuvwxyz012345",
           b"aaaaaaaa", b"aaaaaaaab", b"b\x7f", b"\x00a"]

# (name, phys, precision, scale): every physical type the program pipeline reads; all nullable except "k"
SWEEP_COLUMNS = [("k", "int32", 0, 0), ("i8", "int8", 0, 0), ("i16", "int16", 0, 0), ("i32", "int32", 0, 0), ("i64", "int64", 0, 0),
                 ("dw", "decimal128", 38, 2), ("dn", "decimal128", 18, 2), ("dt", "date32", 0, 0), ("fs", "fsb4", 0, 0),
                 ("f4", "float32", 0, 0), ("f8", "float64", 0, 0), ("s", "utf8", 0, 0), ("u", "utf8", 0, 0)]
INT_COLUMNS = ["i8", "i16", "i32", "i64", "dw", "dn", "fs", "k"]
FLOAT_COLUMNS = ["f4", "f8"]
STRING_COLUMNS = ["s", "u"]


def _value(rng: random.Random, phys: str, precision: int):
    edge = rng.random() < 0.35
    if phys in ("int8", "int16", "int32", "int64", "fsb4"):
        if edge:
            return rng.choice(INT_EDGES[phys])
        bits = {"int8": 8, "int16": 16, "int32": 32, "fsb4": 32, "int64": 64}[phys]
        return rng.randrange(-(1 << (bits - 1)), 1 << (bits - 1)) if rng.random() < 0.5 else rng.randrange(-100, 100)
    if phys == "decimal128":
        if precision < 19:
            return rng.choice(NARROW_DEC_EDGES) if edge else rng.randrange(-10**precision + 1, 10**precision)
        return rng.choice(WIDE_EDGES) if edge else rng.choice([rng.randrange(-10**6, 10**6), rng.randrange(I128_MIN, I128_MAX), rng.randrange(-(1 << 80), 1 << 80)])
    if phys == "date32":
        return rng.choice(DATE_EDGES) if edge else rng.choice([rng.randrange(-719162, 2932897), rng.randrange(8000, 11000), rng.randrange(I32_MIN, I32_MAX)])
    if phys == "float32":
        v = rng.choice(FLOAT32_EDGES) if edge else rng.choice([rng.uniform(-100, 100), float(rng.randrange(-50, 50)), rng.uniform(-1e30, 1e30)])
        return float(np.float32(v))
    if phys == "float64":
        return rng.choice(FLOAT_EDGES) if edge else rng.choice([rng.uniform(-100, 100), float(rng.randrange(-50, 50)), rng.uniform(-1e300, 1e300), rng.uniform(-1e-300, 1e-300)])
    if phys == "utf8":
        if edge or rng.random() < 0.5:
            return rng.choice(STRINGS)
        return bytes(rng.randrange(0x61 if rng.random() < 0.5 else 0, 0x63 if rng.random() < 0.5 else 256) for _ in range(rng.randrange(0, 12)))
    raise ValueError(phys)


def gen_values(seed: int, n: int, columns=SWEEP_COLUMNS, null_rate: float = 0.15, key_domain: int = 16) -> Dict[str, list]:
    """Seeded column values (None = NULL).  The first rows of every column run through its edge values."""
    rng = random.Random(seed)
    out = {}
    for name, phys, prec, _ in columns:
        vals = []
        edges = {"decimal128": WIDE_EDGES if prec >= 19 else NARROW_DEC_EDGES, "date32": DATE_EDGES, "float32": FLOAT32_EDGES,
                 "float64": FLOAT_EDGES, "utf8": STRINGS}.get(phys, INT_EDGES.get(phys, []))
        for i in range(n):
            if name == "k":
                vals.append(rng.randrange(key_domain))
            elif i < len(edges):
                vals.append(float(np.float32(edges[i])) if phys == "float32" else edges[i])
            elif rng.random() < null_rate:
                vals.append(None)
            else:
                vals.append(_value(rng, phys, prec))
        if name != "k" and n > len(edges):  # one NULL among the first rows of every nullable column
            vals[len(edges)] = None
        out[name] = vals
    return out


def specs_of(columns=SWEEP_COLUMNS) -> List[datagen.ColumnSpec]:
    return [datagen.ColumnSpec(n, p, pr, sc) for n, p, pr, sc in columns]


_NP = {"int8": np.int8, "int16": np.int16, "int32": np.int32, "fsb4": np.int32, "date32": np.int32, "int64": np.int64, "float32": np.float32, "float64": np.float64}


def column_buffers(phys: str, vals: list, offset: int = 0):
    """Arrow buffers of one column with `offset` leading filler rows: values (or (offsets, bytes)) and the validity bitmap (None when
    no value is NULL)"""
    full = [None] * offset + list(vals)
    valid = np.array([v is not None for v in full], bool)
    bitmap = np.packbits(valid, bitorder="little") if not valid[offset:].all() else None
    if bitmap is not None:
        bitmap = np.concatenate([bitmap, np.zeros(1, np.uint8)])  # whole bytes: the scan may read the last partial byte
    if phys == "utf8":
        data = b"".join(v if v is not None else b"" for v in full)
        offs = np.zeros(len(full) + 1, np.int32)
        offs[1:] = np.cumsum([len(v) if v is not None else 0 for v in full])
        return (offs, np.frombuffer(data + b"\0", np.uint8).copy()), bitmap
    if phys == "decimal128":
        cells = b"".join((0 if v is None else v & M128).to_bytes(16, "little") for v in full)
        return np.frombuffer(cells, np.uint8).reshape(-1, 16).copy(), bitmap
    z = 0.0 if phys.startswith("float") else 0
    return np.array([z if v is None else v for v in full], dtype=_NP[phys]), bitmap


def to_table_data(name: str, values: Dict[str, list], columns=SWEEP_COLUMNS, cuts=()) -> datagen.TableData:
    """the values as a TableData cut into batches at `cuts`"""
    td = datagen.TableData(name, specs_of(columns))
    n = len(next(iter(values.values())))
    edges = [0] + list(cuts) + [n]
    for a, b in zip(edges, edges[1:]):
        ch = {}
        for cname, phys, _, _ in columns:
            buf, bm = column_buffers(phys, values[cname][a:b])
            ch[cname] = buf
            if bm is not None:
                ch[cname + "$valid"] = bm
        td.chunks.append(ch)
        td.chunk_rows.append(b - a)
    return td


# ---------------------------------------------------------------------------------------------------- program generator
INT_CONSTS = [0, 1, -1, 2, 7, -3, 100, I8_MIN, I8_MAX, I16_MAX, I32_MIN, I32_MAX, I64_MIN, I64_MAX, 1 << 64, (3 << 64) + 1, I128_MIN, I128_MAX]
FLOAT_CONSTS = [0.0, -0.0, 1.0, -2.5, 0.1, math.inf, -math.inf, math.nan, 5e-324, 1e308]
DATE_CONSTS = [0, -1, 10957, 11016, -719162, 2932896, -25508]
CMP_OPS = ["=", "!=", "<", "<=", ">", ">="]
LIMITS = dict(regs=48, instr=96, columns=12, consts=24, strings=12, tables=4)


class ProgramGen:
    """Seeded, well-typed random expression trees of depth <= `depth` over SWEEP_COLUMNS: 'int' (integers and decimals), 'float',
    'bool' and 'date' trees.  A divisor that could be -1 is guarded so INT128_MIN / -1 never runs."""

    def __init__(self, seed: int, depth: int = 4):
        self.rng, self.depth = random.Random(seed), depth

    def tree(self, ty: str, depth: Optional[int] = None):
        d = self.depth if depth is None else depth
        r = self.rng
        leaf = d <= 1 or r.random() < 0.25
        if ty == "int":
            if leaf:
                c = r.random()
                if c < 0.55:
                    return ("col", r.choice(INT_COLUMNS))
                if c < 0.8:
                    return ("const", r.choice(INT_CONSTS) if r.random() < 0.6 else r.randrange(-1000, 1000))
                if c < 0.9:
                    return ("strkey8", r.choice(STRING_COLUMNS))
                return ("year", ("col", "dt"))
            op = r.choice(["add", "sub", "mul", "div", "neg", "case", "year"])
            if op == "neg":
                return ("neg", self.tree("int", d - 1))
            if op == "case":
                return ("case", self.tree("bool", d - 1), self.tree("int", d - 1), self.tree("int", d - 1))
            if op == "year":
                return ("year", self.tree("date", d - 1))
            a, b = self.tree("int", d - 1), self.tree("int", d - 1)
            if op == "div":
                b = ("case", ("cmp", "=", b, ("const", -1)), ("const", 1), b)
            return (op, a, b)
        if ty == "float":
            if leaf:
                c = r.random()
                if c < 0.6:
                    return ("col", r.choice(FLOAT_COLUMNS))
                if c < 0.85:
                    return ("f64", r.choice(FLOAT_CONSTS) if r.random() < 0.6 else round(r.uniform(-10, 10), 3))
                return ("i2f", ("col", r.choice(INT_COLUMNS)))
            op = r.choice(["fadd", "fsub", "fmul", "fdiv", "case", "i2f"])
            if op == "case":
                return ("case", self.tree("bool", d - 1), self.tree("float", d - 1), self.tree("float", d - 1))
            if op == "i2f":
                return ("i2f", self.tree("int", d - 1))
            return (op, self.tree("float", d - 1), self.tree("float", d - 1))
        if ty == "date":
            if leaf or r.random() < 0.5:
                return ("col", "dt") if r.random() < 0.7 else ("const", r.choice(DATE_CONSTS))
            return ("case", self.tree("bool", d - 1), self.tree("date", d - 1), self.tree("date", d - 1))
        if ty == "bool":
            if leaf:
                c = r.random()
                if c < 0.3:
                    return ("cmp", r.choice(CMP_OPS), ("col", r.choice(INT_COLUMNS)), ("const", r.choice(INT_CONSTS)))
                if c < 0.45:
                    return ("fcmp", r.choice(CMP_OPS), ("col", r.choice(FLOAT_COLUMNS)), ("f64", r.choice(FLOAT_CONSTS)))
                if c < 0.6:
                    return ("strcmp", r.choice(CMP_OPS), r.choice(STRING_COLUMNS), r.choice(PATTERNS))
                if c < 0.75:
                    return ("like", r.choice(["prefix", "suffix", "contains"]), r.choice(STRING_COLUMNS), r.choice(PATTERNS))
                if c < 0.85:
                    return ("cmp", r.choice(CMP_OPS), ("col", "dt"), ("const", r.choice(DATE_CONSTS)))
                return ("isnull", ("col", r.choice(INT_COLUMNS + FLOAT_COLUMNS + ["dt"])))
            op = r.choice(["and", "or", "not", "cmp", "fcmp", "isnull", "cmpdate"])
            if op in ("and", "or"):
                return (op, self.tree("bool", d - 1), self.tree("bool", d - 1))
            if op == "not":
                return ("not", self.tree("bool", d - 1))
            if op == "cmp":
                return ("cmp", r.choice(CMP_OPS), self.tree("int", d - 1), self.tree("int", d - 1))
            if op == "cmpdate":
                return ("cmp", r.choice(CMP_OPS), self.tree("date", d - 1), self.tree("date", d - 1))
            if op == "fcmp":
                return ("fcmp", r.choice(CMP_OPS), self.tree("float", d - 1), self.tree("float", d - 1))
            return ("isnull", self.tree(r.choice(["int", "float"]), d - 1))
        raise ValueError(ty)

    def program(self, ty: Optional[str] = None):
        """(type, expression) that fits the interpreter's limits on its own, next to a ROWID output"""
        while True:
            t = ty or self.rng.choice(["int", "int", "float", "bool", "date"])
            e = self.tree(t)
            if fits([e, ("rowid",)]):
                return t, e


def usage(exprs: list, where=None) -> dict:
    """registers / instructions / columns / constants / strings / tables one Builder needs for these outputs (registers: None = over
    48, or a program the builder refuses)"""
    from lingodb_b200 import program as P
    b = P.Builder()
    try:
        f = b.expr(where) if where is not None else -1
        for e in exprs:
            b.expr(e)
        b.where(f)  # with the conditions an outer probe_each with a residual ANDs into the WHERE
    except ValueError:
        return dict(regs=None)
    return dict(regs=b._next, instr=len(b.instr), columns=len(b.columns) + len(b.side_columns), consts=len(b.consts), strings=len(b.strings),
                tables=len(b.tables))


def fits(exprs: list, where=None) -> bool:
    u = usage(exprs, where)
    return u["regs"] is not None and all(u[k] <= v for k, v in LIMITS.items())


def programs(seed: int, count: int, depth: int = 4) -> list:
    g = ProgramGen(seed, depth)
    return [g.program() for _ in range(count)]


def pack(progs: list, max_out: int = 7) -> List[list]:
    """group (type, expression) pairs into batches that share one materialize call next to a ROWID output"""
    out, cur = [], []
    for p in progs:
        if cur and (len(cur) == max_out or not fits([e for _, e in cur] + [p[1], ("rowid",)])):
            out.append(cur)
            cur = []
        cur.append(p)
    if cur:
        out.append(cur)
    return out
