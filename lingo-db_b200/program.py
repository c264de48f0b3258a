"""Expression trees → register programs of the generic pipeline (include/ldb_gpu.h "program pipelines", csrc/program.cu).

An expression is a nested tuple:
  ("col", name) ("const", int) ("f64", float)
  ("add"|"sub"|"mul"|"div", a, b) ("neg", a)                 exact i128 arithmetic; decimal scales are the writer's job
  ("cmp", "<"|"<="|"="|"!="|">"|">=", a, b) ("between", x, lo, hi)
  ("and", a, b) ("or", a, b) ("not", a) ("isnull", a)       SQL three-valued logic
  ("case", cond, a, b)                                       cond is true ? a : b
  ("i2f", a) ("fadd"|"fsub"|"fmul"|"fdiv", a, b) ("fcmp", op, a, b)
  ("strcmp", op, column, "constant") ("like", "prefix"|"suffix"|"contains", column, "text") ("strkey8", column)
  ("strcode", dict_state, column[, "lookup"])                the string's int32 code in a string dictionary (dict_state): inserted when
                                                             absent, or with "lookup" NULL when absent; a NULL string gives NULL
  ("year", a)                                                extract(year from date32)
  ("probe", join_table_state, key, …)                        payload, or NULL when the key is absent (semi / anti / mark / outer joins);
                                                             a key-tuple table (runtime.join_table_keys) takes one key per component
  ("probe_each", join_table_state, key, …[, "outer"])        payload of EACH match: what follows runs once per match (inner join; "outer":
                                                             a row without a match yields one tuple with a NULL payload).  At most one
                                                             per program; emitted once, never re-evaluated.
                                                             The keys of a tuple go to consecutive registers (moves where needed).
  ("mark", probe, cond)                                      probe: a ("probe", …) or ("probe_each", …) expression.  When cond is TRUE
                                                             and that probe matched, marks the matched build entry; TRUE when it
                                                             marked, else FALSE.  Runs whether WHERE keeps the tuple or not (the
                                                             residual join predicate goes into cond).  A "probe" marks one of a
                                                             multimap key's entries, "probe_each" every one it walks.  join_marks
                                                             reads the markers: reversed semi / anti / mark joins, right / full outer
  ("exists", join_table_state, key, …, cond)                 TRUE when some match of the key satisfies cond, else FALSE (never NULL):
                                                             semi join (WHERE it), anti join (WHERE ("not", it)), mark join (its value).
                                                             cond is the residual, evaluated once per match in probe-run order until one
                                                             is TRUE; inside it ("match", join_table_state) is the current match's
                                                             payload (a "fetch" row).  cond None: TRUE when the key has any match.  No
                                                             exists, probe_each, mark or inserting strcode inside cond; what cond
                                                             evaluates stays inside it (re-evaluated if used again after it).
  ("probe_each", join_table_state, key, …, "outer", ("on", cond))
                                                             left outer join with the residual cond (("match", join_table_state) as in
                                                             exists): each match that satisfies cond, or one tuple with a NULL payload
                                                             when none does.  Emitted as exists + a key NULLed when it fails + an outer
                                                             probe_each, with (cond OR payload IS NULL) ANDed into the WHERE.
  ("rowid",)                                                 the scanned row's number in its table (a build payload for "fetch")
  ("fetch", side_table, row, "column")                       `column` of another table at the row `row` evaluates to (NULL row → NULL);
                                                             accepted wherever a column name is, also as the column of strcmp / like /
                                                             strkey8 / strcode
This is test/bench plumbing over the C-ABI, like runtime.py; in a LingoDB build the sub-operator lowering would emit LdbInstr lists."""
import ctypes as C
import struct
from typing import Dict, List, Optional

from . import capi
from .capi import Error, check

OPS = dict(load=1, const=2, add=3, sub=4, mul=5, div=6, neg=7, cmp=8, **{"and": 9, "or": 10, "not": 11}, isnull=12, select=13, i2f=14, fadd=15, fsub=16, fmul=17,
           fdiv=18, fcmp=19, strcmp=20, strlike=21, year=22, probe=23, strkey8=24, rowid=25, probe_each=26, strcode=27, mark=28, exists=29)
CMP = {"=": 0, "!=": 1, "<": 2, "<=": 3, ">": 4, ">=": 5}
AGG = dict(sum=1, sum_f64=2, count=3, count_star=4, min=5, max=6, min_f64=7, max_f64=8, any=9)
LIKE = dict(prefix=0, suffix=1, contains=2)
SINK_HASHAGG, SINK_JOIN_BUILD, SINK_MATERIALIZE, SINK_NONE = 1, 2, 3, 4
MARKED, UNMARKED, ALL = 1, 0, -1  # join_marks: which entries


class Builder:
    def __init__(self):
        self.instr, self.columns, self.consts, self.strings, self.tables = [], [], [], [], []
        self.side_tables, self.side_columns = [], []  # side tables (handles); side columns as (side table index, column, row register)
        self._cache, self._rows, self._next, self._each = {}, {}, 0, None
        # _match = (table handle, register of the current match) while a residual compiles; _on = the registers to AND into the WHERE
        # (outer probe_each with a residual)
        self._match, self._on = None, []

    def _reg(self):
        r = self._next
        self._next += 1
        if r >= 48:
            raise ValueError("program needs more than 48 registers")
        return r

    def _col(self, name):
        """Column operand: a source column name, or a ("fetch", side_table, row, "column") side column.  Side columns come after
        the source columns, whose number is only known at the end: until instructions() they are numbered -1, -2, …"""
        if isinstance(name, tuple):
            if name[0] != "fetch":
                raise ValueError(f"not a column: {name[0]}")
            h = _handle(name[1])
            if h not in self.side_tables:
                self.side_tables.append(h)
            rk = repr(name[2])  # columns fetched through the same row expression share its register (and its probe)
            if rk not in self._rows:
                self._rows[rk] = self.expr(name[2])
            sc = (self.side_tables.index(h), name[3], self._rows[rk])
            if sc not in self.side_columns:
                self.side_columns.append(sc)
            return -1 - self.side_columns.index(sc)
        if name not in self.columns:
            self.columns.append(name)
        return self.columns.index(name)

    def instructions(self):
        """The LdbInstr tuples with side columns numbered after the source columns."""
        n = len(self.columns)
        fix = lambda c: n - 1 - c if c < 0 else c
        out = []
        for op, dst, a, b, arg in self.instr:
            if op == OPS["load"]:
                arg = fix(arg)
            elif op in (OPS["strcmp"], OPS["strlike"], OPS["strkey8"], OPS["strcode"]):
                a = fix(a)
            out.append((op, dst, a, b, arg))
        return out

    def _emit(self, op, a=0, b=0, arg=0):
        r = self._reg()
        self.instr.append((OPS[op], r, a, b, arg))
        return r

    def _const(self, v: int):
        v &= (1 << 128) - 1
        if v not in self.consts:
            self.consts.append(v)
        return self.consts.index(v)

    def _keys(self, keys) -> int:
        """The first of consecutive registers holding the key expressions: as evaluated when they already are consecutive, else
        copied by moves (SELECT dst, x, x, x: condition, then and else all x) into fresh registers."""
        regs = [self.expr(k) for k in keys]
        if all(r == regs[0] + i for i, r in enumerate(regs)):
            return regs[0]
        return [self._emit("select", r, r, r) for r in regs][0]

    def _string(self, s: str):
        if s not in self.strings:
            self.strings.append(s)
        return self.strings.index(s)

    def _residual(self, table, match: int, cond) -> int:
        """cond with ("match", table) = register `match`.  What it evaluates is cached only while it compiles: inside an exists block
        it is re-evaluated per match, so a later use must not read it after the block."""
        saved = dict(self._cache), dict(self._rows)
        self._match = (_handle(table), match)
        try:
            return self.expr(cond)
        finally:
            self._cache, self._rows = saved
            self._match = None

    def _exists(self, table, key: int, cond) -> int:
        """EXISTS over the keys from register `key` on, its residual block right after it (b = the block's length)"""
        if table not in self.tables:
            self.tables.append(table)
        at = len(self.instr)
        r = self._emit("exists", key, 0, self.tables.index(table))
        if cond is None:
            return r
        res = self._residual(table, r, cond)
        if len(self.instr) == at + 1 or self.instr[-1][1] != res:  # the residual is the block's last write; an empty block means none
            self._emit("select", res, res, res)
        n = len(self.instr) - at - 1
        if n > 255:
            raise ValueError("exists: the residual takes more than 255 instructions")
        op, dst, a, _, arg = self.instr[at]
        self.instr[at] = (op, dst, a, n, arg)
        return r

    def where(self, f: int) -> int:
        """the WHERE register: f (-1: none) ANDed with the conditions outer probe_each residuals add, emitted last"""
        for r in self._on:
            f = r if f < 0 else self._emit("and", f, r)
        self._on = []
        return f

    def expr(self, e) -> int:
        key = repr(e) if not (isinstance(e, tuple) and e and e[0] in ("probe", "match")) else None
        if key is not None and key in self._cache:
            return self._cache[key]
        k = e[0]
        if self._match is not None and (k in ("exists", "probe_each", "mark") or (k == "strcode" and len(e) <= 3)):
            raise ValueError(f"{k} inside the condition of an exists or an outer probe_each (no nesting, no effects per match)")
        if k == "match":
            if self._match is None or _handle(e[1]) != self._match[0]:
                raise ValueError("match: only inside the condition of an exists or an outer probe_each, naming its join table")
            return self._match[1]
        if k == "col":
            r = self._emit("load", arg=self._col(e[1]))
        elif k == "fetch":
            r = self._emit("load", arg=self._col(e))
        elif k == "rowid":
            r = self._emit("rowid")
        elif k == "probe_each":
            if self._each is not None:
                raise ValueError("at most one probe_each per program")
            if e[1] not in self.tables:
                self.tables.append(e[1])
            keys = list(e[2:])
            on = keys.pop()[1] if isinstance(keys[-1], tuple) and len(keys[-1]) == 2 and keys[-1][0] == "on" else None
            outer = keys[-1] == "outer"
            if outer:
                keys.pop()
            if on is None:
                r = self._emit("probe_each", self._keys(keys), int(outer), self.tables.index(e[1]))
            elif not outer:
                raise ValueError("probe_each: a residual ('on', cond) takes the outer form (an inner join's residual is a WHERE term)")
            else:  # v = EXISTS(k, cond); k' = v ? k : NULL; PROBE_EACH(k', outer); WHERE (cond[match] OR payload IS NULL)
                k0 = self._keys(keys)
                v = self._exists(e[1], k0, on)
                null = self.expr(("div", ("const", 0), ("const", 0)))
                kn = [self._emit("select", k0 + i, null, v) for i in range(len(keys))]
                r = self._emit("probe_each", kn[0], 1, self.tables.index(e[1]))
                self._each = r
                res = self._residual(e[1], r, on)
                self._on.append(self._emit("or", res, self._emit("isnull", r)))
            self._each = r
        elif k == "const":
            r = self._emit("const", arg=self._const(int(e[1])))
        elif k == "f64":
            r = self._emit("const", arg=self._const(struct.unpack("<q", struct.pack("<d", float(e[1])))[0] & 0xFFFFFFFFFFFFFFFF))
        elif k in ("add", "sub", "mul", "div", "and", "or", "fadd", "fsub", "fmul", "fdiv"):
            a, b = self.expr(e[1]), self.expr(e[2])
            r = self._emit(k, a, b)
        elif k in ("neg", "not", "isnull", "i2f", "year"):
            r = self._emit(k, self.expr(e[1]))
        elif k in ("cmp", "fcmp"):
            a, b = self.expr(e[2]), self.expr(e[3])
            r = self._emit(k, a, b, CMP[e[1]])
        elif k == "between":
            return self.expr(("and", ("cmp", ">=", e[1], e[2]), ("cmp", "<=", e[1], e[3])))
        elif k == "case":
            c, a, b = self.expr(e[1]), self.expr(e[2]), self.expr(e[3])
            r = self._emit("select", a, b, c)
        elif k == "strcmp":
            r = self._emit("strcmp", self._col(e[2]), CMP[e[1]], self._string(e[3]))
        elif k == "like":
            r = self._emit("strlike", self._col(e[2]), LIKE[e[1]], self._string(e[3]))
        elif k == "strkey8":
            r = self._emit("strkey8", self._col(e[1]))
        elif k == "strcode":
            if len(e) > 3 and e[3] != "lookup":
                raise ValueError(f"strcode mode is 'lookup' or omitted, not {e[3]!r}")
            if e[1] not in self.tables:
                self.tables.append(e[1])
            r = self._emit("strcode", self._col(e[2]), int(len(e) <= 3), self.tables.index(e[1]))
        elif k == "exists":
            if len(e) < 4:
                raise ValueError("exists takes a join table, its keys and a condition (None: no residual)")
            r = self._exists(e[1], self._keys(e[2:-1]), e[-1])
        elif k == "probe":
            if e[1] not in self.tables:
                self.tables.append(e[1])
            r = self._emit("probe", self._keys(e[2:]), 0, self.tables.index(e[1]))
        elif k == "mark":
            probe = e[1] if len(e) == 3 else None
            if not (isinstance(probe, tuple) and probe and probe[0] in ("probe", "probe_each")):
                raise ValueError("mark takes a probe or probe_each expression and a condition")
            if probe[1] in self.tables and any(i[0] == OPS["strcode"] and i[4] == self.tables.index(probe[1]) for i in self.instr):
                raise ValueError("mark: the probed table is a string dictionary")
            c = self.expr(e[2])
            p = self.expr(probe)  # after the condition: the probe the mark refers to is the table's latest one
            t = self.tables.index(probe[1])
            last = [i for i in self.instr if i[0] in (OPS["probe"], OPS["probe_each"]) and i[4] == t][-1]
            if last[1] != p:
                raise ValueError("mark: another probe of the same table runs between the probe and the mark")
            r = self._emit("mark", c, 0, t)
        else:
            raise ValueError(f"unknown expression {k}")
        if key is not None:
            self._cache[key] = r
        return r


def _desc(ctx, table, b: Builder, filter_reg: int):
    keep = []
    filter_reg = b.where(filter_reg)
    d = capi.ProgramDesc()
    d.source = table.h
    cols = [c.encode() for c in b.columns]
    arr = (C.c_char_p * max(1, len(cols)))(*cols)
    d.n_columns, d.columns = len(cols), arr
    ins = (capi.Instr * max(1, len(b.instr)))(*[capi.Instr(*i) for i in b.instructions()])
    d.n_instr, d.instr = len(b.instr), ins
    cs = (capi.I128 * max(1, len(b.consts)))(*[capi.I128(v & 0xFFFFFFFFFFFFFFFF, (v >> 64) - (1 << 64 if v >> 127 else 0)) for v in b.consts])
    d.n_consts, d.consts = len(b.consts), cs
    ss = [s.encode() for s in b.strings]
    sarr = (C.c_char_p * max(1, len(ss)))(*ss)
    d.n_strings, d.strings = len(ss), sarr
    tarr = (C.c_void_p * max(1, len(b.tables)))(*[t.value if isinstance(t, C.c_void_p) else t for t in b.tables])
    d.n_tables, d.tables = len(b.tables), tarr
    d.filter_reg = filter_reg
    keep += [cols, arr, ins, cs, ss, sarr, tarr]
    return d, keep


def _handle(t):
    h = getattr(t, "h", t)
    return h.value if isinstance(h, C.c_void_p) else h


def _run(ctx, d, b: Builder):
    """ldb_gpu_run_program, or ldb_gpu_run_program_ex when the program reads side columns."""
    e = Error()
    if not b.side_columns:
        check(ctx.L.ldb_gpu_run_program(ctx.h, C.byref(d), C.byref(e)), e)
        return
    names = [c.encode() for _, c, _ in b.side_columns]
    j = capi.ProgramJoins()
    tarr = (C.c_void_p * len(b.side_tables))(*b.side_tables)
    sarr = (capi.SideColumn * len(b.side_columns))(*[capi.SideColumn(t, n, r) for (t, _, r), n in zip(b.side_columns, names)])
    j.n_side_tables, j.side_tables = len(b.side_tables), tarr
    j.n_side_columns, j.side_columns = len(b.side_columns), sarr
    check(ctx.L.ldb_gpu_run_program_ex(ctx.h, C.byref(d), C.byref(j), C.byref(e)), e)


def hashagg_state(ctx, n_keys: int, agg_kinds: List[str], expected_groups: int) -> C.c_void_p:
    aggs = (capi.ProgAgg * max(1, len(agg_kinds)))(*[capi.ProgAgg(AGG[k], 0) for k in agg_kinds])
    s, e = C.c_void_p(), Error()
    check(ctx.L.ldb_gpu_hashagg_create(ctx.h, n_keys, len(agg_kinds), aggs, int(expected_groups), C.byref(s), C.byref(e)), e)
    return s


def group_by(ctx, table, keys: list, aggs: list, where=None, expected_groups: int = 1024, state=None) -> C.c_void_p:
    """aggs: [(kind, expr | None)].  Returns the hash-aggregation state (pass `state` to accumulate further tables into it)."""
    b = Builder()
    f = b.expr(where) if where is not None else -1
    kregs = [b.expr(k) for k in keys]
    aregs = [b.expr(x) if x is not None else 0 for _, x in aggs]
    st = state or hashagg_state(ctx, len(keys), [k for k, _ in aggs], expected_groups)
    d, keep = _desc(ctx, table, b, f)
    d.sink_kind, d.sink = SINK_HASHAGG, st
    d.n_keys = len(keys)
    for i, r in enumerate(kregs):
        d.key_regs[i] = r
    d.n_aggs = len(aggs)
    for i, ((kind, _), r) in enumerate(zip(aggs, aregs)):
        d.aggs[i] = capi.ProgAgg(AGG[kind], r)
    _run(ctx, d, b)
    return st


def read_groups(ctx, state, max_rows: int = 1 << 22, f64_aggs=()) -> list:
    """[(keys tuple with None for NULL, aggs list with None for NULL)] — order unspecified."""
    rows = (capi.HashAggRow * max_rows)()
    n, e = C.c_int64(), Error()
    check(ctx.L.ldb_gpu_hashagg_read(state, rows, max_rows, C.byref(n), C.byref(e)), e)
    if n.value > max_rows:
        raise ValueError(f"{n.value} groups, buffer holds {max_rows}")
    nk = None
    out = []
    for r in rows[: n.value]:
        out.append((r.keys[:], r.key_null_mask, r.agg_valid_mask, [(a.lo, a.hi) for a in r.aggs]))
    return out


def decode_groups(raw, n_keys: int, n_aggs: int, f64_aggs=()):
    res = {}
    for keys, knull, avalid, aggs in raw:
        k = tuple(None if (knull >> i) & 1 else int(keys[i]) for i in range(n_keys))
        vals = []
        for a in range(n_aggs):
            if not (avalid >> a) & 1:
                vals.append(None)
            elif a in f64_aggs:
                vals.append(struct.unpack("<d", struct.pack("<Q", aggs[a][0]))[0])
            else:
                vals.append((int(aggs[a][1]) << 64) | int(aggs[a][0]))
        res[k] = vals
    return res


def build_join(ctx, table, join_state, key, payload=None, where=None):
    """key: one expression, or a list of 1..4 key expressions for a key-tuple table (runtime.join_table_keys)."""
    b = Builder()
    f = b.expr(where) if where is not None else -1
    tuple_keys = isinstance(key, list)
    kregs = [b.expr(k) for k in key] if tuple_keys else [b.expr(key)]
    pr = b.expr(payload) if payload is not None else -1
    d, keep = _desc(ctx, table, b, f)
    d.sink_kind, d.sink = SINK_JOIN_BUILD, join_state
    if tuple_keys:
        d.n_keys = len(kregs)
        for i, r in enumerate(kregs):
            d.key_regs[i] = r
        d.build_key_reg = -1
    else:
        d.build_key_reg = kregs[0]
    d.build_payload_reg = pr
    _run(ctx, d, b)


def materialize(ctx, table, outs: list, where=None) -> C.c_void_p:
    """Returns a DEVICE table handle with columns c0..cN (raw i128 cells + validity bytes)."""
    b = Builder()
    f = b.expr(where) if where is not None else -1
    regs = [b.expr(x) for x in outs]
    d, keep = _desc(ctx, table, b, f)
    d.sink_kind = SINK_MATERIALIZE
    d.n_out = len(regs)
    for i, r in enumerate(regs):
        d.out_regs[i] = r
    out = C.c_void_p()
    d.out_table = C.pointer(out)
    _run(ctx, d, b)
    return out


def run_effects(ctx, table, effects: list):
    """A program with no sink (LDB_SINK_NONE): evaluates the expressions in `effects` — ("mark", …), ("strcode", …) inserts — on every
    row of `table` and produces nothing else."""
    b = Builder()
    for x in effects:
        b.expr(x)
    d, keep = _desc(ctx, table, b, -1)
    d.sink_kind = SINK_NONE
    _run(ctx, d, b)


def join_marks(ctx, state, which: int, name="marks") -> "RawTable":
    """The entries of a join table by their markers (which: MARKED, UNMARKED or ALL) as a DEVICE table: "key" (or "k0".."k{n-1}" for a
    key-tuple table) and "payload", int64 (gather with cell_bytes=8); with ALL also "marked", int32 0 / 1 (cell_bytes=4).  Row order
    is unspecified."""
    t, e = C.c_void_p(), Error()
    check(ctx.L.ldb_gpu_join_table_marks(state, int(which), name.encode(), C.byref(t), C.byref(e)), e)
    return RawTable(ctx, t)


def clear_marks(ctx, state):
    """Unmarks every entry of a join table."""
    e = Error()
    check(ctx.L.ldb_gpu_join_table_clear_marks(state, C.byref(e)), e)


class RawTable:
    """Handle-only wrapper (tables created by the library: exported groups, materialised rows)."""

    def __init__(self, ctx, h):
        self.ctx, self.h = ctx, h

    @property
    def num_rows(self):
        return int(self.ctx.L.ldb_gpu_table_num_rows(self.h))

    def order_by(self, column: str, descending=False, limit=-1):
        n = self.num_rows
        ids = (C.c_int64 * max(1, n))()
        m, e = C.c_int64(), Error()
        check(self.ctx.L.ldb_gpu_table_order_by(self.h, column.encode(), int(descending), limit, ids, C.byref(m), C.byref(e)), e)
        return list(ids[: m.value])

    def gather(self, column: str, row_ids: list, cell_bytes=16):
        n = len(row_ids)
        ids = (C.c_int64 * max(1, n))(*row_ids)
        buf = (C.c_uint8 * max(1, n * cell_bytes))()
        valid = (C.c_uint8 * max(1, n))()
        e = Error()
        check(self.ctx.L.ldb_gpu_table_gather(self.h, column.encode(), ids, n, buf, valid, C.byref(e)), e)
        raw = bytes(buf)
        out = []
        for i in range(n):
            if not valid[i]:
                out.append(None)
            else:
                out.append(int.from_bytes(raw[i * cell_bytes:(i + 1) * cell_bytes], "little", signed=True))
        return out

    def order_by_keys(self, keys: list, limit=-1):
        """ORDER BY over [(column, descending), …] (fixed-width or utf8 columns); the first `limit` row ids (all with -1)."""
        n = self.num_rows
        names = [c.encode() for c, _ in keys]
        cols = (C.c_char_p * max(1, len(keys)))(*names)
        desc = (C.c_int32 * max(1, len(keys)))(*[int(bool(d)) for _, d in keys])
        ids = (C.c_int64 * max(1, n))()
        m, e = C.c_int64(), Error()
        check(self.ctx.L.ldb_gpu_table_order_by_keys(self.h, len(keys), cols, desc, limit, ids, C.byref(m), C.byref(e)), e)
        return list(ids[: m.value])

    def gather_strings(self, column: str, row_ids: list, decode=True) -> list:
        """The utf8 cells at `row_ids`: str (bytes with decode=False), None for NULL."""
        n = len(row_ids)
        ids = (C.c_int64 * max(1, n))(*row_ids)
        offs = (C.c_int64 * (n + 1))()
        valid = (C.c_uint8 * max(1, n))()
        need, e = C.c_int64(), Error()
        rc = self.ctx.L.ldb_gpu_table_gather_strings(self.h, column.encode(), ids, n, offs, None, 0, C.byref(need), valid, C.byref(e))
        if rc == capi.LDB_ERR_CAPACITY and need.value > 0:
            buf = (C.c_uint8 * need.value)()
            rc = self.ctx.L.ldb_gpu_table_gather_strings(self.h, column.encode(), ids, n, offs, buf, need.value, C.byref(need), valid, C.byref(e))
            raw = bytes(buf)
        else:
            raw = b""
        check(rc, e)
        out = [raw[offs[i]:offs[i + 1]] if valid[i] else None for i in range(n)]
        return [s.decode() if decode and s is not None else s for s in out]

    def window(self, partition_by=(), order_by=(), frame=None, funcs=(), columns=None, name="window", mode="rows") -> "RawTable":
        """Window functions (ldb_gpu_table_window / _ex) as a new table in window order: the carried `columns` (None: every column), then
        one column per function.  order_by: [(column, descending), …]; frame: (from, to) offsets relative to the current row, None for an
        unbounded end, 0 for CURRENT ROW (default: (None, 0) with ORDER BY, (None, None) without, as the SQL analyzer sets it); mode:
        "rows" or "range" (RANGE offsets are key distances, and (None, 0) is SQL's default frame there); funcs: [(kind, column, name[, n[,
        default]]), …] with kind one of capi.WIN ("row_number", "rank" (the reference's: ROW_NUMBER), "count_star", "count", "sum", "min",
        "max", "sql_rank", "dense_rank", "percent_rank", "cume_dist", "ntile", "lag", "lead", "first_value", "last_value",
        "nth_value"; column None for those without an argument), n the LAG / LEAD offset (default 1), NTILE's buckets or NTH_VALUE's
        position, and default LAG / LEAD's value outside the partition, an int or a float as in nl_join.  AVG is sum / count."""
        if frame is None:
            frame = (None, 0) if order_by else (None, None)
        lo = -(1 << 63) if frame[0] is None else int(frame[0])
        hi = (1 << 63) - 1 if frame[1] is None else int(frame[1])
        enc = lambda xs: (C.c_char_p * max(1, len(xs)))(*[x.encode() for x in xs])
        part, order = list(partition_by), list(order_by)
        desc = (C.c_int32 * max(1, len(order)))(*[int(bool(d)) for _, d in order])
        carried = None if columns is None else enc(list(columns))
        t, e = C.c_void_p(), Error()
        funcs = [tuple(f) for f in funcs]
        if mode == "rows" and all(len(f) == 3 and capi.WIN[f[0]] <= capi.WIN["max"] for f in funcs):
            fs = (capi.WindowFunc * max(1, len(funcs)))(*[capi.WindowFunc(capi.WIN[k], c.encode() if c is not None else None, n.encode()) for k, c, n in funcs])
            check(self.ctx.L.ldb_gpu_table_window(self.h, len(part), enc(part), len(order), enc([c for c, _ in order]), desc, lo, hi, len(funcs), fs,
                                                  0 if columns is None else len(columns), carried, name.encode(), C.byref(t), C.byref(e)), e)
            return RawTable(self.ctx, t)
        fx = []
        for f in funcs:
            kind, col, nm = f[0], f[1], f[2]
            n = int(f[3]) if len(f) > 3 and f[3] is not None else (1 if kind in ("lag", "lead") else 0)
            w = capi.WindowFuncEx(capi.WIN[kind], 0, None if col is None else col.encode(), nm.encode(), n)
            if len(f) > 4 and f[4] is not None:
                # a float argument reads fvalue, any other value: an int sets both, a float its integral value too (as nl_join)
                v = f[4]
                iv = int(v) if isinstance(v, int) or float(v).is_integer() else 0
                iv = iv if -(1 << 127) <= iv < (1 << 127) else 0  # a float beyond i128 (1e300): fvalue only
                w.has_default, w.value, w.fvalue = 1, capi.I128(iv & ((1 << 64) - 1), iv >> 64), float(v)
            fx.append(w)
        fs = (capi.WindowFuncEx * max(1, len(fx)))(*fx)
        fr = capi.WindowFrame(capi.FRAME[mode], 0, lo, hi)
        check(self.ctx.L.ldb_gpu_table_window_ex(self.h, len(part), enc(part), len(order), enc([c for c, _ in order]), desc, C.byref(fr), len(fx), fs,
                                                 0 if columns is None else len(columns), carried, name.encode(), C.byref(t), C.byref(e)), e)
        return RawTable(self.ctx, t)

    def setop(self, other, kind: str, columns=None, other_columns=None, name="setop") -> "RawTable":
        """A set operation (ldb_gpu_table_setop) of this table's rows with `other`'s as a new table: kind one of capi.SETOP ("union_all",
        "union", "intersect", "intersect_all", "except", "except_all"; "distinct" with other=None).  columns / other_columns: the
        positional column lists (None: every column).  Each distinct row comes at its first occurrence in this table's rows followed by
        other's, ALL copies consecutive.  `other` may be a RawTable, a runtime.Table or this table itself."""
        enc = lambda xs: None if xs is None else (C.c_char_p * max(1, len(xs)))(*[x.encode() for x in xs])
        cols = None if columns is None else list(columns)
        ocols = None if other_columns is None else list(other_columns)
        n = len(cols) if cols is not None else len(ocols) if ocols is not None else 0
        t, e = C.c_void_p(), Error()
        check(self.ctx.L.ldb_gpu_table_setop(self.h, None if other is None else other.h, capi.SETOP[kind], n, enc(cols), enc(ocols), name.encode(),
                                             C.byref(t), C.byref(e)), e)
        return RawTable(self.ctx, t)

    def nl_join(self, other, kind: str, conds=(), columns=None, other_columns=None, other_names=None, value_name=None, name="nljoin") -> "RawTable":
        """A nested-loop join (ldb_gpu_table_nl_join) of this table (left) with `other` (right) as a new table: kind one of capi.NLJOIN
        ("inner", "left", "right", "full", "semi", "anti", "mark", "count").  conds: the conjunction of (left column, op, right column)
        triples, op one of "=", "!=", "<", "<=", ">", ">=", with None for one column to compare the other with a constant: (column, op,
        None, value) or (None, op, column, value), value an int (integers, days, char(1) codes, unscaled decimals; float columns
        too) or a float (float columns; against any other column only an integral one).  No conds: a cross product.  columns /
        other_columns: the carried columns (None: every column; other's only for the pair kinds), other_names: their output names; value_name: the MARK (int32 0 / 1) or COUNT (int64) column.  Rows come in left
        row order, then right row order; unmatched right rows of right / full joins last.  `other` may be a RawTable, a runtime.Table
        or this table itself.  Joins with an equality or a range condition over at least 2^24 pairs sort one side and binary-search each
        row's range of matches instead of comparing every pair (DESIGN §7, "Sorted ranges")."""
        cs = []
        for c in conds:
            lcol, op, rcol = c[0], c[1], c[2]
            v = c[3] if len(c) > 3 else 0
            # a float column reads fvalue, any other column value: an int sets both, a float its integral value too, so a non-integral
            # float constant against a non-float column is refused (LDB_ERR_INVALID) instead of being read as 0
            fv = float(v)
            iv = int(v) if isinstance(v, int) or float(v).is_integer() else 0
            cs.append(capi.JoinCond(None if lcol is None else lcol.encode(), capi.OPS[op], None if rcol is None else rcol.encode(),
                                    capi.I128(iv & ((1 << 64) - 1), iv >> 64), fv))
        arr = (capi.JoinCond * max(1, len(cs)))(*cs)
        enc = lambda xs: None if xs is None else (C.c_char_p * max(1, len(xs)))(*[x.encode() for x in xs])
        t, e = C.c_void_p(), Error()
        check(self.ctx.L.ldb_gpu_table_nl_join(self.h, other.h, capi.NLJOIN[kind], len(cs), arr, 0 if columns is None else len(columns), enc(columns),
                                               0 if other_columns is None else len(other_columns), enc(other_columns), enc(other_names),
                                               None if value_name is None else value_name.encode(), name.encode(), C.byref(t), C.byref(e)), e)
        return RawTable(self.ctx, t)

    def distinct(self, columns=None, name="distinct") -> "RawTable":
        """SELECT DISTINCT over `columns` (None: every column), each distinct row at its first occurrence."""
        return self.setop(None, "distinct", columns, None, name)

    def destroy(self):
        if self.h:
            self.ctx.L.ldb_gpu_table_destroy(self.h)
            self.h = C.c_void_p()


def groups_table(ctx, state, name="groups") -> RawTable:
    t, e = C.c_void_p(), Error()
    check(ctx.L.ldb_gpu_hashagg_to_table(state, name.encode(), C.byref(t), C.byref(e)), e)
    return RawTable(ctx, t)


def dict_state(ctx, expected_strings: int, expected_bytes: int) -> C.c_void_p:
    """A string dictionary for ("strcode", state, column): codes 0..n-1, which string gets which code is unspecified."""
    s, e = C.c_void_p(), Error()
    check(ctx.L.ldb_gpu_dict_create(ctx.h, int(expected_strings), int(expected_bytes), C.byref(s), C.byref(e)), e)
    return s


def dict_count(ctx, state) -> int:
    n, e = C.c_int64(), Error()
    check(ctx.L.ldb_gpu_dict_count(state, C.byref(n), C.byref(e)), e)
    return n.value


def dict_table(ctx, state, name="dictionary") -> RawTable:
    """The dictionary as a table, row i = code i: "str" (utf8) and "rank" (int32, the string's position in bytewise order)."""
    t, e = C.c_void_p(), Error()
    check(ctx.L.ldb_gpu_dict_to_table(state, name.encode(), C.byref(t), C.byref(e)), e)
    return RawTable(ctx, t)
