"""Random join programs against the exact evaluator of tests/_progref.py: PROBE, PROBE_EACH (inner, outer, outer with a residual), EXISTS,
MARK and STRCODE composed freely over every join-table kind — plain unique and multimap, direct-address, key-tuple tables of 1–4 keys
(unique and multimap) and a string equi-join table — with the four sinks (materialize, hash aggregation, JOIN_BUILD, no sink), the
markers and the dictionary contents compared after every call; every program-kernel instance (programKernel<KeyTuples, Marks, Exists>)
on the table-free and the join programs; ORDER BY over wide decimals that exported groups and materialized outputs hold."""
import random
from collections import Counter

import numpy as np
import pytest

import _progref as R
from lingodb_b200 import program as P, runtime

pytestmark = pytest.mark.gpu

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))
NULL = ("div", const(0), const(0))

NB = 3000  # build rows
HEAVY = {0: 1200, 1: 300, 2: 100}  # build key → entries in the multimaps: warps whose lanes have thousands, hundreds or no matches
B_COLUMNS = R.SWEEP_COLUMNS + [("bk", "int32", 0, 0), ("b1", "int64", 0, 0), ("b2", "int64", 0, 0), ("uk", "int32", 0, 0), ("rid", "int32", 0, 0)]
A_COLUMNS = R.SWEEP_COLUMNS + [("j", "int64", 0, 0), ("w", "decimal128", 38, 0)]
A_BATCHES = (1, 33, 700, 566)  # ragged probe batches
BIG_BATCHES = (1, 33, 4097, 70_000)  # the 70 000-row HOST batch goes through compressed staging
TUPLE_KEYS = {"u": ["uk", "b1", "b2", "bk"], "m": ["bk", "b1", "b2", "b1"]}  # key-tuple tables: the first n of these build columns
SEEDS, PER_SEED = range(4), 60


def _stage(ctx, name, values, columns, batches):
    cuts = list(np.cumsum(batches)[:-1])
    return ctx.table_from_host(R.to_table_data(name, values, columns, cuts))


def _build_values(seed):
    rng = random.Random(seed)
    v = R.gen_values(seed, NB, B_COLUMNS)
    bk = [k for k, n in HEAVY.items() for _ in range(n)]
    bk += [rng.choice([None] + list(range(3, 600))) for _ in range(NB - len(bk))]
    rng.shuffle(bk)
    v["bk"] = bk
    v["b1"] = [rng.choice([0, 1, 2, None, R.I64_MIN, R.I64_MAX]) for _ in range(NB)]
    v["b2"] = [rng.choice([0, 1, None, -5]) for _ in range(NB)]
    uk = list(range(-3, NB - 3))
    rng.shuffle(uk)
    v["uk"], v["rid"] = uk, list(range(NB))
    return v


def _probe_values(seed, n):
    rng = random.Random(seed)
    v = R.gen_values(seed, n, A_COLUMNS)

    def key():
        c = rng.random()
        if c < 0.003:
            return 0
        if c < 0.015:
            return 1
        if c < 0.04:
            return 2
        if c < 0.12:
            return None
        if c < 0.15:
            return rng.choice([R.I32_MIN, R.I32_MAX, -1, -3, -4, NB, NB - 4])
        return rng.randrange(3, 700)  # 600..699: no build entry

    v["k"] = [key() for _ in range(n)]
    v["j"] = [rng.choice([0, 1, 2, None, R.I64_MIN, R.I64_MAX, 3]) for _ in range(n)]
    v["w"] = [rng.choice([0, 1, 2, None, 1 << 64, -(1 << 64), R.I128_MAX, R.I64_MAX, R.I64_MAX + 1, -1, 7 << 64]) for _ in range(n)]
    return v


class Env:
    """the build table B (side table of every fetch), its join tables and their models, the dictionaries"""

    def __init__(self, ctx):
        self.ctx = ctx
        self.bv = _build_values(7)
        self.B = _stage(ctx, "fz_b", self.bv, B_COLUMNS, (7, 1493, 1500))
        self.side = R.Side(self.bv)
        self.h, self.model = {}, {}  # name → join state; handle value → Join
        bv = self.bv
        rows = range(NB)

        def add(name, js, model):
            self.h[name], self.model[js.value] = js, model

        for name, key, unique in (("pu", "uk", True), ("pm", "bk", False)):
            js = runtime.join_table(ctx, NB, unique=unique)
            P.build_join(ctx, self.B, js, col(key), payload=("rowid",))
            add(name, js, R.Join("plain", [(bv[key][r], r) for r in rows]))
        js = runtime.join_table_direct(ctx, -3, NB - 4)
        runtime.run_pipeline(ctx, "scan_build", self.B, build_key="uk", build_payload="rid", sink=js)
        add("dr", js, R.Join("direct", [(bv["uk"][r], r) for r in rows], lo=-3, hi=NB - 4))
        for n in range(1, 5):
            for kind, cols in TUPLE_KEYS.items():
                js = runtime.join_table_keys(ctx, n, NB, unique=kind == "u")
                P.build_join(ctx, self.B, js, [col(c) for c in cols[:n]], payload=("rowid",))
                add(f"t{n}{kind}", js, R.Join("tuple", [(tuple(bv[c][r] for c in cols[:n]), r) for r in rows], n_keys=n))
        # a string equi-join: the build inserts its strings into `dl`, the probes look theirs up
        self.dl = P.dict_state(ctx, 4096, 1 << 16)
        P.run_effects(ctx, self.B, [("strcode", self.dl, "s"), ("strcode", self.dl, "u")])
        self.dl_map = self.read_dict(self.dl, {s for c in ("s", "u") for s in bv[c] if s is not None})
        js = runtime.join_table(ctx, NB, unique=False)
        P.build_join(ctx, self.B, js, ("strcode", self.dl, "s", "lookup"), payload=("rowid",))
        add("sj", js, R.Join("plain", [(self.dl_map.get(bv["s"][r]), r) for r in rows]))
        self.di = P.dict_state(ctx, 1 << 15, 1 << 20)  # filled by the programs' inserting STRCODEs
        self.di_keys = set()
        self.tuple_handles = {self.h[n].value for n in self.h if n[0] == "t"}
        # empty tables: the inert tails that select a kernel instance
        self.empty_tuple = runtime.join_table_keys(ctx, 1, 16)
        self.empty_mark = runtime.join_table(ctx, 16)
        self.empty_exists = runtime.join_table(ctx, 16, unique=False)
        self.tuple_handles.add(self.empty_tuple.value)
        self.model[self.empty_tuple.value] = R.Join("tuple", [], n_keys=1)
        self.model[self.empty_mark.value] = R.Join("plain", [])
        self.model[self.empty_exists.value] = R.Join("plain", [])

    def read_dict(self, d, keys) -> dict:
        t = P.dict_table(self.ctx, d)
        ids = list(range(t.num_rows))
        strings = t.gather_strings("str", ids, decode=False) if ids else []
        ranks = _read(self.ctx, t, ["rank"], 4)[0]
        return R.check_dictionary(strings, ranks, keys)

    def marked(self, js) -> set:
        return set(_read(self.ctx, P.join_marks(self.ctx, js, P.MARKED), ["payload"], 8)[0])

    def destroy(self):
        for js in list(self.h.values()) + [self.empty_tuple, self.empty_mark, self.empty_exists, self.dl, self.di]:
            runtime.state_destroy(self.ctx, js)


@pytest.fixture(scope="module")
def env(gpu_ctx):
    e = Env(gpu_ctx)
    yield e
    e.destroy()


@pytest.fixture(scope="module")
def probe(gpu_ctx):
    values = _probe_values(11, sum(A_BATCHES))
    return _stage(gpu_ctx, "fz_a", values, A_COLUMNS, A_BATCHES), values


# ---------------------------------------------------------------------------------------------------- program generator
def walk(e):
    if isinstance(e, tuple) and e and isinstance(e[0], str):
        yield e
        for x in e[1:]:
            yield from walk(x)


def flags(exprs, tuple_handles) -> tuple:
    """(KeyTuples, Marks, Exists) of the interpreter instance launchProgram picks for these expressions: a key-tuple table named by a
    probe, a MARK, an EXISTS (an outer probe_each with a residual compiles to one)"""
    kt = mk = ex = False
    for e in exprs:
        for x in walk(e):
            if x[0] in ("probe", "probe_each", "exists") and R.Evaluator._h(x[1]) in tuple_handles:
                kt = True
            mk |= x[0] == "mark"
            ex |= x[0] == "exists" or (x[0] == "probe_each" and isinstance(x[-1], tuple) and x[-1][:1] == ("on",))
    return kt, mk, ex


def tails(env, want) -> list:
    """inert WHERE terms (always TRUE) that select the instance flags in `want` = (KeyTuples, Marks, Exists)"""
    out = []
    if want[0]:
        out.append(("isnull", ("probe", env.empty_tuple, const(0))))
    if want[1]:
        out.append(("not", ("mark", ("probe", env.empty_mark, const(0)), const(0))))
    if want[2]:
        out.append(("not", ("exists", env.empty_exists, const(0), None)))
    return out


def conj(terms):
    terms = [t for t in terms if t is not None]
    if not terms:
        return None
    out = terms[0]
    for t in terms[1:]:
        out = ("and", out, t)
    return out


class JoinGen(R.ProgramGen):
    """Seeded random join programs over the probe table A (the SWEEP_COLUMNS plus j int64 and w decimal(38)) and the build table B of
    an Env.  Atoms: PROBE of unique, direct and tuple-unique tables with FETCH through the payload inside the ProgramGen trees, chained
    (a key fetched through another probe's payload); 0–3 EXISTS with residuals over the match and the probe columns, as a value, a WHERE
    term and NOT; at most one PROBE_EACH (inner, outer, outer with ("on", cond)), EXISTS placed before and after it (after it keyed by a
    fetched build value); MARK through PROBE and PROBE_EACH with random, NULL, FALSE and EXISTS conditions; STRCODE lookups and inserts
    over source and side columns and the string equi-join table.  PROBE of a multimap appears only as a semi / anti join (ISNULL) or
    under a MARK, where the payload it picks does not matter.

    Effects must not depend on where the builder places an instruction, since the evaluator works on expressions: an instruction before
    the PROBE_EACH runs once per source row, one after it once per tuple.  So in a program with an inner PROBE_EACH, every MARK and
    inserting STRCODE depends on the PROBE_EACH's payload (it is emitted after it and runs once per tuple, as the evaluator sees it);
    otherwise the PROBE_EACH is outer, which yields at least one tuple per row, so both placements give the same effects.  An outer
    PROBE_EACH with ("on", cond) walks every match of a key with a passing one and its WHERE drops the rejected matches' tuples, but
    effects run on them: there only a MARK through the PROBE_EACH itself (whose walk the evaluator models) reads the payload.  A marked
    table is probed by its MARK only (a MARK marks the latest probe of its table, and not one inside an EXISTS block)."""

    def __init__(self, seed, env, depth=3):
        super().__init__(seed, depth)
        self.env = env

    # -- atoms
    def fetch(self, row, c):
        return ("fetch", self.env.B, row, c)

    def _key(self, pos):
        """key component `pos` of a probe: the first from k (or a unique build value fetched through a payload in reach), the others
        from j, w (values past int64) or fetched build values; the heavy keys come from k alone, so few rows of a warp expand"""
        r = self.rng
        rows = [x for x in self.rows if x[0] != "match"]
        if rows and r.random() < (0.7 if self.after_each else 0.3):
            return self.fetch(r.choice(rows), r.choice(["uk", "uk", "bk"] if pos == 0 else ["b1", "b2", "bk"]))
        if pos == 0:
            return r.choice([col("k"), col("k"), ("add", col("k"), const(r.choice([-1, 1, 600])))])
        return r.choice([col("j"), col("w"), const(0), const(1), ("neg", col("j"))])

    def keys(self, name):
        n = int(name[1]) if name[0] == "t" else 1
        if name == "sj":
            r = self.rng
            rows = [x for x in self.rows if x[0] != "match"]
            s = self.fetch(r.choice(rows), "s") if rows and r.random() < 0.5 else r.choice(R.STRING_COLUMNS)
            return [("strcode", self.env.dl, s, "lookup")]
        return [self._key(i) for i in range(n)]

    def tree(self, ty, depth=None):
        d = self.depth if depth is None else depth
        r = self.rng
        if ty in ("int", "float", "bool") and self.rows and r.random() < 0.3:
            row = r.choice(self.rows)
            if ty == "int":
                return self.fetch(row, r.choice(R.INT_COLUMNS + ["bk", "b1", "dt"]))
            if ty == "float":
                return self.fetch(row, r.choice(R.FLOAT_COLUMNS))
            c = r.random()
            if c < 0.4:
                return ("strcmp", r.choice(R.CMP_OPS), self.fetch(row, r.choice(R.STRING_COLUMNS)), r.choice(R.PATTERNS))
            if c < 0.7:
                return ("cmp", r.choice(R.CMP_OPS), self.fetch(row, r.choice(["i32", "bk", "b1", "dw"])), self.tree("int", d - 1))
            return ("isnull", self.fetch(row, r.choice(R.INT_COLUMNS)))
        if ty == "int" and r.random() < 0.05:
            rows = [x for x in self.rows if x[0] != "match"]
            s = self.fetch(r.choice(rows), r.choice(R.STRING_COLUMNS)) if rows and r.random() < 0.5 else r.choice(R.STRING_COLUMNS)
            return ("strcode", self.env.dl, s, "lookup")
        if ty == "bool" and not self.in_cond and self.exists_left > 0 and r.random() < 0.2:
            self.exists_left -= 1
            e = self.exists()
            return ("not", e) if r.random() < 0.3 else e
        if ty == "bool" and not self.in_cond and r.random() < 0.05:
            t = r.choice(["pm", "t2m", "sj"])
            self.probed.add(t)
            return ("isnull", ("probe", self.env.h[t], *self.keys(t)))
        return super().tree(ty, depth)

    def cond(self, t):
        """a residual over ("match", t), the probe columns and the payloads in reach"""
        self.in_cond = True
        self.rows.append(("match", self.env.h[t]))
        try:
            return self.tree("bool", 3)
        finally:
            self.rows.pop()
            self.in_cond = False

    def exists(self):
        r = self.rng
        t = r.choice(["pm", "pu", "dr", "sj"] + [f"t{n}{k}" for n in range(1, 5) for k in "um"])
        self.probed.add(t)
        keys = self.keys(t)
        return ("exists", self.env.h[t], *keys, None if r.random() < 0.25 else self.cond(t))

    def mark_cond(self):
        r = self.rng
        c = r.random()
        if c < 0.15:
            return const(0)  # FALSE
        if c < 0.3:
            return ("cmp", "=", col("i32"), NULL)  # NULL
        if c < 0.5 and self.exists_left > 0:
            self.exists_left -= 1
            e = self.exists()
            return ("not", e) if r.random() < 0.3 else e
        return self.tree("bool", 3)

    def join_program(self):
        """a dict: outs [(type, expression)], where, marks (expressions), inserts (inserting STRCODEs), each (the probe_each or None)"""
        r, env = self.rng, self.env
        self.rows, self.in_cond, self.after_each, self.probed = [], False, False, set()
        self.exists_left = r.randrange(0, 4)
        for i in range(r.randrange(0, 3)):  # PROBE of unique tables; the second keyed through the first's payload (Q7's shape)
            t = r.choice(["pu", "dr", "t1u", "t2u", "t3u", "t4u"])
            self.probed.add(t)
            if i and r.random() < 0.7:
                keys = [self.fetch(self.rows[-1], "uk")] + [self.fetch(self.rows[-1], c) for c in TUPLE_KEYS["u"][1:int(t[1]) if t[0] == "t" else 1]]
            else:
                keys = self.keys(t)
            self.rows.append(("probe", env.h[t], *keys))
        pre = [("bool", self.exists())] if self.exists_left and r.random() < 0.5 else []  # before the probe_each in the builder's order
        each, form = None, None
        if r.random() < 0.6:
            t = r.choice(["pm", "pu", "dr", "sj", "t1m", "t2m", "t3m", "t4m", "t2u"])
            self.probed.add(t)
            form = r.choice(["inner", "outer", "on"])
            each = ("probe_each", env.h[t], *self.keys(t)) + (() if form == "inner" else ("outer",)) + ((("on", self.cond(t)),) if form == "on" else ())
            self.rows.append(each)
            self.after_each = True
        outs = pre + [(ty, self.tree(ty)) for ty in (r.choice(["int", "int", "float", "bool"]) for _ in range(r.randrange(1, 4)))]
        if each is not None:
            outs.append(("int", each) if r.random() < 0.5 else ("int", self.fetch(each, r.choice(["i64", "dw", "bk"]))))
        while self.exists_left > 0 and r.random() < 0.7:
            self.exists_left -= 1
            outs.append(("bool", self.exists()))
        where = self.tree("bool") if r.random() < 0.5 else None
        # effects
        inner = form == "inner"
        marks = []
        for _ in range(r.randrange(0, 3)):
            if each is not None and r.random() < 0.4 and not any(x[1] == each for x in marks):
                marks.append(("mark", each, self.mark_cond()))
                continue
            if form == "on":  # the walk also reaches the matches the residual rejects: other effects stay off the payload
                self.rows.remove(each)
            c = self.mark_cond()
            t = r.choice(["pm", "pu", "dr", "sj", "t1m", "t2u", "t3m", "t4u", "t4m"])
            keys = self.keys(t)
            if form == "on":
                self.rows.append(each)
            if inner:
                keys = [self.fetch(each, "uk" if t in ("pu", "dr") or t.endswith("u") else "bk")] + keys[1:] if t != "sj" else \
                       [("strcode", env.dl, self.fetch(each, "s"), "lookup")]
            marks.append(("mark", ("probe", env.h[t], *keys), c))
        inserts = []
        if r.random() < 0.35:
            rows = [x for x in self.rows if x[0] != "match" and (form != "on" or x != each)]
            if inner:
                s = self.fetch(each, r.choice(R.STRING_COLUMNS))
            else:
                s = self.fetch(r.choice(rows), r.choice(R.STRING_COLUMNS)) if rows and r.random() < 0.5 else r.choice(R.STRING_COLUMNS)
            inserts.append(("strcode", env.di, s))
        return dict(outs=outs, where=where, marks=marks, inserts=inserts, each=each, form=form)

    @staticmethod
    def valid(p, extra=()) -> bool:
        """fits the interpreter's limits, and a marked table is probed by its MARK only"""
        exprs = [e for _, e in p["outs"]] + p["marks"] + p["inserts"] + list(extra) + [("rowid",)]
        if not R.fits(exprs, p["where"]):
            return False
        marked = [m[1] for m in p["marks"]]
        for m in marked:
            h = R.Evaluator._h(m[1])
            others = {repr(x) for e in exprs + [p["where"]] for x in walk(e) if x[0] in ("probe", "probe_each", "exists") and R.Evaluator._h(x[1]) == h}
            if others != {repr(m)} or marked.count(m) > 1 and m[0] == "probe":
                return False
        return len({R.Evaluator._h(m[1][1]) for m in p["marks"]}) == len(p["marks"])

    def programs(self, count):
        out = []
        while len(out) < count:
            p = self.join_program()
            if self.valid(p):
                out.append(p)
        return out


# ---------------------------------------------------------------------------------------------------- running and checking
def _norm(ty, v):
    """a reference value as a comparable cell: floats by their bits, any NaN as one token"""
    if v is None:
        return None
    if ty == "float":
        return "nan" if v != v else R.f64_bits(v)
    return R.cell(v)


def _norm_got(ty, g):
    if g is not None and ty == "float" and g >> 64 == 0 and R.bits_f64(g) != R.bits_f64(g):
        return "nan"
    return g


def _read(ctx, t, columns, cell_bytes=16):
    ids = list(range(t.num_rows))
    out = [t.gather(c, ids, cell_bytes=cell_bytes) for c in columns] if ids else [[] for _ in columns]
    t.destroy()
    return out


def _int64_value(e) -> bool:
    """an expression whose values fit int64: payloads, string codes, verdicts, int32 / int64 build columns"""
    return e[0] in ("probe_each", "strcode", "exists", "mark", "isnull", "cmp", "strcmp", "not") or (e[0] == "fetch" and e[3] in ("bk", "i32", "i64", "i8", "uk"))


def agg_shape(env, p):
    """hash aggregation: up to 3 int64 keys from the outputs (payloads, fetched values, codes, verdicts); ANY of every effect first
    (so the builder emits them), then every other aggregate kind"""
    ints = [e for ty, e in p["outs"] if ty in ("int", "bool")]
    keys = [e for e in ints if _int64_value(e)][:3] or [("isnull", col("i32"))]
    aggs = [("any", x) for x in p["marks"] + p["inserts"]] + [("count_star", None)]
    aggs += [(k, e) for e in [x for x in ints if x not in keys][:1] for k in ("sum", "min", "max", "count")]
    aggs += [(k, ("i2f", ("fetch", env.B, p["each"], "i8") if p["each"] is not None else col("i8"))) for k in ("sum_f64", "min_f64", "max_f64")]
    return keys, aggs[:8]


def build_shape(p):
    """JOIN_BUILD into a fresh 2-key multimap: int64 keys from the outputs (or the probe keys), the PROBE_EACH payload or ROWID"""
    keys = ([e for ty, e in p["outs"] if _int64_value(e)] + [col("k"), col("j")])[:2]
    return keys, p["each"] if p["each"] is not None else ("rowid",)


def run_and_check(env, table, values, p, sink, tail=()):
    """one program through `sink` on the device, then its result, the markers of the tables it marks and the insert dictionary against
    the evaluator"""
    ctx = env.ctx
    marked = [m[1][1] for m in p["marks"]]
    for js in marked:
        P.clear_marks(ctx, js)
        env.model[js.value].clear_marks()
    where = conj([p["where"]] + list(tail))
    effects = p["marks"] + p["inserts"]
    types = ["int"] + [ty for ty, _ in p["outs"]] + ["int"] * len(effects)
    exprs = [("rowid",)] + [e for _, e in p["outs"]] + effects
    if sink == "materialize":
        got = _read(ctx, P.RawTable(ctx, P.materialize(ctx, table, exprs, where=where)), [f"c{i}" for i in range(len(exprs))])
    elif sink == "hashagg":
        keys, aggs = agg_shape(env, p)
        st = P.group_by(ctx, table, keys, aggs, where=where, expected_groups=1 << 14)
        f64 = tuple(i for i, (k, _) in enumerate(aggs) if k.endswith("_f64"))
        got = P.decode_groups(P.read_groups(ctx, st, 1 << 17), len(keys), len(aggs), f64_aggs=f64)
        runtime.state_destroy(ctx, st)
    elif sink == "join_build":
        keys, pay = build_shape(p)
        jt = runtime.join_table_keys(ctx, 2, 1 << 18, unique=False)
        b = P.Builder()
        f = b.expr(where) if where is not None else -1
        kregs = [b.expr(k) for k in keys]
        pr = b.expr(pay)
        for x in effects:
            b.expr(x)
        d, keep = P._desc(ctx, table, b, f)
        d.sink_kind, d.sink, d.n_keys, d.build_key_reg, d.build_payload_reg = P.SINK_JOIN_BUILD, jt, 2, -1, pr
        for i, r in enumerate(kregs):
            d.key_regs[i] = r
        P._run(ctx, d, b)
        got = Counter(zip(*_read(ctx, P.join_marks(ctx, jt, P.ALL), ["k0", "k1", "payload"], 8)))
        runtime.state_destroy(ctx, jt)
    else:
        P.run_effects(ctx, table, effects + list(tail))
    t = P.dict_table(ctx, env.di)
    ids = list(range(t.num_rows))
    strings = t.gather_strings("str", ids, decode=False) if ids else []
    ranks = _read(ctx, t, ["rank"], 4)[0]
    ev = R.Evaluator(values, joins=env.model, sides={env.B.h.value: env.side},
                     dicts={env.dl.value: env.dl_map, env.di.value: {s: i for i, s in enumerate(strings)}})
    what = (sink, p["outs"], p["where"], effects)
    if sink == "materialize":
        want = Counter(tuple(_norm(t, v) for t, v in zip(types, row)) for row in zip(*ev.run(exprs, where)[0]))
        have = Counter(tuple(_norm_got(t, g) for t, g in zip(types, row)) for row in zip(*got))
        assert have == want, (what, list((have - want).items())[:3], list((want - have).items())[:3])
    elif sink == "hashagg":
        vals = [x for _, x in aggs if x is not None]
        cols, src = ev.run(keys + vals, where)
        it = iter(cols[len(keys):])
        want = R.group_by(len(src), cols[:len(keys)], [(k, None if x is None else next(it)) for k, x in aggs])
        assert set(got) == set(want), (what, sorted(map(repr, set(got) ^ set(want)))[:5])
        for g, w in want.items():
            for i, (k, _) in enumerate(aggs):
                gv = got[g][i]
                assert (gv is None and w[i] is None) or (gv in w[i] if k == "any" else gv == w[i]), (what, g, k, gv, w[i])
    elif sink == "join_build":
        cols, _ = ev.run(keys + [pay] + effects, where)
        want = Counter((a, b, 0 if c is None else c) for a, b, c in zip(*cols[:3]) if a is not None and b is not None)
        assert got == want, (what, list((got - want).items())[:3], list((want - got).items())[:3])
    else:
        ev.run(effects)
    for js in marked:
        env.model[js.value].marks.check(env.model[js.value], env.marked(js), (what, js.value))
    env.di_keys |= ev.inserted.get(env.di.value, set())
    R.check_dictionary(strings, ranks, env.di_keys)


ALL_INSTANCES = {(kt, mk, ex) for kt in (False, True) for mk in (False, True) for ex in (False, True)}  # DESIGN §7: programKernel<KeyTuples, Marks, Exists>
SINKS = ["materialize", "hashagg", "join_build", "none"]


def _instance(env, p, tail=()):
    return flags([e for _, e in p["outs"]] + p["marks"] + p["inserts"] + [p["where"]] + list(tail), env.tuple_handles)


# ---------------------------------------------------------------------------------------------------- 1. random join programs
@pytest.mark.parametrize("seed", SEEDS)
def test_random_join_programs(env, probe, seed):
    """every program through one sink in its own instance; the materialize ones also in each instance that adds flags it lacks (inert
    tails), the same results each time"""
    table, values = probe
    reached = set()
    for i, p in enumerate(JoinGen(500 + seed, env).programs(PER_SEED)):
        sink = SINKS[i % len(SINKS)]
        own = _instance(env, p)
        run_and_check(env, table, values, p, sink)
        reached.add(own)
        if sink != "materialize":
            continue
        for want in ALL_INSTANCES:
            if want == own or not all(w or not o for w, o in zip(want, own)):
                continue
            t = tails(env, [w and not o for w, o in zip(want, own)])
            if JoinGen.valid(p, extra=t):
                assert _instance(env, p, t) == want
                run_and_check(env, table, values, p, sink, t)
                reached.add(want)
    assert reached == ALL_INSTANCES, sorted(ALL_INSTANCES - reached)


def test_join_programs_over_ragged_and_compressed_batches(env, gpu_ctx):
    """a probe table in batches of 1, 33, 4 097 and 70 000 rows (the last through compressed staging), programs without a PROBE_EACH
    expansion so the evaluator stays quick"""
    values = _probe_values(12, sum(BIG_BATCHES))
    table = _stage(gpu_ctx, "fz_big", values, A_COLUMNS, BIG_BATCHES)
    progs = [p for p in JoinGen(900, env).programs(60) if p["each"] is None and not p["inserts"]][:6]  # the insert dictionary stays small
    assert len(progs) >= 4
    for i, p in enumerate(progs):
        run_and_check(env, table, values, p, ["materialize", "hashagg"][i % 2])
    table.clear()


def test_regrown_materialize_reads_as_one_run(env, probe):
    """an inner expansion far larger than the source (the heavy keys) with a MARK and an inserting STRCODE on every tuple: the rerun after
    the output grows must leave the markers, the dictionary and the rows as one run would"""
    table, values = probe
    h = env.h
    each = ("probe_each", h["pm"], col("k"))
    f = lambda c: ("fetch", env.B, each, c)
    p = dict(outs=[("int", each), ("int", f("i64")), ("bool", ("exists", h["t2m"], f("bk"), f("b1"), ("cmp", "!=", ("match", h["t2m"]), each)))],
             where=None, marks=[("mark", ("probe", h["pu"], f("uk")), ("cmp", "<", f("i16"), const(0)))], inserts=[("strcode", env.di, f("s"))],
             each=each, form="inner")
    assert sum(len(env.model[h["pm"].value].hits((k,))) for k in values["k"]) > 5 * len(values["k"])
    run_and_check(env, table, values, p, "materialize")


# ---------------------------------------------------------------------------------------------------- 2. every kernel instance
@pytest.fixture(scope="module")
def sweep(gpu_ctx):
    values = R.gen_values(101, 3000)
    return gpu_ctx.table_from_host(R.to_table_data("fz_sweep", values, cuts=(1000,))), R.Evaluator(values)


def test_table_free_programs_in_every_instance(env, gpu_ctx, sweep):
    """the opcode edge programs and random programs under all eight instances, the instance chosen by inert WHERE tails"""
    from test_gpu_program_ops import _edge_programs
    tab, ev = sweep
    every = tails(env, (True, True, True))
    progs = _edge_programs() + R.programs(1000, 50) + R.programs(1001, 50)
    batches, cur = [], []
    for p in progs:
        if cur and (len(cur) == 7 or not R.fits([e for _, e in cur] + [p[1], ("rowid",)], conj(every))):
            batches.append(cur)
            cur = []
        cur.append(p)
    batches.append(cur)
    reached = set()
    for batch in batches:
        exprs = [e for _, e in batch]
        want = ev.run(exprs)[0]
        for inst in sorted(ALL_INSTANCES):
            t = tails(env, inst)
            assert flags(exprs + t, env.tuple_handles) == inst
            reached.add(inst)
            got = _read(gpu_ctx, P.RawTable(gpu_ctx, P.materialize(gpu_ctx, tab, [("rowid",)] + exprs, where=conj(t))), [f"c{i}" for i in range(len(exprs) + 1)])
            assert sorted(got[0]) == list(range(ev.n)), inst
            for j, e in enumerate(exprs):
                for rid, g in zip(got[0], got[j + 1]):
                    assert R.same_cell(g, want[j][rid]), (inst, e, rid, g, want[j][rid])
    assert reached == ALL_INSTANCES


# ---------------------------------------------------------------------------------------------------- 3. ORDER BY on 16-byte cells
def test_order_by_wide_group_sums_and_materialized_outputs(env, gpu_ctx, probe):
    table, values = probe
    st = P.group_by(gpu_ctx, table, [col("i8")], [("sum", col("w")), ("sum", ("mul", col("w"), col("i16")))], where=("not", ("isnull", col("w"))))
    k, a, b = R.Evaluator(values).run([col("i8"), col("w"), ("mul", col("w"), col("i16"))], ("not", ("isnull", col("w"))))[0]
    want = R.group_by(len(k), [k], [("sum", a), ("sum", b)])
    gt = P.groups_table(gpu_ctx, st)
    ids = list(range(gt.num_rows))
    cols = [gt.gather("k0", ids, cell_bytes=8)] + [gt.gather(c, ids) for c in ("a0", "a1")]
    assert {(k,): [a, b] for k, a, b in zip(*cols)} == want
    assert any(v is not None and not R.I64_MIN <= v <= R.I64_MAX for v in cols[1]), "no group sum outside int64"
    for c, cells in (("a0", cols[1]), ("a1", cols[2])):
        if None in cells:
            continue  # a NULL orders by the cell it holds
        for desc in (False, True):
            assert gt.order_by(c, descending=desc) == R.order_rows(cells, desc), (c, desc)
    gt.destroy()
    runtime.state_destroy(gpu_ctx, st)
    for ty, e in R.programs(31, 40):
        if ty == "bool":
            continue
        mt = P.RawTable(gpu_ctx, P.materialize(gpu_ctx, table, [e], where=("not", ("isnull", e))))
        cells = mt.gather("c0", list(range(mt.num_rows)))
        for desc in (False, True):
            assert mt.order_by("c0", descending=desc) == R.order_rows(cells, desc), (e, desc)
        mt.destroy()
