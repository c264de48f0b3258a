"""The double aggregates (SUM_F64, MIN_F64, MAX_F64) and contended hash-aggregation states against the order-independent rules of
tests/_progref.py (aggregate): SUM_F64 within gamma_m * sum|x| of the exact sum, MIN_F64 / MAX_F64 to the bit (NaN ignored unless a
group has nothing else, -0.0 below +0.0).  Value families put NaN, ±0, ±inf, subnormals, rounding and cancelling sums and one-sign
overflow into nullable float64 and float32 columns, each family in groups of its own under 0–4 nullable keys.  Under contention
(keyless, one, four and more than 100 000 groups over up to 2^22 rows, HOST and DEVICE batches) every input is larger than twice its
group's bound, so one lost or doubled atomic update fails the check, and the 128-bit SUM / MIN / MAX run on values whose halves carry
and disagree.  Every read path (hashagg_read, the exported table read by a second program, HAVING over it with NaN rows), every
programKernel instance, and the merge across 1, 2, 3 and 8 in-process ranks.

Order-dependent overflow (finite inputs of mixed signs beyond DBL_MAX / 2) is deliberately not generated: the model refuses it."""
import random
from types import SimpleNamespace

import numpy as np
import pytest

import _progref as R
from lingodb_b200 import program as P, runtime
from test_gpu_hashagg_exchange import run_ranks, shard_bounds, slice_values
from test_gpu_exchange import ranks
from test_gpu_program_fuzz import ALL_INSTANCES, conj, flags, tails

pytestmark = pytest.mark.gpu
col, const = (lambda n: ("col", n)), (lambda v: ("const", v))

COLUMNS = [("fam", "int32", 0, 0), ("g1", "int64", 0, 0), ("g2", "int8", 0, 0), ("g3", "int16", 0, 0), ("d", "float64", 0, 0), ("s", "float32", 0, 0)]
KEYS = ["fam", "g1", "g2", "g3"]
AGGS = [("sum_f64", "d"), ("min_f64", "d"), ("max_f64", "d"), ("count", "d"), ("sum_f64", "s"), ("min_f64", "s"), ("max_f64", "s"), ("count_star", None)]
F64_AT = tuple(i for i, (k, _) in enumerate(AGGS) if k.endswith("_f64"))
nan, inf = float("nan"), float("inf")
F32_MAX = 3.4028234663852886e38


def _wide(rng, f32):
    """a double of random sign with a binary exponent anywhere from the subnormals up to ~1e300 (float32: its own range)"""
    lo, hi = (-149, 120) if f32 else (-1074, 996)
    return rng.choice([1.0, -1.0]) * rng.random() * 2.0 ** rng.randrange(lo, hi)


def family(name, rng, n, f32):
    """n values of one family, in row order (float32 columns: values float32 holds exactly)"""
    edges = R.FLOAT32_EDGES if f32 else [x for x in R.FLOAT_EDGES if x != R.DBL_MAX]  # DBL_MAX goes to the one-sign overflow families
    if name == "edges":
        v = [rng.choice(edges) for _ in range(n)]
    elif name == "finite_edges":
        v = [rng.choice([x for x in edges if abs(x) < inf]) for _ in range(n)]
    elif name == "wide":
        v = [_wide(rng, f32) for _ in range(n)]
    elif name == "cancel":  # x, -x pairs of large magnitude plus tiny terms: the exact sum is the tiny ones'
        v = []
        while len(v) < n:
            x = rng.uniform(1e10, 1e20) * rng.choice([1, -1])
            v += [x, rng.uniform(-1e-3, 1e-3), -x]
        v = v[:n]
    elif name == "subnormal":
        v = [rng.choice([1, -1]) * rng.randrange(1, 1 << (23 if f32 else 52)) * (2.0 ** -149 if f32 else 5e-324) for _ in range(n)]
    elif name == "negzero":
        v = [-0.0] * n
    elif name == "latezero":  # +0.0 in the first rows, one -0.0 last: MIN must still be -0.0
        v = [0.0] * (n - 1) + [-0.0]
    elif name == "nanonly":
        v = [rng.choice([nan, -nan]) for _ in range(n)]
    elif name == "nanmix":
        v = [nan if rng.random() < 0.5 else rng.uniform(-100, 100) for _ in range(n)]
    elif name == "posinf":
        v = [inf] * n
    elif name == "infs":
        v = [rng.choice([inf, -inf, 1.5, -0.0]) for _ in range(n)]
    elif name in ("overflow", "overflow_neg"):
        # one sign, each in [0.26, 0.3] DBL_MAX: up to three stay finite, four or more overflow in every order; DBL_MAX shares its
        # keys with the next row (family_values), so it never stands alone (float32: finite as double sums)
        v = [F32_MAX if f32 else R.DBL_MAX] + [F32_MAX * rng.uniform(0.26, 1.0) if f32 else R.DBL_MAX * rng.uniform(0.26, 0.3) for _ in range(n - 1)]
        v = [-x for x in v] if name == "overflow_neg" else v
    elif name == "allnull":
        return [None] * n
    else:
        raise ValueError(name)
    return [float(np.float32(x)) for x in v] if f32 else v


FAMILIES = ["edges", "finite_edges", "wide", "cancel", "subnormal", "negzero", "latezero", "nanonly", "nanmix", "posinf", "infs", "overflow",
            "overflow_neg", "allnull"]
NO_NULLS = {"negzero", "latezero", "overflow", "overflow_neg"}  # keep their designed rows intact


def family_values(seed: int, per_family: int = 240) -> dict:
    """the families in consecutive row blocks (fam = its index), nullable keys g1..g3 over small domains"""
    rng = random.Random(seed)
    out = {c: [] for c, *_ in COLUMNS}
    for f, name in enumerate(FAMILIES):
        d, s = family(name, rng, per_family, False), family(name, rng, per_family, True)
        for i in range(per_family):
            null = name not in NO_NULLS and rng.random() < 0.1
            out["fam"].append(f)
            keys = [rng.choice([None, -1, R.I64_MAX]), rng.choice([None, 0, 1]), rng.choice([None, 7])]
            if i == 1 and name in ("overflow", "overflow_neg"):
                keys = [out[g][-1] for g in ("g1", "g2", "g3")]  # row 0 (±DBL_MAX) and row 1 share every group
            for g, k in zip(("g1", "g2", "g3"), keys):
                out[g].append(k)
            out["d"].append(None if null else d[i])
            out["s"].append(None if null or (name not in NO_NULLS and rng.random() < 0.1) else s[i])
    return out


def model(v: dict, keys: list, aggs=AGGS, where=None) -> dict:
    rows = [i for i in range(len(v["fam"])) if where is None or where(i)]
    pick = lambda c: [v[c][i] for i in rows]
    return R.group_by(len(rows), [pick(k) for k in keys], [(k, None if x is None else pick(x)) for k, x in aggs])


def read(ctx, st, n_keys, aggs=AGGS, max_rows=1 << 12):
    f64 = tuple(i for i, (k, _) in enumerate(aggs) if k.endswith("_f64"))
    return P.decode_groups(P.read_groups(ctx, st, max_rows), n_keys, len(aggs), f64_aggs=f64)


def assert_groups(got: dict, want: dict, aggs=AGGS, what=""):
    assert set(got) == set(want), (what, sorted(map(repr, set(got) ^ set(want)))[:6])
    bad = [(g, aggs[i], got[g][i], w[i]) for g, w in want.items() for i in range(len(aggs))
           if not ((got[g][i] is None and w[i] is None) or (got[g][i] is not None and w[i] is not None and w[i] == got[g][i]))]
    assert not bad, (what, len(bad), bad[:6])


def run(ctx, tab, keys, aggs=AGGS, where=None, expected=1024):
    return P.group_by(ctx, tab, [col(k) for k in keys], [(k, None if x is None else col(x)) for k, x in aggs], where=where, expected_groups=expected)


@pytest.fixture(scope="module")
def fam_table(gpu_ctx):
    v = family_values(41)
    n = len(v["fam"])
    return gpu_ctx.table_from_host(R.to_table_data("fam", v, COLUMNS, cuts=(1, 777, n - 5))), v


# ---------------------------------------------------------------------------------------------------- 1. families, every read path
def test_families_cover_what_they_claim(fam_table):
    _, v = fam_table
    want = model(v, ["fam"])
    at = {name: want[(f,)] for f, name in enumerate(FAMILIES)}
    assert R.f64_bits(at["latezero"][1]) == R.f64_bits(-0.0) and R.f64_bits(at["latezero"][2]) == R.f64_bits(0.0)
    assert R.f64_bits(at["negzero"][0]) == R.f64_bits(0.0) and R.f64_bits(at["negzero"][2]) == R.f64_bits(-0.0)
    assert all(np.isnan(at["nanonly"][i]) for i in (0, 1, 2, 4, 5, 6)) and not np.isnan(at["nanmix"][1])
    assert at["overflow"][0] == inf and at["overflow_neg"][0] == -inf and at["infs"][0] == nan and at["posinf"][1] == inf
    assert float(at["cancel"][0].bound) > 1.0 and 0 < float(at["wide"][0].bound) and at["allnull"][:4] == [None, None, None, 0]
    assert any(x is not None and 0 < abs(x) < 2.2250738585072014e-308 for x in v["d"])


@pytest.mark.parametrize("n_keys", range(5))
def test_families_through_every_read_path(gpu_ctx, fam_table, n_keys):
    """hashagg_read, the exported table read back by a second program's materialize sink, HAVING fcmp over the exported doubles; with
    no key, one keyless program per family (WHERE fam = f)"""
    tab, v = fam_table
    keys = KEYS[:n_keys]
    filters = [(("cmp", "=", col("fam"), const(f)), lambda i, f=f: v["fam"][i] == f) for f in range(len(FAMILIES))] if n_keys == 0 else [(None, None)]
    for where, test in filters:
        st = run(gpu_ctx, tab, keys, where=where)
        got = read(gpu_ctx, st, n_keys)
        want = model(v, keys, where=test)
        what = (n_keys, where)
        assert_groups(got, want, what=what)
        gt = P.groups_table(gpu_ctx, st)
        outs = [col(f"k{k}") for k in range(n_keys)]
        for part in range(0, len(AGGS), 8 - n_keys):
            cols = list(range(len(AGGS)))[part:part + 8 - n_keys]
            mt = P.RawTable(gpu_ctx, P.materialize(gpu_ctx, gt, outs + [col(f"a{i}") for i in cols]))
            rows = [mt.gather(f"c{j}", list(range(mt.num_rows))) for j in range(n_keys + len(cols))]
            mt.destroy()
            back = {}
            for r in zip(*rows):
                back[tuple(r[:n_keys])] = [None if x is None else R.bits_f64(x) if i in F64_AT else x for i, x in zip(cols, r[n_keys:])]
            assert_groups(back, {g: [w[i] for i in cols] for g, w in want.items()}, [AGGS[i] for i in cols], ("exported",) + what)
        # HAVING over the exported doubles: NaN rows fail every fcmp (so NOT (a < 0) keeps them and a >= 0 drops them), -0.0 = 0.0
        for i in F64_AT:
            for pred, keep in ((("fcmp", ">=", col(f"a{i}"), ("f64", 0.0)), lambda x: x >= 0.0),
                               (("not", ("fcmp", "<", col(f"a{i}"), ("f64", 0.0))), lambda x: not x < 0.0),
                               (("fcmp", "=", col(f"a{i}"), ("f64", -0.0)), lambda x: x == 0.0)):
                mt = P.RawTable(gpu_ctx, P.materialize(gpu_ctx, gt, outs + [col(f"a{i}")], where=pred))
                kept = sorted(map(repr, zip(*[mt.gather(f"c{j}", list(range(mt.num_rows))) for j in range(n_keys)]))) if n_keys else ["()"] * mt.num_rows
                mt.destroy()
                expect = sorted(repr(g) if n_keys else "()" for g, row in got.items() if row[i] is not None and keep(row[i]))
                assert kept == expect, ("having", what, i, pred)
        gt.destroy()
        runtime.state_destroy(gpu_ctx, st)


# ---------------------------------------------------------------------------------------------------- 2. contention
BIG_N = 1 << 22
BIG_CUTS = (1, 4097, 2 ** 20 + 3)
BIG_COLUMNS = [("d", "float64", 0, 0), ("ws", "decimal128", 38, 0), ("wm", "decimal128", 38, 0), ("g4", "int32", 0, 0), ("gb", "int32", 0, 0)]
BIG_AGGS = [("sum_f64", "d"), ("min_f64", "d"), ("max_f64", "d"), ("sum", "ws"), ("min", "wm"), ("max", "wm"), ("count", "d"), ("count_star", None)]
MANY_N, MANY_GROUPS = 1 << 18, 100_003


class Big:
    """2^22 rows: d = ±(1 + k 2^-30) (5 % NULL), so sum|x| ~ 2^22 and the SUM_F64 bound ~ 2^-9 is far below one input; ws near 2^64 - 1
    or small negatives (almost every add carries into the high word); wm = k 2^64 + (2^64 - 1) or (k + 1) 2^64 (halves that disagree);
    g4 = row mod 4; gb = a hash of the row into MANY_GROUPS groups."""

    def __init__(self, seed=7):
        rng = np.random.default_rng(seed)
        n = BIG_N
        self.d = np.where(rng.random(n) < 0.5, -1.0, 1.0) * (1.0 + rng.integers(0, 1 << 20, n) * 2.0 ** -30)
        self.valid = rng.random(n) >= 0.05
        pos = rng.random(n) < 0.7
        a, b = rng.integers(0, 1000, n), rng.integers(1, 1000, n)
        self.ws = np.stack([np.where(pos, -1 - a, -b), np.where(pos, 0, -1)], axis=1).astype(np.int64)  # (lo, hi) words
        k = rng.integers(-3, 3, n)
        low = rng.random(n) < 0.5
        self.wm = np.stack([np.where(low, -1, 0), np.where(low, k, k + 1)], axis=1).astype(np.int64)
        self.g4 = (np.arange(n) % 4).astype(np.int32)
        self.gb = ((np.arange(n, dtype=np.int64) * 2654435761) % MANY_GROUPS).astype(np.int32)
        self._py = None

    @staticmethod
    def i128(words):
        return [(h << 64) + (lo & R.M128 >> 64) for lo, h in words.tolist()]

    def values(self, lo=0, hi=BIG_N):
        d = [x if ok else None for x, ok in zip(self.d[lo:hi].tolist(), self.valid[lo:hi].tolist())]
        return {"d": d, "ws": self.i128(self.ws[lo:hi]), "wm": self.i128(self.wm[lo:hi]), "g4": self.g4[lo:hi].tolist(), "gb": self.gb[lo:hi].tolist()}

    def py(self):
        if self._py is None:
            self._py = self.values()
        return self._py

    def chunk(self, lo, hi):
        valid = np.concatenate([np.packbits(self.valid[lo:hi], bitorder="little"), np.zeros(1, np.uint8)])
        return {"d": self.d[lo:hi].copy(), "d$valid": valid, "ws": self.ws[lo:hi].view(np.uint8).reshape(-1, 16).copy(),
                "wm": self.wm[lo:hi].view(np.uint8).reshape(-1, 16).copy(), "g4": self.g4[lo:hi].copy(), "gb": self.gb[lo:hi].copy()}

    def table(self, ctx, device: bool, n=BIG_N, cuts=BIG_CUTS):
        import torch
        t = runtime.Table(ctx, "big", R.specs_of(BIG_COLUMNS))
        edges = [0] + [c for c in cuts if c < n] + [n]
        for lo, hi in zip(edges, edges[1:]):
            ch = self.chunk(lo, hi)
            if device:
                dev = {k: torch.from_numpy(x).cuda() for k, x in ch.items()}
                torch.cuda.synchronize()
                t.append_device(dev, hi - lo)
            else:
                t.append_host(ch, hi - lo)
        torch.cuda.synchronize()
        return t


def one_group(vals: dict, aggs=BIG_AGGS):
    return [R.aggregate(k, [None] * len(vals["d"]) if x is None else vals[x]) for k, x in aggs]


@pytest.fixture(scope="module")
def big():
    b = Big()
    v = b.py()
    b.want_one = one_group(v)
    b.want_four = {(g,): one_group({c: x[g::4] for c, x in v.items()}) for g in range(4)}
    return b


def test_the_contention_data_detects_one_lost_update(big):
    w = big.want_one
    bound = float(w[0].bound)
    assert bound < 2.0 ** -8 and all(abs(x) > 2 * bound for x in big.d[:1000])
    some = next(x for x, ok in zip(big.d.tolist(), big.valid.tolist()) if ok)
    assert w[0] == float(w[0]) and w[0] != float(w[0]) - some and w[0] != float(w[0]) + some
    ws = big.py()["ws"]
    assert sum(1 for x in ws[:1000] if x >= 1 << 63) > 500 and sum(1 for x in ws[:1000] if x < 0) > 200
    assert w[4] % (1 << 64) == (1 << 64) - 1 and w[5] % (1 << 64) == 0  # MIN / MAX: the halves disagree


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_contended_groups(gpu_ctx, big, device):
    """keyless, one group (a constant key), four groups; the same table once"""
    t = big.table(gpu_ctx, device)
    for keys, want in (([], {(): big.want_one}), ([const(7)], {(7,): big.want_one}), ([col("g4")], big.want_four)):
        st = P.group_by(gpu_ctx, t, keys, [(k, None if x is None else col(x)) for k, x in BIG_AGGS], expected_groups=8)
        assert_groups(read(gpu_ctx, st, len(keys), BIG_AGGS), want, BIG_AGGS, (device, keys))
        runtime.state_destroy(gpu_ctx, st)
    t.clear()


def test_more_than_100_000_groups(gpu_ctx, big):
    v = big.values(0, MANY_N)
    want = R.group_by(MANY_N, [v["gb"]], [(k, None if x is None else v[x]) for k, x in BIG_AGGS])
    assert len(want) == MANY_GROUPS
    t = big.table(gpu_ctx, False, MANY_N, cuts=(1, 4097))
    st = P.group_by(gpu_ctx, t, [col("gb")], [(k, None if x is None else col(x)) for k, x in BIG_AGGS], expected_groups=MANY_GROUPS)
    assert_groups(read(gpu_ctx, st, 1, BIG_AGGS, max_rows=MANY_GROUPS + 16), want, BIG_AGGS)
    runtime.state_destroy(gpu_ctx, st)
    t.clear()


# ---------------------------------------------------------------------------------------------------- 3. every kernel instance
def test_hot_group_in_every_instance(gpu_ctx, big):
    """the keyless hot group once in each programKernel<KeyTuples, Marks, Exists> instance, chosen by inert WHERE terms"""
    env = SimpleNamespace(empty_tuple=runtime.join_table_keys(gpu_ctx, 1, 16), empty_mark=runtime.join_table(gpu_ctx, 16),
                          empty_exists=runtime.join_table(gpu_ctx, 16, unique=False))
    env.tuple_handles = {env.empty_tuple.value}
    t = big.table(gpu_ctx, False)
    aggs = [(k, None if x is None else col(x)) for k, x in BIG_AGGS]
    reached = set()
    for inst in sorted(ALL_INSTANCES):
        tl = tails(env, inst)
        assert flags([x for _, x in aggs if x is not None] + tl, env.tuple_handles) == inst
        st = P.group_by(gpu_ctx, t, [], aggs, where=conj(tl))
        assert_groups(read(gpu_ctx, st, 0, BIG_AGGS), {(): big.want_one}, BIG_AGGS, inst)
        runtime.state_destroy(gpu_ctx, st)
        reached.add(inst)
    assert reached == ALL_INSTANCES
    t.clear()
    for js in (env.empty_tuple, env.empty_mark, env.empty_exists):
        runtime.state_destroy(gpu_ctx, js)


# ---------------------------------------------------------------------------------------------------- 4. the exchange
def rank_values(v: dict, world: int, seed: int) -> list:
    """ragged shards (one empty) of the family rows; every non-empty rank adds a row of group (fam 100) — NaN on the first non-empty
    rank, its rank number elsewhere — and of group (fam 101) — +0.0 on the first non-empty rank, -0.0 elsewhere"""
    out = []
    first = None
    for r, (lo, hi) in enumerate(shard_bounds(len(v["fam"]), world, seed)):
        if hi == lo:
            out.append(None)
            continue
        first = r if first is None else first
        sv = slice_values(v, lo, hi)
        for fam, x in ((100, nan if r == first else float(r)), (101, 0.0 if r == first else -0.0)):
            for c, y in (("fam", fam), ("g1", 0), ("g2", 0), ("g3", 0), ("d", x), ("s", x)):
                sv[c].append(y)
        out.append(sv)
    return out


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_families_across_ranks(world):
    v = family_values(60 + world, per_family=90)
    with ranks(world, user_bytes=8 << 20) as (ctxs, comms):
        parts = rank_values(v, world, world * 7)
        assert world == 1 or None in parts
        whole = {c: sum((p[c] for p in parts if p is not None), []) for c in v}
        shards = [c.table_from_host(R.to_table_data(f"s{r}", p, COLUMNS, cuts=(len(p["fam"]) // 3,) if len(p["fam"]) > 3 else ()))
                  if p is not None else None for r, (c, p) in enumerate(zip(ctxs, parts))]
        for keys in (["fam"], ["fam", "g1", "g2"], KEYS):
            want = model(whole, keys)
            _, _, got = run_ranks(ctxs, comms, shards, keys, AGGS, expected=4096)
            merged = {}
            for g in got:
                for k, row in g.items():
                    assert k not in merged, ("group on two ranks", k)
                    merged[k] = row
            assert_groups(merged, want, what=(world, keys))
        # keyless: one family per exchange, every rank's owned row is the whole answer
        for fam in (FAMILIES.index("nanonly"), FAMILIES.index("latezero"), FAMILIES.index("wide"), FAMILIES.index("allnull"), 100, 101):
            sub = [None if p is None else {c: [x for x, f in zip(p[c], p["fam"]) if f == fam] for c in p} for p in parts]
            tabs = [c.table_from_host(R.to_table_data(f"k{r}", p, COLUMNS)) if p and p["fam"] else None for r, (c, p) in enumerate(zip(ctxs, sub))]
            want = model({c: [x for x, f in zip(whole[c], whole["fam"]) if f == fam] for c in whole}, [])
            _, _, got = run_ranks(ctxs, comms, tabs, [], AGGS, expected=1)
            for g in got:
                assert_groups(g, want, what=(world, "keyless", fam))
