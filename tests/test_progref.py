"""The reference evaluator of tests/_progref.py against values worked out by hand, and its generators' determinism and limits.  The
GPU opcode tests (test_gpu_program_ops.py) trust this evaluator, so it is pinned here on a CPU-only machine."""
import math

import pytest

import _progref as R

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))


def _ev(cols, e):
    return R.Evaluator(cols).eval(e)


def test_three_valued_connectives():
    vals = [1, 0, None]
    a = [x for x in vals for _ in vals]
    b = [y for _ in vals for y in vals]
    cols = {"a": a, "b": b}
    T, F, N = 1, 0, None
    assert _ev(cols, ("and", col("a"), col("b"))) == [T, F, N, F, F, F, N, F, N]
    assert _ev(cols, ("or", col("a"), col("b"))) == [T, T, T, T, F, N, T, N, N]
    assert _ev({"a": vals}, ("not", col("a"))) == [F, T, N]
    assert _ev({"a": vals}, ("isnull", col("a"))) == [F, F, T]
    # CASE with a NULL condition takes the else branch
    assert _ev({"a": vals}, ("case", col("a"), const(10), const(20))) == [10, 20, 20]


def test_truncating_division_and_wrapping():
    cols = {"a": [7, -7, 7, -7, 7, None, 0, R.I128_MIN], "b": [2, 2, -2, -2, 0, 1, -5, 1]}
    assert _ev(cols, ("div", col("a"), col("b"))) == [3, -3, -3, 3, None, None, 0, R.I128_MIN]
    assert _ev({"a": [R.I128_MAX, R.I128_MIN]}, ("add", col("a"), const(1))) == [R.I128_MIN, R.I128_MIN + 1]
    assert _ev({"a": [R.I128_MIN, 0]}, ("neg", col("a"))) == [R.I128_MIN, 0]
    assert _ev({"a": [1 << 64]}, ("mul", col("a"), col("a"))) == [0]  # 2^128 wraps to 0
    assert _ev({"a": [(1 << 64) + 3]}, ("mul", col("a"), const(1 << 63))) == [R.wrap128((1 << 127) + (3 << 63))]


def test_year_at_calendar_edges():
    days = {"1900-02-28": -25510, "1900-03-01": -25509, "2000-02-29": 11016, "2000-03-01": 11017, "1969-12-31": -1, "1970-01-01": 0,
            "0001-01-01": -719162, "9999-12-31": 2932896}
    for s, d in days.items():
        assert R.year_of_days(d) == int(s[:4]), s
    # beyond datetime's range: the proleptic Gregorian calendar continues (year 0 = 1 BC, 400-year cycles of 146 097 days)
    assert R.year_of_days(-719163) == 0  # 0000-12-31
    assert R.year_of_days(-719162 - 366) == 0  # 0000-01-01 (year 0 is a leap year)
    assert R.year_of_days(-719162 - 367) == -1
    assert R.year_of_days(2932897) == 10000
    assert R.year_of_days(2932896 + 146097) == 9999 + 400
    assert _ev({"d": [11016, None]}, ("year", col("d"))) == [2000, None]


def test_int_to_double_rounds_to_nearest_even():
    got = _ev({"a": [2**53 + 1, 2**64 - 1, -(2**53 + 3), R.I128_MAX]}, ("i2f", col("a")))
    assert got == [9007199254740992.0, 18446744073709551616.0, -9007199254740996.0, 2.0**127]
    assert R.f64_bits(got[0]) == 0x4340000000000000


def test_double_ops_are_ieee():
    cols = {"x": [1.0, -1.0, 0.0, -0.0, math.inf, math.nan], "y": [0.0, 0.0, 0.0, 0.0, math.inf, 1.0]}
    q = _ev(cols, ("fdiv", col("x"), col("y")))
    assert q[0] == math.inf and q[1] == -math.inf and math.isnan(q[2]) and math.isnan(q[3]) and math.isnan(q[4]) and math.isnan(q[5])
    assert _ev({"x": [-1.0]}, ("fdiv", col("x"), ("f64", -0.0))) == [math.inf]
    assert math.isnan(_ev({"x": [math.inf]}, ("fsub", col("x"), col("x")))[0])
    # NaN compares false except !=
    assert [_ev({"x": [math.nan]}, ("fcmp", op, col("x"), col("x")))[0] for op in R.CMP_OPS] == [0, 1, 0, 0, 0, 0]
    assert _ev({"x": [0.1]}, ("fadd", col("x"), ("f64", 0.2))) == [0.30000000000000004]


def test_strings_and_keys():
    cols = {"s": [b"", b"a", b"ab", b"\xc3\xa9", b"b", None]}
    assert _ev(cols, ("strcmp", "<", "s", "ab")) == [1, 1, 0, 0, 0, None]
    assert _ev(cols, ("strcmp", ">", "s", "b")) == [0, 0, 0, 1, 0, None]  # bytes >= 0x80 sort after ASCII
    assert _ev(cols, ("like", "suffix", "s", "b")) == [0, 0, 1, 0, 1, None]
    assert _ev(cols, ("like", "contains", "s", "")) == [1, 1, 1, 1, 1, None]
    assert _ev(cols, ("like", "prefix", "s", "é")) == [0, 0, 0, 1, 0, None]
    k = _ev({"s": [b"ab", b"abcdefghij", b"\xff", b""]}, ("strkey8", "s"))
    assert k == [0x6162 << 48, int.from_bytes(b"abcdefgh", "big"), -(1 << 56), 0]


def test_probe_fetch_and_expansion():
    jt = 17
    ev = R.Evaluator({"k": [1, 2, None, 1 << 32 | 1, 3]}, joins={jt: {1: [10, 11], 2: [20], (1 << 32) | 1: [99]}},
                     sides={5: R.Side({"v": [100, None, 300]})})
    outs, src = ev.run([col("k"), ("probe_each", jt, col("k"))])
    assert src == [0, 0, 1] and outs[1] == [10, 11, 20]  # a key outside int32 never matches
    outs, src = ev.run([("probe_each", jt, col("k"), "outer")])
    assert src == [0, 0, 1, 2, 3, 4] and outs[0] == [10, 11, 20, None, None, None]
    ev2 = R.Evaluator({"r": [0, 1, 2, 3, None, -1]}, sides={5: R.Side({"v": [100, None, 300]})})
    assert ev2.eval(("fetch", 5, col("r"), "v")) == [100, None, 300, None, None, None]
    outs, src = ev2.run([("rowid",)], where=("cmp", ">", col("r"), const(0)))
    assert outs == [[1, 2, 3]]


def test_aggregates():
    assert R.group_by(0, [], [("count_star", None), ("sum", []), ("min", [])]) == {(): [0, None, None]}
    g = R.group_by(4, [[1, None, 1, None]], [("min", [-5, None, 3, None]), ("count", [1, None, 2, None]), ("max", [R.I64_MIN - 1, 2, None, None])])
    assert g == {(1,): [-5, 2, R.I64_MIN - 1], (None,): [None, 0, 2]}


def test_cells_compare_bit_for_bit():
    assert R.same_cell(R.f64_bits(math.nan) | 1, math.nan)
    assert not R.same_cell(R.f64_bits(0.0), -0.0)
    assert R.same_cell(-1, -1) and not R.same_cell((1 << 128) - 1, 1)
    assert R.same_cell(None, None) and not R.same_cell(0, None)


def test_table_generator_is_deterministic_and_round_trips():
    a, b = R.gen_values(3, 300), R.gen_values(3, 300)
    assert a == b or all(repr(a[k]) == repr(b[k]) for k in a)  # NaN != NaN: compare the representation
    assert repr(R.gen_values(4, 300)) != repr(a)
    td = R.to_table_data("t", a, cuts=(1, 33, 200))
    back = R.decode_table(td)
    for name, *_ in R.SWEEP_COLUMNS:
        assert repr(back[name]) == repr(a[name]), name
    # every physical type the program pipeline reads, NULLs in every nullable column, and the edge values
    assert {p for _, p, _, _ in R.SWEEP_COLUMNS} == {"int8", "int16", "int32", "int64", "decimal128", "date32", "fsb4", "float32", "float64", "utf8"}
    for name, *_ in R.SWEEP_COLUMNS:
        assert (None in a[name]) == (name != "k"), name
    assert R.I128_MIN in a["dw"] and (7 << 64) + 3 in a["dw"] and R.I64_MAX in a["dn"]
    assert any(isinstance(x, float) and math.isnan(x) for x in a["f8"]) and 5e-324 in a["f8"] and -0.0 in a["f8"]
    assert -719162 in a["dt"] and 2932896 in a["dt"] and -10**6 in a["dt"]
    assert b"" in a["s"] and b"abcdefghijklmnopqrstuvwxyz012345" in a["s"] and any(x and max(x) >= 0x80 for x in a["s"])


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_program_generator_is_deterministic_and_within_limits(seed):
    ps = R.programs(seed, 60)
    assert repr(ps) == repr(R.programs(seed, 60))
    assert repr(ps) != repr(R.programs(seed + 100, 60))
    assert {t for t, _ in ps} == {"int", "float", "bool", "date"}
    for batch in R.pack(ps):
        u = R.usage([e for _, e in batch] + [("rowid",)])
        assert u["regs"] is not None and all(u[k] <= v for k, v in R.LIMITS.items()), u
    # the programs evaluate over a generated table without error (no INT128_MIN / -1: divisors that may be -1 are guarded)
    cols = R.gen_values(seed, 200)
    ev = R.Evaluator(cols)
    for _, e in ps:
        assert len(ev.eval(e)) == 200


def test_opcode_coverage_of_the_generated_programs():
    ops = set()

    def walk(e):
        if isinstance(e, tuple) and e and isinstance(e[0], str):
            ops.add(e[0])
            for x in e[1:]:
                walk(x)

    for _, e in R.programs(7, 300):
        walk(e)
    assert {"col", "const", "f64", "add", "sub", "mul", "div", "neg", "cmp", "and", "or", "not", "isnull", "case", "i2f", "fadd", "fsub", "fmul", "fdiv",
            "fcmp", "strcmp", "like", "year", "strkey8"} <= ops
