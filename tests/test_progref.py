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


def test_probe_on_every_table_kind():
    plain = R.Join("plain", [(1, 10), (2, 20), (2, 21), (R.I32_MAX, 30)])
    direct = R.Join("direct", [(k, 100 + k) for k in range(-2, 3)], lo=-2, hi=2)
    tup = R.Join("tuple", [((1, R.I64_MAX), 7), ((1, R.I64_MIN), 8), ((0, 0), 9), ((0, 0), 10)], n_keys=2)
    ev = R.Evaluator({"k": [1, R.I32_MAX, R.I32_MAX + 1, None, 3, -2, 2], "a": [1, 1, 1, None, 0, 0, 1 << 64],
                      "b": [R.I64_MAX, R.I64_MIN, 0, 0, 0, 0, 0]}, joins={1: plain, 2: direct, 3: tup})
    assert ev.eval(("probe", 1, col("k"))) == [10, 30, None, None, None, None, R.OneOf([20, 21])]
    assert ev.eval(("probe", 2, col("k"))) == [101, None, None, None, None, 98, 102]  # outside [min, max]: no match
    # a NULL component, or one outside int64 (2^64), never matches; a multimap key's payload is any of its entries
    assert ev.eval(("probe", 3, col("a"), col("b"))) == [7, 8, None, None, R.OneOf([9, 10]), R.OneOf([9, 10]), None]
    assert R.same_cell(21, R.OneOf([20, 21])) and not R.same_cell(22, R.OneOf([20, 21])) and not R.same_cell(None, R.OneOf([20]))
    outs, src = ev.run([("probe_each", 3, col("a"), col("b"), "outer")])
    assert src == [0, 1, 2, 3, 4, 4, 5, 5, 6] and outs[0] == [7, 8, None, None, 9, 10, 9, 10, None]


def test_exists_and_the_outer_join_with_a_residual():
    mm = R.Join("plain", [(1, 0), (1, 1), (1, 2), (2, 3), (3, 4)])
    side = R.Side({"v": [None, None, 5, None, 1]})  # key 1: NULL, NULL, then TRUE; key 2: NULL only; key 3: FALSE
    ev = R.Evaluator({"k": [1, 2, 3, 4, None], "x": [5, 5, 5, 5, 5]}, joins={9: mm}, sides={8: side})
    cond = ("cmp", "=", ("fetch", 8, ("match", 9), "v"), col("x"))
    assert ev.eval(("exists", 9, col("k"), cond)) == [1, 0, 0, 0, 0]  # NULL is not TRUE; never NULL
    assert ev.eval(("exists", 9, col("k"), None)) == [1, 1, 1, 0, 0]
    assert ev.eval(("not", ("exists", 9, col("k"), cond))) == [0, 1, 1, 1, 1]
    outs, src = ev.run([("rowid",), ("exists", 9, col("k"), cond)], where=("exists", 9, col("k"), None))
    assert outs == [[0, 1, 2], [1, 0, 0]]
    # each passing match, or exactly one NULL tuple
    m = ("probe_each", 9, col("k"), "outer", ("on", cond))
    outs, src = ev.run([("rowid",), m, ("fetch", 8, m, "v")])
    assert src == [0, 1, 2, 3, 4] and outs[1] == [2, None, None, None, None] and outs[2] == [5, None, None, None, None]
    # a residual that reads the PROBE_EACH payload, and an EXISTS keyed by a value fetched through it
    e = ("probe_each", 9, col("k"))
    inner = ("exists", 9, ("add", ("fetch", 8, e, "v"), const(-4)), ("cmp", "!=", ("match", 9), e))
    outs, src = ev.run([e, inner])
    assert src == [0, 0, 0, 1, 2] and outs == [[0, 1, 2, 3, 4], [0, 0, 1, 0, 0]]  # v = 5 → key 1, whose matches 0, 1 differ from 2


def test_mark_values_and_effects():
    mm = R.Join("plain", [(1, 0), (1, 1), (2, 2)])
    uq = R.Join("tuple", [((1, 1 << 40), 5), ((2, 0), 6)], n_keys=2)
    ev = R.Evaluator({"k": [1, 2, 3, None, 1], "c": [1, None, 1, 1, 0]}, joins={1: mm, 2: uq})
    t = ("cmp", "=", col("c"), const(1))  # TRUE, NULL, TRUE, TRUE, FALSE
    # through PROBE on a multimap: at least one entry of key 1; key 2's condition is NULL, key 3 has no entry
    assert ev.eval(("mark", ("probe", 1, col("k")), t)) == [1, 0, 0, 0, 0]
    assert mm.marks.must == set() and mm.marks.some == {(1,)}
    mm.marks.check(mm, {0})
    mm.marks.check(mm, {0, 1})
    for bad in (set(), {2}, {0, 2}):
        with pytest.raises(AssertionError):
            mm.marks.check(mm, bad)
    # through PROBE_EACH: every walked match with a TRUE condition
    outs, _ = ev.run([("mark", ("probe_each", 1, col("k")), t)])
    assert outs == [[1, 1, 0, 0, 0]] and mm.marks.must == {0, 1}  # rows 0 (two matches), 1 (NULL condition), 4 (two, FALSE)
    with pytest.raises(AssertionError):
        mm.marks.check(mm, {0})
    mm.marks.check(mm, {0, 1})
    # through an outer PROBE_EACH with a residual: the walk reaches the rejected matches of a key with a passing one
    mm.clear_marks()
    on = ("probe_each", 1, col("k"), "outer", ("on", ("cmp", "=", ("match", 1), const(1))))
    outs, src = ev.run([on, ("mark", on, const(1))])
    assert outs == [[1, None, None, None, 1], [1, 0, 0, 0, 1]] and mm.marks.must == {0, 1}  # entry 0 is walked, not kept
    # through PROBE of a key-tuple table: the one entry; markers accumulate until cleared
    ev2 = R.Evaluator({"a": [1, 2, 2], "b": [1 << 40, 0, 1 << 64]}, joins={2: uq})
    assert ev2.eval(("mark", ("probe", 2, col("a"), col("b")), const(1))) == [1, 1, 0]
    assert ev2.eval(("mark", ("probe", 2, col("a"), col("b")), ("cmp", "=", col("a"), const(1)))) == [1, 0, 0]
    assert uq.marks.must == {5, 6}
    uq.clear_marks()
    assert uq.marks.must == set()


def test_string_codes():
    d = {b"a": 1, b"bc": 0}
    ev = R.Evaluator({"s": [b"a", b"bc", b"zz", None], "i": [1, 0, 1, 1]}, dicts={4: d})
    assert ev.eval(("strcode", 4, "s", "lookup")) == [1, 0, None, None]  # absent strings are NULL
    assert ev.inserted == {}
    outs, src = ev.run([("strcode", 4, "s")], where=("cmp", "=", col("i"), const(1)))
    assert ev.inserted == {4: {b"a", b"bc", b"zz"}}  # what the inserting STRCODE saw, WHERE or not
    assert R.check_dictionary([b"bc", b"a"], [1, 0], {b"a", b"bc"}) == d
    for strings, ranks, keys in (([b"bc", b"a"], [0, 1], {b"a", b"bc"}), ([b"a", b"a"], [0, 1], {b"a"}), ([b"a"], [0], {b"a", b"b"})):
        with pytest.raises(AssertionError):
            R.check_dictionary(strings, ranks, keys)


def test_order_by_is_a_stable_sort_over_the_whole_i128():
    vals = [1 << 64, 1, -1, -(1 << 64), R.I128_MIN, R.I128_MAX]
    assert R.order_rows(vals) == [4, 3, 2, 1, 0, 5]
    assert R.order_rows(vals, descending=True) == [5, 0, 1, 2, 3, 4]
    ties = [2, -(1 << 64), 2, 1 << 64, -(1 << 64)]
    assert R.order_rows(ties) == [1, 4, 0, 2, 3] and R.order_rows(ties, descending=True) == [3, 0, 2, 1, 4]


def test_reference_order_puts_nulls_last_ascending_and_first_descending():
    vals = [3, None, -1, None, 3, R.I128_MIN]
    assert R.reference_order([vals], [(0, False)]) == [5, 2, 0, 4, 1, 3]
    assert R.reference_order([vals], [(0, True)]) == [1, 3, 0, 4, 2, 5]
    assert R.order_rows(vals) == [5, 2, 0, 4, 1, 3] and R.order_rows(vals, descending=True) == [1, 3, 0, 4, 2, 5]
    assert R.reference_order([[]], [(0, False)]) == [] and R.reference_order([[None] * 3], [(0, True)]) == [0, 1, 2]


def test_reference_order_lets_the_next_key_decide_between_nulls():
    cols = {"a": [None, 1, None, None, 1], "b": [5, 0, -2, 5, None]}
    assert R.reference_order(cols, [("a", False), ("b", False)]) == [1, 4, 2, 0, 3]
    assert R.reference_order(cols, [("a", False), ("b", True)]) == [4, 1, 0, 3, 2]
    assert R.reference_order(cols, [("a", True), ("b", False)]) == [2, 0, 3, 1, 4]
    assert R.reference_order(cols, [("b", True), ("a", True)]) == [4, 0, 3, 1, 2]


def test_reference_order_of_strings_is_bytewise_with_null_after_the_empty_string():
    s = [b"b", None, b"", b"a\x80", b"a\x7f", b"a", b"\xff", b"a\0", None, b""]
    assert R.reference_order([s], [(0, False)]) == [2, 9, 5, 7, 4, 3, 0, 6, 1, 8]
    assert R.reference_order([s], [(0, True)]) == [1, 8, 6, 0, 3, 4, 7, 5, 2, 9]


def test_aggregates():
    assert R.group_by(0, [], [("count_star", None), ("sum", []), ("min", [])]) == {(): [0, None, None]}
    g = R.group_by(4, [[1, None, 1, None]], [("min", [-5, None, 3, None]), ("count", [1, None, 2, None]), ("max", [R.I64_MIN - 1, 2, None, None])])
    assert g == {(1,): [-5, 2, R.I64_MIN - 1], (None,): [None, 0, 2]}


def test_sum_f64_specials():
    s = lambda vs: R.aggregate("sum_f64", vs)
    nan, inf = math.nan, math.inf
    for vs in ([1.0, nan], [nan], [inf, -inf], [-inf, 2.0, inf], [nan, inf]):
        assert s(vs) == nan and s(vs) == -nan and s(vs) != inf and s(vs) != 0.0, vs
    assert s([inf, 1.0, -5e-324]) == inf and s([inf, 1.0]) != -inf and s([inf]) != nan and s([inf]) != R.DBL_MAX
    assert s([-inf, -inf, 3.0]) == -inf and s([-inf]) != inf
    assert s([None, 1.0]) is not None and R.aggregate("sum_f64", [None, None]) is None
    assert not s([1.0]).__eq__(None) and s([1.0]) != 1  # only doubles compare equal


def test_sum_f64_error_bound():
    s = lambda vs: R.aggregate("sum_f64", vs)
    # exact sums: bound gamma_2 * 3 = 6.7e-16 admits one ulp of 3 (4.4e-16), not two
    assert s([1.0, 2.0]) == 3.0 and s([1.0, 2.0]) == 3.0 + 2.0 ** -51 and s([1.0, 2.0]) != 3.0 + 2.0 ** -50 and s([1.0, 2.0]) != 3.0 - 2.0 ** -50
    # a rounding sum: S = 1 + 2^-52; left to right gives 1.0 (two ties to even), the other order gives S; both are within the bound
    r = s([1.0, 2.0 ** -53, 2.0 ** -53])
    assert r.exact == 1 + R.Fraction(1, 1 << 52) and r == 1.0 and r == 1.0 + 2.0 ** -52 and r != 1.0 + 2.0 ** -50
    # catastrophic cancellation: S = 1, sum|x| = 2e16 + 1, bound gamma_3 * (2e16 + 1) = 6.66; 1e16 + 1 rounds to 1e16, so 0.0 is a result
    r = s([1e16, 1.0, -1e16])
    assert r == 1.0 and r == 0.0 and r == 6.0 and r != 8.0 and r != -8.0 and 6.6 < float(r.bound) < 6.7
    # a zero sum is +0.0: the sum starts from +0.0 and x + (-x) is +0.0
    assert s([-0.0]) == 0.0 and s([-0.0]) != -0.0 and s([-0.0, -0.0]) != -0.0 and s([2.5, -2.5]) != -0.0 and s([-0.0, 0.0]) == 0.0
    # subnormals add without rounding: 3 * 2^-1074 exactly
    assert s([5e-324] * 3) == 1.5e-323 and s([5e-324] * 3) != 1e-323 and s([5e-324, -5e-324, 5e-324]) == 5e-324
    # the bound grows with m and sum|x|: 2^20 inputs of 1 + 2^-30 at 2^-53 each
    r = s([1.0 + 2.0 ** -30] * (1 << 20))
    assert r.exact == (1 << 20) + R.Fraction(1, 1 << 10) and r.bound == R.sum_bound(1 << 20, r.exact)
    assert 2.0 ** -14 < float(r.bound) < 2.0 ** -12
    assert r == float(r.exact) + 2.0 ** -14 and r != float(r.exact) + 2.0 ** -12 and r != float(r.exact) - 1.0  # one update lost is off by ~1


def test_sum_f64_overflow():
    s = lambda vs: R.aggregate("sum_f64", vs)
    big = R.DBL_MAX
    assert s([big, big]) == math.inf and s([big, big]) != big and s([-big, -big * 0.75]) == -math.inf
    assert s([big * 0.51, big * 0.5]) == math.inf  # |S| - bound > DBL_MAX: every order overflows
    assert s([big / 4, big / 8]) == big * 0.375  # sum|x| <= DBL_MAX / 2: finite in every order
    assert s([big * 0.3, big * 0.3, big * 0.3]) == big * 0.9 and s([-big * 0.7, -0.0]) == -big * 0.7  # one sign, |S| + bound <= DBL_MAX: finite
    for vs in ([big, -big, big], [big * 0.6, big * 0.5, -1.0], [math.inf, big, big], [big * 0.6, -big * 0.1], [big, big * 1e-17]):
        with pytest.raises(ValueError):  # the order decides whether it overflows: not modelled
            s(vs)


def test_exact_sum_is_exact():
    rng = __import__("random").Random(5)
    for n in (0, 1, 7, 255, 256, 3000):
        xs = [rng.choice([1.0, -1.0]) * rng.random() * 2.0 ** rng.randrange(-1074, 1000) for _ in range(n)] + [5e-324, -0.0, R.DBL_MAX / 4]
        assert R.exact_sum(xs) == sum(map(R.Fraction, xs), R.Fraction(0)), n
    assert R.exact_sum([R.DBL_MAX] * 300 + [-R.DBL_MAX] * 299) == R.Fraction(R.DBL_MAX)


def test_min_max_f64_ignore_nan_and_order_signed_zeros():
    mn = lambda vs: R.aggregate("min_f64", vs)
    mx = lambda vs: R.aggregate("max_f64", vs)
    nan, inf = math.nan, math.inf
    assert mn([nan, 1.0, nan]) == 1.0 and mx([nan, 1.0, nan]) == 1.0 and mn([nan, 1.0]) != nan
    assert mn([nan, nan]) == nan and mx([nan]) == nan and mn([nan]) != inf and mx([nan]) != -inf
    for vs in ([0.0, -0.0], [-0.0, 0.0], [0.0, -0.0, 0.0, nan]):
        assert mn(vs) == -0.0 and mn(vs) != 0.0 and mx(vs) == 0.0 and mx(vs) != -0.0, vs
    assert mn([inf, -inf, nan, 3.0]) == -inf and mx([nan, inf, -inf]) == inf and mn([inf, nan]) == inf and mx([-inf]) == -inf
    assert mn([5e-324, 0.0]) == 0.0 and mn([-5e-324, -0.0]) == -5e-324 and mx([1.0]) != 1.0 + 2.0 ** -52
    assert mn([None, nan, None]) == nan and mn([None]) is None
    # the result does not depend on the input order, to the bit
    vals = [nan, 0.0, -0.0, 5.0, nan, -0.0, 0.0]
    for k in range(len(vals)):
        rot = vals[k:] + vals[:k]
        assert R.f64_bits(mn(rot)) == R.f64_bits(-0.0) and R.f64_bits(mx(rot)) == R.f64_bits(5.0)
        assert R.f64_bits(mx([x for x in rot if x != 5.0])) == R.f64_bits(0.0)


def test_cells_compare_bit_for_bit():
    assert R.same_cell(R.f64_bits(0.0), R.aggregate("sum_f64", [1.0, -1.0])) and not R.same_cell(R.f64_bits(-0.0), R.aggregate("sum_f64", [-0.0]))
    assert R.same_cell(R.f64_bits(-0.0), R.aggregate("min_f64", [0.0, -0.0])) and not R.same_cell(R.f64_bits(0.0), R.aggregate("min_f64", [0.0, -0.0]))
    assert R.same_cell(R.f64_bits(math.nan), R.aggregate("max_f64", [math.nan])) and not R.same_cell(1 << 64, R.aggregate("max_f64", [0.0]))
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
