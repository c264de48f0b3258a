"""The window model (tests/_windowref.py) against the reference's own answers (uni.test queries c-f over studenten) and hand-worked
frames: the clamping of finite bounds, UNBOUNDED FOLLOWING as the partition end, NULL keys as one partition and NULL arguments."""
import json
import os
from fractions import Fraction

import _windowref as W

HERE = os.path.dirname(os.path.abspath(__file__))
UNI = json.load(open(os.path.join(HERE, "golden", "uni_windows.json")))


def studenten() -> dict:
    rows = UNI["studenten"]["rows"]
    return {"matrnr": [r[0] for r in rows], "name": [r[1].encode() for r in rows], "semester": [r[2] for r in rows]}


# each uni query as (partition_by, order_by, funcs) and how its output row is made from the window's columns
UNI_WINDOWS = {
    "c": (["semester"], [], [("sum", "matrnr", "s"), ("count", "matrnr", "c")]),
    "d": ([], [("matrnr", False)], [("rank", None, "r")]),
    "e": (["semester"], [("matrnr", False)], [("rank", None, "r")]),
    "f": (["semester"], [("matrnr", False)], [("sum", "matrnr", "s")]),
}


def uni_rows(q: str, cols: dict, order: list, out: dict) -> list:
    """the query's output rows, cell by cell as exact values (AVG as SUM / COUNT)"""
    rows = []
    for i, r in enumerate(order):
        m, sem = cols["matrnr"][r], cols["semester"][r]
        if q == "c":
            rows.append((m, sem, Fraction(out["s"][i], out["c"][i])))
        elif q == "d":
            rows.append((m, out["r"][i]))
        elif q == "e":
            rows.append((m, sem, out["r"][i]))
        else:
            rows.append((m, sem, out["s"][i]))
    return sorted(rows)


def expected_uni(q: str) -> list:
    return sorted(tuple(Fraction(x) for x in r) for r in UNI["queries"][q]["rows"])


def test_model_reproduces_the_uni_window_answers():
    cols = studenten()
    for q, (part, order, funcs) in UNI_WINDOWS.items():
        frame = (None, 0) if order else (None, None)
        o, out = W.window(cols, part, order, frame, funcs)
        assert uni_rows(q, cols, o, out) == expected_uni(q), q


def test_clamped_frames_by_hand():
    cols = {"v": [1, 2, 3, 4, 5, 6]}
    run = lambda frame, kind="sum": W.window(cols, [], [("v", False)], frame, [(kind, "v", "x")])[1]["x"]
    # 2 FOLLOWING .. 5 FOLLOWING: the last rows clamp onto the partition end and aggregate the last row
    assert run((2, 5)) == [3 + 4 + 5 + 6, 4 + 5 + 6, 5 + 6, 6, 6, 6]
    # 5 PRECEDING .. 2 PRECEDING: the first rows clamp onto the first row
    assert run((-5, -2)) == [1, 1, 1, 1 + 2, 1 + 2 + 3, 1 + 2 + 3 + 4]
    assert run((-3, 2)) == [6, 10, 15, 21, 20, 18]
    assert run((0, 0)) == [1, 2, 3, 4, 5, 6]
    # UNBOUNDED FOLLOWING is the partition end for every row (no i64 wrap)
    assert run((-2, None)) == [21, 21, 21, 20, 18, 15]
    assert run((None, 3)) == [10, 15, 21, 21, 21, 21]
    assert run((None, None), "max") == [6] * 6
    assert run((-1, 1), "min") == [1, 1, 2, 3, 4, 5]
    # ROW_NUMBER is i - lo + 1 with the clamped frame start, COUNT(*) the clamped width
    rn = W.window(cols, [], [("v", False)], (2, 5), [("row_number", None, "r"), ("count_star", None, "c")])[1]
    assert rn["r"] == [-1, -1, -1, -1, 0, 1]
    assert rn["c"] == [4, 3, 2, 1, 1, 1]


def test_null_keys_form_one_partition_and_null_arguments_are_skipped():
    cols = {"p": [None, 1, None, 1, 2], "o": [5, None, 3, 1, 7], "a": [None, 10, None, None, 4]}
    order, out = W.window(cols, ["p"], [("o", True)], (None, 0), [("sum", "a", "s"), ("count", "a", "c"), ("min", "a", "m"), ("row_number", None, "r")])
    # p ascending with NULL last; o DESC puts its NULL first
    assert order == [1, 3, 4, 0, 2]
    assert out["r"] == [1, 2, 1, 1, 2]
    assert out["c"] == [1, 1, 1, 0, 0]
    assert out["s"] == [10, 10, 4, None, None]
    assert out["m"] == [10, 10, 4, None, None]


def test_sum_wraps_to_signed_128_bits():
    big = (1 << 127) - 1
    out = W.window({"a": [big, 1, 1]}, [], [], (None, None), [("sum", "a", "s")])[1]["s"]
    assert out == [W.wrap128(big + 2)] * 3 == [-(1 << 127) + 1] * 3
