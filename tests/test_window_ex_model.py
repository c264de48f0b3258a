"""The model of the RANGE frames and the ranking, offset and value window functions (tests/_windowref_ex.py) pinned to hand-worked
answers, and its ROWS mode to tests/_windowref.py on seeded tables."""
import random

import pytest

import _windowref as W
import _windowref_ex as X

# source rows 0..7; PARTITION BY p ORDER BY o puts them at window positions 0..7 as rows 0, 1, 2, 4, 3 | 5, 6 | 7 (NULLs last, ties in
# source order), so x reads 1, 2, 3, 5, 4 | 6, NULL | 8 in window order; under o DESC the order is rows 3, 4, 1, 2, 0 | 5, 6 | 7
T = {"p": [1, 1, 1, 1, 1, 2, 2, None], "o": [10, 20, 20, None, 30, 5, 5, 1], "x": [1, 2, 3, 4, 5, 6, None, 8]}
ASC, DESC = [("o", False)], [("o", True)]


def run(frame, funcs, order=ASC, mode="range"):
    return X.window_ex(T, ["p"], order, frame, funcs, mode)[1]


def test_order_of_the_small_table():
    assert X.window_ex(T, ["p"], ASC, (None, 0), [("row_number", None, "rn")])[0] == [0, 1, 2, 4, 3, 5, 6, 7]
    assert X.window_ex(T, ["p"], DESC, (None, 0), [("row_number", None, "rn")])[0] == [3, 4, 1, 2, 0, 5, 6, 7]


def test_ranking_functions():
    r = run((None, 0), [("sql_rank", None, "rk"), ("dense_rank", None, "dr"), ("percent_rank", None, "pr"), ("cume_dist", None, "cd"),
                        ("row_number", None, "rn")])
    assert r["rk"] == [1, 2, 2, 4, 5, 1, 1, 1]
    assert r["dr"] == [1, 2, 2, 3, 4, 1, 1, 1]
    assert r["pr"] == [0.0, 0.25, 0.25, 0.75, 1.0, 0.0, 0.0, 0.0]  # the last partition has one row: 0
    assert r["cd"] == [0.2, 0.6, 0.6, 0.8, 1.0, 1.0, 1.0, 1.0]
    assert r["rn"] == [1, 2, 3, 4, 5, 1, 2, 1]  # RANGE: the position in the partition
    # the ranks ignore the frame and the mode; without order keys a partition is one peer group
    assert run((-1, 1), [("sql_rank", None, "rk")], mode="rows")["rk"] == r["rk"]
    nok = X.window_ex(T, ["p"], [], (None, None), [("sql_rank", None, "rk"), ("dense_rank", None, "dr"), ("cume_dist", None, "cd")])[1]
    assert nok == {"rk": [1] * 8, "dr": [1] * 8, "cd": [1.0] * 8}


def test_ntile():
    assert run((None, 0), [("ntile", None, "t", 2)])["t"] == [1, 1, 1, 2, 2, 1, 2, 1]  # len 5 % 2: the first bucket holds 3
    assert run((None, 0), [("ntile", None, "t", 7)])["t"] == [1, 2, 3, 4, 5, 1, 2, 1]  # len < n: 1..len
    assert run((None, 0), [("ntile", None, "t", 1)])["t"] == [1] * 8
    assert [X._ntile(j, 10, 3) for j in range(10)] == [1, 1, 1, 1, 2, 2, 2, 3, 3, 3]


def test_lag_lead():
    r = run((None, 0), [("lag", "x", "l1"), ("lag", "x", "ld", 1, -1), ("lead", "x", "e2", 2), ("lag", "x", "l0", 0), ("lead", "x", "ed", 1, 99)])
    assert r["l1"] == [None, 1, 2, 3, 5, None, 6, None]
    assert r["ld"] == [-1, 1, 2, 3, 5, -1, 6, -1]  # the default only outside the partition
    assert r["e2"] == [3, 5, 4, None, None, None, None, None]
    assert r["l0"] == [1, 2, 3, 5, 4, 6, None, 8]
    assert r["ed"] == [2, 3, 5, 4, 99, None, 99, 99]  # LEAD into the NULL x of row 6 stays NULL


def test_value_functions_over_the_default_range_frame():
    r = run((None, 0), [("first_value", "x", "f"), ("last_value", "x", "l"), ("nth_value", "x", "n2", 2), ("nth_value", "x", "n9", 9)])
    assert r["f"] == [1, 1, 1, 1, 1, 6, 6, 8]
    assert r["l"] == [1, 3, 3, 5, 4, None, None, 8]  # RESPECT NULLS: the last peer's NULL
    assert r["n2"] == [None, 2, 2, 2, 2, None, None, None]
    assert r["n9"] == [None] * 8
    rows = run((None, 0), [("last_value", "x", "l")], mode="rows")
    assert rows["l"] == [1, 2, 3, 5, 4, 6, None, 8]


def test_default_range_frame_includes_every_peer():
    r = run((None, 0), [("sum", "x", "s"), ("count_star", None, "c"), ("count", "x", "cx"), ("min", "x", "mn"), ("max", "x", "mx")])
    assert r["s"] == [1, 6, 6, 11, 15, 6, 6, 8]
    assert r["c"] == [1, 3, 3, 4, 5, 2, 2, 1]
    assert r["cx"] == [1, 3, 3, 4, 5, 1, 1, 1]
    assert r["mn"] == [1, 1, 1, 1, 1, 6, 6, 8]
    assert r["mx"] == [1, 3, 3, 5, 5, 6, 6, 8]
    assert run((None, 0), [("sum", "x", "s")], mode="rows")["s"] == [1, 3, 6, 11, 15, 6, 6, 8]
    assert run((0, 0), [("sum", "x", "s")])["s"] == [1, 5, 5, 5, 4, 6, 6, 8]  # the peers alone


def test_range_offsets_asc():
    r = run((-10, 0), [("sum", "x", "s"), ("count_star", None, "c")])
    assert r["s"] == [1, 6, 6, 10, 4, 6, 6, 8]  # the NULL-key row: its NULL peers
    assert r["c"] == [1, 3, 3, 3, 1, 2, 2, 1]
    # 1 FOLLOWING AND 5 FOLLOWING: no such key anywhere, so every non-NULL row's frame is empty
    r = run((1, 5), [("sum", "x", "s"), ("count_star", None, "c"), ("count", "x", "cx"), ("max", "x", "m"), ("first_value", "x", "f"),
                     ("last_value", "x", "l"), ("nth_value", "x", "n", 1)])
    assert r["s"] == [None, None, None, None, 4, None, None, None]
    assert r["c"] == [0, 0, 0, 0, 1, 0, 0, 0]
    assert r["cx"] == r["c"]
    assert r["m"] == r["s"] == r["f"] == r["l"] == r["n"]
    # 1 FOLLOWING AND UNBOUNDED FOLLOWING: the head stops at the NULL rows after the keys (they are after every key), as in PostgreSQL
    r = run((1, None), [("sum", "x", "s"), ("count_star", None, "c")])
    assert r["s"] == [14, 9, 9, 4, 4, None, None, None]
    assert r["c"] == [4, 2, 2, 1, 1, 0, 0, 0]
    # 10 PRECEDING AND 10 FOLLOWING
    assert run((-10, 10), [("sum", "x", "s")])["s"] == [6, 11, 11, 10, 4, 6, 6, 8]


def test_range_offsets_desc():
    # window order x: 4, 5, 2, 3, 1 | 6, NULL | 8 with o NULL, 30, 20, 20, 10 | 5, 5 | 1; 10 PRECEDING reaches keys up to key + 10
    r = run((-10, 0), [("sum", "x", "s")], order=DESC)
    assert r["s"] == [4, 5, 10, 10, 6, 6, 6, 8]
    # UNBOUNDED PRECEDING AND 5 PRECEDING: keys >= key + 5 and the NULL rows before them
    r = run((None, -5), [("sum", "x", "s"), ("count_star", None, "c")], order=DESC)
    assert r["s"] == [4, 4, 9, 9, 14, None, None, None]
    assert r["c"] == [1, 1, 2, 2, 4, 0, 0, 0]
    # 0 AND 10 FOLLOWING: the current peers down to key - 10
    assert run((0, 10), [("sum", "x", "s")], order=DESC)["s"] == [4, 10, 6, 6, 1, 6, 6, 8]


def test_range_offsets_at_the_extremes():
    big = (1 << 63) - 1
    t = {"k": [big, big - 3, -big - 1, None, 0], "x": [1, 2, 3, 4, 5]}
    # order: -2^63, 0, 2^63 - 4, 2^63 - 1, NULL; key + 5 of the last key is past every key, not a wrapped negative
    r = X.window_ex(t, [], [("k", False)], (0, 5), [("sum", "x", "s")], "range")[1]
    assert r["s"] == [3, 5, 3, 1, 4]
    r = X.window_ex(t, [], [("k", False)], (-5, 0), [("sum", "x", "s")], "range")[1]
    assert r["s"] == [3, 5, 2, 3, 4]
    r = X.window_ex(t, [], [("k", True)], (-5, 0), [("sum", "x", "s")], "range")[1]  # DESC: NULL first, then 2^63 - 1 ...
    assert r["s"] == [4, 1, 3, 5, 3]


def test_rows_mode_equals_the_rows_model():
    frames = [(None, 0), (None, None), (-3, 2), (0, 0), (2, 5), (-5, -2), (None, 3), (-2, None)]
    funcs = [("row_number", None, "rn"), ("count_star", None, "cs"), ("count", "a", "c"), ("sum", "a", "s"), ("min", "a", "mn"), ("max", "a", "mx")]
    for seed in range(12):
        rng = random.Random(seed)
        n = rng.randrange(0, 60)
        cols = {"p": [rng.choice([None, 1, 2, 3]) for _ in range(n)], "o": [rng.choice([None, 1, 2, 3, 4]) for _ in range(n)],
                "a": [rng.choice([None, rng.randrange(-100, 100)]) for _ in range(n)]}
        for frame in frames:
            for order in ([("o", False)], [("o", True)], []):
                assert X.window_ex(cols, ["p"], order, frame, funcs, "rows") == W.window(cols, ["p"], order, frame, funcs), (seed, frame, order)


@pytest.mark.parametrize("desc", [False, True])
def test_range_frames_against_a_brute_force_reading(desc):
    """every frame of every row as the set of rows PostgreSQL's frame head and tail walk over, on seeded tables with NULL keys"""
    for seed in range(8):
        rng = random.Random(seed)
        n = rng.randrange(1, 40)
        cols = {"p": [rng.choice([None, 1, 2]) for _ in range(n)], "o": [rng.choice([None] + list(range(-6, 7))) for _ in range(n)],
                "a": list(range(n))}
        order = [("o", desc)]
        perm = W.window_order(cols, ["p"], order)
        for frame in [(-3, 0), (-2, 2), (1, 4), (-4, -1), (None, 2), (-2, None), (0, 3)]:
            got = X.window_ex(cols, ["p"], order, frame, [("count_star", None, "c"), ("first_value", "a", "f")], "range")[1]
            for i in range(n):
                ri = perm[i]
                same = [q for q in range(n) if cols["p"][perm[q]] == cols["p"][ri]]
                k = cols["o"][ri]

                def before(q, off):  # row q lies before the bound key + off (in the order's direction)
                    kq = cols["o"][perm[q]]
                    if k is None:
                        return kq is not None and not desc  # NULLs: last ASC, first DESC; a NULL row's offset bound is its peers
                    if kq is None:
                        return desc
                    return kq > k - off if desc else kq < k + off

                def after(q, off):
                    kq = cols["o"][perm[q]]
                    if k is None:
                        return kq is not None and desc
                    if kq is None:
                        return not desc
                    return kq < k - off if desc else kq > k + off
                fr, to = frame
                rows = [q for q in same if (fr is None or not before(q, fr)) and (to is None or not after(q, to))]
                assert got["c"][i] == len(rows), (seed, frame, i)
                assert got["f"][i] == (cols["a"][perm[rows[0]]] if rows else None), (seed, frame, i)
