"""The factored Q1 kernel (kernels.cu scanQ1FactoredKernel) on shapes of its own: two TMA stages in flight per CTA, single-buffered
cell words folded after every frame (a stage of kEncFrames tiles, or one tail tile read with plain loads), register keys compared as
one packed word, and the shared / HBM fallback for groups past the register set.  Every case is exact against tests/_piperef.py, with
the encoded copy and with Arrow cells, and counts the batches that ran the factored kernel (kernel family "scan_groupby_factored")."""
import numpy as np
import pytest

from test_gpu_encoded_scan import COLS, SCHEMA, Q1, check, ctx, read_groups, rt, sig_aggs, table  # noqa: F401
from test_gpu_encoded_scan_bounds import SHIPDATE
from test_gpu_encoded_scan_factored import check_q1
from test_gpu_encoded_scan_stages import STAGE_ROWS, tpch_values
import _piperef as P

pytestmark = pytest.mark.gpu
TILE_ROWS = STAGE_ROWS // 4


def fast_tpch_values(seed, n):
    """TPC-H-shaped rows drawn with numpy (large tables): 4 groups, 11 discounts, 9 taxes, shipdates around Q1's cut"""
    rng = np.random.default_rng(seed)
    cut = P.date32("1998-09-02")
    ints = lambda lo, hi: [int(x) for x in rng.integers(lo, hi, n, endpoint=True)]  # noqa: E731
    v = {"k": ints(0, 1), "k2": ints(0, 1), "i": ints(-100, 100), "dt": ints(cut - 2000, cut + 100), "fs": ints(0, 1000),
         "a": ints(100, 5000), "b": ints(90_000, 10_500_000), "c": ints(0, 10), "d": ints(0, 8), "s": [b"x"] * n}
    assert set(v) == {c for c, _, _, _ in COLS}
    return v


def test_stage_counts_not_a_multiple_of_the_pipeline(ctx):
    """an odd number of full stages above twice any resident grid: some CTA runs an odd number of stages (3) through the two-stage
    ring, then the tail tiles"""
    n = 793 * STAGE_ROWS + 2 * TILE_ROWS + 333
    vals = fast_tpch_values(80, n)
    check_q1(ctx, table(ctx, vals), vals, factored=1, filters=(SHIPDATE,))


@pytest.mark.parametrize("stages,tiles,rest", [(0, 1, 0), (0, 3, 77), (0, 0, 300), (2, 1, 0), (2, 2, 5), (3, 3, 511), (1, 0, 1)])
def test_tail_classes(ctx, stages, tiles, rest):
    """0 or more full stages, then 0 to 3 full tiles and a partial tile read with plain loads"""
    vals = tpch_values(81 + stages, stages * STAGE_ROWS + tiles * TILE_ROWS + rest)
    check_q1(ctx, table(ctx, vals), vals, factored=1)


def test_fifth_group_in_the_last_stage(ctx):
    """4 register groups everywhere; a 5th group appears first in the table's last full stage (some CTA's last) and in the tail"""
    n = 5 * STAGE_ROWS + TILE_ROWS + 9
    vals = tpch_values(82, n)
    for r in range(n):
        vals["k"][r], vals["k2"][r] = r % 2, (r // 2) % 2
    last = 4 * STAGE_ROWS
    for r in list(range(last + 100, last + 140)) + [n - 3]:
        vals["k"][r], vals["k2"][r] = 7, 1
    check_q1(ctx, table(ctx, vals), vals, factored=1)


def test_register_groups_fill_up_mid_stage(ctx):
    """stage 0 starts with one group; from its middle on rows cycle through 7, so the register groups fill up inside the stage and the
    rest go to the shared sums"""
    n = 3 * STAGE_ROWS + 17
    vals = tpch_values(83, n)
    for r in range(n):
        g = 0 if r < STAGE_ROWS // 2 else r % 7
        vals["k"][r], vals["k2"][r] = g, g % 3
    check_q1(ctx, table(ctx, vals), vals, factored=1)


def test_captured_replays_over_stages_and_tail(ctx):
    vals = tpch_values(84, 7 * STAGE_ROWS + 3 * TILE_ROWS + 100)
    src = table(ctx, vals)
    keys, aggs = sig_aggs(Q1)
    filters = list(SHIPDATE)
    want = P.scan_groupby(vals, SCHEMA, filters, keys, aggs)
    check(ctx, src, vals, keys, aggs, filters)  # eager, and builds the copy outside the capture
    ctx.graph_begin()
    s = rt().groupby_state(ctx, len(keys), len(aggs), 64)
    rt().run_pipeline(ctx, "scan_groupby", src, filters=filters, keys=keys, aggs=aggs, sink=s)
    g = ctx.graph_end()
    try:
        for _ in range(4):
            g.launch()
            assert read_groups(ctx, s, len(aggs)) == want
    finally:
        g.destroy()
        rt().state_destroy(ctx, s)
