"""The factored stage path of the encoded Q1 scan (kernels.cu scanGroupByKernel, FAC): when a batch's discount (c) and tax (d) take at
most kCells / 4 (c, d) pairs, its b and a ranges fit the word budgets (max - min below 2^28 and 2^21) and its bounds prove the 64-bit
product bound, the register groups sum per (group, c, d) cell in 32-bit shared words and the products run once per cell.  Every other
batch runs the per-row stage instance.  Each case runs with the encoded copy and with Arrow cells, both against the exact reference of
tests/_piperef.py, and counts the batches that ran the factored instance (kernel family "scan_groupby_factored")."""
import pytest

from test_gpu_encoded_scan import BLOCK_ROWS, Q1, SCHEMA, check, ctx, read_groups, rt, sig_aggs, table, values  # noqa: F401
from test_gpu_encoded_scan_bounds import SHIPDATE, fill, tpch_block
from test_gpu_encoded_scan_stages import STAGE_ROWS, tpch_values
import _piperef as P

pytestmark = pytest.mark.gpu


def check_q1(ctx, src, vals, factored, filters=((), SHIPDATE)):
    """each query exact; `factored` = how many of the table's batches run the factored instance under Q1's one-column filter (without
    a filter the encoded scan runs the descriptor-filter instance, which has no stage path)"""
    keys, aggs = sig_aggs(Q1)
    for f in filters:
        ctx.kernel_time_reset(True)
        try:
            check(ctx, src, vals, keys, aggs, list(f))
            assert ctx.kernel_time("scan_groupby_factored")[1] == (factored if list(f) == SHIPDATE else 0)
        finally:
            ctx.kernel_time_reset(False)


def block_cuts(n):
    return tuple(range(BLOCK_ROWS, n, BLOCK_ROWS))


def test_tpch_shaped_batches(ctx):
    """TPC-H domains (11 discounts, 9 taxes) over several blocks and batches, with and without Q1's filter"""
    vals = tpch_values(61, 3 * BLOCK_ROWS + 5 * STAGE_ROWS + 77)
    check_q1(ctx, table(ctx, vals, cuts=(BLOCK_ROWS + 3 * STAGE_ROWS,)), vals, factored=2)


@pytest.mark.parametrize("c_lo,d_hi,factored", [(85, 7, 1), (85, 8, 0), (-27, 0, 1), (-28, 0, 0), (100, 127, 1)])
def test_factor_domains_around_the_cell_count(ctx, c_lo, d_hi, factored):
    """4 * 16 * 8, 4 * 128 * 1 and 4 * 1 * 128 cells fill kCells exactly; 4 * 16 * 9 and 4 * 129 * 1 are one step past it (per-row
    path).  c stays <= 100, so 1 - c keeps the 64-bit proof"""
    n = 2 * BLOCK_ROWS + 3 * STAGE_ROWS + 100
    vals = tpch_values(62, n)
    for blk in range(3):
        fill(vals, "c", blk, c_lo, 100, 70 + blk)
        fill(vals, "d", blk, 0, d_hi, 80 + blk)
    check_q1(ctx, table(ctx, vals), vals, factored)


@pytest.mark.parametrize("name,lo,hi,factored", [("b", 90_000, 90_000 + (1 << 28) - 1, 1), ("b", 90_000, 90_000 + (1 << 28), 0),
                                                 ("b", 90_000, 90_000 + (1 << 29), 0), ("a", -7, -7 + (1 << 21) - 1, 1),
                                                 ("a", -7, -7 + (1 << 21), 0)])
def test_batch_ranges_at_the_word_budgets(ctx, name, lo, hi, factored):
    """TPC-H discounts and taxes with b or a spanning just inside or past its word budget across the batch (each block on its own
    inside it): a batch past it runs the per-row instance, register sums and all"""
    vals = tpch_values(72, 2 * BLOCK_ROWS + 300)
    mid = (lo + hi) // 2
    fill(vals, name, 0, lo, mid, 73)
    fill(vals, name, 1, mid, hi, 74)
    fill(vals, name, 2, mid, mid + 10, 75)
    check_q1(ctx, table(ctx, vals), vals, factored)


def test_negative_values_and_batch_minima(ctx):
    """negative discounts, taxes and quantities (factored: min * count is added back), then negative prices (no 64-bit proof: the batch
    runs the per-row instance); each batch has its own minima"""
    n = 3 * BLOCK_ROWS + 400
    vals = tpch_values(63, n)
    fill(vals, "c", 0, -5, 5, 90)
    fill(vals, "d", 0, -4, 4, 91)
    fill(vals, "a", 0, -2000, 3000, 92)
    fill(vals, "c", 1, 3, 13, 93)
    fill(vals, "d", 1, -8, 0, 94)
    fill(vals, "b", 2, -50_000, 9_000_000, 95)
    fill(vals, "c", 2, -10, 0, 96)
    fill(vals, "c", 3, 20, 30, 97)
    check_q1(ctx, table(ctx, vals, cuts=(BLOCK_ROWS, 2 * BLOCK_ROWS, 3 * BLOCK_ROWS)), vals, factored=3)


def one_cell(vals, blk, b_lo, b_top, seed):
    """block `blk` entirely in one (group, c, d) cell, b and a near the top of their words: the per-stage sums nearly fill them"""
    a, z = blk * BLOCK_ROWS, min((blk + 1) * BLOCK_ROWS, len(vals["b"]))
    for name, v in (("k", 1), ("k2", 2), ("c", 7), ("d", 3), ("i", 0)):
        vals[name][a:z] = [v] * (z - a)
    vals["dt"][a:z] = [P.date32("1995-06-17")] * (z - a)
    fill(vals, "b", blk, b_top - 1000, b_top, seed)
    vals["b"][a] = b_lo
    fill(vals, "a", blk, (1 << 21) - 500, (1 << 21) - 1, seed + 1)
    vals["a"][a] = 0


def test_every_row_in_one_cell_at_the_word_budgets(ctx):
    """batches 0 and 2: b - min b reaches 2^28 - 1 (factored, every stage's words near full, folded every stage); batch 1 reaches 2^28
    (one past the budget: the per-row instance)"""
    vals = values(64, 3 * BLOCK_ROWS, "tpch")
    lo = 1_000_000
    for blk, top in ((0, lo + (1 << 28) - 1), (1, lo + (1 << 28)), (2, lo + (1 << 28) - 1)):
        one_cell(vals, blk, lo, top, 100 + 10 * blk)
    check_q1(ctx, table(ctx, vals, cuts=block_cuts(3 * BLOCK_ROWS)), vals, factored=2)


def test_unproven_batches_between_factored_ones(ctx):
    """batch 1's b reaches 2^31 (no 64-bit proof) and batch 3's a spans more than 2^21: both run the per-row instance between factored
    batches of one table"""
    vals = tpch_values(65, 5 * BLOCK_ROWS + 3)
    fill(vals, "b", 1, (1 << 31) - 300, 1 << 31, 66)
    fill(vals, "a", 3, 0, 1 << 21, 67)
    check_q1(ctx, table(ctx, vals, cuts=block_cuts(5 * BLOCK_ROWS + 3)), vals, factored=4)


@pytest.mark.parametrize("key_domain", [2, 10])
def test_groups_beyond_the_register_set(ctx, key_domain):
    """6 groups (2 past the register groups, in shared sums) or 30 (past the CTA's 16, in the HBM table) next to factored groups"""
    vals = values(68, 2 * BLOCK_ROWS + 3 * STAGE_ROWS + 1, "tpch", key_domain=key_domain)
    for blk in range(3):
        tpch_block(vals, blk, 110 + 10 * blk)
    assert len(set(zip(vals["k"], vals["k2"]))) > (4 if key_domain == 2 else 16)
    check_q1(ctx, table(ctx, vals), vals, factored=1)


@pytest.mark.parametrize("n", [3 * STAGE_ROWS + 511, 3 * STAGE_ROWS + 1, STAGE_ROWS - 1, 100])
def test_partial_tail_tiles(ctx, n):
    vals = tpch_values(69, n)
    check_q1(ctx, table(ctx, vals), vals, factored=1)


def test_captured_query_replays(ctx):
    vals = tpch_values(70, BLOCK_ROWS + 3 * STAGE_ROWS + 700)
    fill(vals, "c", 1, -3, 7, 71)  # the second batch has other minima, baked into its launch
    src = table(ctx, vals, cuts=(BLOCK_ROWS + 5,))
    keys, aggs = sig_aggs(Q1)
    filters = list(SHIPDATE)
    want = P.scan_groupby(vals, SCHEMA, filters, keys, aggs)
    check(ctx, src, vals, keys, aggs, filters)  # eager, and builds the copy outside the capture
    ctx.graph_begin()
    s = rt().groupby_state(ctx, len(keys), len(aggs), 64)
    rt().run_pipeline(ctx, "scan_groupby", src, filters=filters, keys=keys, aggs=aggs, sink=s)
    g = ctx.graph_end()
    try:
        for _ in range(3):
            g.launch()
            assert read_groups(ctx, s, len(aggs)) == want
    finally:
        g.destroy()
        rt().state_destroy(ctx, s)
