"""The stage path of the encoded Q1 scan (kernels.cu scanGroupByKernel, encodedStages): a TMA stage holds FRAMES consecutive 512-row
tiles, the full tiles after the last full stage and the partial tail tile are read tile by tile, the filter and the key compares run on the
raw fields and the 64-bit proof admits products below 2^63 / (2 * FRAMES).  Each case runs with the encoded copy and with Arrow cells, both
against the exact reference of tests/_piperef.py, for Q1 with and without its one-column filter and for Q6."""
import pytest

import _piperef as P
from test_gpu_encoded_scan import BLOCK_ROWS, Q1, Q6, SCHEMA, TILE_ROWS, check, ctx, read_groups, rt, sig_aggs, table, values  # noqa: F401
from test_gpu_encoded_scan_bounds import SHIPDATE, check_q1_q6, fill, tpch_block

pytestmark = pytest.mark.gpu
FRAMES = 4  # kernels.cu kEncFrames
STAGE_ROWS = TILE_ROWS * FRAMES


def tpch_values(seed, n, key_domain=4):
    vals = values(seed, n, "tpch", key_domain=key_domain)
    for blk in range((n + BLOCK_ROWS - 1) // BLOCK_ROWS):
        tpch_block(vals, blk, seed + 10 * blk)
    return vals


@pytest.mark.parametrize("n", [3 * STAGE_ROWS - 1, 3 * STAGE_ROWS, 3 * STAGE_ROWS + 1, 3 * STAGE_ROWS + 511,
                               STAGE_ROWS - 1, TILE_ROWS + 3, 100])
def test_row_counts_around_a_stage(ctx, n):
    """full stages, then up to FRAMES - 1 full tiles and a partial tail tile; and batches shorter than one stage"""
    vals = tpch_values(41, n)
    check_q1_q6(ctx, table(ctx, vals), vals)


def test_odd_device_batches_in_one_table(ctx):
    cuts = (STAGE_ROWS + 7, 2 * STAGE_ROWS + 300, 5 * STAGE_ROWS + 301, 5 * STAGE_ROWS + 302)
    vals = tpch_values(42, 7 * STAGE_ROWS + 999)
    check_q1_q6(ctx, table(ctx, vals, cuts=cuts), vals)


def test_unproven_block_next_to_proven_ones(ctx):
    """block 1's b reaches 2^31, so its stages take the i128 path between proven stages of blocks 0 and 2"""
    vals = tpch_values(43, 2 * BLOCK_ROWS + 3 * STAGE_ROWS + 5)
    fill(vals, "b", 1, (1 << 31) - 300, 1 << 31, 44)
    check_q1_q6(ctx, table(ctx, vals), vals)


def test_products_at_the_stage_bound(ctx):
    """block 0's largest product is just below 2^63 / (2 * FRAMES) = 2^60 (proven, the 64-bit sums fold every stage), block 1's is
    exactly 2^60 (one past the bound)"""
    assert 2 * FRAMES == 8
    vals = tpch_values(45, 2 * BLOCK_ROWS)
    for blk, d_hi in ((0, (1 << 15) - 101), (1, (1 << 15) - 100)):
        fill(vals, "b", blk, (1 << 30) - 5, 1 << 30, 46 + blk)
        fill(vals, "c", blk, 100 - (1 << 15), 0, 48 + blk)
        fill(vals, "d", blk, 0, d_hi, 50 + blk)
    assert (1 << 30) * (1 << 15) * (100 + (1 << 15) - 100) == 1 << 60
    check_q1_q6(ctx, table(ctx, vals), vals, filters_q6=())


@pytest.mark.parametrize("key_domain", [2, 10])
def test_many_groups_inside_one_stage(ctx, key_domain):
    """(k, k2) spans 6 groups (past the 4 register groups) or 30 (past the CTA's 16) inside every stage"""
    vals = tpch_values(52, 2 * STAGE_ROWS + 1, key_domain=key_domain)
    assert len(set(zip(vals["k"][:STAGE_ROWS], vals["k2"][:STAGE_ROWS]))) > (4 if key_domain == 2 else 16)
    check_q1_q6(ctx, table(ctx, vals), vals, filters_q6=())


def test_filter_ops_on_the_raw_field(ctx):
    """every compare of the one-column filter, with constants inside, below and above a block's range"""
    vals = tpch_values(53, BLOCK_ROWS + 2 * STAGE_ROWS + 17)
    vals["i"] = [(j * 7919) % 1000 - 500 for j in range(len(vals["i"]))]
    filters = [[("i", op, c)] for op in ("=", "!=", "<", "<=", ">", ">=") for c in (-501, -500, 0, 499, 500, P.I32_MIN, P.I32_MAX)]
    filters += [[("dt", "<", "1970-01-01")], [("dt", ">=", "1970-01-01")]]
    keys, aggs = sig_aggs(Q1)
    src = table(ctx, vals)
    for f in filters:
        check(ctx, src, vals, keys, aggs, f)


def test_captured_query_replays(ctx):
    vals = tpch_values(54, 3 * STAGE_ROWS + 700)
    src = table(ctx, vals, cuts=(STAGE_ROWS + 3,))
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
