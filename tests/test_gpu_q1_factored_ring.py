"""The factored Q1 kernel's stage ring and row runs (kernels.cu scanQ1FactoredKernel): STAGES stages of FRAMES tiles in shared memory,
each thread decoding runs of RUN adjacent rows of one tile from one shared load per column, and cell words folded after every frame (a
stage, or one tile read with plain loads, two rows per thread).  Every case is exact against tests/_piperef.py, with the encoded copy and
with Arrow cells, and counts the batches that ran the factored kernel (kernel family "scan_groupby_factored")."""
import pytest

from test_gpu_encoded_scan import BLOCK_ROWS, Q1, SCHEMA, TILE_ROWS, check, ctx, read_groups, rt, sig_aggs, table, values  # noqa: F401
from test_gpu_encoded_scan_bounds import SHIPDATE
from test_gpu_encoded_scan_factored import check_q1, one_cell
from test_gpu_encoded_scan_stages import tpch_values
from test_gpu_q1_factored_kernel import fast_tpch_values
import _piperef as P

pytestmark = pytest.mark.gpu
FRAMES, STAGES, RUN = 4, 2, 4  # kernels.cu kFacTiles, kFacStages and the factored kernel's RUN
RING_ROWS = FRAMES * TILE_ROWS  # rows of one stage


def resident_grid(ctx):
    """CTAs of the factored kernel at TPC-H widths: three per SM"""
    return 3 * ctx.info()["sm_count"]


def test_stage_counts_not_a_multiple_of_the_ring(ctx):
    """every CTA wraps the ring: a third of them run STAGES + 2 stages, the others STAGES + 1, then the tail tiles"""
    grid = resident_grid(ctx)
    n = ((STAGES + 1) * grid + grid // 3) * RING_ROWS + (FRAMES - 1) * TILE_ROWS + 5
    vals = fast_tpch_values(90, n)
    check_q1(ctx, table(ctx, vals), vals, factored=1, filters=(SHIPDATE,))


@pytest.mark.parametrize("stages", [0, 2 * STAGES + 1])
@pytest.mark.parametrize("tiles", range(FRAMES))
def test_tail_classes(ctx, stages, tiles):
    """0 or more full stages, then 0 to FRAMES - 1 full tiles and a partial tile, all read with plain loads after the ring"""
    vals = tpch_values(91 + tiles, stages * RING_ROWS + tiles * TILE_ROWS + 300 + 53 * tiles)
    check_q1(ctx, table(ctx, vals), vals, factored=1)


def test_consecutive_frames_at_the_word_budget(ctx):
    """every row of one block in one (group, d, t) cell with ep - min and qty - min up to 2^28 - 1 and 2^21 - 1: each frame fills
    the cell's words as far as they go, frame after frame, stages and tail tiles alike"""
    n = (4 * STAGES + 1) * RING_ROWS + 3 * TILE_ROWS + 17
    assert n <= BLOCK_ROWS
    vals = values(92, n, "tpch")
    lo = 1_000_000
    one_cell(vals, 0, lo, lo + (1 << 28) - 1, 93)
    vals["b"][1], vals["b"][n - 1] = lo + (1 << 28) - 1, lo + (1 << 28) - 1
    vals["a"][2], vals["a"][n - 2] = (1 << 21) - 1, (1 << 21) - 1
    check_q1(ctx, table(ctx, vals), vals, factored=1)


def test_fifth_group_in_odd_and_even_frames(ctx):
    """CTA 0 sees a 5th group first in its second frame, CTA 1 in its third; from the middle of CTA 2's second frame on, rows cycle
    through 7 groups, so its register groups fill up inside that frame"""
    grid = resident_grid(ctx)
    n = (2 * grid + 3) * RING_ROWS + TILE_ROWS + 11
    vals = fast_tpch_values(94, n)
    for r in range(0, 2 * RING_ROWS, 97):
        vals["k"][grid * RING_ROWS + r], vals["k2"][grid * RING_ROWS + r] = 7, 1
        vals["k"][(2 * grid + 1) * RING_ROWS + r], vals["k2"][(2 * grid + 1) * RING_ROWS + r] = 7, 1
    start = (grid + 2) * RING_ROWS + RING_ROWS // 2
    for r in range(start, start + RING_ROWS):
        g = r % 7
        vals["k"][r], vals["k2"][r] = g, g % 3
    check_q1(ctx, table(ctx, vals), vals, factored=1, filters=(SHIPDATE,))


@pytest.mark.parametrize("n", [RING_ROWS, TILE_ROWS, 100])
def test_one_frame(ctx, n):
    """one stage, one full tile or one partial tile: the kernel's only frame is folded at the flush"""
    vals = tpch_values(95, n)
    check_q1(ctx, table(ctx, vals), vals, factored=1)


def test_runs_next_to_the_tile_edges(ctx):
    """the RUN-row runs on either side of every tile edge inside a stage carry groups, discounts, taxes and filter values of their
    own, so a run that read across an edge or into a tile's header would show"""
    n = 3 * RING_ROWS + 7
    vals = tpch_values(96, n)
    cut = P.date32("1998-09-02")
    for s in range(3):
        for f in range(1, FRAMES):
            edge = s * RING_ROWS + f * TILE_ROWS
            for i, r in enumerate(range(edge - RUN, edge + RUN)):
                vals["k"][r], vals["k2"][r] = 5 + (i % 2), 1 + f
                vals["c"][r], vals["d"][r] = (3 * i + f) % 11, (5 * i + s) % 9
                vals["dt"][r] = cut + (i % 3) - 1
    check_q1(ctx, table(ctx, vals), vals, factored=1)


def test_captured_replays(ctx):
    vals = tpch_values(97, (3 * STAGES + 1) * RING_ROWS + 2 * TILE_ROWS + 99)
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
        for _ in range(3):
            g.launch()
            assert read_groups(ctx, s, len(aggs)) == want
    finally:
        g.destroy()
        rt().state_destroy(ctx, s)
