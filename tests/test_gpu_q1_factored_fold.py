"""The factored Q1 kernel's fold interval (kernels.cu scanQ1FactoredKernel, factoredFold): the launcher splits ep - min_ep into its low s
bits and the rest and folds the four cell words {L, H, Q, N} into 64-bit sums only every K frames, s and K chosen from the batch's
ranges so that no word overflows in K frames of 2048 rows.  Every case is exact against tests/_piperef.py and counts the batches that
ran the factored kernel (kernel family "scan_groupby_factored")."""
import numpy as np
import pytest

from test_gpu_encoded_scan import Q1, SCHEMA, TILE_ROWS, ctx, read_groups, rt, sig_aggs, table  # noqa: F401
from test_gpu_encoded_scan_bounds import SHIPDATE
from test_gpu_encoded_scan_factored import check_q1
from test_gpu_q1_factored_kernel import fast_tpch_values
from test_gpu_q1_factored_ring import RING_ROWS, resident_grid
import _piperef as P

pytestmark = pytest.mark.gpu
MAX_WORD = (1 << 32) - 1


def fold_of(ep_range, qty_range):
    """(s, K) as factoredFold chooses them: the smallest s in [0, 28] that allows the largest K"""
    best = (20, 0)
    for s in range(29):
        k = MAX_WORD // (max((1 << s) - 1, ep_range >> s, qty_range, 1) * RING_ROWS)
        if k > best[1]:
            best = (s, k)
    return best


def batch_fold(vals, a, z):
    span = lambda name: max(vals[name][a:z]) - min(vals[name][a:z])  # noqa: E731
    return fold_of(span("b"), span("a"))


def spread(vals, name, a, z, lo, hi, seed):
    """rows a..z of column `name` uniform in [lo, hi], both ends present"""
    xs = [int(x) for x in np.random.default_rng(seed).integers(lo, hi, z - a, endpoint=True)]
    xs[0], xs[-1] = lo, hi
    vals[name][a:z] = xs


def one_cell_at_the_top(vals, a, z, ep_lo, ep_range, qty_range):
    """rows a..z in one (group, c, d) cell, ep and qty at the top of their ranges except for the minima in row a: every frame adds as
    much to the cell's words as the batch bounds allow"""
    for name, v in (("k", 1), ("k2", 0), ("c", 7), ("d", 3)):
        vals[name][a:z] = [v] * (z - a)
    vals["dt"][a:z] = [P.date32("1995-06-17")] * (z - a)
    vals["b"][a:z] = [ep_lo + ep_range] * (z - a)
    vals["a"][a:z] = [qty_range] * (z - a)
    vals["b"][a], vals["a"][a] = ep_lo, 0


@pytest.mark.parametrize("k,qty_range,s,extra,tiles", [(1, (1 << 21) - 1, 7, 3, 2), (2, (1 << 20) - 1, 8, 7, 1),
                                                       (3, MAX_WORD // (3 * RING_ROWS), 9, 5, 3)])
def test_words_at_their_limit_across_k_frames(ctx, k, qty_range, s, extra, tiles):
    """ep - min_ep at 2^28 - 1 and qty - min_qty at the top of the range that gives K on every row, all in one cell: K frames fill the
    H and Q words to within one frame of 2^32, so a fold one frame late overflows.  K * grid + extra stages: CTAs 0 .. extra - 1 fold at
    stage K (ring slot K % 2: 1, 0 and 1), the others run exactly K stages, and the tail tiles go to CTAs extra, extra + 1, .., which
    fold directly before them"""
    grid = resident_grid(ctx)
    n = (k * grid + extra) * RING_ROWS + tiles * TILE_ROWS + 300
    vals = fast_tpch_values(200 + k, n)
    one_cell_at_the_top(vals, 0, n, 1_000_000, (1 << 28) - 1, qty_range)
    assert batch_fold(vals, 0, n) == (s, k)
    check_q1(ctx, table(ctx, vals), vals, factored=1, filters=(SHIPDATE,))


def test_tpch_batch_folds_only_at_the_flush(ctx):
    """TPC-H ranges give s = 12 and K = 427, more frames than any CTA runs here: the words are folded only at the end"""
    grid = resident_grid(ctx)
    n = (grid + grid // 2) * RING_ROWS + 2 * TILE_ROWS + 41
    vals = fast_tpch_values(210, n)
    assert batch_fold(vals, 0, n) == (12, 427)
    check_q1(ctx, table(ctx, vals), vals, factored=1, filters=(SHIPDATE,))


@pytest.mark.parametrize("ep_range,fold", [((1 << 28) - 1, (14, 128)), (3, (0, 427))])
def test_split_at_both_ends(ctx, ep_range, fold):
    """ep - min_ep up to 2^28 - 1 (s = 14, both ep words bind K) or up to 3 (s = 0: L is always 0 and H holds the whole offset), with
    TPC-H quantities"""
    n = 200 * RING_ROWS + TILE_ROWS + 7
    vals = fast_tpch_values(220, n)
    spread(vals, "b", 0, n, 90_000, 90_000 + ep_range, 221)
    assert batch_fold(vals, 0, n) == fold
    check_q1(ctx, table(ctx, vals), vals, factored=1, filters=(SHIPDATE,))


def test_fifth_group_right_after_a_fold(ctx):
    """K = 2: CTAs 0 and 1 run 3 stages and fold at the start of stage 2; a 5th group appears first in the middle of CTA 0's stage 2
    and in the first row of CTA 1's"""
    grid = resident_grid(ctx)
    n = (2 * grid + 2) * RING_ROWS + TILE_ROWS + 5
    vals = fast_tpch_values(230, n)
    spread(vals, "a", 0, n, 0, (1 << 20) - 1, 231)
    assert batch_fold(vals, 0, n) == (4, 2)
    for r in list(range(2 * grid * RING_ROWS + RING_ROWS // 2, (2 * grid + 1) * RING_ROWS, 13)) + [(2 * grid + 1) * RING_ROWS]:
        vals["k"][r], vals["k2"][r] = 7, 1
    check_q1(ctx, table(ctx, vals), vals, factored=1, filters=(SHIPDATE,))


def test_captured_replays_over_batches_with_different_folds(ctx):
    """a TPC-H batch (s = 12, K = 427) and a batch with its words at the limit of K = 2 (s = 8), each launch with its own s and K"""
    grid = resident_grid(ctx)
    n0 = 3 * RING_ROWS + 2 * TILE_ROWS + 99
    n = n0 + (2 * grid + 3) * RING_ROWS + TILE_ROWS + 17
    vals = fast_tpch_values(240, n)
    spread(vals, "a", 0, n0, 100, 5000, 241)
    spread(vals, "b", 0, n0, 90_000, 10_500_000, 242)
    one_cell_at_the_top(vals, n0, n, 500_000, (1 << 28) - 1, (1 << 20) - 1)
    assert batch_fold(vals, 0, n0) == (12, 427) and batch_fold(vals, n0, n) == (8, 2)
    src = table(ctx, vals, cuts=(n0,))
    keys, aggs = sig_aggs(Q1)
    filters = list(SHIPDATE)
    want = P.scan_groupby(vals, SCHEMA, filters, keys, aggs)
    check_q1(ctx, src, vals, factored=2, filters=(SHIPDATE,))  # eager, and builds the copy outside the capture
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
