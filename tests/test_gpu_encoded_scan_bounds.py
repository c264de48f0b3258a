"""The per-tile 64-bit path of the encoded Q1 scan with a one-column int32 filter (kernels.cu scanGroupByKernel, aggBound64): a
tile whose header bounds prove every product a non-negative int64 below 2^61 sums in 64-bit registers, folded into the i128 sums
before they could overflow; every other tile, the tail tile and other filters take the general path (Q6 runs on the same data as a
check of that path).  Each case runs with the encoded copy and with Arrow cells, both against the exact reference of
tests/_piperef.py."""
import numpy as np
import pytest

from test_gpu_encoded_scan import BLOCK_ROWS, Q1, Q6, check, ctx, sig_aggs, table, values  # noqa: F401  (ctx is a fixture)

pytestmark = pytest.mark.gpu
SHIPDATE = [("dt", "<=", "1998-09-02")]  # Q1's filter: one int32 column against one constant


def fill(vals, name, block, lo, hi, seed):
    """block `block` of column `name` uniform in [lo, hi], both ends present, so the block's header bounds are exactly lo and hi"""
    rng = np.random.default_rng(seed)
    a, b = block * BLOCK_ROWS, min((block + 1) * BLOCK_ROWS, len(vals[name]))
    xs = [int(x) for x in rng.integers(lo, hi, b - a, endpoint=True)]
    xs[0], xs[-1] = lo, hi
    vals[name][a:b] = xs


def tpch_block(vals, block, seed):
    fill(vals, "a", block, 100, 5000, seed)
    fill(vals, "b", block, 90_000, 10_500_000, seed + 1)
    fill(vals, "c", block, 0, 10, seed + 2)
    fill(vals, "d", block, 0, 8, seed + 3)


def check_q1_q6(ctx, src, vals, filters_q1=((), SHIPDATE), filters_q6=((),)):
    for f in filters_q1:
        keys, aggs = sig_aggs(Q1)
        check(ctx, src, vals, keys, aggs, list(f))
    for f in filters_q6:
        keys, aggs = sig_aggs(Q6)
        check(ctx, src, vals, keys, aggs, list(f))


def test_negative_bases_and_wide_columns(ctx):
    """block 0 proven; block 1 has a negative base in b; block 2 an 8-byte-wide d (its copy is W = 8 throughout)"""
    vals = values(31, 3 * BLOCK_ROWS + 300, "tpch")
    for blk in range(4):
        tpch_block(vals, blk, 100 + 10 * blk)
    fill(vals, "b", 1, -5_000, 9_000_000, 7)
    fill(vals, "d", 2, -10**17, 10**17, 8)
    check_q1_q6(ctx, table(ctx, vals), vals)


def test_operands_at_the_edge_of_the_proof(ctx):
    """each block puts one operand of b*(1-c)*(1+d) just inside or just outside [0, 2^31), or the product just below or above 2^61"""
    top = (1 << 31) - 1
    cases = [
        dict(b=(top - 300, top)),                                     # largest b the proof admits
        dict(b=(top - 300, top + 1)),                                 # b reaches 2^31
        dict(c=(0, 100)),                                             # 1 - c reaches 0
        dict(c=(0, 101)),                                             # 1 - c reaches -1
        dict(b=(0, 100), d=((1 << 31) - 102, top - 100)),             # 1 + d reaches 2^31 - 1
        dict(b=(0, 100), d=((1 << 31) - 102, top - 99)),              # 1 + d reaches 2^31
        dict(b=(top - 5, top), c=(100 - (1 << 15), 0), d=(0, (1 << 15) - 100)),      # product just below 2^61
        dict(b=(top - 5, top), c=(100 - (1 << 15), 0), d=(0, (1 << 15) - 99)),       # product just above 2^61
    ]
    vals = values(32, len(cases) * BLOCK_ROWS, "tpch")
    for blk, case in enumerate(cases):
        tpch_block(vals, blk, 200 + 10 * blk)
        for name, (lo, hi) in case.items():
            fill(vals, name, blk, lo, hi, 300 + blk)
    check_q1_q6(ctx, table(ctx, vals), vals, filters_q1=(SHIPDATE,))


def test_several_headroom_folds(ctx):
    """every product near 2^61: the 64-bit sums of a thread fold into i128 every other tile, over many tiles per CTA"""
    n = 17 * BLOCK_ROWS
    vals = values(33, n, "tpch")
    for blk in range(17):
        fill(vals, "a", blk, 100, 5000, 400 + blk)
        fill(vals, "b", blk, (1 << 30) + (1 << 29), (1 << 31) - 1, 500 + blk)
        fill(vals, "c", blk, 100 - (1 << 15), 100 - (1 << 14), 600 + blk)
        fill(vals, "d", blk, 1 << 14, (1 << 15) - 100, 700 + blk)
    check_q1_q6(ctx, table(ctx, vals), vals, filters_q1=(SHIPDATE,), filters_q6=())


@pytest.mark.parametrize("key_domain", [2, 10])
def test_groups_beyond_the_register_set(ctx, key_domain):
    """(k, k2) spans 6 groups (shared-memory sums past the 4 register groups) or 30 (the group table past the CTA's 16)"""
    vals = values(34, 2 * BLOCK_ROWS + 700, "tpch", key_domain=key_domain)
    for blk in range(3):
        tpch_block(vals, blk, 800 + 10 * blk)
    assert len(set(zip(vals["k"], vals["k2"]))) > (4 if key_domain == 2 else 16)
    check_q1_q6(ctx, table(ctx, vals), vals, filters_q6=())


def test_partial_tail_tile(ctx):
    """a proven batch whose last tile holds 265 rows, next to a batch smaller than one tile"""
    vals = values(35, BLOCK_ROWS + 777 + 100, "tpch")
    for blk in range(2):
        tpch_block(vals, blk, 900 + 10 * blk)
    check_q1_q6(ctx, table(ctx, vals, cuts=(BLOCK_ROWS + 777,)), vals)


def test_filters_outside_the_shaped_instance(ctx):
    """a constant outside int32, a range, a filter on a group key and two filter columns take the descriptor-driven filter"""
    vals = values(36, BLOCK_ROWS + 1000, "tpch")
    for blk in range(2):
        tpch_block(vals, blk, 1000 + 10 * blk)
    filters = [[("i", "<", 1 << 40)], [("i", ">", -(1 << 40))], [("i", ">", -50), ("i", "<=", 50)], [("k", "<", 3)],
               [("dt", "<=", "1998-09-02"), ("i", ">", 0)], [("i", ">=", -(1 << 31))], [("fs", "<=", "B")]]
    check_q1_q6(ctx, table(ctx, vals), vals, filters_q1=filters, filters_q6=filters[:2])
