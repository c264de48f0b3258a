"""Pins the exchange reference (tests/_exchref.py) on hand-worked values: the partition function against the oracle's hash, the Bloom
bits of a few keys, K10's semi-join rule, the receive-side arithmetic and a 64-bit merge whose low words carry into the high word."""
from collections import Counter

import pytest

import _exchref as X
import _piperef as P


def test_part_of_takes_the_top_bits_of_the_oracle_hash(oracle):
    # h64(1) = m ^ bswap(m), m = 0x9E3779B97F4A7C55: 0xCB4B33C6C6334BCB; the top word 0xCB4B33C6 = 3410703302
    assert X.h64(1) == 0xCB4B33C6C6334BCB
    assert [X.part_of(1, n) for n in (1, 2, 3, 7, 8, 64)] == [0, 1, 2, 5, 6, 50]  # floor(3410703302 * n / 2^32)
    assert X.h64(0) == 0 and all(X.part_of(0, n) == 0 for n in (1, 7, 64))
    for k in (1, -1, 0, 12345, P.I32_MIN, P.I32_MAX, 10**9):
        h = oracle.lib.oracle_hash_i64(k) % (1 << 64)
        assert X.h64(k) == h
        for n in (1, 2, 3, 7, 8, 64):
            assert X.part_of(k, n) == (h >> 32) * n // (1 << 32)


def test_bloom_bits_of_a_few_keys():
    # key 0: h = 0, g = 0 → word 0, the three bit positions all 0
    assert X.bloom_word_bits(0, 1024) == (0, 1)
    # key 1: word = 0xCB4B33C6 & 1023 = 966; g = h * 0xD6E8FEB86659FD93 mod 2^64 has g >> 59 = 31, (g >> 54) & 31 = 21, (g >> 49) & 31 = 27
    g = (0xCB4B33C6C6334BCB * 0xD6E8FEB86659FD93) % (1 << 64)
    assert (g >> 59, (g >> 54) & 31, (g >> 49) & 31) == (31, 21, 27)
    assert X.bloom_word_bits(1, 1024) == (966, (1 << 31) | (1 << 27) | (1 << 21))
    assert X.bloom_word_bits(1, 4096) == (0xCB4B33C6 & 4095, (1 << 31) | (1 << 27) | (1 << 21))
    # a filter holds exactly the bits of its keys; the OR of two filters answers for both key sets
    f0, f1 = X.bloom_filter([0], 1024), X.bloom_filter([1], 1024)
    assert sum(bin(w).count("1") for w in f0) == 1 and sum(bin(w).count("1") for w in f1) == 3
    both = X.or_reduce([f0, f1])
    assert X.bloom_may_contain(both, 0) and X.bloom_may_contain(both, 1)
    assert not X.bloom_may_contain(f0, 1) and not X.bloom_may_contain(f1, 0)
    assert X.bloom_may_contain(None, 7)  # no filter: every key passes
    # geometry of create_shared_bloom: nextPow2(max(n, 2048) * 2) / 4 words
    assert [X.shared_bloom_words(n) for n in (0, 2048, 2049, 5000)] == [1024, 1024, 2048, 4096]
    # a plain table has a filter from 4096 directory slots (nextPow2(2 * expected)) on, a quarter word per slot
    assert [X.table_bloom_words(n) for n in (1000, 1024, 1025, 4096)] == [0, 0, 1024, 2048]


def test_partition_offsets_and_payloads():
    offs, parts = X.partition([1, 1, 0, -1], [[10, 11, 12, 13]], 2)
    assert offs == [0, 1, 4]  # part_of(0, 2) = 0; part_of(1, 2) = part_of(-1, 2) = 1
    assert parts[0] == Counter({(0, 12): 1}) and parts[1] == Counter({(1, 10): 1, (1, 11): 1, (-1, 13): 1})
    with pytest.raises(P.PipeError):
        X.partition([1], [], 65)


def test_k10_full_probe_is_a_semi_join():
    schema = {"k": ("int32", 0, 0), "v": ("int32", 0, 0), "a": ("decimal128", 18, 2)}
    cols = {"k": [5, 6, 7], "v": [50, 60, 70], "a": [-1, 2, 3]}
    multi = P.JoinTable("hash", 64, unique=False)
    for k, p in ((5, 1), (5, 2), (7, 3)):
        multi.insert(k, p)
    out = X.partition_send(cols, schema, [], ["k", "v", "a"], 1, probe=(multi, "k"))
    # row 5 matches twice but ships once; row 6 has no match; the decimal ships as its low 64 bits
    assert out == [[(X.pack(5, 50), (1 << 64) - 1), (X.pack(7, 70), 3)]]
    with pytest.raises(P.PipeError) as e:
        X.partition_send(cols, schema, [], ["k", "$payload"], 1, probe=(multi, "k"))
    assert e.value.code == P.LDB_ERR_UNSUPPORTED
    uniq = P.JoinTable("hash", 64)
    uniq.insert(5, -9)
    want = [[], []]
    want[X.part_of(5, 2)].append((X.pack(5, -9),))
    assert X.partition_send(cols, schema, [], ["k", "$payload"], 2, probe=(uniq, "k")) == want
    assert X.pack(-1, -1) == (1 << 64) - 1 and X.unpack(X.pack(P.I32_MIN, 7)) == (P.I32_MIN, 7)
    assert X.stored([()] * 5, 3) == (5, True, 3) and X.stored([()] * 3, 3) == (3, False, 3)


def test_receive_side_arithmetic():
    assert X.publish_counts([[1, 2], [3, 4]]) == [[1, 3], [2, 4]]
    a, b = P.JoinTable("hash", 64), P.JoinTable("hash", 64)
    a.insert(1, 9)
    b.insert(2, 9)
    b.insert(3, 8)
    tup = [(X.pack(1, 2), 300, 25), (X.pack(1, 3), 7, 0), (X.pack(1, 2), (-4) % (1 << 64), 1)]
    # payloads agree only for (1, 2): 300 * (100 - 25) + (-4) * (100 - 1)
    assert X.probe_received_groupby(a, b, tup, 2) == {(9, 0): [300 * 75 - 4 * 99]}
    assert X.probe_received_groupby(a, b, tup[:1], 0) == {(9, 0): [300 * (1 - 25)]}
    s = P.JoinTable("hash", 64, unique=False)
    s.insert(4, 1)
    s.insert(4, 2)
    v = -(1 << 100)
    got = X.probe_received_groupby2(s, [(X.pack(4, -1), v % (1 << 64), (v >> 64) % (1 << 64))])
    assert got == {(-1, 1): [v], (-1, 2): [v]}
    assert X.received([[(1,), (2,), (3,)], [(4,)]], [2, 5], 3) == [(1,), (2,), (4,)]


def test_merge_reads_each_lane_at_the_target_width():
    # two 64-bit partials whose low words carry: 0xFFFF_FFFF_FFFF_FFFF (-1) + 1 → low word 0 with a carry into the high word;
    # a 64-bit lane reads the low word (0), a 128-bit lane the whole sum (2^64)
    shards = [{(1, 0): [(1 << 64) - 1, (1 << 64) - 1]}, {(1, 0): [1, 1]}]
    assert X.merge(shards, [True, False]) == {(1, 0): [0, 1 << 64]}
    # negative 64-bit sums sign-extended: -5 from two ranks' -2 and -3 stored as raw 128-bit cells
    assert X.merge([{(2, 0): [-2]}, {(2, 0): [-3]}, {}], [True]) == {(2, 0): [-5]}
    assert X.merge([{}, {}], [True, False], keyless=True) == {(): [0, 0]}
    assert X.merge([{(0, 0): [(1 << 127)]}, {(0, 0): [(1 << 127)]}], [False]) == {(0, 0): [0]}  # 128-bit sums wrap
    with pytest.raises(P.PipeError) as e:
        X.merge([{(k, 0): [1] for k in range(17)}], [True], capacity=16)
    assert e.value.code == P.LDB_ERR_CAPACITY
    assert X.allgather_small([b"a" * 16, b"b" * 16]) == [b"a" * 16, b"b" * 16]
    with pytest.raises(P.PipeError):
        X.allgather_small([b"a" * 8])
