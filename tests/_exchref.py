"""Exact reference for the multi-GPU exchange layer (include/ldb_gpu.h "repartition (K6)", K10 LDB_PIPE_SCAN_PARTITION_SEND, K11
LDB_PIPE_SCAN_STAR_PROBE_SEND, the receive side, the K7 merges and the peer collectives) — plain Python, no GPU.

Written from the header's contract, restated:
  - a tuple goes to partition part_of(key, n) = ((h64(key) >> 32) * n) >> 32: the top bits of the reference hash;
  - the join tables' blocked Bloom filter: word (h >> 32) & mask, three bits of g = h * 0xD6E8FEB86659FD93 (g >> 59, (g >> 54) & 31,
    (g >> 49) & 31).  A table made by ldb_gpu_join_table_create_shared_bloom has nextPow2(max(n, 2048) * 2) / 4 words;
  - K10 ships {key | second << 32, low 64 bits of each decimal} per qualifying row; its full probe is a semi-join (one tuple per row
    with at least one match), so "$payload" needs a unique table.  A destination's cursor counts every tuple, the first `capacity` are
    stored and the rest set the overflow flag (cursor word 8);
  - K11 ships {kO | g0 << 32, lo, hi} per (match c of P, match g0 of S) with the i128 a * (1 - b) - c * d;
  - the receiver reads counts[s] = the cursor source s kept for it; insert_received inserts {key, payload} into a join table,
    probe_received_groupby sums a * (10^scale - b) over the pairs of matches whose payloads agree, _groupby2 groups by (g0, g1);
  - K7 adds the 128-bit cells per key; a lane is read at its target's width (a 64-bit lane as its low word, sign-extended);
  - allgather_small places rank r's block at r * slot; or_reduce ORs the ranks' words.
Multisets are collections.Counter of tuples; errors raise _piperef.PipeError with the LdbStatus the C-ABI reports."""
from collections import Counter
from typing import Dict, List, Optional, Sequence

import numpy as np

import _piperef as P
import _progref as R
from _piperef import LDB_ERR_CAPACITY, LDB_ERR_INVALID, LDB_ERR_UNSUPPORTED, PipeError, wrap64
from _progref import wrap128

M32 = (1 << 32) - 1
M64 = (1 << 64) - 1
BLOOM_MUL = 0xD6E8FEB86659FD93
SLOT_BYTES = 256 << 10
MAX_PEERS = 8


def h64(key: int) -> int:
    return int(P.h64([key])[0])


def part_of(key: int, n: int) -> int:
    return ((h64(key) >> 32) * n) >> 32


def parts_of(keys, n: int) -> np.ndarray:
    """part_of of an array of int32 keys (vectorised)"""
    top = P.h64(keys) >> np.uint64(32)
    return ((top * np.uint64(n)) >> np.uint64(32)).astype(np.int64)  # top < 2^32, n <= 64: no overflow


def pack(lo32: int, hi32: int) -> int:
    """one tuple word {lo32 : 32 | hi32 : 32} (both int32, stored as their bits)"""
    return (lo32 & M32) | ((hi32 & M32) << 32)


def unpack(w: int):
    lo, hi = w & M32, w >> 32
    return lo - (1 << 32) if lo >> 31 else lo, hi - (1 << 32) if hi >> 31 else hi


# ---------------------------------------------------------------------------------------------------- Bloom filter
def next_pow2(n: int) -> int:
    return 1 << (n - 1).bit_length()


def shared_bloom_words(expected_rows: int) -> int:
    return next_pow2(max(expected_rows, 2048) * 2) // 4


def table_bloom_words(expected_rows: int) -> int:
    """words of the filter of ldb_gpu_join_table_create / _create_pair (0: no filter below 4096 slots)"""
    slots = P.table_slots(expected_rows)
    return slots // 4 if slots >= 4096 else 0


def bloom_word_bits(key: int, words: int):
    h = h64(key)
    g = (h * BLOOM_MUL) & M64
    return (h >> 32) & (words - 1), (1 << (g >> 59)) | (1 << ((g >> 54) & 31)) | (1 << ((g >> 49) & 31))


def bloom_filter(keys, words: int) -> List[int]:
    f = [0] * words
    for k in keys:
        w, b = bloom_word_bits(k, words)
        f[w] |= b
    return f


def bloom_may_contain(f: Optional[List[int]], key: int) -> bool:
    if not f:
        return True  # a table without a filter passes every key
    w, b = bloom_word_bits(key, len(f))
    return f[w] & b == b


def or_reduce(filters: Sequence[Sequence[int]]) -> List[int]:
    out = [0] * len(filters[0])
    for f in filters:
        out = [a | b for a, b in zip(out, f)]
    return out


# ---------------------------------------------------------------------------------------------------- K6
def partition(keys: Sequence[int], payloads: Sequence[Sequence], n_parts: int):
    """ldb_gpu_partition_tuples: (offsets [n_parts + 1], [Counter of (key, payload...)] per partition)"""
    if not 1 <= n_parts <= 64:
        raise PipeError(LDB_ERR_INVALID, "n_parts must be in [1, 64]")
    parts = [Counter() for _ in range(n_parts)]
    dest = parts_of(list(keys), n_parts) if len(keys) else []
    for i, k in enumerate(keys):
        parts[dest[i]][(k,) + tuple(col[i] for col in payloads)] += 1
    offsets = [0]
    for p in parts:
        offsets.append(offsets[-1] + sum(p.values()))
    return offsets, parts


# ---------------------------------------------------------------------------------------------------- K10 / K11
def partition_send(cols, schema, filters, out_columns: Sequence[str], world: int, probe: Optional[tuple] = None, bloom_only: bool = False,
                   bloom: Optional[List[int]] = None, year: bool = False) -> List[List[tuple]]:
    """K10 of one source rank: the tuples (word tuples) it ships to each destination, in row order.  probe = (JoinTable, key column);
    with bloom_only the row is kept when `bloom` (the probe table's filter) may contain its key."""
    if not 2 <= len(out_columns) <= 4:
        raise PipeError(LDB_ERR_INVALID, "partition-send ships {key, second[, decimal[, decimal]]}")
    payload = out_columns[1] == "$payload"
    if payload and (probe is None or bloom_only):
        raise PipeError(LDB_ERR_INVALID, "$payload needs a full probe")
    if payload and not probe[0].unique:
        raise PipeError(LDB_ERR_UNSUPPORTED, "$payload over a probe table that is not unique")
    if year and payload:
        raise PipeError(LDB_ERR_INVALID, "the year expression applies to a shipped date32 column")
    for c in out_columns[2:]:
        if schema[c][0] != "decimal128":
            raise PipeError(LDB_ERR_UNSUPPORTED, "decimal tuple column")
    keep = P.filter_rows(cols, schema, filters)
    idx = probe[0].index() if probe is not None and not bloom_only else None
    out: List[List[tuple]] = [[] for _ in range(world)]
    dest = parts_of(cols[out_columns[0]], world) if keep else []
    for i, ok in enumerate(keep):
        if not ok:
            continue
        key = cols[out_columns[0]][i]
        second = None if payload else cols[out_columns[1]][i]
        if year:
            second = R.year_of_days(second)
        if probe is not None:
            pk = cols[probe[1]][i]
            if bloom_only:
                if not bloom_may_contain(bloom, pk):
                    continue
            else:
                hits = idx.get(pk, [])
                if not hits:
                    continue
                if payload:
                    second = hits[0][1] & 0x7FFFFFFF if probe[0].wide else hits[0][1]
        out[dest[i]].append((pack(key, second),) + tuple(cols[c][i] & M64 for c in out_columns[2:]))
    return out


def star_probe_send(cols, schema, filters, table_p: P.JoinTable, keys_p: tuple, table_s: P.JoinTable, key_s: str, key_o: str, values: tuple,
                    world: int) -> List[List[tuple]]:
    """K11 of one source rank: {kO | g0 << 32, lo, hi} per (match c of P, match g0 of S), to part_of(kO)"""
    if table_p.kind != "pair":
        raise PipeError(LDB_ERR_INVALID, "probe 0 of a star-probe-send pipeline is a composite-key table")
    if table_s.kind == "pair":
        raise PipeError(LDB_ERR_INVALID, "probe 1 of a star-probe-send pipeline is a single-key table")
    keep = P.filter_rows(cols, schema, filters)
    ip, is_ = table_p.index(), table_s.index()
    a, b, d = values
    out: List[List[tuple]] = [[] for _ in range(world)]
    for i, ok in enumerate(keep):
        if not ok:
            continue
        ko = cols[key_o][i]
        for ep in ip.get((cols[keys_p[0]][i], cols[keys_p[1]][i]), []):
            for es in is_.get(cols[key_s][i], []):
                g0 = es[1] & 0x7FFFFFFF if table_s.wide else es[1]
                v = wrap128(P.agg_term("mul_1minus_minus_paymul", wrap64(cols[a][i]), wrap64(cols[b][i]), pay=ep[1], d=wrap64(cols[d][i])))
                out[part_of(ko, world)].append((pack(ko, g0), v & M64, (v >> 64) & M64))
    return out


def stored(sent: List[tuple], capacity: int):
    """(cursor, overflow?, number of stored tuples) of one destination"""
    return len(sent), len(sent) > capacity, min(len(sent), capacity)


# ---------------------------------------------------------------------------------------------------- receive side
def publish_counts(cursors: Sequence[Sequence[int]]) -> List[List[int]]:
    """cursors[s][d] (tuples source s sent to d) → counts[d][s] (what rank d reads for source s)"""
    world = len(cursors)
    return [[cursors[s][d] for s in range(world)] for d in range(world)]


def received(regions: Sequence[Sequence[tuple]], counts: Sequence[int], capacity: int) -> List[tuple]:
    """the tuples a receiver reads: the first min(counts[s], capacity) of each source's sub-region"""
    out = []
    for s, reg in enumerate(regions):
        out.extend(reg[: min(counts[s], capacity)])
    return out


def insert_received(table: P.JoinTable, tuples: Sequence[tuple]):
    for t in tuples:
        k, p = unpack(t[0])
        table.insert(k, p)


def _groups_cap(sums: dict, capacity: int):
    if len(sums) > P.group_slots(capacity):
        raise PipeError(LDB_ERR_CAPACITY, "group-by table overflow")


def probe_received_groupby(table_a: P.JoinTable, table_b: P.JoinTable, tuples: Sequence[tuple], scale: int, capacity: int = 64) -> Dict[tuple, list]:
    """{keyA | keyB << 32, a, b}: every pair (match of A, match of B) with equal payloads adds a * (10^scale - b) to group (payload, 0)"""
    if not 0 <= scale <= 18:
        raise PipeError(LDB_ERR_INVALID, "decimal scale out of range")
    ia, ib = table_a.index(), table_b.index()
    one = 10**scale
    sums: Dict[tuple, int] = {}
    for w0, a, b in tuples:
        ka, kb = unpack(w0)
        a, b = wrap64(a), wrap64(b)
        for ea in ia.get(ka, []):
            for eb in ib.get(kb, []):
                if ea[1] == eb[1]:
                    sums[(eb[1], 0)] = sums.get((eb[1], 0), 0) + a * (one - b)
    _groups_cap(sums, capacity)
    return {g: [wrap128(v)] for g, v in sums.items()}


def probe_received_groupby2(table: P.JoinTable, tuples: Sequence[tuple], capacity: int = 1024) -> Dict[tuple, list]:
    """{key | g0 << 32, lo, hi}: per match g1 of `table` on key, group (g0, g1) += the shipped i128"""
    idx = table.index()
    sums: Dict[tuple, int] = {}
    for w0, lo, hi in tuples:
        k, g0 = unpack(w0)
        for e in idx.get(k, []):
            sums[(g0, e[1])] = sums.get((g0, e[1]), 0) + (lo | (hi << 64))
    _groups_cap(sums, capacity)
    return {g: [wrap128(v)] for g, v in sums.items()}


# ---------------------------------------------------------------------------------------------------- K7
def merge(shards: Sequence[Dict[tuple, list]], widths64: Sequence[bool], capacity: int = 64, keyless: bool = False) -> Dict[tuple, list]:
    """shards: {key: [raw 128-bit cells (ints, any sign)]} → the merged groups read at the target's lane widths (widths64[a]: lane a is
    a 64-bit lane).  A keyless (SIMPLE) target has the one group () even when every shard is empty."""
    total: Dict[tuple, list] = {(): [0] * len(widths64)} if keyless else {}
    for sh in shards:
        for k, cells in sh.items():
            acc = total.setdefault(k, [0] * len(widths64))
            for a, v in enumerate(cells):
                acc[a] += v
    if not keyless:
        _groups_cap(total, capacity)
    return {k: [wrap64(v) if w else wrap128(v) for v, w in zip(acc, widths64)] for k, acc in total.items()}


# ---------------------------------------------------------------------------------------------------- collectives
def allgather_small(blocks: Sequence[bytes], slot: int = SLOT_BYTES) -> List[bytes]:
    """the gathered region of every rank: block r at r * slot (only the first len(block) bytes of a slot are defined)"""
    if not blocks or len(blocks) > MAX_PEERS:
        raise PipeError(LDB_ERR_INVALID, "rank/world out of range")
    n = len(blocks[0])
    if n <= 0 or n > slot or n % 16 or any(len(b) != n for b in blocks):
        raise PipeError(LDB_ERR_INVALID, "all-gather blocks are 16..262144 bytes, multiples of 16")
    return list(blocks)
