"""The device hashes of csrc/keyhash.cuh restated in Python, scalar and numpy forms, and solvers that invert them.

- mix64 / unmix64: the splitmix finaliser and its inverse (each xor-shift by 33 undoes itself, both multipliers are odd);
- str_hash: strHash, 8-byte little-endian chunks (the last one zero padded) folded through mix64, seeded with the length;
- key_tuple_hash: keyTupleHash over int64 keys and a 32-bit seed (hash aggregation seeds it with its key-NULL bits);
- the set operations' cell words (NULL_WORD, int_word, f64_word, cell_word) and their row hash (row_hash, the fold setRowFold);
- solvers: last_word sets the last cell word of a row so the row hash is a chosen 64-bit value, and the *_for functions make a cell of
  a given type whose word is a chosen word (decimal128 and utf8 of at least 8 bytes always, float64 unless the word is a NaN other than
  the canonical one or -0.0, int64 always, since mix64(-1) < 2^63).

tests/test_keyhash_pin.py compiles keyhash.cuh with g++ and pins every function here to it."""
import struct

import numpy as np

M64 = (1 << 64) - 1
_C1, _C2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53
_C1_INV, _C2_INV = pow(_C1, -1, 1 << 64), pow(_C2, -1, 1 << 64)
SEED = 0x9E3779B97F4A7C55       # keyTupleHash and the row fold
STR_SEED = 0x9E3779B97F4A7C15   # strHash
STEP = 0x632BE59BD9B4E019       # added after each mix64 of a fold, times the 1-based position (strHash: once per chunk)
NULL_WORD = 0x2545F4914F6CDD1D  # kSetNullWord: a NULL cell's word
NAN_WORD = 0x7FF8000000000000   # every NaN's word


# ---------------------------------------------------------------------------------------------------- scalar
def mix64(x: int) -> int:
    x &= M64
    x ^= x >> 33
    x = (x * _C1) & M64
    x ^= x >> 33
    x = (x * _C2) & M64
    return x ^ (x >> 33)


def unmix64(x: int) -> int:
    x &= M64
    x ^= x >> 33
    x = (x * _C2_INV) & M64
    x ^= x >> 33
    x = (x * _C1_INV) & M64
    return x ^ (x >> 33)


def _chunks(b: bytes) -> list:
    return [int.from_bytes(b[i:i + 8].ljust(8, b"\0"), "little") for i in range(0, len(b), 8)]


def _str_seed(n: int) -> int:
    return STR_SEED ^ ((n & 0xFFFFFFFF) * _C1 & M64)


def str_hash(b: bytes) -> int:
    h = _str_seed(len(b))
    for w in _chunks(b):
        h = (mix64(h ^ w) + STEP) & M64
    return mix64(h)


def key_tuple_hash(keys: list, seed: int = 0) -> int:
    """keys: ints taken as int64 (their low 64 bits)"""
    h = SEED ^ (seed & 0xFFFFFFFF)
    for k, v in enumerate(keys):
        h = (mix64(h ^ (v & M64)) + STEP * (k + 1)) & M64
    return h


def int_word(v: int) -> int:
    """an integer, date, char(1) or decimal cell: its value sign-extended to 128 bits, lo ^ mix64(hi)"""
    return (v & M64) ^ mix64((v >> 64) & M64)


def f64_word(x) -> int:
    """a float cell (a Python float; float32 values widen exactly): -0.0 as +0.0, every NaN as one NaN"""
    x = float(x)
    if x == 0.0:
        return 0
    if x != x:
        return NAN_WORD
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def cell_word(phys: str, v) -> int:
    """setCellWord of a cell of physical type `phys` (None = NULL)"""
    if v is None:
        return NULL_WORD
    if phys == "utf8":
        return str_hash(v)
    if phys in ("float32", "float64"):
        return f64_word(v)
    return int_word(v)


def row_hash(words: list) -> int:
    """setRowFold over the cell words of a row"""
    h = SEED
    for c, w in enumerate(words):
        h = (mix64(h ^ w) + STEP * (c + 1)) & M64
    return mix64(h)


def row_hash_of(phys: list, row) -> int:
    return row_hash([cell_word(p, v) for p, v in zip(phys, row)])


# ---------------------------------------------------------------------------------------------------- solvers
def last_word(words: list, target: int) -> int:
    """the word w such that row_hash(words + [w]) == target"""
    h = SEED
    for c, w in enumerate(words):
        h = (mix64(h ^ w) + STEP * (c + 1)) & M64
    return unmix64((unmix64(target) - STEP * (len(words) + 1)) & M64) ^ h


def decimal_for(word: int, hi: int = 0) -> int:
    """the decimal128 value (signed 128-bit) with high half `hi` whose word is `word`: always exists"""
    lo = word ^ mix64(hi & M64)
    v = ((hi & M64) << 64) | lo
    return v - (1 << 128) if v >> 127 else v


def int64_for(word: int):
    """the int64 whose word is `word`, or None: a value >= 0 has word v, a negative one v ^ mix64(-1) (which is >= 2^63, as
    mix64(-1) < 2^63: every word has exactly one int64)"""
    if word >> 63 == 0:
        return word
    lo = word ^ mix64(M64)
    return lo - (1 << 64) if lo >> 63 else None


def f64_for(word: int):
    """the float64 whose word is `word`, or None for -0.0 and NaNs other than the canonical one"""
    if word == 1 << 63:
        return None
    x = struct.unpack("<d", struct.pack("<Q", word))[0]
    if x != x and word != NAN_WORD:
        return None
    return x


def utf8_for(word: int, template: bytes, chunk: int = 0) -> bytes:
    """`template` (at least 8 * (chunk + 1) bytes) with its 8-byte chunk `chunk` replaced so that str_hash is `word`: the chunks
    before it fold forwards from the seed, the ones after it unfold backwards from the word"""
    assert len(template) >= 8 * (chunk + 1)
    ws = _chunks(template)
    h = _str_seed(len(template))
    for w in ws[:chunk]:
        h = (mix64(h ^ w) + STEP) & M64
    g = unmix64(word)  # the fold's value after the last chunk
    for w in reversed(ws[chunk + 1:]):
        g = unmix64((g - STEP) & M64) ^ w
    x = unmix64((g - STEP) & M64) ^ h
    return template[:8 * chunk] + x.to_bytes(8, "little") + template[8 * chunk + 8:]


def cell_for(phys: str, word: int, free=0):
    """a cell of `phys` whose word is `word`, or None when the type cannot realise it; `free` picks among the many solutions (the
    decimal's high half, or the string template)"""
    if phys == "decimal128":
        return decimal_for(word, free)
    if phys == "utf8":
        return utf8_for(word, free if isinstance(free, bytes) else b"\0" * 8 + int(free).to_bytes(8, "little"))
    if phys == "float64":
        return f64_for(word)
    if phys == "int64":
        return int64_for(word)
    raise ValueError(phys)


# ---------------------------------------------------------------------------------------------------- numpy
def _u64(x) -> np.ndarray:
    return np.asarray(x).astype(np.uint64) if np.asarray(x).dtype != np.uint64 else np.asarray(x)


def mix64_np(x) -> np.ndarray:
    x = _u64(x).copy()
    with np.errstate(over="ignore"):
        x ^= x >> np.uint64(33)
        x *= np.uint64(_C1)
        x ^= x >> np.uint64(33)
        x *= np.uint64(_C2)
        x ^= x >> np.uint64(33)
    return x


def unmix64_np(x) -> np.ndarray:
    x = _u64(x).copy()
    with np.errstate(over="ignore"):
        x ^= x >> np.uint64(33)
        x *= np.uint64(_C2_INV)
        x ^= x >> np.uint64(33)
        x *= np.uint64(_C1_INV)
        x ^= x >> np.uint64(33)
    return x


def key_tuple_hash_np(keys: list, seed=0) -> np.ndarray:
    """keys: int64 (or uint64) arrays of one length; seed: a scalar or an array of 32-bit seeds"""
    n = len(keys[0])
    h = np.full(n, SEED, np.uint64) ^ (np.broadcast_to(np.asarray(seed, np.uint64), (n,)) & np.uint64(0xFFFFFFFF))
    with np.errstate(over="ignore"):
        for k, v in enumerate(keys):
            v = np.asarray(v)
            w = v.view(np.uint64) if v.dtype.itemsize == 8 else v.astype(np.int64).view(np.uint64)
            h = mix64_np(h ^ w) + np.uint64((STEP * (k + 1)) & M64)
    return h


def str_hash_np(s: np.ndarray, n: int) -> np.ndarray:
    """strHash of equal-length strings: s is (rows, n) uint8"""
    rows = s.shape[0]
    pad = np.zeros((rows, (n + 7) // 8 * 8), np.uint8)
    pad[:, :n] = s
    words = pad.view("<u8")
    h = np.full(rows, _str_seed(n), np.uint64)
    with np.errstate(over="ignore"):
        for j in range(words.shape[1]):
            h = mix64_np(h ^ words[:, j]) + np.uint64(STEP)
    return mix64_np(h)


def int_word_np(v) -> np.ndarray:
    """int64 cells (sign-extended): the word of each"""
    v = np.asarray(v, np.int64)
    return v.view(np.uint64) ^ mix64_np((v >> np.int64(63)).view(np.uint64))


def row_hash_np(words: list) -> np.ndarray:
    """setRowFold over per-column word arrays"""
    h = np.full(len(words[0]), SEED, np.uint64)
    with np.errstate(over="ignore"):
        for c, w in enumerate(words):
            h = mix64_np(h ^ _u64(w)) + np.uint64((STEP * (c + 1)) & M64)
    return mix64_np(h)
