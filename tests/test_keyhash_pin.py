"""tests/_keyhash.py against csrc/keyhash.cuh itself (no GPU): a small C++ driver compiled with g++ against the header
(-D__device__= -D__forceinline__=inline), fed fixed and random inputs, every output compared with the Python copy.  The set
operations' collision tests build their rows with that copy's solvers, so without this pin a change to the device hash would quietly
turn them back into random tests."""
import os
import random
import struct
import subprocess

import numpy as np
import pytest

import _keyhash as K

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "lingo-db_b200", "csrc")
M64 = K.M64

DRIVER = r"""
#include "keyhash.cuh"
#include <cstdio>
#include <cstring>
#include <iostream>
#include <string>
#include <vector>
using namespace ldb;
// one request per line, numbers in hex, one answer per line:
//   m x | s len hexbytes | k seed n keys... | i lo hi | f bits | r n words... | z
int main() {
   std::string op;
   while (std::cin >> op) {
      unsigned long long out = 0;
      if (op == "m") {
         unsigned long long x;
         std::cin >> std::hex >> x;
         out = mix64(x);
      } else if (op == "s") {
         int n;
         std::string hex;
         std::cin >> std::dec >> n >> hex;
         std::vector<uint8_t> b(n + 1);
         for (int i = 0; i < n; i++) b[i] = (uint8_t) std::stoi(hex.substr(2 * i, 2), nullptr, 16);
         out = strHash(b.data(), n);
      } else if (op == "k") {
         unsigned long long seed;
         int n;
         std::cin >> std::hex >> seed >> std::dec >> n;
         std::vector<int64_t> keys(n + 1);
         for (int i = 0; i < n; i++) {
            unsigned long long v;
            std::cin >> std::hex >> v;
            keys[i] = (int64_t) v;
         }
         out = keyTupleHash(keys.data(), n, (uint32_t) seed);
      } else if (op == "i") {
         unsigned long long lo, hi;
         std::cin >> std::hex >> lo >> hi;
         out = setIntWord(lo, hi);
      } else if (op == "f") {
         unsigned long long bits;
         std::cin >> std::hex >> bits;
         double d;
         std::memcpy(&d, &bits, 8);
         out = setF64Bits(d);
      } else if (op == "r") {
         int n;
         std::cin >> std::dec >> n;
         std::vector<uint64_t> w(n + 1);
         for (int i = 0; i < n; i++) {
            unsigned long long v;
            std::cin >> std::hex >> v;
            w[i] = v;
         }
         out = setRowFold(n, [&](int c) { return w[c]; });
      } else if (op == "z") {
         out = kSetNullWord;
      } else {
         return 2;
      }
      std::printf("%llx\n", out);
   }
   return 0;
}
"""


@pytest.fixture(scope="module")
def device_hash(tmp_path_factory):
    """run(lines) -> the header's answers, one int per request line"""
    d = tmp_path_factory.mktemp("keyhash")
    src, exe = d / "driver.cpp", d / "driver"
    src.write_text(DRIVER)
    cxx = os.environ.get("CXX", "g++")
    subprocess.run([cxx, "-std=c++17", "-O2", "-D__device__=", "-D__forceinline__=inline", "-I", CSRC, str(src), "-o", str(exe)], check=True)

    def run(lines):
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout.split()
        assert len(out) == len(lines)
        return [int(x, 16) for x in out]
    return run


def bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


EDGE64 = [0, 1, 2, 0x7F, 0x80, 0xFF, 1 << 31, (1 << 32) - 1, 1 << 32, (1 << 63) - 1, 1 << 63, M64, M64 - 1, K.NULL_WORD, K.SEED, K.STEP]


def rand64(rng, n):
    return [rng.getrandbits(64) for _ in range(n)] + [rng.getrandbits(rng.randrange(1, 64)) for _ in range(n)]


def test_mix64_and_its_inverse(device_hash):
    rng = random.Random(1)
    xs = EDGE64 + rand64(rng, 500)
    assert device_hash([f"m {x:x}" for x in xs]) == [K.mix64(x) for x in xs]
    assert all(K.unmix64(K.mix64(x)) == x and K.mix64(K.unmix64(x)) == x for x in xs)
    a = np.array(xs, np.uint64)
    assert K.mix64_np(a).tolist() == [K.mix64(x) for x in xs]
    assert K.unmix64_np(a).tolist() == [K.unmix64(x) for x in xs]
    assert K.mix64(0) == 0


def test_str_hash_lengths_0_to_70(device_hash):
    rng = random.Random(2)
    strs = [b"", b"\0", b"\0" * 8, b"\xff" * 9, b"COLLIDE#imldaaaa"]
    for n in range(71):
        strs += [bytes(rng.randrange(256) for _ in range(n)) for _ in range(3)]
    got = device_hash([f"s {len(s)} {s.hex() or '-'}" for s in strs])
    assert got == [K.str_hash(s) for s in strs]
    for n in (0, 1, 7, 8, 9, 16, 23, 70):  # the numpy form, over equal-length strings
        same = [s for s in strs if len(s) == n]
        arr = np.array([list(s) for s in same], np.uint8).reshape(len(same), n)
        assert K.str_hash_np(arr, n).tolist() == [K.str_hash(s) for s in same], n


def test_key_tuple_hash_with_null_seed_bits(device_hash):
    rng = random.Random(3)
    cases = [([], 0), ([0], 0), ([0], 1), ([7], 0), ([-1], 0), ([M64], 5)]
    for _ in range(300):
        n = rng.randrange(0, 5)
        keys = [rng.choice([rng.getrandbits(64), rng.randrange(-1000, 1000)]) for _ in range(n)]
        cases.append((keys, rng.getrandbits(n) if n else rng.getrandbits(32)))
    lines = [f"k {seed:x} {len(keys)} " + " ".join(f"{v & M64:x}" for v in keys) for keys, seed in cases]
    assert device_hash(lines) == [K.key_tuple_hash(keys, seed) for keys, seed in cases]
    for n in (1, 2, 4):  # the numpy form, seeds per row
        rows = [(keys, seed) for keys, seed in cases if len(keys) == n]
        cols = [np.array([keys[k] & M64 for keys, _ in rows], np.uint64) for k in range(n)]
        seeds = np.array([seed for _, seed in rows], np.uint64)
        assert K.key_tuple_hash_np(cols, seeds).tolist() == [K.key_tuple_hash(keys, seed) for keys, seed in rows], n


def test_set_cell_words_and_row_fold(device_hash):
    rng = random.Random(4)
    assert device_hash(["z"]) == [K.NULL_WORD]
    ints = [0, 1, -1, (1 << 63) - 1, -(1 << 63), (1 << 64) - 1, 1 << 64, -(1 << 64), (1 << 127) - 1, -(1 << 127), K.NULL_WORD]
    ints += [rng.randrange(-(1 << 127), 1 << 127) for _ in range(300)] + [rng.randrange(-(1 << 63), 1 << 63) for _ in range(300)]
    assert device_hash([f"i {v & M64:x} {(v >> 64) & M64:x}" for v in ints]) == [K.int_word(v) for v in ints]
    assert K.int_word_np(np.array([v for v in ints if -(1 << 63) <= v < 1 << 63], np.int64)).tolist() == [K.int_word(v) for v in ints if -(1 << 63) <= v < 1 << 63]
    floats = [0.0, -0.0, 1.0, -1.5, float("inf"), float("-inf"), 5e-324, 1.7976931348623157e308, struct.unpack("<d", struct.pack("<Q", K.NULL_WORD))[0]]
    fbits = [bits(x) for x in floats] + [0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0x7FF8000000000123, 0xFFFFFFFFFFFFFFFF]
    fbits += rand64(rng, 200)
    want = [K.f64_word(struct.unpack("<d", struct.pack("<Q", b))[0]) for b in fbits]
    assert device_hash([f"f {b:x}" for b in fbits]) == want
    assert K.f64_word(-0.0) == 0 and K.f64_word(float("nan")) == K.NAN_WORD
    rows = [[]] + [[rng.getrandbits(64) for _ in range(rng.randrange(1, 17))] for _ in range(300)] + [[K.NULL_WORD] * 16]
    assert device_hash([f"r {len(r)} " + " ".join(f"{w:x}" for w in r) for r in rows]) == [K.row_hash(r) for r in rows]
    for n in (1, 3, 16):
        same = [r for r in rows if len(r) == n]
        if same:
            assert K.row_hash_np([np.array([r[c] for r in same], np.uint64) for c in range(n)]).tolist() == [K.row_hash(r) for r in same]


def test_solvers_hit_their_targets(device_hash):
    """every solver's cell has the chosen word and every solved row the chosen hash, checked by the header, not by the Python copy"""
    rng = random.Random(5)
    targets = [0, M64, K.NULL_WORD, (rng.getrandbits(32) << 32) | 0xFFFFFFFF] + rand64(rng, 40)
    lines, want = [], []
    for t in targets:
        prefix = [rng.getrandbits(64) for _ in range(rng.randrange(0, 4))]
        w = K.last_word(prefix, t)
        lines.append(f"r {len(prefix) + 1} " + " ".join(f"{x:x}" for x in prefix + [w]))
        want.append(t)
        for hi in (0, 1, M64, rng.getrandbits(64)):
            v = K.decimal_for(w, hi)
            assert -(1 << 127) <= v < 1 << 127 and (v >> 64) & M64 == hi
            lines.append(f"i {v & M64:x} {(v >> 64) & M64:x}")
            want.append(w)
        for n, chunk in ((8, 0), (16, 0), (16, 1), (21, 1), (40, 2)):
            s = K.utf8_for(w, bytes(rng.randrange(256) for _ in range(n)), chunk)
            assert len(s) == n
            lines.append(f"s {n} {s.hex()}")
            want.append(w)
        x = K.f64_for(w)
        if x is not None:
            lines.append(f"f {bits(x):x}")
            want.append(w)
        v = K.int64_for(w)
        if v is not None:
            assert -(1 << 63) <= v < 1 << 63
            lines.append(f"i {v & M64:x} {(v >> 64) & M64:x}")
            want.append(w)
    assert device_hash(lines) == want
    # the NULL word is realisable by every type the set operations hash this way
    assert K.int64_for(K.NULL_WORD) == K.NULL_WORD and K.f64_word(K.f64_for(K.NULL_WORD)) == K.NULL_WORD
    assert K.int_word(K.decimal_for(K.NULL_WORD, 3)) == K.NULL_WORD and K.str_hash(K.utf8_for(K.NULL_WORD, b"12345678")) == K.NULL_WORD
    # the float words that cannot be made: -0.0 and the non-canonical NaNs.  int64 makes every word: mix64(-1) < 2^63, so the
    # negative values' words are exactly the words of 2^63 and above
    assert K.f64_for(1 << 63) is None and K.f64_for(0x7FF0000000000001) is None and K.f64_for(K.NAN_WORD) is not None
    assert K.mix64(M64) >> 63 == 0 and all(K.int64_for(w) is not None for w in targets)
