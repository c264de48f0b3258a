// keyhash.cuh — the key-tuple hash shared by the program interpreter (program.cu: hash aggregation, key-tuple join tables, the owner
// of an exchanged group) and the table exchange (peer.cu: the owner of a row).  One definition, so that a row and a group with the same
// key values land on the same rank.  The set operations (setop.cu) build their whole-row hash from the same pieces.
// The header also compiles as plain C++ (-D__device__= -D__forceinline__=inline): tests/test_keyhash_pin.py checks the Python copy
// in tests/_keyhash.py against it.
#pragma once
#include <cstdint>

namespace ldb {

__device__ __forceinline__ uint64_t mix64(uint64_t x) {
   x ^= x >> 33;
   x *= 0xff51afd7ed558ccdull;
   x ^= x >> 33;
   x *= 0xc4ceb9fe1a85ec53ull;
   x ^= x >> 33;
   return x;
}
// placement hash of a tuple of int64 keys: every key goes through mix64, so correlated tuples ((partkey, suppkey) pairs whose
// components grow together) do not cluster the way an XOR combine of per-key hashes does.  Shared by the hash-aggregation table (seeded
// with its key-NULL bits), the key-tuple join table and the table exchange.
__device__ __forceinline__ uint64_t keyTupleHash(const int64_t* keys, int n, uint32_t seed) {
   uint64_t h = 0x9E3779B97F4A7C55ull ^ seed;
   for (int k = 0; k < n; k++) h = mix64(h ^ (uint64_t) keys[k]) + 0x632BE59BD9B4E019ull * (k + 1);
   return h;
}
// placement hash of a byte string: 8-byte little-endian chunks (the last one zero padded) folded through mix64, seeded with the
// length.  Internal: codes and results never depend on it.  The string dictionary (program.cu) and the set operations (setop.cu).
__device__ __forceinline__ uint64_t strHash(const uint8_t* s, int32_t n) {
   uint64_t h = 0x9E3779B97F4A7C15ull ^ ((uint64_t) (uint32_t) n * 0xff51afd7ed558ccdull);
   for (int32_t i = 0; i < n; i += 8) {
      uint64_t w = 0;
      for (int j = 0; j < 8 && i + j < n; j++) w |= (uint64_t) s[i + j] << (8 * j);
      h = mix64(h ^ w) + 0x632BE59BD9B4E019ull;
   }
   return mix64(h);
}
// the rank of `world` that owns a key tuple with hash h: its high 32 bits, scaled (the low bits place the tuple inside a table)
__device__ __forceinline__ int keyOwner(uint64_t h, int world) { return (int) (((h >> 32) * (uint64_t) world) >> 32); }

// The set operations' whole-row hash (setop.cu): one 64-bit word per cell, equal cells giving equal words, folded in column order.
// setCellWord (setop.cu) picks the case and loads the cell; the values' rules are here, next to the pieces they are made of.
// A NULL cell's word.  An int64 holding this number has the same word (mix64(0) == 0), so only the NULL test tells them apart.
constexpr uint64_t kSetNullWord = 0x2545F4914F6CDD1Dull;
// an integer, date, char(1) or decimal cell by its value sign-extended to 128 bits: the low word, xor the mixed high word (0 or -1 for
// every value of 64 bits, so a narrowed decimal cell has the word of the same value in a 16-byte cell)
__device__ __forceinline__ uint64_t setIntWord(uint64_t lo, uint64_t hi) { return lo ^ mix64(hi); }
// a double's bits, on the device and in a host build of this header
__device__ __forceinline__ uint64_t f64Bits(double d) {
#ifdef __CUDA_ARCH__
   return (uint64_t) __double_as_longlong(d);
#else
   uint64_t bits;
   __builtin_memcpy(&bits, &d, 8);
   return bits;
#endif
}
// a float's bits (float32 arrives widened to double) with -0.0 as +0.0 and every NaN as the one quiet NaN
__device__ __forceinline__ uint64_t setF64Bits(double d) { return d == 0.0 ? 0ull : d != d ? 0x7ff8000000000000ull : f64Bits(d); }
// the row hash over n cells, word(c) the word of cell c: keyTupleHash's step, then mix64
template <class Word>
__device__ __forceinline__ uint64_t setRowFold(int n, Word word) {
   uint64_t h = 0x9E3779B97F4A7C55ull;
   for (int c = 0; c < n; c++) h = mix64(h ^ word(c)) + 0x632BE59BD9B4E019ull * (c + 1);
   return mix64(h);
}

} // namespace ldb
