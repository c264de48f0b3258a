// keyhash.cuh — the key-tuple hash shared by the program interpreter (program.cu: hash aggregation, key-tuple join tables, the owner
// of an exchanged group) and the table exchange (peer.cu: the owner of a row).  One definition, so that a row and a group with the same
// key values land on the same rank.  The set operations (setop.cu) build their whole-row hash from the same pieces.
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

} // namespace ldb
