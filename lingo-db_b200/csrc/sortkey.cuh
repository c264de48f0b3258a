// sortkey.cuh — the value of a fixed-width ORDER BY key cell, as one definition: the radix sort's key words (program.cu
// buildSortWordsKernel) and the sort exchange's sample tuples and range owners (peer.cu) read a cell through it, so the splitters that
// cut the rows across ranks and the sort that orders each rank's slice agree on the order by construction.
#pragma once
#include <cstdint>

namespace ldb {

// A key cell's value sign-extended to 128 bits: a 4-byte cell (int32, date32, char(1)) and an 8-byte cell (int64, a narrowed decimal) as
// their signed integer (sortNarrowValue), a 16-byte cell (decimal128) as its two words (sortWideWord).  The same value whatever width a
// shard staged the column at.
__device__ __forceinline__ int64_t sortNarrowValue(const uint8_t* col, int elemBytes, int64_t row) {
   return elemBytes == 4 ? (int64_t) ((const int32_t*) col)[row] : *(const int64_t*) (col + (size_t) row * elemBytes);
}
__device__ __forceinline__ unsigned long long sortWideWord(const uint8_t* col, int64_t row, int hi) { return ((const unsigned long long*) (col + (size_t) row * 16))[hi]; }
struct SortCell {
   unsigned long long lo, hi;
};
__device__ __forceinline__ SortCell sortCell(const uint8_t* col, int elemBytes, int64_t row) {
   if (elemBytes == 16) return SortCell{sortWideWord(col, row, 0), sortWideWord(col, row, 1)};
   const int64_t v = sortNarrowValue(col, elemBytes, row);
   return SortCell{(unsigned long long) v, (unsigned long long) (v >> 63)};
}

} // namespace ldb
