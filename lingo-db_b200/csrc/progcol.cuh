// progcol.cuh — how a program column's cell becomes a value (ProgCol, program.h): the interpreter's loads (program.cu) and the table
// exchange's key reads (peer.cu) share these definitions, so a row's key value, and with it its owner rank, is the value the
// aggregation sink groups by.
#pragma once
#include "program.h"
#include "../../include/ldb_gpu.h"

namespace ldb {

typedef __int128 s128;
struct Val {
   s128 v;    // integers, decimals (raw), dates (days), booleans (0/1); doubles live in the low 64 bits
   bool null;
};
__device__ __forceinline__ double asF64(const Val& x) { return __longlong_as_double((long long) (uint64_t) x.v); }
__device__ __forceinline__ Val fromF64(double d, bool null) { return Val{(s128) (uint64_t) __double_as_longlong(d), null}; }

__device__ __forceinline__ bool colIsNull(const ProgCol& c, int64_t row) {
   if (c.validBytes) return c.validBytes[row] == 0;
   if (!c.validity) return false;
   const int64_t bit = c.bitOffset + row;
   return !((c.validity[bit >> 3] >> (bit & 7)) & 1u);
}
// LoadArrowOp lowering (ArrowToStd.cpp:67-173, LowerToStd.cpp:111-209): physical cell → value register
__device__ __forceinline__ Val loadCol(const ProgCol& c, int64_t row) {
   Val r;
   r.null = colIsNull(c, row);
   switch (c.type) {
      case LDB_INT32:
      case LDB_DATE32:
      case LDB_FSB4: r.v = (s128) ((const int32_t*) c.data)[row]; break;
      case LDB_INT64: r.v = (s128) ((const int64_t*) c.data)[row]; break;
      case LDB_INT8: r.v = (s128) ((const int8_t*) c.data)[row]; break;
      case LDB_INT16: r.v = (s128) ((const int16_t*) c.data)[row]; break;
      // at the column's cell width: exported float aggregates keep 16-byte cells (the double's bits in the low 8 bytes)
      case LDB_FLOAT32: return fromF64((double) *(const float*) (c.data + (size_t) row * c.elemBytes), r.null);
      case LDB_FLOAT64: return fromF64(*(const double*) (c.data + (size_t) row * c.elemBytes), r.null);
      case LDB_DECIMAL128:
         if (c.elemBytes == 16) {
            const ulonglong2 cell = ((const ulonglong2*) c.data)[row];
            r.v = (s128) (((unsigned __int128) cell.y << 64) | cell.x);
         } else {
            r.v = (s128) ((const int64_t*) c.data)[row]; // narrowed HOST batch (p < 19): sign-extend
         }
         break;
      default: r.v = 0; r.null = true;
   }
   return r;
}

} // namespace ldb
