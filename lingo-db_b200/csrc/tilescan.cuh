// tilescan.cuh — a device-wide inclusive scan over n positions for any associative Op: per tile a reduction, one CTA's exclusive scan
// of the tile totals, then each tile rescanned from its prefix.  The window operator (window.cu) and the set operations (setop.cu).
//
// An Op has T, identity(), combine(a, b), load(k) (the value at scan position k) and store(k, inclusive scan at k).  T needs a
// tileShflUp(T, offset) overload: uint32_t's is here, an Op's own struct brings its own (found by argument-dependent lookup).
#pragma once
#include "context.h"

namespace ldb {

constexpr int kTileScanThreads = 256, kTileScanItems = 8;
constexpr int64_t kTileScanTile = (int64_t) kTileScanThreads * kTileScanItems;

__device__ __forceinline__ uint32_t tileShflUp(uint32_t v, int o) { return __shfl_up_sync(0xffffffffu, v, o); }
// the exclusive scan of one value per thread across the CTA; *total = the CTA's combined value
template <class Op>
__device__ __forceinline__ typename Op::T tileBlockScan(const Op& op, typename Op::T v, typename Op::T* total) {
   using T = typename Op::T;
   __shared__ T warpTot[kTileScanThreads / 32];
   const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
   T x = v;
   for (int o = 1; o < 32; o <<= 1) {
      const T y = tileShflUp(x, o);
      if (lane >= o) x = op.combine(y, x);
   }
   T ex = tileShflUp(x, 1);
   if (lane == 0) ex = op.identity();
   if (lane == 31) warpTot[warp] = x;
   __syncthreads();
   T pre = op.identity(), all = op.identity();
   for (int w = 0; w < kTileScanThreads / 32; w++) {
      if (w < warp) pre = op.combine(pre, warpTot[w]);
      all = op.combine(all, warpTot[w]);
   }
   __syncthreads(); // warpTot is free for the next call
   *total = all;
   return op.combine(pre, ex);
}
template <class Op>
__global__ void __launch_bounds__(kTileScanThreads) tileScanReduceKernel(const __grid_constant__ Op op, int64_t n, typename Op::T* tileAgg) {
   using T = typename Op::T;
   const int64_t base = (int64_t) blockIdx.x * kTileScanTile + (int64_t) threadIdx.x * kTileScanItems;
   T a = op.identity();
#pragma unroll
   for (int q = 0; q < kTileScanItems; q++)
      if (base + q < n) a = op.combine(a, op.load(base + q));
   T total;
   tileBlockScan(op, a, &total);
   if (threadIdx.x == 0) tileAgg[blockIdx.x] = total;
}
// one CTA: the exclusive scan of the tile totals, in place
template <class Op>
__global__ void __launch_bounds__(kTileScanThreads) tileScanTilesKernel(const __grid_constant__ Op op, int64_t nTiles, typename Op::T* tileAgg) {
   using T = typename Op::T;
   T carry = op.identity(); // the same in every thread
   for (int64_t b = 0; b < nTiles; b += kTileScanThreads) {
      const int64_t i = b + threadIdx.x;
      T total;
      const T ex = tileBlockScan(op, i < nTiles ? tileAgg[i] : op.identity(), &total);
      if (i < nTiles) tileAgg[i] = op.combine(carry, ex);
      carry = op.combine(carry, total);
   }
}
template <class Op>
__global__ void __launch_bounds__(kTileScanThreads) tileScanDownKernel(const __grid_constant__ Op op, int64_t n, const typename Op::T* tileAgg) {
   using T = typename Op::T;
   const int64_t base = (int64_t) blockIdx.x * kTileScanTile + (int64_t) threadIdx.x * kTileScanItems;
   T item[kTileScanItems];
   T a = op.identity();
#pragma unroll
   for (int q = 0; q < kTileScanItems; q++) {
      item[q] = base + q < n ? op.load(base + q) : op.identity();
      a = op.combine(a, item[q]);
   }
   T total;
   T run = op.combine(tileAgg[blockIdx.x], tileBlockScan(op, a, &total));
#pragma unroll
   for (int q = 0; q < kTileScanItems; q++) {
      run = op.combine(run, item[q]);
      if (base + q < n) op.store(base + q, run);
   }
}
// the three launches of one scan over n > 0 positions, counted under the kernel family `family`
template <class Op>
static void tileScan(LdbContext* ctx, Scratch& tmp, const Op& op, int64_t n, const char* family) {
   using T = typename Op::T;
   const int64_t tiles = (n + kTileScanTile - 1) / kTileScanTile;
   T* agg = tmp.alloc<T>((size_t) tiles * sizeof(T));
   ctx->launch(family, [&] {
      tileScanReduceKernel<Op><<<(unsigned) tiles, kTileScanThreads, 0, ctx->compute>>>(op, n, agg);
      tileScanTilesKernel<Op><<<1, kTileScanThreads, 0, ctx->compute>>>(op, tiles, agg);
      tileScanDownKernel<Op><<<(unsigned) tiles, kTileScanThreads, 0, ctx->compute>>>(op, n, agg);
   });
}

} // namespace ldb
