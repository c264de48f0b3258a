// tilescan.cuh — a device-wide inclusive scan over n positions for any associative Op: per tile a reduction, one CTA's exclusive scan
// of the tile totals, then each tile rescanned from its prefix.  The window operator (window.cu) and the set operations (setop.cu).
// And rowScanKernel, the one-launch exclusive sum of short rows: the radix sort's digit counts (program.cu), the table exchange's
// histograms and the permute's byte sums (peer.cu).
//
// An Op has T, identity(), combine(a, b), load(k) (the value at scan position k) and store(k, inclusive scan at k).  T needs a
// tileShflUp(T, offset) overload: uint32_t's is here, an Op's own struct brings its own (found by argument-dependent lookup).
#pragma once
#include "context.h"

namespace ldb {

constexpr int kTileScanThreads = 256, kTileScanItems = 8;
constexpr int64_t kTileScanTile = (int64_t) kTileScanThreads * kTileScanItems;

__device__ __forceinline__ uint32_t tileShflUp(uint32_t v, int o) { return __shfl_up_sync(0xffffffffu, v, o); }
__device__ __forceinline__ unsigned long long tileShflUp(unsigned long long v, int o) { return __shfl_up_sync(0xffffffffu, v, o); }
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

// CTA r: the exclusive sum of row r (rows[r n .. r n + n)), in place, with a 64-bit carry across its 1024-element chunks; totals[r] =
// the row's sum (totals null: none).  One launch, a CTA per row: for the few, short rows its callers scan, tileScan's three launches cost more.
template <class T>
__global__ void __launch_bounds__(1024) rowScanKernel(T* rows, int64_t n, unsigned long long* totals) {
   __shared__ T warpSums[32];
   __shared__ unsigned long long carry;
   T* h = rows + (size_t) blockIdx.x * n;
   if (threadIdx.x == 0) carry = 0;
   __syncthreads();
   T next = threadIdx.x < n ? h[threadIdx.x] : T(0);
   for (int64_t base = 0; base < n; base += 1024) {
      const int64_t i = base + threadIdx.x;
      const T v = next;
      next = i + 1024 < n ? h[i + 1024] : T(0); // the next chunk's load overlaps this chunk's scan: the loop is latency-bound
      T x = v;
      for (int o = 1; o < 32; o <<= 1) {
         const T y = __shfl_up_sync(0xffffffffu, x, o);
         if ((threadIdx.x & 31) >= o) x += y;
      }
      if ((threadIdx.x & 31) == 31) warpSums[threadIdx.x >> 5] = x;
      __syncthreads();
      if (threadIdx.x < 32) {
         const T w = warpSums[threadIdx.x];
         T ws = w;
         for (int o = 1; o < 32; o <<= 1) {
            const T y = __shfl_up_sync(0xffffffffu, ws, o);
            if (threadIdx.x >= o) ws += y;
         }
         warpSums[threadIdx.x] = ws - w;
      }
      __syncthreads();
      const unsigned long long excl = carry + warpSums[threadIdx.x >> 5] + (x - v);
      if (i < n) h[i] = (T) excl;
      __syncthreads();
      if (threadIdx.x == 1023) carry = excl + v;
      __syncthreads();
   }
   if (totals && threadIdx.x == 0) totals[blockIdx.x] = carry;
}

} // namespace ldb
