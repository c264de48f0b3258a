// encode.cu — frame-of-reference encoded copies of DEVICE-resident columns for the K1/K2 scan (kernels.h kEncodeTileHeader).
//
// A Q1 pass over Arrow cells reads 76 B/row, 64 of them the four decimal128 cells of which the kernels use only the low 8
// bytes.  The values are small (quantities, discounts, taxes, flags, dates over a few thousand days), so per block of
// kEncodeBlockRows rows they fit in 1-4 bytes above the block minimum: Q1 reads ~12 B/row from the copy, Q6 ~9.  The copy is
// built once per (batch, column), on the first K1/K2 pipeline that needs it, on a stream of its own with host waits — never
// as part of a captured graph — and lives until the table is cleared.
#include "context.h"

#include <algorithm>
#include <climits>

namespace ldb {

constexpr uint64_t kSign64 = 1ull << 63;

__device__ __forceinline__ int64_t encodeSource(const uint8_t* src, bool isI32, int64_t r) {
   return isI32 ? (int64_t) ((const int32_t*) src)[r] : ((const int64_t*) src)[2 * r]; // decimal128: its low 8 bytes
}

// one CTA per block: blockMin[b], blockRange[b] = max - min, and the column's stats (kEncodeStats words): the largest range of all
// blocks, and the batch minimum and maximum as order-preserving unsigned keys, so all three reduce with an unsigned atomicMax from zero
__global__ void encodeRangeKernel(const uint8_t* src, bool isI32, int64_t n, int64_t* blockMin, int64_t* blockRange, unsigned long long* stats) {
   __shared__ int64_t sLo[32], sHi[32];
   const int64_t r0 = (int64_t) blockIdx.x * kEncodeBlockRows, r1 = min(n, r0 + kEncodeBlockRows);
   int64_t lo = LLONG_MAX, hi = LLONG_MIN;
   for (int64_t r = r0 + threadIdx.x; r < r1; r += blockDim.x) {
      const int64_t v = encodeSource(src, isI32, r);
      lo = min(lo, v);
      hi = max(hi, v);
   }
   for (int o = 16; o > 0; o >>= 1) {
      lo = min(lo, (int64_t) __shfl_xor_sync(0xffffffffu, (long long) lo, o));
      hi = max(hi, (int64_t) __shfl_xor_sync(0xffffffffu, (long long) hi, o));
   }
   const int warp = threadIdx.x / 32, nWarps = blockDim.x / 32;
   if ((threadIdx.x & 31) == 0) {
      sLo[warp] = lo;
      sHi[warp] = hi;
   }
   __syncthreads();
   if (threadIdx.x == 0) {
      for (int w = 1; w < nWarps; w++) {
         lo = min(lo, sLo[w]);
         hi = max(hi, sHi[w]);
      }
      blockMin[blockIdx.x] = lo;
      blockRange[blockIdx.x] = (int64_t) ((uint64_t) hi - (uint64_t) lo);
      atomicMax(&stats[0], (unsigned long long) ((uint64_t) hi - (uint64_t) lo));
      atomicMax(&stats[1], (unsigned long long) ~((uint64_t) lo ^ kSign64));
      atomicMax(&stats[2], (unsigned long long) ((uint64_t) hi ^ kSign64));
   }
}

// one thread per row: the value's offset from its block minimum in `width` bytes, and the header {block min, block range} of every
// tile — the range bounds every value of the tile, so K1/K2 can prove per tile that its products fit 64 bits
__global__ void encodePackKernel(const uint8_t* src, bool isI32, int64_t n, const int64_t* blockMin, const int64_t* blockRange, int width, int tileRows,
                                 uint8_t* dst) {
   const int64_t tileStride = kEncodeTileHeader + (int64_t) tileRows * width;
   for (int64_t r = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t) gridDim.x * blockDim.x) {
      const int64_t t = r / tileRows, lr = r - t * tileRows;
      const int64_t base = blockMin[r / kEncodeBlockRows];
      uint8_t* tile = dst + t * tileStride;
      if (lr == 0) {
         ((int64_t*) tile)[0] = base;
         ((int64_t*) tile)[1] = blockRange[r / kEncodeBlockRows];
      }
      const uint64_t d = (uint64_t) encodeSource(src, isI32, r) - (uint64_t) base;
      uint8_t* p = tile + kEncodeTileHeader + lr * width;
      switch (width) {
         case 1: *p = (uint8_t) d; break;
         case 2: *(uint16_t*) p = (uint16_t) d; break;
         case 4: *(uint32_t*) p = (uint32_t) d; break;
         default: *(uint64_t*) p = d; break;
      }
   }
}

void launchEncodeRange(const uint8_t* src, bool isI32, int64_t n, int64_t* blockMin, int64_t* blockRange, unsigned long long* stats, cudaStream_t s) {
   const int64_t blocks = (n + kEncodeBlockRows - 1) / kEncodeBlockRows;
   encodeRangeKernel<<<(unsigned) blocks, 256, 0, s>>>(src, isI32, n, blockMin, blockRange, stats);
}
void launchEncodePack(const uint8_t* src, bool isI32, int64_t n, const int64_t* blockMin, const int64_t* blockRange, int width, int tileRows, uint8_t* dst,
                      cudaStream_t s) {
   const int64_t grid = std::min<int64_t>((n + 255) / 256, 8192);
   encodePackKernel<<<(unsigned) grid, 256, 0, s>>>(src, isI32, n, blockMin, blockRange, width, tileRows, dst);
}

static int encodedWidth(uint64_t range) { return range < (1ull << 8) ? 1 : range < (1ull << 16) ? 2 : range < (1ull << 32) ? 4 : 8; }

} // namespace ldb

using namespace ldb;

bool ldb_gpu_encode_batch_internal(LdbContext* ctx, LdbTable* t, LdbBatch& b, const int* cols, int n, int tileRows) {
   if (!b.borrowed || b.nRows == 0) return false;
   if (b.enc.size() < t->columns.size()) b.enc.resize(t->columns.size());
   int todo[kMaxStagedCols], nTodo = 0;
   for (int i = 0; i < n; i++) {
      const LdbBatch::Encoded& e = b.enc[cols[i]];
      if (e.failed) return false; // the batch is scanned in Arrow layout; a failed column is not retried until the table is cleared
      if (e.data) {
         if (e.tileRows != tileRows) return false;
         continue;
      }
      bool dup = false;
      for (int k = 0; k < nTodo; k++) dup |= todo[k] == cols[i];
      if (!dup) todo[nTodo++] = cols[i];
   }
   if (nTodo == 0) return true;
   for (int k = 0; k < nTodo; k++) {
      const LdbColumn& c = t->columns[todo[k]];
      const bool ok = c.type == LDB_INT32 || c.type == LDB_DATE32 || c.type == LDB_FSB4 || (c.type == LDB_DECIMAL128 && c.precision < 19 && b.elemBytes[todo[k]] == 16);
      if (!ok) return false;
   }
   auto failAll = [&] {
      cudaGetLastError(); // an allocation failure is not a query failure
      for (int k = 0; k < nTodo; k++) b.enc[todo[k]].failed = true;
      return false;
   };
   const int64_t rows = b.nRows, blocks = (rows + kEncodeBlockRows - 1) / kEncodeBlockRows;
   if (!ctx->encodeStream) LDB_CUDA(cudaStreamCreateWithFlags(&ctx->encodeStream, cudaStreamNonBlocking));
   cudaStream_t s = ctx->encodeStream;
   // the build runs OUTSIDE any capture: on its own stream, ordered after the compute stream's earlier work (inside a capture the
   // compute stream was drained by ldb_gpu_graph_begin), finished with host waits, so a replayed graph never re-encodes
   if (!ctx->capturing) {
      LDB_CUDA(cudaEventRecord(ctx->computeDone, ctx->compute));
      LDB_CUDA(cudaStreamWaitEvent(s, ctx->computeDone, 0));
   }
   void* scratch = nullptr;
   const size_t scratchBytes = (size_t) nTodo * (size_t) blocks * 16 + (size_t) nTodo * kEncodeStats * 8;
   if (cudaMalloc(&scratch, scratchBytes) != cudaSuccess) return failAll();
   int64_t* blockMin = (int64_t*) scratch;
   int64_t* blockRange = blockMin + (size_t) nTodo * blocks;
   unsigned long long* stats = (unsigned long long*) (blockRange + (size_t) nTodo * blocks);
   uint64_t st[kMaxStagedCols][kEncodeStats];
   try {
      LDB_CUDA(cudaMemsetAsync(stats, 0, (size_t) nTodo * kEncodeStats * 8, s));
      for (int k = 0; k < nTodo; k++) {
         const bool isI32 = t->columns[todo[k]].type != LDB_DECIMAL128;
         launchEncodeRange((const uint8_t*) b.data[todo[k]], isI32, rows, blockMin + (size_t) k * blocks, blockRange + (size_t) k * blocks,
                           stats + (size_t) k * kEncodeStats, s);
         LDB_CUDA(cudaGetLastError());
      }
      LDB_CUDA(cudaMemcpyAsync(st, stats, (size_t) nTodo * kEncodeStats * 8, cudaMemcpyDeviceToHost, s));
      LDB_CUDA(cudaStreamSynchronize(s));
      ctx->encodeLaunches += nTodo;
      bool all = true;
      for (int k = 0; k < nTodo; k++) {
         LdbBatch::Encoded& e = b.enc[todo[k]];
         const int width = encodedWidth(st[k][0]);
         const int64_t bytes = encodedColumnBytes(rows, width, tileRows);
         void* data = nullptr;
         if (ctx->encodedBytes + bytes > ctx->encodedBudget || cudaMalloc(&data, (size_t) bytes) != cudaSuccess) {
            cudaGetLastError();
            e.failed = true;
            all = false;
            continue;
         }
         const bool isI32 = t->columns[todo[k]].type != LDB_DECIMAL128;
         launchEncodePack((const uint8_t*) b.data[todo[k]], isI32, rows, blockMin + (size_t) k * blocks, blockRange + (size_t) k * blocks, width, tileRows,
                          (uint8_t*) data, s);
         LDB_CUDA(cudaGetLastError());
         ctx->encodeLaunches++;
         e.data = (uint8_t*) data;
         e.width = width;
         e.bytes = bytes;
         e.tileRows = tileRows;
         e.min = (int64_t) (~st[k][1] ^ kSign64);
         e.max = (int64_t) (st[k][2] ^ kSign64);
         ctx->encodedBytes += bytes;
      }
      LDB_CUDA(cudaStreamSynchronize(s));
      cudaFree(scratch);
      return all;
   } catch (...) {
      cudaStreamSynchronize(s);
      cudaFree(scratch);
      throw;
   }
}

void ldb_gpu_free_encoded_internal(LdbContext* ctx, LdbBatch& b) {
   for (auto& e : b.enc) {
      if (e.data) {
         cudaFree(e.data);
         ctx->encodedBytes -= e.bytes;
      }
   }
   b.enc.clear();
}
