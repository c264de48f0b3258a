// window.cu — window functions over a single-batch table (ldb_gpu_table_window, include/ldb_gpu.h): the reference's WindowLowering
// (RelAlgToSubOp.cpp:2193-2553) over a sorted buffer, a continuous view with frame offsets (SubOpToControlFlow.cpp:3834-3881) and a
// SegmentTreeView (src/runtime/SegmentTreeView.cpp).
//
// Semantics, rule by rule:
//   Partitions: rows equal on every partition key under `isa` (IS NOT DISTINCT FROM, RelAlgToSubOp.cpp:142-153), so NULL keys form one
//     partition.  Within a partition rows follow the order keys in the order of ldb_gpu_table_order_by_keys (a NULL greater than any
//     value, DESC swaps); rows that tie on every key keep their source row order (our stable rule; the reference's sort leaves it open).
//   Frames: ROWS frames with constant offsets [from, to] relative to the current row (sql_analyzer.cpp:2424-2500); INT64_MIN is
//     UNBOUNDED PRECEDING, INT64_MAX UNBOUNDED FOLLOWING (BoundWindowFrame, ast/bound/bound_expression.h:114-115).
//   Clamping: for the row at position j of a partition of length len, each finite bound becomes min(len - 1, max(0, j + offset))
//     (SubOpToControlFlow.cpp:3861-3879), so a frame is never empty: ROWS BETWEEN 2 FOLLOWING AND 5 FOLLOWING on the last row
//     aggregates the last row.  Mirrored exactly.
//   UNBOUNDED FOLLOWING is the partition end.  DIVERGENCE: the reference feeds INT64_MAX through the same i64 add
//     (RelAlgToSubOp.cpp:2512-2530 with SubOpToControlFlow.cpp:3870), which wraps for every row past the first, so its frame end
//     collapses to 0 (or SegmentTreeView::lookup throws "from must be <= to"); only (UNBOUNDED, UNBOUNDED) escapes through the static
//     aggregate branch (RelAlgToSubOp.cpp:2496-2498).  We implement the SQL meaning instead of the wrap.
//   Functions (RelAlgToSubOp.cpp:2204-2247, sql_mlir_translator.cpp:1476-1481):
//     ROW_NUMBER = entries_between(frame start, current) + 1 = i - lo + 1 with the clamped frame start lo (RankWindowFunc, :2043-2058;
//       the reference's RANK is this same function, without tie handling);
//     COUNT(*) = hi - lo + 1;  COUNT(col) = the non-NULL values in [lo, hi];
//     SUM, MIN, MAX over the non-NULL values, NULL when the frame holds none (results nullable, sql_analyzer.cpp:2495-2502); SUM is
//       exact modulo 2^128 (the wrapping of LDB_AGG_SUM).
//
// Device work after the sort (every read of a source cell goes through the sort's row ids):
//   1. winHeadsKernel: row ids[i] against ids[i - 1] on every partition key (cells and NULL flags; bytes for utf8) → head flags;
//   2. two scans of the heads: partition start (max-scan of head ? i : 0) and partition end (min-scan from the last row);
//   3. SUM / COUNT(col): one global inclusive scan of (i128 sum of the non-NULL values, their count); a frame's value is
//      S[hi] - S[lo - 1], exact modulo 2^128.  The scan needs no segments because [lo, hi] never leaves its partition;
//   4. MIN / MAX: a segment tree over the sorted argument (NULL = the identity, plus an "any value" flag per node), built bottom-up
//      one launch per level over a power-of-two leaf array, queried per row by the iterative O(log width) walk;
//   5. winFramesKernel: per row its frame [lo, hi] by the clamping rule and every function's value.
// The scans are the tile scans of tilescan.cuh: per tile a reduction, one CTA's exclusive scan of the tile totals, then each tile
// rescanned from its prefix.
#include "context.h"
#include "progcol.cuh"
#include "sortkey.cuh"
#include "tilescan.cuh"

#include <algorithm>
#include <climits>

namespace ldb {

constexpr int kWinThreads = 256;
constexpr int kWinMaxFuncs = 8, kWinMaxCarried = 16;

__device__ __forceinline__ int64_t winRow(const uint32_t* ids, int64_t i) { return ids ? (int64_t) ids[i] : i; }

// ---------------------------------------------------------------- partition heads
struct WinKeys {
   ProgCol col[kProgMaxKeys];
   int32_t n, pad;
};
__device__ __forceinline__ bool winSameKey(const ProgCol& c, int64_t a, int64_t b) {
   const bool na = colIsNull(c, a), nb = colIsNull(c, b);
   if (na || nb) return na == nb;
   if (c.type == LDB_UTF8) {
      const int32_t* o = (const int32_t*) c.data;
      const int32_t a0 = o[a], b0 = o[b], len = o[a + 1] - a0;
      if (o[b + 1] - b0 != len) return false;
      for (int32_t x = 0; x < len; x++)
         if (c.bytes[a0 + x] != c.bytes[b0 + x]) return false;
      return true;
   }
   const SortCell x = sortCell(c.data, c.elemBytes, a), y = sortCell(c.data, c.elemBytes, b);
   return x.lo == y.lo && x.hi == y.hi;
}
__global__ void __launch_bounds__(kWinThreads) winHeadsKernel(const __grid_constant__ WinKeys k, const uint32_t* ids, int64_t n, uint8_t* head) {
   for (int64_t i = (int64_t) blockIdx.x * kWinThreads + threadIdx.x; i < n; i += (int64_t) gridDim.x * kWinThreads) {
      bool h = i == 0;
      if (!h) {
         const int64_t a = winRow(ids, i), b = winRow(ids, i - 1);
         for (int q = 0; q < k.n && !h; q++) h = !winSameKey(k.col[q], a, b);
      }
      head[i] = h ? 1 : 0;
   }
}

// ---------------------------------------------------------------- the scans' Ops (tilescan.cuh)
struct WinSum {
   unsigned long long lo, hi, cnt; // i128 sum of the non-NULL values (wrapping), their count
};
__device__ __forceinline__ WinSum tileShflUp(const WinSum& v, int o) {
   return WinSum{__shfl_up_sync(0xffffffffu, v.lo, o), __shfl_up_sync(0xffffffffu, v.hi, o), __shfl_up_sync(0xffffffffu, v.cnt, o)};
}
// partition start of row k: the last head at or before k
struct WinStartOp {
   using T = uint32_t;
   const uint8_t* head;
   uint32_t* start;
   __device__ T identity() const { return 0; }
   __device__ T combine(T a, T b) const { return max(a, b); }
   __device__ T load(int64_t k) const { return head[k] ? (T) k : 0u; }
   __device__ void store(int64_t k, T v) const { start[k] = v; }
};
// partition end of row i: scan position k is row n - 1 - k, so the scan runs from the last row back; a row ends its partition when it
// is the last row or the next row is a head (n - 1 < 2^32 - 1, so no row index equals the identity)
struct WinEndOp {
   using T = uint32_t;
   const uint8_t* head;
   uint32_t* end;
   int64_t n;
   __device__ T identity() const { return 0xffffffffu; }
   __device__ T combine(T a, T b) const { return min(a, b); }
   __device__ T load(int64_t k) const {
      const int64_t i = n - 1 - k;
      return i == n - 1 || head[i + 1] ? (T) i : 0xffffffffu;
   }
   __device__ void store(int64_t k, T v) const { end[n - 1 - k] = v; }
};
// the running (sum, count) of the non-NULL argument values in window order
struct WinSumOp {
   using T = WinSum;
   ProgCol arg;
   const uint32_t* ids;
   unsigned long long* sums;   // 2 words per row, or null (COUNT(col) needs only the counts)
   unsigned long long* counts;
   __device__ T identity() const { return WinSum{0, 0, 0}; }
   __device__ T combine(const T& a, const T& b) const {
      WinSum r;
      r.lo = a.lo + b.lo;
      r.hi = a.hi + b.hi + (r.lo < a.lo ? 1ull : 0ull);
      r.cnt = a.cnt + b.cnt;
      return r;
   }
   __device__ T load(int64_t k) const {
      const int64_t row = winRow(ids, k);
      if (colIsNull(arg, row)) return identity();
      if (!sums) return WinSum{0, 0, 1}; // COUNT(col) reads only the NULL flag: a column of any type
      const unsigned __int128 u = (unsigned __int128) loadCol(arg, row).v;
      return WinSum{(unsigned long long) u, (unsigned long long) (u >> 64), 1};
   }
   __device__ void store(int64_t k, const T& v) const {
      if (sums) *(ulonglong2*) (sums + 2 * k) = make_ulonglong2(v.lo, v.hi);
      counts[k] = v.cnt;
   }
};
// ---------------------------------------------------------------- MIN / MAX segment tree
// node k (1 <= k < 2 leaves) covers leaves [k << d, (k + 1) << d) of its level; leaf `leaves + i` is row i in window order.  A NULL
// leaf (and the padding past n) holds the identity of the operation, and any[k] says whether the node covers a non-NULL value.
template <class V>
__device__ __forceinline__ V winIdentity(int isMax);
template <>
__device__ __forceinline__ long long winIdentity<long long>(int isMax) { return isMax ? LLONG_MIN : LLONG_MAX; }
template <>
__device__ __forceinline__ s128 winIdentity<s128>(int isMax) {
   const unsigned __int128 top = (unsigned __int128) 1 << 127;
   return isMax ? (s128) top : (s128) (top - 1);
}
template <class V>
__device__ __forceinline__ V winPick(V a, V b, int isMax) { return isMax ? (a > b ? a : b) : (a < b ? a : b); }
template <class V>
__global__ void __launch_bounds__(kWinThreads) winTreeLeavesKernel(ProgCol arg, const uint32_t* ids, int64_t n, uint64_t leaves, int isMax, V* val, uint8_t* any) {
   for (uint64_t i = (uint64_t) blockIdx.x * kWinThreads + threadIdx.x; i < leaves; i += (uint64_t) gridDim.x * kWinThreads) {
      bool has = false;
      V v = winIdentity<V>(isMax);
      if (i < (uint64_t) n) {
         const Val x = loadCol(arg, winRow(ids, (int64_t) i));
         if (!x.null) {
            has = true;
            v = (V) x.v;
         }
      }
      val[leaves + i] = v;
      any[leaves + i] = has ? 1 : 0;
   }
}
// the m nodes of one level, [m, 2m), from the level below
template <class V>
__global__ void __launch_bounds__(kWinThreads) winTreeLevelKernel(uint64_t m, int isMax, V* val, uint8_t* any) {
   for (uint64_t k = m + (uint64_t) blockIdx.x * kWinThreads + threadIdx.x; k < 2 * m; k += (uint64_t) gridDim.x * kWinThreads) {
      val[k] = winPick(val[2 * k], val[2 * k + 1], isMax);
      any[k] = any[2 * k] | any[2 * k + 1];
   }
}
template <class V>
__device__ __forceinline__ void winTreeQuery(const V* val, const uint8_t* any, uint64_t leaves, uint64_t lo, uint64_t hi, int isMax, V& acc, bool& has) {
   acc = winIdentity<V>(isMax);
   has = false;
   for (uint64_t l = lo + leaves, r = hi + leaves + 1; l < r; l >>= 1, r >>= 1) {
      if (l & 1) {
         acc = winPick(acc, val[l], isMax);
         has |= any[l] != 0;
         l++;
      }
      if (r & 1) {
         --r;
         acc = winPick(acc, val[r], isMax);
         has |= any[r] != 0;
      }
   }
}

// ---------------------------------------------------------------- frames and function values
struct WinFunc {
   int32_t kind, width, wide, pad; // width: output cell bytes (MIN / MAX); wide: the tree holds i128 nodes
   uint8_t* out;
   uint8_t* valid;                  // SUM, MIN, MAX
   const unsigned long long* sums;  // SUM: the scan's i128 prefix sums
   const unsigned long long* counts; // SUM, COUNT: the scan's prefix counts
   const void* tree;                 // MIN, MAX
   const uint8_t* any;
};
struct WinFrameParams {
   const uint32_t* start;
   const uint32_t* end;
   int64_t n, from, to; // offsets already limited to +-2^40 (|j| < 2^32, so the clamp gives the same bounds)
   int32_t fromUnbounded, toUnbounded, nFuncs, pad;
   uint64_t leaves;
   WinFunc f[kWinMaxFuncs];
};
__device__ __forceinline__ void winStoreCell(uint8_t* out, int width, int64_t i, s128 v) {
   uint8_t* p = out + (size_t) i * width;
   switch (width) {
      case 16: *(ulonglong2*) p = make_ulonglong2((unsigned long long) v, (unsigned long long) ((unsigned __int128) v >> 64)); break;
      case 8: *(long long*) p = (long long) v; break;
      case 4: *(int32_t*) p = (int32_t) v; break;
      case 2: *(int16_t*) p = (int16_t) v; break;
      default: *(int8_t*) p = (int8_t) v;
   }
}
__global__ void __launch_bounds__(kWinThreads) winFramesKernel(const __grid_constant__ WinFrameParams p) {
   for (int64_t i = (int64_t) blockIdx.x * kWinThreads + threadIdx.x; i < p.n; i += (int64_t) gridDim.x * kWinThreads) {
      const int64_t s = p.start[i], len = (int64_t) p.end[i] - s + 1, j = i - s;
      const int64_t lo = s + (p.fromUnbounded ? 0 : min(len - 1, max((int64_t) 0, j + p.from)));
      const int64_t hi = p.toUnbounded ? s + len - 1 : s + min(len - 1, max((int64_t) 0, j + p.to));
      for (int q = 0; q < p.nFuncs; q++) {
         const WinFunc& f = p.f[q];
         switch (f.kind) {
            case LDB_WIN_ROW_NUMBER: ((int64_t*) f.out)[i] = i - lo + 1; break;
            case LDB_WIN_COUNT_STAR: ((int64_t*) f.out)[i] = hi - lo + 1; break;
            case LDB_WIN_COUNT: ((int64_t*) f.out)[i] = (int64_t) (f.counts[hi] - (lo ? f.counts[lo - 1] : 0ull)); break;
            case LDB_WIN_SUM: {
               const unsigned long long c = f.counts[hi] - (lo ? f.counts[lo - 1] : 0ull);
               const ulonglong2 a = *(const ulonglong2*) (f.sums + 2 * hi);
               const ulonglong2 b = lo ? *(const ulonglong2*) (f.sums + 2 * (lo - 1)) : make_ulonglong2(0, 0);
               const unsigned long long dlo = a.x - b.x, dhi = a.y - b.y - (a.x < b.x ? 1ull : 0ull);
               *(ulonglong2*) (f.out + (size_t) i * 16) = c ? make_ulonglong2(dlo, dhi) : make_ulonglong2(0, 0);
               f.valid[i] = c ? 1 : 0;
               break;
            }
            default: { // MIN, MAX
               const int isMax = f.kind == LDB_WIN_MAX;
               bool has;
               s128 v;
               if (f.wide) {
                  winTreeQuery((const s128*) f.tree, f.any, p.leaves, (uint64_t) lo, (uint64_t) hi, isMax, v, has);
               } else {
                  long long w;
                  winTreeQuery((const long long*) f.tree, f.any, p.leaves, (uint64_t) lo, (uint64_t) hi, isMax, w, has);
                  v = w;
               }
               winStoreCell(f.out, f.width, i, has ? v : (s128) 0);
               f.valid[i] = has ? 1 : 0;
            }
         }
      }
   }
}

// ---------------------------------------------------------------- host side
static unsigned winGrid(const LdbContext* ctx, uint64_t items) {
   return (unsigned) std::max<uint64_t>(1, std::min<uint64_t>((items + kWinThreads - 1) / kWinThreads, (uint64_t) ctx->smCount * 16));
}
template <class V>
static void winTree(LdbContext* ctx, const ProgCol& arg, const uint32_t* ids, int64_t n, uint64_t leaves, int isMax, V* val, uint8_t* any) {
   ctx->launch("window_tree", [&] {
      winTreeLeavesKernel<V><<<winGrid(ctx, leaves), kWinThreads, 0, ctx->compute>>>(arg, ids, n, leaves, isMax, val, any);
      for (uint64_t m = leaves / 2; m >= 1; m /= 2) winTreeLevelKernel<V><<<winGrid(ctx, m), kWinThreads, 0, ctx->compute>>>(m, isMax, val, any);
   });
}

static bool winKeyType(int type) { return type == LDB_INT32 || type == LDB_DATE32 || type == LDB_FSB4 || type == LDB_INT64 || type == LDB_DECIMAL128 || type == LDB_UTF8; }
static bool winSumType(int type) { return type == LDB_INT8 || type == LDB_INT16 || type == LDB_INT32 || type == LDB_INT64 || type == LDB_DECIMAL128; }

static void tableWindow(LdbTable* src, int32_t n_partition, const char* const* partition_columns, int32_t n_order, const char* const* order_columns,
                        const int32_t* descending, int64_t frame_from, int64_t frame_to, int32_t n_funcs, const LdbWindowFunc* funcs, int32_t n_columns,
                        const char* const* columns, const char* name, LdbTable** out) {
   // everything is checked before the first launch
   if (!src || !out || (n_partition > 0 && !partition_columns) || (n_order > 0 && (!order_columns || !descending)) || (n_funcs > 0 && !funcs))
      fail(LDB_ERR_INVALID, "null argument");
   if (n_partition < 0 || n_partition > kProgMaxKeys || n_order < 0 || n_order > kProgMaxKeys) fail(LDB_ERR_INVALID, "a window takes 0..4 partition keys and 0..4 order keys");
   if (n_funcs < 1 || n_funcs > kWinMaxFuncs) fail(LDB_ERR_INVALID, "a window computes 1..8 functions");
   if (n_columns < 0 || (columns && n_columns > kWinMaxCarried)) fail(LDB_ERR_INVALID, "a window carries 0..16 columns");
   if (frame_from > frame_to || frame_from == INT64_MAX || frame_to == INT64_MIN)
      fail(LDB_ERR_INVALID, "bad frame: from must be <= to, from may not be UNBOUNDED FOLLOWING (INT64_MAX) nor to UNBOUNDED PRECEDING (INT64_MIN)");
   auto column = [&](const char* c, const char* what) {
      const int ci = src->colIndex(c);
      if (ci < 0) fail(LDB_ERR_INVALID, std::string("unknown ") + what + " column " + (c ? c : "(null)"));
      return ci;
   };
   std::vector<std::pair<int, int>> keys; // partition keys ascending, then the order keys
   for (int k = 0; k < n_partition + n_order; k++) {
      const bool part = k < n_partition;
      const int ci = column(part ? partition_columns[k] : order_columns[k - n_partition], part ? "partition" : "order");
      if (!winKeyType(src->columns[ci].type))
         fail(LDB_ERR_UNSUPPORTED, "window keys are int32, date32, char(1), int64, decimal or utf8 columns (column " + src->columns[ci].name + ")");
      keys.push_back({ci, part ? 0 : (descending[k - n_partition] ? 1 : 0)});
   }
   std::vector<int> argCol(n_funcs, -1);
   for (int q = 0; q < n_funcs; q++) {
      const int kind = funcs[q].kind;
      if (kind < LDB_WIN_ROW_NUMBER || kind > LDB_WIN_MAX) fail(LDB_ERR_INVALID, "unknown window function kind " + std::to_string(kind));
      if (!funcs[q].name) fail(LDB_ERR_INVALID, "a window function needs an output column name");
      if (kind == LDB_WIN_ROW_NUMBER || kind == LDB_WIN_COUNT_STAR) continue;
      const int ci = argCol[q] = column(funcs[q].column, "argument");
      const int type = src->columns[ci].type;
      if (kind == LDB_WIN_SUM && !winSumType(type))
         fail(LDB_ERR_UNSUPPORTED, "window SUM takes int8..int64 or decimal columns (column " + src->columns[ci].name + ")");
      if ((kind == LDB_WIN_MIN || kind == LDB_WIN_MAX) && !winSumType(type) && type != LDB_DATE32 && type != LDB_FSB4)
         fail(LDB_ERR_UNSUPPORTED, "window MIN / MAX take int8..int64, decimal, date32 or char(1) columns (column " + src->columns[ci].name + ")");
   }
   std::vector<int> carried;
   if (columns) {
      for (int j = 0; j < n_columns; j++) carried.push_back(column(columns[j], "carried"));
   } else {
      for (int ci = 0; ci < (int) src->columns.size(); ci++) carried.push_back(ci);
      if (carried.size() > (size_t) kWinMaxCarried) fail(LDB_ERR_INVALID, "a window carries 0..16 columns: name them (the table has more)");
   }
   // every column of the result is found by its name (the first match), so no two may share one: a function named like a carried
   // column, two functions of one name or a column carried twice would leave a column that no later call can read
   const size_t nCarried = carried.size();
   for (size_t a = 0; a < nCarried + n_funcs; a++) {
      const std::string na = a < nCarried ? src->columns[carried[a]].name : std::string(funcs[a - nCarried].name);
      for (size_t b = 0; b < a; b++) {
         const std::string nb = b < nCarried ? src->columns[carried[b]].name : std::string(funcs[b - nCarried].name);
         if (na != nb) continue;
         const char* what = a < nCarried ? "a column carried twice" : b < nCarried ? "a function named like a carried column" : "two functions of one name";
         fail(LDB_ERR_INVALID, "window output column " + na + " is named twice (" + what + ")");
      }
   }
   if (src->batches.size() > 1) fail(LDB_ERR_UNSUPPORTED, "windows run over single-batch tables (materialised results, exported groups, received or sorted tables)");
   const int64_t n = src->numRows;
   if (n >= (int64_t) 1 << 32) fail(LDB_ERR_UNSUPPORTED, "a window handles up to 2^32 - 1 rows");
   LdbContext* ctx = src->ctx;
   if (ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "the window operator sizes its sort on the host and cannot be captured");

   LDB_CUDA(cudaSetDevice(ctx->device));
   if (!src->batches.empty()) ldb_gpu_wait_batch_internal(ctx, &src->batches[0]);
   Scratch sorted(ctx), cols(ctx), tmp(ctx);
   const uint32_t* ids = n > 0 && !keys.empty() ? sortRows(sorted, src, keys, n) : nullptr; // null: source order
   std::vector<int32_t> widths;
   for (int ci : carried) widths.push_back(shipCellBytes(src->columns[ci].type));
   LdbBatch ob;
   if (!carried.empty()) {
      ob = permuteRows(src, carried, widths.data(), ids, n, cols, "window");
   } else {
      ob.nRows = n;
   }
   std::vector<LdbColumn> outCols;
   for (int ci : carried) outCols.push_back(src->columns[ci]);

   const size_t rows = (size_t) std::max<int64_t>(n, 1);
   WinFrameParams fp{};
   fp.n = n;
   fp.fromUnbounded = frame_from == INT64_MIN;
   fp.toUnbounded = frame_to == INT64_MAX;
   constexpr int64_t kLimit = (int64_t) 1 << 40;
   fp.from = std::min(kLimit, std::max(-kLimit, frame_from));
   fp.to = std::min(kLimit, std::max(-kLimit, frame_to));
   fp.nFuncs = n_funcs;
   fp.leaves = nextPow2((uint64_t) std::max<int64_t>(n, 1));
   for (int q = 0; q < n_funcs; q++) {
      const int kind = funcs[q].kind;
      WinFunc& f = fp.f[q];
      f.kind = kind;
      const LdbColumn* a = argCol[q] >= 0 ? &src->columns[argCol[q]] : nullptr;
      const int32_t argBytes = argCol[q] >= 0 && !src->batches.empty() ? src->batches[0].elemBytes[argCol[q]] : (a ? shipCellBytes(a->type) : 8);
      if (kind == LDB_WIN_SUM) {
         f.width = 16;
         outCols.push_back({funcs[q].name, LDB_DECIMAL128, 38, a->type == LDB_DECIMAL128 ? a->scale : 0});
      } else if (kind == LDB_WIN_MIN || kind == LDB_WIN_MAX) {
         f.width = argBytes;
         f.wide = argBytes == 16;
         outCols.push_back({funcs[q].name, a->type, a->precision, a->scale});
      } else {
         f.width = 8;
         outCols.push_back({funcs[q].name, LDB_INT64, 0, 0});
      }
      f.out = cols.alloc<uint8_t>(std::max<size_t>(rows * f.width, 16));
      const bool nullable = kind == LDB_WIN_SUM || kind == LDB_WIN_MIN || kind == LDB_WIN_MAX;
      if (nullable) f.valid = cols.alloc<uint8_t>(std::max<size_t>(rows, 16));
      ob.data.push_back(f.out);
      ob.bytes.push_back(nullptr);
      ob.elemBytes.push_back(f.width);
      ob.validBytes.push_back(f.valid);
   }

   if (n > 0) {
      // partition bounds
      uint32_t* start = tmp.alloc<uint32_t>(rows * 4);
      uint32_t* end = tmp.alloc<uint32_t>(rows * 4);
      uint8_t* head = tmp.alloc<uint8_t>(rows);
      WinKeys wk{};
      wk.n = n_partition;
      for (int k = 0; k < n_partition; k++) {
         bindColumn(wk.col[k], src->batches[0], keys[k].first);
         wk.col[k].type = src->columns[keys[k].first].type;
      }
      ctx->launch("window_partition", [&] { winHeadsKernel<<<winGrid(ctx, (uint64_t) n), kWinThreads, 0, ctx->compute>>>(wk, ids, n, head); });
      tileScan(ctx, tmp, WinStartOp{head, start}, n, "window_scan");
      tileScan(ctx, tmp, WinEndOp{head, end, n}, n, "window_scan");
      fp.start = start;
      fp.end = end;
      // per function its scan or its tree
      for (int q = 0; q < n_funcs; q++) {
         WinFunc& f = fp.f[q];
         if (argCol[q] < 0) continue;
         ProgCol arg{};
         bindColumn(arg, src->batches[0], argCol[q]);
         arg.type = src->columns[argCol[q]].type;
         if (f.kind == LDB_WIN_SUM || f.kind == LDB_WIN_COUNT) {
            unsigned long long* sums = f.kind == LDB_WIN_SUM ? tmp.alloc<unsigned long long>(rows * 16) : nullptr;
            unsigned long long* counts = tmp.alloc<unsigned long long>(rows * 8);
            tileScan(ctx, tmp, WinSumOp{arg, ids, sums, counts}, n, "window_scan");
            f.sums = sums;
            f.counts = counts;
         } else {
            const int isMax = f.kind == LDB_WIN_MAX;
            uint8_t* any = tmp.alloc<uint8_t>(2 * fp.leaves);
            if (f.wide) {
               s128* val = tmp.alloc<s128>(2 * fp.leaves * 16);
               winTree(ctx, arg, ids, n, fp.leaves, isMax, val, any);
               f.tree = val;
            } else {
               long long* val = tmp.alloc<long long>(2 * fp.leaves * 8);
               winTree(ctx, arg, ids, n, fp.leaves, isMax, val, any);
               f.tree = val;
            }
            f.any = any;
         }
      }
      ctx->launch("window_frames", [&] { winFramesKernel<<<winGrid(ctx, (uint64_t) n), kWinThreads, 0, ctx->compute>>>(fp); });
   }
   ctx->syncStream(ctx->compute); // the sort's and the scans' temporaries go back to the pool
   *out = addResultTable(ctx, name ? name : "window", std::move(outCols), std::move(ob), cols);
}

} // namespace ldb

static_assert(sizeof(ldb::WinFrameParams) <= 4096, "the frames kernel's parameters");

extern "C" int ldb_gpu_table_window(LdbTable* src, int32_t n_partition, const char* const* partition_columns, int32_t n_order, const char* const* order_columns,
                                    const int32_t* descending, int64_t frame_from, int64_t frame_to, int32_t n_funcs, const LdbWindowFunc* funcs, int32_t n_columns,
                                    const char* const* columns, const char* name, LdbTable** out, LdbError* err) {
   return ldb::guarded(err, [&] {
      ldb::tableWindow(src, n_partition, partition_columns, n_order, order_columns, descending, frame_from, frame_to, n_funcs, funcs, n_columns, columns, name, out);
   });
}
