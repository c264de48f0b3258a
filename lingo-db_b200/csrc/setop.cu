// setop.cu — set operations over whole rows (ldb_gpu_table_setop, include/ldb_gpu.h): SELECT DISTINCT (ProjectionDistinctLowering,
// RelAlgToSubOp.cpp:337-394), UNION ALL (UnionAllLowering, :622-634), UNION (UnionDistinctLowering, :636-727) and INTERSECT [ALL] /
// EXCEPT [ALL] (CountingSetOperationLowering, :728-916).  The reference lowers each to a subop::MapType keyed on the whole row
// (LookupOrInsertOp), with two counters per entry for the counting operations; this file is that map on the device.
//
// Semantics, rule by rule:
//   Row equality: compareKeys (:142-153) is db.cmp isa, IS NOT DISTINCT FROM, on every column: NULL equals NULL and never a value, the
//     bytes under a NULL cell are not read.  utf8 compares by length and bytes; integers, dates, char(1) and decimals by their value
//     sign-extended to 128 bits (loadCol), so a narrowed 8-byte decimal cell equals the same value in a 16-byte cell; floats by their
//     bits after -0.0 -> +0.0 and every NaN -> one NaN (setF64Bits).  The float rule is OUR DEFINITION: the reference compares floats
//     with oeq but hashes their bits, so its answer on zeros and NaN depends on the hash.
//   Multiplicities (:849-913), cL / cR the occurrences of a row in left / right: DISTINCT and UNION 1; UNION ALL every row of both
//     sides; INTERSECT 1 if cL > 0 && cR > 0; EXCEPT 1 if cL > 0 && cR == 0; INTERSECT ALL min(cL, cR); EXCEPT ALL max(cL - cR, 0).
//   Order: the reference scans its hash map, so its order is unspecified.  Ours: each distinct row at the position of its first
//     occurrence in the left rows followed by the right rows, its ALL copies consecutive, its cells those of that first occurrence.
//
// Device work, over a view whose batches are left's, then right's (row i of the view is row i of left for i < nL):
//   1. setInsertKernel: per row its whole-row hash (mix64 over per-column words, utf8 through strHash), then a lookup-or-insert into
//      an open-addressing directory of nextPow2(2 x inserted rows) slot words tag << 32 | (row + 1).  A slot is claimed by one CAS: the
//      row's cells are in memory already and never change, so an entry is complete once claimed and no reader waits.  A tag match
//      compares the two rows cell by cell.  Each row records its entry (the row that claimed the slot, its "representative"); the
//      entry's first row (atomicMin) and its counter of the row's side (+1) are updated once per warp and entry (__match_any_sync:
//      the lowest lane holds the smallest row, the leader adds the popcount), so many equal rows do not serialise on one address.
//      DISTINCT and UNION insert every row.  INTERSECT and EXCEPT insert the left rows, then the right rows only probe (a second launch)
//      and count their hits; a right row that matches nothing makes no entry.
//   2. setCountKernel: per emitting row (every row for DISTINCT / UNION, the left rows otherwise) its entry's multiplicity if it is the
//      entry's first row, else 0.
//   3. The tile scan (tilescan.cuh) of the counts; its store writes each row's ids into its output range, rows of more than kSetDirect
//      copies are listed and written by setBigKernel, one CTA per row.
//   4. permuteRows (peer.cu) gathers the ids' cells into the result batch.  UNION ALL is steps 4 alone, over the view in order.
#include "context.h"
#include "keyhash.cuh"
#include "progcol.cuh"
#include "tilescan.cuh"

#include <algorithm>

namespace ldb {

constexpr int kSetThreads = 256, kSetMaxCols = 16;
constexpr uint32_t kSetNone = 0xffffffffu; // no entry: a right row that matched nothing (rows are <= 2^32 - 2)
constexpr uint32_t kSetDirect = 64;        // copies of a row the scan's store writes itself; more go to setBigKernel

struct SetBatch {
   ProgCol cols[kSetMaxCols];
   int64_t firstRow;
};
struct SetParams {
   const SetBatch* dir; // device, sorted by firstRow, non-empty batches only
   int32_t nBatches, nCols;
   unsigned long long* slots; // the directory: tag << 32 | (representative row + 1), 0 = empty
   uint64_t mask;             // slots - 1
   uint32_t* entry;           // per row: its entry's representative row, or kSetNone
   uint32_t* first;           // per representative row: the entry's first row (0xffffffff until set)
   uint32_t* counts;          // per representative row: left and right occurrences, or null (DISTINCT, UNION)
   unsigned int* error;       // set when a lookup ran past the directory
};

__device__ __forceinline__ const SetBatch& setBatchOf(const SetParams& p, int64_t row) {
   int lo = 0, hi = p.nBatches - 1;
   while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (p.dir[mid].firstRow <= row) lo = mid;
      else hi = mid - 1;
   }
   return p.dir[lo];
}
__device__ __forceinline__ bool setIsFloat(int type) { return type == LDB_FLOAT32 || type == LDB_FLOAT64; }
// a cell's word for the row hash (the value rules are keyhash.cuh's): equal cells (by the rule above) give equal words
__device__ __forceinline__ uint64_t setCellWord(const ProgCol& c, int64_t r) {
   if (colIsNull(c, r)) return kSetNullWord;
   if (c.type == LDB_UTF8) {
      const int32_t* o = (const int32_t*) c.data;
      return strHash(c.bytes + o[r], o[r + 1] - o[r]);
   }
   const Val v = loadCol(c, r);
   if (setIsFloat(c.type)) return setF64Bits(asF64(v));
   return setIntWord((uint64_t) v.v, (uint64_t) (v.v >> 64));
}
__device__ __forceinline__ bool setCellEq(const ProgCol& a, int64_t ra, const ProgCol& b, int64_t rb) {
   const bool na = colIsNull(a, ra), nb = colIsNull(b, rb);
   if (na || nb) return na == nb;
   if (a.type == LDB_UTF8) {
      const int32_t* oa = (const int32_t*) a.data;
      const int32_t* ob = (const int32_t*) b.data;
      const int32_t a0 = oa[ra], b0 = ob[rb], len = oa[ra + 1] - a0;
      if (ob[rb + 1] - b0 != len) return false;
      for (int32_t x = 0; x < len; x++)
         if (a.bytes[a0 + x] != b.bytes[b0 + x]) return false;
      return true;
   }
   const Val x = loadCol(a, ra), y = loadCol(b, rb);
   if (setIsFloat(a.type)) return setF64Bits(asF64(x)) == setF64Bits(asF64(y));
   return x.v == y.v;
}
// the whole-row hash: keyTupleHash's step over the cell words, in column order
__device__ __forceinline__ uint64_t setRowHash(const SetParams& p, const SetBatch& b, int64_t r) {
   return setRowFold(p.nCols, [&](int c) { return setCellWord(b.cols[c], r); });
}
__device__ __forceinline__ bool setRowsEqual(const SetParams& p, const SetBatch& b, int64_t r, int64_t other) {
   const SetBatch& o = setBatchOf(p, other);
   const int64_t ro = other - o.firstRow;
   for (int c = 0; c < p.nCols; c++)
      if (!setCellEq(b.cols[c], r, o.cols[c], ro)) return false;
   return true;
}

// rows [begin, end) of the view: look up (insert: or insert) each row's entry, then count it on `side` (0 left, 1 right)
__global__ void __launch_bounds__(kSetThreads) setInsertKernel(const __grid_constant__ SetParams p, int64_t begin, int64_t end, int insert, int side) {
   const int lane = threadIdx.x & 31;
   for (int64_t base = begin + (int64_t) blockIdx.x * kSetThreads; base < end; base += (int64_t) gridDim.x * kSetThreads) {
      const int64_t i = base + threadIdx.x;
      uint32_t rep = kSetNone;
      if (i < end) {
         const SetBatch& b = setBatchOf(p, i);
         const int64_t r = i - b.firstRow;
         const uint64_t h = setRowHash(p, b, r);
         const unsigned long long tag = (h >> 32) << 32;
         uint64_t s = h & p.mask;
         for (uint64_t probes = 0; probes <= p.mask; probes++) {
            unsigned long long w = *(volatile unsigned long long*) (p.slots + s);
            if (w == 0) {
               if (!insert) break;
               w = atomicCAS(p.slots + s, 0ull, tag | (unsigned long long) (i + 1));
               if (w == 0) {
                  rep = (uint32_t) i;
                  break;
               }
            }
            if ((w & 0xffffffff00000000ull) == tag && setRowsEqual(p, b, r, (int64_t) (uint32_t) w - 1)) {
               rep = (uint32_t) w - 1;
               break;
            }
            s = (s + 1) & p.mask;
         }
         if (insert && rep == kSetNone) atomicExch(p.error, 1u);
         p.entry[i] = rep;
      }
      // once per warp and entry: lanes hold consecutive rows, so the lowest lane of a group holds its smallest row
      const unsigned peers = __match_any_sync(0xffffffffu, rep);
      if (rep != kSetNone && lane == __ffs(peers) - 1) {
         if (insert && p.first[rep] > (uint32_t) i) atomicMin(p.first + rep, (uint32_t) i);
         if (p.counts) atomicAdd(p.counts + 2 * (size_t) rep + side, (uint32_t) __popc(peers));
      }
   }
}
// per emitting row: its entry's multiplicity if it is the entry's first row, else 0
__global__ void __launch_bounds__(kSetThreads) setCountKernel(const __grid_constant__ SetParams p, int kind, int64_t n, uint32_t* cnt) {
   for (int64_t i = (int64_t) blockIdx.x * kSetThreads + threadIdx.x; i < n; i += (int64_t) gridDim.x * kSetThreads) {
      const uint32_t rep = p.entry[i];
      uint32_t c = 0;
      if (rep != kSetNone && p.first[rep] == (uint32_t) i) {
         const uint32_t cl = p.counts ? p.counts[2 * (size_t) rep] : 1u, cr = p.counts ? p.counts[2 * (size_t) rep + 1] : 0u;
         switch (kind) {
            case LDB_SET_INTERSECT: c = cr > 0; break;
            case LDB_SET_EXCEPT: c = cr == 0; break;
            case LDB_SET_INTERSECT_ALL: c = min(cl, cr); break;
            case LDB_SET_EXCEPT_ALL: c = cl > cr ? cl - cr : 0u; break;
            default: c = 1; // DISTINCT, UNION
         }
      }
      cnt[i] = c;
   }
}
// the scan of the counts; its store writes row k's ids into [incl - cnt[k], incl), or lists the row when it has many copies
struct SetExpandOp {
   using T = uint32_t;
   const uint32_t* cnt;
   uint32_t* ids;
   uint32_t* big;      // rows of more than kSetDirect copies, and where their ranges end
   uint32_t* bigEnd;
   unsigned int* ctr;  // [1] rows listed in big, [2] the total
   int64_t n;
   __device__ T identity() const { return 0; }
   __device__ T combine(T a, T b) const { return a + b; }
   __device__ T load(int64_t k) const { return cnt[k]; }
   __device__ void store(int64_t k, T v) const {
      const uint32_t c = cnt[k];
      if (k == n - 1) ctr[2] = v;
      if (c <= kSetDirect) {
         for (uint32_t j = 0; j < c; j++) ids[v - c + j] = (uint32_t) k;
      } else {
         const unsigned at = atomicAdd(ctr + 1, 1u);
         big[at] = (uint32_t) k;
         bigEnd[at] = v;
      }
   }
};
__global__ void __launch_bounds__(kSetThreads) setBigKernel(const uint32_t* cnt, const uint32_t* big, const uint32_t* bigEnd, const unsigned int* ctr, uint32_t* ids) {
   for (unsigned b = blockIdx.x; b < ctr[1]; b += gridDim.x) {
      const uint32_t k = big[b], c = cnt[k], e = bigEnd[b];
      for (uint32_t j = threadIdx.x; j < c; j += kSetThreads) ids[e - c + j] = k;
   }
}

// ---------------------------------------------------------------- host side
static unsigned setGrid(const LdbContext* ctx, uint64_t items) {
   return (unsigned) std::max<uint64_t>(1, std::min<uint64_t>((items + kSetThreads - 1) / kSetThreads, (uint64_t) ctx->smCount * 16));
}
static bool setType(int type) {
   switch (type) {
      case LDB_INT8:
      case LDB_INT16:
      case LDB_INT32:
      case LDB_INT64:
      case LDB_DATE32:
      case LDB_FSB4:
      case LDB_DECIMAL128:
      case LDB_FLOAT32:
      case LDB_FLOAT64:
      case LDB_UTF8: return true;
      default: return false;
   }
}
static std::vector<int> setColumns(const LdbTable* t, int32_t n, const char* const* names, const char* side) {
   std::vector<int> cols;
   if (!names) {
      for (int ci = 0; ci < (int) t->columns.size(); ci++) cols.push_back(ci);
      return cols;
   }
   for (int j = 0; j < n; j++) {
      const int ci = t->colIndex(names[j]);
      if (ci < 0) fail(LDB_ERR_INVALID, std::string("unknown ") + side + " column " + (names[j] ? names[j] : "(null)"));
      cols.push_back(ci);
   }
   return cols;
}
// the view's batches for `cols` of t: the batch's pointers for those columns only, nothing owned
static void setViewBatches(LdbTable& view, const LdbTable* t, const std::vector<int>& cols) {
   for (const LdbBatch& b : t->batches) {
      LdbBatch v;
      v.nRows = b.nRows;
      for (int ci : cols) {
         v.data.push_back(b.data[ci]);
         v.bytes.push_back(b.bytes[ci]);
         v.elemBytes.push_back(b.elemBytes[ci]);
         v.validity.push_back(ci < (int) b.validity.size() ? b.validity[ci] : nullptr);
         v.validityBitOffset.push_back(ci < (int) b.validityBitOffset.size() ? b.validityBitOffset[ci] : 0);
         v.validBytes.push_back(ci < (int) b.validBytes.size() ? b.validBytes[ci] : nullptr);
      }
      view.batches.push_back(std::move(v));
   }
}

static void tableSetop(LdbTable* left, LdbTable* right, int32_t kind, int32_t n_columns, const char* const* left_columns, const char* const* right_columns,
                       const char* name, LdbTable** out) {
   // everything is checked before the first launch
   if (!left || !out) fail(LDB_ERR_INVALID, "null argument");
   if (kind < LDB_SET_DISTINCT || kind > LDB_SET_EXCEPT_ALL) fail(LDB_ERR_INVALID, "unknown set operation kind " + std::to_string(kind));
   if (kind == LDB_SET_DISTINCT && (right || right_columns)) fail(LDB_ERR_INVALID, "DISTINCT takes no right table");
   if (kind != LDB_SET_DISTINCT && !right) fail(LDB_ERR_INVALID, "null argument: the set operation needs a right table");
   if (right && right->ctx != left->ctx) fail(LDB_ERR_INVALID, "left and right tables belong to different contexts");
   if ((left_columns || right_columns) && (n_columns < 1 || n_columns > kSetMaxCols)) fail(LDB_ERR_INVALID, "a set operation takes 1..16 columns");
   const std::vector<int> lc = setColumns(left, n_columns, left_columns, "left");
   const std::vector<int> rc = right ? setColumns(right, n_columns, right_columns, "right") : lc;
   if (lc.size() != rc.size()) fail(LDB_ERR_INVALID, "the column lists of a set operation have different lengths (" + std::to_string(lc.size()) + " and " + std::to_string(rc.size()) + ")");
   if (lc.empty() || lc.size() > (size_t) kSetMaxCols) fail(LDB_ERR_INVALID, "a set operation takes 1..16 columns (it has " + std::to_string(lc.size()) + ")");
   // the result takes left's names, and later calls find a column by its first match: a repeated left name would be unreadable (right
   // names are positional and may repeat)
   for (size_t j = 0; j < lc.size(); j++)
      for (size_t k = 0; k < j; k++)
         if (left->columns[lc[j]].name == left->columns[lc[k]].name)
            fail(LDB_ERR_INVALID, "the set operation's result would have two columns named " + left->columns[lc[j]].name + " (left columns " +
                                     std::to_string(k) + " and " + std::to_string(j) + ")");
   const LdbTable* rt = right ? right : left;
   std::vector<LdbColumn> outCols;
   std::vector<int32_t> widths;
   for (size_t j = 0; j < lc.size(); j++) {
      const LdbColumn& a = left->columns[lc[j]];
      const LdbColumn& b = rt->columns[rc[j]];
      if (!setType(a.type)) fail(LDB_ERR_UNSUPPORTED, "set operations take integer, date, char(1), decimal, float or utf8 columns (column " + a.name + ")");
      if (a.type != b.type) fail(LDB_ERR_UNSUPPORTED, "set operation columns " + a.name + " and " + b.name + " have different physical types");
      if (a.type == LDB_DECIMAL128 && a.scale != b.scale)
         fail(LDB_ERR_UNSUPPORTED, "set operation columns " + a.name + " and " + b.name + " are decimals of different scales (cast one)");
      LdbColumn c = a;
      if (a.type == LDB_DECIMAL128) c.precision = std::max(a.precision, b.precision);
      outCols.push_back(c);
      widths.push_back(shipCellBytes(a.type));
   }
   const int64_t nL = left->numRows, nR = right ? right->numRows : 0, n = nL + nR;
   if (n >= (int64_t) 1 << 32) fail(LDB_ERR_UNSUPPORTED, "a set operation handles fewer than 2^32 rows on both sides together");
   LdbContext* ctx = left->ctx;
   if (ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "a set operation reads its output size on the host and cannot be captured");

   LDB_CUDA(cudaSetDevice(ctx->device));
   for (auto& b : left->batches) ldb_gpu_wait_batch_internal(ctx, &b);
   if (right && right != left)
      for (auto& b : right->batches) ldb_gpu_wait_batch_internal(ctx, &b);
   LdbTable view{};
   view.ctx = ctx;
   view.numRows = n;
   view.columns = outCols;
   setViewBatches(view, left, lc);
   if (right) setViewBatches(view, right, rc);
   std::vector<int> all;
   for (size_t j = 0; j < lc.size(); j++) all.push_back((int) j);

   Scratch bufs(ctx), tmp(ctx);
   const bool counting = kind != LDB_SET_DISTINCT && kind != LDB_SET_UNION && kind != LDB_SET_UNION_ALL;
   const int64_t nIns = counting ? nL : n, nEmit = nIns;
   uint32_t* ids = nullptr;
   int64_t total = n;
   if (kind != LDB_SET_UNION_ALL) {
      total = 0;
      if (nEmit > 0) {
         std::vector<SetBatch> dir;
         int64_t firstRow = 0;
         for (const LdbBatch& b : view.batches) {
            if (b.nRows > 0) {
               SetBatch sb{};
               for (size_t j = 0; j < lc.size(); j++) {
                  bindColumn(sb.cols[j], b, (int) j);
                  sb.cols[j].type = outCols[j].type;
               }
               sb.firstRow = firstRow;
               dir.push_back(sb);
            }
            firstRow += b.nRows;
         }
         SetParams p{};
         p.nBatches = (int32_t) dir.size();
         p.nCols = (int32_t) lc.size();
         const uint64_t nSlots = nextPow2((uint64_t) std::max<int64_t>(2 * nIns, 2));
         p.mask = nSlots - 1;
         SetBatch* dd = tmp.alloc<SetBatch>(dir.size() * sizeof(SetBatch));
         p.dir = dd;
         p.slots = tmp.alloc<unsigned long long>(nSlots * 8);
         p.entry = tmp.alloc<uint32_t>((size_t) n * 4);
         p.first = tmp.alloc<uint32_t>((size_t) n * 4);
         p.counts = counting ? tmp.alloc<uint32_t>((size_t) n * 8) : nullptr;
         unsigned int* ctr = tmp.alloc<unsigned int>(16); // [0] error, [1] rows of many copies, [2] the total
         p.error = ctr;
         uint32_t* cnt = tmp.alloc<uint32_t>((size_t) nEmit * 4);
         const size_t bigCap = (size_t) nEmit / (kSetDirect + 1) + 1;
         uint32_t* big = tmp.alloc<uint32_t>(bigCap * 4);
         uint32_t* bigEnd = tmp.alloc<uint32_t>(bigCap * 4);
         ids = tmp.alloc<uint32_t>(std::max<size_t>((size_t) n, 1) * 4);
         LDB_CUDA(cudaMemcpyAsync(dd, dir.data(), dir.size() * sizeof(SetBatch), cudaMemcpyHostToDevice, ctx->compute));
         LDB_CUDA(cudaMemsetAsync(p.slots, 0, nSlots * 8, ctx->compute));
         LDB_CUDA(cudaMemsetAsync(p.first, 0xff, (size_t) n * 4, ctx->compute));
         if (p.counts) LDB_CUDA(cudaMemsetAsync(p.counts, 0, (size_t) n * 8, ctx->compute));
         LDB_CUDA(cudaMemsetAsync(ctr, 0, 16, ctx->compute));
         ctx->launch("setop_insert", [&] {
            setInsertKernel<<<setGrid(ctx, (uint64_t) nIns), kSetThreads, 0, ctx->compute>>>(p, 0, nIns, 1, 0);
            if (counting && nR > 0) setInsertKernel<<<setGrid(ctx, (uint64_t) nR), kSetThreads, 0, ctx->compute>>>(p, nL, n, 0, 1);
         });
         ctx->launch("setop_count", [&] { setCountKernel<<<setGrid(ctx, (uint64_t) nEmit), kSetThreads, 0, ctx->compute>>>(p, kind, nEmit, cnt); });
         tileScan(ctx, tmp, SetExpandOp{cnt, ids, big, bigEnd, ctr, nEmit}, nEmit, "setop_scan");
         ctx->launch("setop_scan", [&] { setBigKernel<<<(unsigned) ctx->smCount * 4, kSetThreads, 0, ctx->compute>>>(cnt, big, bigEnd, ctr, ids); });
         unsigned int* host = (unsigned int*) ctx->scratch();
         LDB_CUDA(cudaMemcpyAsync(host, ctr, 16, cudaMemcpyDeviceToHost, ctx->compute));
         ctx->syncStream(ctx->compute);
         if (host[0]) fail(LDB_ERR_CAPACITY, "set operation: a lookup ran past the device set's directory");
         total = host[2];
      }
   }
   LdbBatch ob = permuteRows(&view, all, widths.data(), ids, total, bufs, "set operation");
   *out = addResultTable(ctx, name ? name : "setop", std::move(outCols), std::move(ob), bufs);
}

} // namespace ldb

static_assert(sizeof(ldb::SetParams) <= 4096, "the set kernels' parameters");

extern "C" int ldb_gpu_table_setop(LdbTable* left, LdbTable* right, int32_t kind, int32_t n_columns, const char* const* left_columns,
                                   const char* const* right_columns, const char* name, LdbTable** out, LdbError* err) {
   return ldb::guarded(err, [&] { ldb::tableSetop(left, right, kind, n_columns, left_columns, right_columns, name, out); });
}
