// nljoin.cu — nested-loop joins (ldb_gpu_table_nl_join, include/ldb_gpu.h): the reference's translateNLJ (RelAlgToSubOp.cpp:948) for
// inner, semi, anti, mark, outer and single joins, translateNLJWithMarker (:1217) for the joins that keep the build side (right and full
// outer, whose unmatched rows come from the marker flag) and CrossProductLowering (:1306) for a join without a predicate.  The reference
// materialises one side into a buffer and, for every row of the other, scans that buffer (NestedMapOp) and evaluates the predicate;
// here every pair of a left tile and a right chunk is one CTA's loop over words kept on chip.
//
// Semantics, rule by rule:
//   Predicate: the conjunction of the conditions (the ON expression's db.and); a pair matches when every condition is TRUE.  A NULL
//     operand makes a db.cmp NULL (Restrictions.cpp's nullable lowering), which the selection does not take.  Floats: the ordered
//     predicates of translateFPredicate (LowerToStd.cpp:876-894), so a NaN operand is never TRUE, not even for <> (ONE), and -0.0 =
//     +0.0 (IEEE).  A condition on one side is part of the ON predicate evaluated per pair, so under an outer, anti, mark or count join
//     a left row failing it is unmatched, not dropped.
//   Output rows: translateNLJ's NestedMapOp walks the right rows for each left row, so pairs come in left row order, then right row
//     order; the left outer join's "no match" row follows its left row's (absent) matches; translateNLJWithMarker's unmatched right rows
//     come from a scan of the marked buffer after the loop, so they are appended in right row order.  Mark joins produce the marker
//     as a boolean without NULL (as LDB_OP_EXISTS does).
//
// Device work:
//   1. nljWordsKernel, per side: each column-to-column operand as a contiguous order-preserving word array, whatever the batches —
//      int64 for integers, dates, char(1), decimals in 8-byte cells and floats (-0.0 -> +0.0, then the sign-flip map of the double's
//      bits), a (lo, hi) pair when a 16-byte decimal cell is involved — and one "can match" byte per row: no NULL operand, no NaN, and
//      every condition of this side against its constant TRUE.
//   2. nljLoopKernel<NC, Wide, Write>, a CTA per (left tile of kNljLeftTile rows, right chunk): each thread keeps kNljRows left rows'
//      words in registers, the right chunk streams through shared memory in tiles of kNljRightTile rows read by every thread at one
//      address (a broadcast), so one shared word serves kNljRows compares.  An op is a 3-bit mask {lt, eq, gt} per condition, no switch
//      per pair.  Count pass: per (left row, chunk) its matches; semi, anti and mark CTAs leave once every row of theirs matched; right
//      and full outer joins set a byte per matched right row, OR'ed over the CTA per tile, then stored once.  Write pass: the same loop
//      writes each match's (left id, right id) at its offset.
//   3. nljRowKernel: per left row its total (COUNT's value, MARK's flag, SEMI / ANTI's keep flag); a left row without a match under a
//      left / full outer join counts 1.  Then the tile scan (tilescan.cuh) of the (left row, chunk) counts gives every pair its offset,
//      a scan of the unmarked right rows their places after the pairs, the host reads the totals and allocates the result, the write
//      pass and nljFillKernel (the NULL-extended rows) write the id pairs, and permuteRows (peer.cu) gathers each side's cells, an id
//      of 0xffffffff giving NULL cells.  COUNT, MARK, SEMI and ANTI need no pairs: their rows are left rows.
//   Step 2's passes give way to the sorted ranges (nljoin_sorted.cu) when an equality or range condition can key a sort and the
//   sides hold at least kNljSortMinPairs pairs: they produce the same per-left-row counts and right markers (as one chunk), and step 3
//   runs on them unchanged.
#include "nljoin.cuh"
#include "progcol.cuh"
#include "tilescan.cuh"

#include <algorithm>
#include <cmath>

namespace ldb {

constexpr int kNljThreads = 256, kNljRows = 4; // a thread's left rows
constexpr int64_t kNljLeftTile = (int64_t) kNljThreads * kNljRows;
constexpr int kNljRightTile = 512;                          // right rows per shared-memory tile
constexpr int64_t kNljMinChunk = 2 * kNljRightTile;          // right rows of a chunk at least

// ---------------------------------------------------------------- 1. words
struct NljSideBatch {
   ProgCol pair[kNljMaxPairs];     // this side's operand of each column-to-column condition
   ProgCol single[kNljMaxConds];   // the column of each condition of this side against a constant
   int64_t firstRow;
};
struct NljSideParams {
   const NljSideBatch* dir; // device, sorted by firstRow, non-empty batches only
   int32_t nBatches, nPair, nSingle, pad;
   int32_t pairFloat[kNljMaxPairs];
   int32_t singleOp[kNljMaxConds];    // read as  column OP constant
   int32_t singleFloat[kNljMaxConds];
   s128 singleValue[kNljMaxConds];
   double singleF[kNljMaxConds];
   int64_t n;
   int64_t* lo; // [nPair][n]
   int64_t* hi; // [nPair][n], or null: every operand fits 64 bits
   uint8_t* ok; // [n]
};
__device__ __forceinline__ const NljSideBatch& nljBatchOf(const NljSideParams& p, int64_t row) {
   int lo = 0, hi = p.nBatches - 1;
   while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (p.dir[mid].firstRow <= row) lo = mid;
      else hi = mid - 1;
   }
   return p.dir[lo];
}
template <class T>
__device__ __forceinline__ bool nljCmp(int op, T a, T b) {
   switch (op) {
      case LDB_EQ: return a == b;
      case LDB_NEQ: return a != b;
      case LDB_LT: return a < b;
      case LDB_LTE: return a <= b;
      case LDB_GT: return a > b;
      default: return a >= b;
   }
}
// the order-preserving int64 of a double that is not NaN: -0.0 as +0.0, then negative values' magnitude bits flipped
__device__ __forceinline__ int64_t nljF64Word(double d) {
   if (d == 0.0) d = 0.0;
   const long long x = __double_as_longlong(d);
   return x ^ ((x >> 63) & 0x7fffffffffffffffll);
}
__global__ void __launch_bounds__(256) nljWordsKernel(const __grid_constant__ NljSideParams p) {
   for (int64_t i = (int64_t) blockIdx.x * 256 + threadIdx.x; i < p.n; i += (int64_t) gridDim.x * 256) {
      const NljSideBatch& b = nljBatchOf(p, i);
      const int64_t r = i - b.firstRow;
      bool ok = true;
      for (int c = 0; c < p.nSingle; c++) {
         const Val v = loadCol(b.single[c], r);
         if (v.null) ok = false;
         else if (p.singleFloat[c]) ok = ok && !isnan(asF64(v)) && !isnan(p.singleF[c]) && nljCmp(p.singleOp[c], asF64(v), p.singleF[c]);
         else ok = ok && nljCmp(p.singleOp[c], v.v, p.singleValue[c]);
      }
      for (int c = 0; c < p.nPair; c++) {
         const Val v = loadCol(b.pair[c], r);
         int64_t lo, hi;
         if (p.pairFloat[c]) {
            const double d = asF64(v);
            if (isnan(d)) ok = false;
            lo = nljF64Word(d);
            hi = lo >> 63;
         } else {
            lo = (int64_t) v.v;
            hi = (int64_t) (v.v >> 64);
         }
         if (v.null) ok = false;
         p.lo[(size_t) c * p.n + i] = lo;
         if (p.hi) p.hi[(size_t) c * p.n + i] = hi;
      }
      p.ok[i] = ok ? 1 : 0;
   }
}

// ---------------------------------------------------------------- 2. the loop
struct NljLoopParams {
   const int64_t *lLo, *lHi, *rLo, *rHi; // the sides' words ([cond][row]; hi only when Wide)
   const uint8_t *lOk, *rOk;
   int64_t nL, nR, chunkRows;
   int32_t nChunks, exists;             // exists: semi / anti / mark, a CTA may stop once all its rows matched
   uint32_t mask[kNljMaxPairs];         // per condition: bit 0 TRUE when left < right, bit 1 when equal, bit 2 when greater
   uint32_t* counts;                    // [nL][nChunks]: the count pass's matches per (left row, chunk)
   uint8_t* rightMark;                  // per right row: 1 once some left row matched it (right / full outer), or null
   const unsigned long long* offs;      // write pass: [nL][nChunks] where each (left row, chunk)'s pairs start
   uint32_t *outL, *outR;               // write pass: the pairs' ids
};
template <bool Wide>
struct NljWord {
   int64_t lo, hi;
};
template <>
struct NljWord<false> {
   int64_t lo;
};
template <bool Wide>
__device__ __forceinline__ bool nljTest(const NljWord<Wide>& a, const NljWord<Wide>& b, uint32_t mask) {
   bool lt, eq;
   if constexpr (Wide) {
      lt = a.hi < b.hi || (a.hi == b.hi && (uint64_t) a.lo < (uint64_t) b.lo);
      eq = a.hi == b.hi && a.lo == b.lo;
   } else {
      lt = a.lo < b.lo;
      eq = a.lo == b.lo;
   }
   return (mask >> (lt ? 0 : eq ? 1 : 2)) & 1u;
}
template <int NC, bool Wide, bool Write>
__global__ void __launch_bounds__(kNljThreads, 2) nljLoopKernel(const __grid_constant__ NljLoopParams p) {
   __shared__ NljWord<Wide> sw[NC > 0 ? NC : 1][kNljRightTile];
   __shared__ uint8_t sOk[kNljRightTile], sMark[kNljRightTile];
   const int lane = threadIdx.x & 31;
   const int chunk = blockIdx.y;
   const int64_t rBegin = (int64_t) chunk * p.chunkRows, rEnd = min(rBegin + p.chunkRows, p.nR);
   NljWord<Wide> a[kNljRows][NC > 0 ? NC : 1];
   bool active[kNljRows];
   uint32_t cnt[kNljRows];
   unsigned long long pos[kNljRows];
   bool any = false;
#pragma unroll
   for (int k = 0; k < kNljRows; k++) {
      const int64_t l = (int64_t) blockIdx.x * kNljLeftTile + (int64_t) k * kNljThreads + threadIdx.x;
      active[k] = l < p.nL && p.lOk[l];
      any |= active[k];
      cnt[k] = 0;
      pos[k] = 0;
#pragma unroll
      for (int c = 0; c < NC; c++) {
         a[k][c].lo = active[k] ? p.lLo[(size_t) c * p.nL + l] : 0;
         if constexpr (Wide) a[k][c].hi = active[k] ? p.lHi[(size_t) c * p.nL + l] : 0;
      }
      if constexpr (Write)
         if (active[k]) pos[k] = p.offs[(size_t) l * p.nChunks + chunk];
   }
   const bool markRight = p.rightMark != nullptr;
   // a CTA none of whose left rows can match counts nothing (and marks nothing)
   if (__syncthreads_or(any)) {
      for (int64_t base = rBegin; base < rEnd; base += kNljRightTile) {
         const int n = (int) min((int64_t) kNljRightTile, rEnd - base);
         __syncthreads(); // the previous tile is read
         for (int j = threadIdx.x; j < n; j += kNljThreads) {
            sOk[j] = p.rOk[base + j];
            sMark[j] = 0;
#pragma unroll
            for (int c = 0; c < NC; c++) {
               sw[c][j].lo = p.rLo[(size_t) c * p.nR + base + j];
               if constexpr (Wide) sw[c][j].hi = p.rHi[(size_t) c * p.nR + base + j];
            }
         }
         __syncthreads();
         for (int j = 0; j < n; j++) {
            if (!sOk[j]) continue; // the same j in every thread: no divergence
            NljWord<Wide> w[NC > 0 ? NC : 1];
#pragma unroll
            for (int c = 0; c < NC; c++) w[c] = sw[c][j];
            bool hit = false;
#pragma unroll
            for (int k = 0; k < kNljRows; k++) {
               bool m = true;
#pragma unroll
               for (int c = 0; c < NC; c++) m = m && nljTest<Wide>(a[k][c], w[c], p.mask[c]);
               if constexpr (Write) {
                  if (m && active[k]) {
                     const int64_t l = (int64_t) blockIdx.x * kNljLeftTile + (int64_t) k * kNljThreads + threadIdx.x;
                     p.outL[pos[k]] = (uint32_t) l;
                     p.outR[pos[k]] = (uint32_t) (base + j);
                     pos[k]++;
                  }
               } else {
                  cnt[k] += m ? 1u : 0u; // masked by `active` at the end: no AND per pair
                  hit |= m && active[k];
               }
            }
            if constexpr (!Write)
               if (markRight && __any_sync(0xffffffffu, hit) && lane == 0) sMark[j] = 1;
         }
         if constexpr (!Write) {
            if (markRight) {
               __syncthreads();
               for (int j = threadIdx.x; j < n; j += kNljThreads)
                  if (sMark[j]) p.rightMark[base + j] = 1;
            }
            if (p.exists) {
               bool done = true;
#pragma unroll
               for (int k = 0; k < kNljRows; k++) done = done && (!active[k] || cnt[k] > 0);
               if (__syncthreads_and(done)) break;
            }
         }
      }
   }
   if constexpr (!Write) {
#pragma unroll
      for (int k = 0; k < kNljRows; k++) {
         const int64_t l = (int64_t) blockIdx.x * kNljLeftTile + (int64_t) k * kNljThreads + threadIdx.x;
         if (l < p.nL) p.counts[(size_t) l * p.nChunks + chunk] = active[k] ? cnt[k] : 0u;
      }
   }
}

// ---------------------------------------------------------------- 3. rows, offsets and the NULL-extended rows
// per left row: its total over the chunks; value = COUNT's int64 or MARK's int32, keep = SEMI / ANTI's flag; under a left / full outer
// join a row without a match counts 1 (its NULL-extended row), in its first chunk's count, and is flagged in `unmatched`
__global__ void __launch_bounds__(256) nljRowKernel(uint32_t* counts, int64_t nL, int32_t nChunks, int kind, void* value, uint32_t* keep, uint8_t* unmatched) {
   for (int64_t l = (int64_t) blockIdx.x * 256 + threadIdx.x; l < nL; l += (int64_t) gridDim.x * 256) {
      unsigned long long t = 0;
      for (int c = 0; c < nChunks; c++) t += counts[(size_t) l * nChunks + c];
      switch (kind) {
         case LDB_NLJ_COUNT: ((long long*) value)[l] = (long long) t; break;
         case LDB_NLJ_MARK: ((int32_t*) value)[l] = t > 0; break;
         case LDB_NLJ_SEMI: keep[l] = t > 0; break;
         case LDB_NLJ_ANTI: keep[l] = t == 0; break;
         case LDB_NLJ_LEFT_OUTER:
         case LDB_NLJ_FULL_OUTER:
            unmatched[l] = t == 0;
            if (t == 0) counts[(size_t) l * nChunks] = 1;
            break;
         default: break;
      }
   }
}
// the scan of the (left row, chunk) counts: offs[k] = where position k's pairs start; total[0] = every pair
struct NljOffsetOp {
   using T = unsigned long long;
   const uint32_t* cnt;
   unsigned long long* offs;
   unsigned long long* total;
   int64_t n;
   __device__ T identity() const { return 0; }
   __device__ T combine(T a, T b) const { return a + b; }
   __device__ T load(int64_t k) const { return cnt[k]; }
   __device__ void store(int64_t k, T v) const {
      offs[k] = v - cnt[k];
      if (k == n - 1) *total = v;
   }
};
// the scan of 0 / 1 flags: at[k] = the flagged positions before k; total[0] = every flagged position; ids (non-null) gets each flagged k
struct NljCompactOp {
   using T = uint32_t;
   const uint8_t* mark;     // flag = mark[k] == 0 (unmatched right rows), or
   const uint32_t* keep;    // flag = keep[k] (semi / anti)
   uint32_t* at;
   uint32_t* ids;
   unsigned long long* total;
   int64_t n;
   __device__ T identity() const { return 0; }
   __device__ T combine(T a, T b) const { return a + b; }
   __device__ T load(int64_t k) const { return keep ? keep[k] : mark[k] == 0; }
   __device__ void store(int64_t k, T v) const {
      const uint32_t f = load(k);
      if (at) at[k] = v - f;
      if (ids && f) ids[v - 1] = (uint32_t) k;
      if (k == n - 1) *total = v;
   }
};
// the NULL-extended rows: a left row without a match at its offset, an unmatched right row at pairs + its place among them
__global__ void __launch_bounds__(256) nljFillKernel(const uint8_t* unmatched, const unsigned long long* offs, int64_t nL, int32_t nChunks,
                                                      const uint8_t* rightMark, const uint32_t* rightAt, const unsigned long long* pairs, int64_t nR,
                                                      uint32_t* outL, uint32_t* outR) {
   const int64_t n = max(nL, nR);
   for (int64_t i = (int64_t) blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t) gridDim.x * 256) {
      if (unmatched && i < nL && unmatched[i]) {
         const unsigned long long at = offs[(size_t) i * nChunks];
         outL[at] = (uint32_t) i;
         outR[at] = kNljNone;
      }
      if (rightMark && i < nR && !rightMark[i]) {
         const unsigned long long at = *pairs + rightAt[i];
         outL[at] = kNljNone;
         outR[at] = (uint32_t) i;
      }
   }
}

// ---------------------------------------------------------------- host side
// the comparable families: 1 integers, 2 date32, 3 char(1), 4 decimal, 5 float; 0 none (utf8 and anything else)
static int nljFamily(int type) {
   switch (type) {
      case LDB_INT8:
      case LDB_INT16:
      case LDB_INT32:
      case LDB_INT64: return 1;
      case LDB_DATE32: return 2;
      case LDB_FSB4: return 3;
      case LDB_DECIMAL128: return 4;
      case LDB_FLOAT32:
      case LDB_FLOAT64: return 5;
      default: return 0;
   }
}
static int nljSwap(int op) {
   switch (op) {
      case LDB_LT: return LDB_GT;
      case LDB_LTE: return LDB_GTE;
      case LDB_GT: return LDB_LT;
      case LDB_GTE: return LDB_LTE;
      default: return op;
   }
}
static uint32_t nljMask(int op) {
   switch (op) {
      case LDB_EQ: return 2;
      case LDB_NEQ: return 5;
      case LDB_LT: return 1;
      case LDB_LTE: return 3;
      case LDB_GT: return 4;
      default: return 6; // GTE
   }
}
static std::vector<int> nljCarried(const LdbTable* t, int32_t n, const char* const* names, const char* side) {
   std::vector<int> cols;
   if (!names) {
      for (int ci = 0; ci < (int) t->columns.size(); ci++) cols.push_back(ci);
   } else {
      if (n < 0 || n > kNljMaxCols) fail(LDB_ERR_INVALID, std::string("a nested-loop join carries 0..16 ") + side + " columns (" + std::to_string(n) + " given)");
      for (int j = 0; j < n; j++) {
         const int ci = t->colIndex(names[j]);
         if (ci < 0) fail(LDB_ERR_INVALID, std::string("unknown ") + side + " column " + (names[j] ? names[j] : "(null)"));
         cols.push_back(ci);
      }
   }
   if (cols.size() > (size_t) kNljMaxCols)
      fail(LDB_ERR_INVALID, std::string("a nested-loop join carries 0..16 ") + side + " columns (table " + t->name + " has " + std::to_string(cols.size()) + "; name them)");
   return cols;
}
static bool nljAnyWideCell(const LdbTable* t, int ci) {
   for (const LdbBatch& b : t->batches)
      if (b.nRows > 0 && b.elemBytes[ci] == 16) return true;
   return false;
}

struct NljSide {
   std::vector<int> pairCols, singleCols, singleOps;
   std::vector<s128> singleValues;
   std::vector<double> singleF;
};
// one side's words and "can match" bytes, in `tmp`
static void nljWords(LdbContext* ctx, Scratch& tmp, const LdbTable* t, const NljSide& s, const std::vector<int>& pairFloat, bool wide,
                     int64_t** lo, int64_t** hi, uint8_t** ok) {
   const int64_t n = t->numRows;
   const size_t np = s.pairCols.size();
   *lo = tmp.alloc<int64_t>(std::max<size_t>(np * (size_t) n * 8, 16));
   *hi = wide ? tmp.alloc<int64_t>(std::max<size_t>(np * (size_t) n * 8, 16)) : nullptr;
   *ok = tmp.alloc<uint8_t>(std::max<size_t>((size_t) n, 16));
   if (n == 0) return;
   std::vector<NljSideBatch> dir;
   int64_t first = 0;
   for (const LdbBatch& b : t->batches) {
      if (b.nRows > 0) {
         NljSideBatch sb{};
         for (size_t c = 0; c < np; c++) {
            bindColumn(sb.pair[c], b, s.pairCols[c]);
            sb.pair[c].type = t->columns[s.pairCols[c]].type;
         }
         for (size_t c = 0; c < s.singleCols.size(); c++) {
            bindColumn(sb.single[c], b, s.singleCols[c]);
            sb.single[c].type = t->columns[s.singleCols[c]].type;
         }
         sb.firstRow = first;
         dir.push_back(sb);
      }
      first += b.nRows;
   }
   NljSideParams p{};
   NljSideBatch* dd = tmp.alloc<NljSideBatch>(dir.size() * sizeof(NljSideBatch));
   LDB_CUDA(cudaMemcpyAsync(dd, dir.data(), dir.size() * sizeof(NljSideBatch), cudaMemcpyHostToDevice, ctx->compute));
   p.dir = dd;
   p.nBatches = (int32_t) dir.size();
   p.nPair = (int32_t) np;
   p.nSingle = (int32_t) s.singleCols.size();
   for (size_t c = 0; c < np; c++) p.pairFloat[c] = pairFloat[c];
   for (size_t c = 0; c < s.singleCols.size(); c++) {
      p.singleOp[c] = s.singleOps[c];
      p.singleFloat[c] = nljFamily(t->columns[s.singleCols[c]].type) == 5;
      p.singleValue[c] = s.singleValues[c];
      p.singleF[c] = s.singleF[c];
   }
   p.n = n;
   p.lo = *lo;
   p.hi = *hi;
   p.ok = *ok;
   ctx->launch("nljoin_words", [&] { nljWordsKernel<<<nljGrid(ctx, (uint64_t) n), 256, 0, ctx->compute>>>(p); });
   // the directory goes back to the pool with `tmp`, after the call has synchronised
}

template <int NC, bool Wide, bool Write>
static void nljLaunch(LdbContext* ctx, dim3 grid, const NljLoopParams& p) {
   nljLoopKernel<NC, Wide, Write><<<grid, kNljThreads, 0, ctx->compute>>>(p);
}
template <bool Wide, bool Write>
static void nljLaunchNC(LdbContext* ctx, int nc, dim3 grid, const NljLoopParams& p) {
   switch (nc) {
      case 0: nljLaunch<0, false, Write>(ctx, grid, p); break;
      case 1: nljLaunch<1, Wide, Write>(ctx, grid, p); break;
      case 2: nljLaunch<2, Wide, Write>(ctx, grid, p); break;
      case 3: nljLaunch<3, Wide, Write>(ctx, grid, p); break;
      default: nljLaunch<4, Wide, Write>(ctx, grid, p); break;
   }
}
static void nljLoop(LdbContext* ctx, int nc, bool wide, bool write, dim3 grid, const NljLoopParams& p) {
   if (wide) write ? nljLaunchNC<true, true>(ctx, nc, grid, p) : nljLaunchNC<true, false>(ctx, nc, grid, p);
   else write ? nljLaunchNC<false, true>(ctx, nc, grid, p) : nljLaunchNC<false, false>(ctx, nc, grid, p);
}

static void tableNlJoin(LdbTable* left, LdbTable* right, int32_t kind, int32_t n_conds, const LdbJoinCond* conds, int32_t n_left_columns,
                        const char* const* left_columns, int32_t n_right_columns, const char* const* right_columns, const char* const* right_names,
                        const char* value_name, const char* name, LdbTable** out) {
   // everything is checked before the first launch
   if (!left || !right || !out || (n_conds > 0 && !conds)) fail(LDB_ERR_INVALID, "null argument");
   if (kind < LDB_NLJ_INNER || kind > LDB_NLJ_COUNT) fail(LDB_ERR_INVALID, "unknown nested-loop join kind " + std::to_string(kind));
   if (right->ctx != left->ctx) fail(LDB_ERR_INVALID, "left and right tables belong to different contexts");
   if (n_conds < 0 || n_conds > kNljMaxConds) fail(LDB_ERR_INVALID, "a nested-loop join takes 0..8 conditions (" + std::to_string(n_conds) + " given)");
   const bool leftOnly = kind >= LDB_NLJ_SEMI;
   const bool valued = kind == LDB_NLJ_MARK || kind == LDB_NLJ_COUNT;
   if (leftOnly && (right_columns || right_names || n_right_columns))
      fail(LDB_ERR_INVALID, "semi, anti, mark and count joins carry no right columns");
   if (valued && (!value_name || !*value_name)) fail(LDB_ERR_INVALID, "a mark or count join needs value_name");
   if (!valued && value_name) fail(LDB_ERR_INVALID, "value_name is for mark and count joins only");

   // the conditions
   NljSide ls, rs;
   std::vector<uint32_t> masks;
   std::vector<int> pairFloat;
   std::vector<std::string> pairNames;
   bool wide = false;
   for (int c = 0; c < n_conds; c++) {
      const LdbJoinCond& jc = conds[c];
      if (jc.op < LDB_EQ || jc.op > LDB_GTE) fail(LDB_ERR_INVALID, "condition " + std::to_string(c) + ": unknown op " + std::to_string(jc.op));
      if (!jc.left && !jc.right) fail(LDB_ERR_INVALID, "condition " + std::to_string(c) + " names no column");
      const int li = jc.left ? left->colIndex(jc.left) : -1, ri = jc.right ? right->colIndex(jc.right) : -1;
      if (jc.left && li < 0) fail(LDB_ERR_INVALID, std::string("condition ") + std::to_string(c) + ": unknown left column " + jc.left);
      if (jc.right && ri < 0) fail(LDB_ERR_INVALID, std::string("condition ") + std::to_string(c) + ": unknown right column " + jc.right);
      const LdbColumn* a = li >= 0 ? &left->columns[li] : nullptr;
      const LdbColumn* b = ri >= 0 ? &right->columns[ri] : nullptr;
      if (a && b) {
         const int fa = nljFamily(a->type), fb = nljFamily(b->type);
         if (!fa || fa != fb || (fa == 4 && a->scale != b->scale))
            fail(LDB_ERR_UNSUPPORTED, "a nested-loop join cannot compare left column " + a->name + " with right column " + b->name +
                                         (fa == 4 && fa == fb ? " (decimals of different scales: cast one)" : " (their types do not compare)"));
         if ((int) masks.size() == kNljMaxPairs) fail(LDB_ERR_INVALID, "a nested-loop join takes at most 4 column-to-column conditions");
         masks.push_back(nljMask(jc.op));
         pairFloat.push_back(fa == 5);
         ls.pairCols.push_back(li);
         rs.pairCols.push_back(ri);
         if (fa == 4 && (nljAnyWideCell(left, li) || nljAnyWideCell(right, ri))) wide = true;
      } else {
         const LdbColumn* col = a ? a : b;
         if (!nljFamily(col->type)) fail(LDB_ERR_UNSUPPORTED, "a nested-loop join cannot compare column " + col->name + " (utf8 and its type do not compare) with a constant");
         // the constant is `value` for every family but floats, whose constant is `fvalue`; a caller that sets both must set one
         // number (a non-integral fvalue against an integer column would otherwise be read as `value`, silently)
         const s128 v = (s128) (((unsigned __int128) (uint64_t) jc.value.hi << 64) | jc.value.lo);
         const bool isFloat = nljFamily(col->type) == 5;
         if (isFloat ? (v != 0 && (double) v != jc.fvalue) : (jc.fvalue != 0.0 && jc.fvalue != (double) v))
            fail(LDB_ERR_INVALID, "condition " + std::to_string(c) + ": the constant's value and fvalue differ; column " + col->name + " reads " +
                                     (isFloat ? "fvalue" : "value") + " (set the other to 0 or to the same number)");
         NljSide& s = a ? ls : rs;
         s.singleCols.push_back(a ? li : ri);
         s.singleOps.push_back(a ? jc.op : nljSwap(jc.op)); // value OP right.col  ==  right.col swap(OP) value
         s.singleValues.push_back(v);
         s.singleF.push_back(jc.fvalue);
      }
   }

   // the output columns
   const std::vector<int> lc = nljCarried(left, n_left_columns, left_columns, "left");
   const std::vector<int> rc = leftOnly ? std::vector<int>{} : nljCarried(right, n_right_columns, right_columns, "right");
   std::vector<LdbColumn> outCols;
   for (int ci : lc) outCols.push_back(left->columns[ci]);
   for (size_t j = 0; j < rc.size(); j++) {
      LdbColumn c = right->columns[rc[j]];
      if (right_names) {
         if (!right_names[j]) fail(LDB_ERR_INVALID, "right_names[" + std::to_string(j) + "] is null");
         c.name = right_names[j];
      }
      outCols.push_back(c);
   }
   if (valued) outCols.push_back(LdbColumn{value_name, kind == LDB_NLJ_MARK ? LDB_INT32 : LDB_INT64, 0, 0});
   for (size_t j = 0; j < outCols.size(); j++)
      for (size_t k = 0; k < j; k++)
         if (outCols[j].name == outCols[k].name)
            fail(LDB_ERR_INVALID, "the nested-loop join's result would have two columns named " + outCols[j].name + " (output columns " + std::to_string(k) +
                                     " and " + std::to_string(j) + "; name the right columns with right_names)");
   std::vector<int32_t> lw, rw;
   size_t rowBytes = !leftOnly ? 8 : 0;
   for (int ci : lc) lw.push_back(shipCellBytes(left->columns[ci].type)), rowBytes += lw.back() + 1;
   for (int ci : rc) rw.push_back(shipCellBytes(right->columns[ci].type)), rowBytes += rw.back() + 1;
   const int64_t nL = left->numRows, nR = right->numRows;
   if (nL >= (int64_t) kNljNone || nR >= (int64_t) kNljNone) fail(LDB_ERR_UNSUPPORTED, "a nested-loop join takes sides of fewer than 2^32 - 1 rows");
   LdbContext* ctx = left->ctx;
   if (ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "a nested-loop join reads its output size on the host and cannot be captured");

   LDB_CUDA(cudaSetDevice(ctx->device));
   for (auto& b : left->batches) ldb_gpu_wait_batch_internal(ctx, &b);
   if (right != left)
      for (auto& b : right->batches) ldb_gpu_wait_batch_internal(ctx, &b);

   Scratch bufs(ctx), tmp(ctx);
   const int nc = (int) masks.size();
   const bool pairs = !leftOnly;
   const bool markRight = kind == LDB_NLJ_RIGHT_OUTER || kind == LDB_NLJ_FULL_OUTER;
   const bool keepLeft = kind == LDB_NLJ_LEFT_OUTER || kind == LDB_NLJ_FULL_OUTER;
   unsigned long long* ctr = tmp.alloc<unsigned long long>(32); // [0] pairs, [1] unmatched right rows, [2] kept left rows
   LDB_CUDA(cudaMemsetAsync(ctr, 0, 32, ctx->compute));
   void* value = nullptr;
   uint8_t* valueValid = nullptr;
   if (valued) {
      value = bufs.alloc<uint8_t>(std::max<size_t>((size_t) nL * (kind == LDB_NLJ_MARK ? 4 : 8), 16));
      valueValid = bufs.alloc<uint8_t>(std::max<size_t>((size_t) nL, 16));
      LDB_CUDA(cudaMemsetAsync(value, 0, std::max<size_t>((size_t) nL * (kind == LDB_NLJ_MARK ? 4 : 8), 16), ctx->compute));
      LDB_CUDA(cudaMemsetAsync(valueValid, 1, std::max<size_t>((size_t) nL, 16), ctx->compute));
   }

   // the count pass
   const int64_t leftTiles = (nL + kNljLeftTile - 1) / kNljLeftTile;
   int64_t nChunks = std::max<int64_t>(1, ((int64_t) ctx->smCount * 8 + leftTiles - 1) / std::max<int64_t>(leftTiles, 1));
   nChunks = std::min<int64_t>({nChunks, std::max<int64_t>(1, (nR + kNljMinChunk - 1) / kNljMinChunk), 65535});
   int64_t chunkRows = (nR + nChunks - 1) / nChunks;
   chunkRows = std::max<int64_t>(kNljRightTile, (chunkRows + kNljRightTile - 1) / kNljRightTile * kNljRightTile);
   nChunks = std::max<int64_t>(1, (nR + chunkRows - 1) / chunkRows);
   NljLoopParams p{};
   p.nL = nL;
   p.nR = nR;
   p.chunkRows = chunkRows;
   p.nChunks = (int32_t) nChunks;
   p.exists = kind == LDB_NLJ_SEMI || kind == LDB_NLJ_ANTI || kind == LDB_NLJ_MARK;
   for (int c = 0; c < nc; c++) p.mask[c] = masks[c];
   int64_t nPos = nL * nChunks;
   uint32_t* keep = nullptr;
   uint8_t* unmatched = nullptr;
   unsigned long long* offs = nullptr;
   uint32_t* rightAt = nullptr;
   uint32_t* ids = nullptr; // semi / anti: the kept left rows
   NljSortedRun sr(ctx);
   bool sorted = false;
   if (nL > 0 && nR > 0) {
      int64_t *lLo, *lHi, *rLo, *rHi;
      uint8_t *lOk, *rOk;
      nljWords(ctx, tmp, left, ls, pairFloat, wide, &lLo, &lHi, &lOk);
      nljWords(ctx, tmp, right, rs, pairFloat, wide, &rLo, &rHi, &rOk);
      p.lLo = lLo;
      p.lHi = lHi;
      p.rLo = rLo;
      p.rHi = rHi;
      p.lOk = lOk;
      p.rOk = rOk;
      // the sorted ranges when some condition keys a sort, the pairs are many and its scratch fits where the loop's does
      if (nljSortedPlan(nc, masks.data(), ls.pairCols.data(), rs.pairCols.data(), nL, nR, &sr.plan) && (double) nL * (double) nR >= kNljSortMinPairs) {
         const int64_t nS = sr.plan.sLeft ? nL : nR, nP = sr.plan.sLeft ? nR : nL;
         const double sortBytes = (double) nS * (24 + 16 * (wide ? 2 : 1) * (sr.plan.nEq + 1)) + (double) nP * 20 + (double) nL * 4;
         const double loopBytes = (double) nPos * 12;
         size_t freeB = 0, totalB = 0;
         LDB_CUDA(cudaMemGetInfo(&freeB, &totalB));
         if (sortBytes <= (double) freeB || loopBytes > (double) freeB) {
            sr.left = NljWordsRef{lLo, lHi, lOk, nL};
            sr.right = NljWordsRef{rLo, rHi, rOk, nR};
            sr.wide = wide;
            sr.kind = kind;
            sr.resultRowBytes = (double) rowBytes;
            sorted = nljSortedCount(ctx, tmp, sr);
            if (!sorted) { // the loop's scratch comes next: the sorted path's goes back to the device first
               sr.keep.toDevice();
               sr.sortOnly.toDevice();
            }
         }
      }
      if (sorted) {
         nChunks = 1;
         nPos = nL;
         p.nChunks = 1;
         p.counts = sr.counts;
         p.rightMark = sr.rightMark;
      } else {
         p.counts = tmp.alloc<uint32_t>((size_t) nPos * 4);
         if (markRight) {
            p.rightMark = tmp.alloc<uint8_t>((size_t) nR);
            LDB_CUDA(cudaMemsetAsync(p.rightMark, 0, (size_t) nR, ctx->compute));
         }
         const dim3 grid((unsigned) leftTiles, (unsigned) nChunks);
         ctx->launch("nljoin_count", [&] { nljLoop(ctx, nc, wide, false, grid, p); });
      }
   } else if (nL > 0) {
      p.counts = tmp.alloc<uint32_t>((size_t) nPos * 4); // no right rows: no matches
      LDB_CUDA(cudaMemsetAsync(p.counts, 0, (size_t) nPos * 4, ctx->compute));
   }
   if (nR > 0 && markRight && !p.rightMark) { // no left rows: every right row is unmatched
      p.rightMark = tmp.alloc<uint8_t>((size_t) nR);
      LDB_CUDA(cudaMemsetAsync(p.rightMark, 0, (size_t) nR, ctx->compute));
   }
   if (nL > 0) {
      if (kind == LDB_NLJ_SEMI || kind == LDB_NLJ_ANTI) {
         keep = tmp.alloc<uint32_t>((size_t) nL * 4);
         ids = tmp.alloc<uint32_t>((size_t) nL * 4);
      }
      if (keepLeft) unmatched = tmp.alloc<uint8_t>((size_t) nL);
      ctx->launch("nljoin_rows", [&] { nljRowKernel<<<nljGrid(ctx, (uint64_t) nL), 256, 0, ctx->compute>>>(p.counts, nL, p.nChunks, kind, value, keep, unmatched); });
      if (pairs) {
         offs = tmp.alloc<unsigned long long>((size_t) nPos * 8);
         tileScan(ctx, tmp, NljOffsetOp{p.counts, offs, ctr, nPos}, nPos, "nljoin_scan");
      }
      if (keep) tileScan(ctx, tmp, NljCompactOp{nullptr, keep, nullptr, ids, ctr + 2, nL}, nL, "nljoin_scan");
   }
   if (markRight && nR > 0) {
      rightAt = tmp.alloc<uint32_t>((size_t) nR * 4);
      tileScan(ctx, tmp, NljCompactOp{p.rightMark, nullptr, rightAt, nullptr, ctr + 1, nR}, nR, "nljoin_scan");
   }
   unsigned long long* host = (unsigned long long*) ctx->scratch();
   LDB_CUDA(cudaMemcpyAsync(host, ctr, 24, cudaMemcpyDeviceToHost, ctx->compute));
   ctx->syncStream(ctx->compute);
   const unsigned long long nPairs = host[0], nRightOnly = host[1], nKept = host[2];

   // the result's rows
   const int64_t total = pairs ? (int64_t) (nPairs + nRightOnly) : kind == LDB_NLJ_SEMI || kind == LDB_NLJ_ANTI ? (int64_t) nKept : nL;
   size_t freeB = 0, totalB = 0;
   LDB_CUDA(cudaMemGetInfo(&freeB, &totalB));
   if ((double) total * (double) rowBytes > (double) freeB && !sr.sortOnly.empty()) { // the sort's buffers are done with: give them back
      sr.sortOnly.toDevice();
      LDB_CUDA(cudaMemGetInfo(&freeB, &totalB));
   }
   if ((double) total * (double) rowBytes > (double) freeB)
      fail(LDB_ERR_CAPACITY, "the nested-loop join's result has " + std::to_string(total) + " rows, which need " + std::to_string((double) total * rowBytes / 1e9) +
                                " GB of device memory; " + std::to_string(freeB / 1e9) + " GB are free");
   uint32_t *outL = nullptr, *outR = nullptr;
   if (pairs && total > 0) {
      outL = tmp.alloc<uint32_t>((size_t) total * 4);
      outR = tmp.alloc<uint32_t>((size_t) total * 4);
      if (sorted) {
         nljSortedWrite(ctx, tmp, sr, offs, outL, outR);
      } else if (nPairs > 0 && nR > 0) {
         p.offs = offs;
         p.outL = outL;
         p.outR = outR;
         const dim3 grid((unsigned) leftTiles, (unsigned) nChunks);
         NljLoopParams w = p;
         w.rightMark = nullptr;
         w.exists = 0;
         ctx->launch("nljoin_write", [&] { nljLoop(ctx, nc, wide, true, grid, w); });
      }
      if (unmatched || (markRight && nR > 0))
         ctx->launch("nljoin_write", [&] {
            nljFillKernel<<<nljGrid(ctx, (uint64_t) std::max(nL, nR)), 256, 0, ctx->compute>>>(unmatched, offs, unmatched ? nL : 0, p.nChunks, markRight ? p.rightMark : nullptr,
                                                                                                rightAt, ctr, markRight ? nR : 0, outL, outR);
         });
      if (sorted) nljSortedOrder(ctx, tmp, sr, (int64_t) nPairs, outL, outR);
   }

   // the cells
   LdbBatch ob;
   ob.nRows = total;
   auto append = [&](LdbBatch&& b) {
      for (size_t j = 0; j < b.data.size(); j++) {
         ob.data.push_back(b.data[j]);
         ob.bytes.push_back(b.bytes[j]);
         ob.elemBytes.push_back(b.elemBytes[j]);
         ob.validBytes.push_back(b.validBytes[j]);
      }
   };
   if (!lc.empty()) append(permuteRows(left, lc, lw.data(), pairs ? outL : ids, total, bufs, "nested-loop join"));
   if (!rc.empty()) append(permuteRows(right, rc, rw.data(), outR, total, bufs, "nested-loop join"));
   if (valued) {
      ob.data.push_back(value);
      ob.bytes.push_back(nullptr);
      ob.elemBytes.push_back(kind == LDB_NLJ_MARK ? 4 : 8);
      ob.validBytes.push_back(valueValid);
   }
   ctx->syncStream(ctx->compute); // the scratch buffers go back to the pool
   *out = addResultTable(ctx, name ? name : "nljoin", std::move(outCols), std::move(ob), bufs);
}

} // namespace ldb

static_assert(sizeof(ldb::NljSideParams) <= 4096, "the nested-loop join's word kernel parameters");
static_assert(sizeof(ldb::NljLoopParams) <= 4096, "the nested-loop join's loop kernel parameters");

extern "C" int ldb_gpu_table_nl_join(LdbTable* left, LdbTable* right, int32_t kind, int32_t n_conds, const LdbJoinCond* conds, int32_t n_left_columns,
                                     const char* const* left_columns, int32_t n_right_columns, const char* const* right_columns,
                                     const char* const* right_names, const char* value_name, const char* name, LdbTable** out, LdbError* err) {
   return ldb::guarded(err, [&] {
      ldb::tableNlJoin(left, right, kind, n_conds, conds, n_left_columns, left_columns, n_right_columns, right_columns, right_names, value_name, name, out);
   });
}
