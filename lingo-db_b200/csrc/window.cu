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
//
// ldb_gpu_table_window_ex adds RANGE frames and the ranking, offset and value functions, which the reference does not have (standard
// SQL as PostgreSQL implements it; the header comment in include/ldb_gpu.h states the rules).  Only a call that uses them runs:
//   peer heads (winHeadsKernel over the order keys, OR-ed with the partition heads) and their start / end scans; DENSE_RANK's add-scan;
//   for RANGE bounds the order key's words (winKeyWordsKernel) and winRangeKernel's per-row [lo, hiEx) by binary search;
//   winFramesKernel<true>, which also handles empty frames, the ranks and NTILE, and writes the value functions' source rows;
//   one permuteRows per value function, then winDefaultKernel for LAG / LEAD defaults.
// Every other call runs winFramesKernel<false>, the ROWS-only instance, and launches what it always did.
#include "context.h"
#include "progcol.cuh"
#include "sortkey.cuh"
#include "tilescan.cuh"

#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>

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
// head[i] = 1 when row i starts a run: the first row, a flag of `base` (null: none) or a key differing from the previous row's.  The
// partition heads (base null, the partition keys) and the peer heads (base = the partition heads, the order keys)
__global__ void __launch_bounds__(kWinThreads) winHeadsKernel(const __grid_constant__ WinKeys k, const uint32_t* ids, int64_t n, const uint8_t* base, uint8_t* head) {
   for (int64_t i = (int64_t) blockIdx.x * kWinThreads + threadIdx.x; i < n; i += (int64_t) gridDim.x * kWinThreads) {
      bool h = i == 0 || (base && base[i]);
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
// DENSE_RANK: the running count of the peer heads (the row's peer group is dense[i] - dense[partition start] + 1)
struct WinCountOp {
   using T = uint32_t;
   const uint8_t* head;
   uint32_t* out;
   __device__ T identity() const { return 0; }
   __device__ T combine(T a, T b) const { return a + b; }
   __device__ T load(int64_t k) const { return head[k]; }
   __device__ void store(int64_t k, T v) const { out[k] = v; }
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

// ---------------------------------------------------------------- RANGE frame bounds
// The single order key in window order as contiguous order-preserving words (sortCell's value: int64 for 4- and 8-byte cells, i128 for
// 16-byte decimals) and its NULL flags, so the bound search reads words, not a gather through the sort's ids per probe.
template <class K>
__global__ void __launch_bounds__(kWinThreads) winKeyWordsKernel(ProgCol key, const uint32_t* ids, int64_t n, K* words, uint8_t* null) {
   for (int64_t i = (int64_t) blockIdx.x * kWinThreads + threadIdx.x; i < n; i += (int64_t) gridDim.x * kWinThreads) {
      const int64_t row = winRow(ids, i);
      const SortCell c = sortCell(key.data, key.elemBytes, row);
      words[i] = sizeof(K) == 16 ? (K) (s128) ((unsigned __int128) c.hi << 64 | c.lo) : (K) (long long) c.lo;
      null[i] = colIsNull(key, row) ? 1 : 0;
   }
}
enum WinBound : int32_t { kWinUnbounded = 0, kWinPeer = 1, kWinOffset = 2 };
struct WinRangeParams {
   const uint32_t* start;     // partition
   const uint32_t* end;
   const uint32_t* peerStart; // first / last peer
   const uint32_t* peerEnd;
   const uint8_t* null;       // the key's NULL flags in window order (offset bounds)
   uint32_t* lo;              // out: the frame [lo[i], hiEx[i]), empty when lo >= hiEx
   uint32_t* hiEx;
   int64_t n, from, to;
   int32_t fromKind, toKind, desc, pad;
};
// key + d without wrapping: the sum, or past the i128 range `past` = +1 (above every key) / -1 (below every key); an int64 key never
// gets there
__device__ __forceinline__ s128 winTarget(s128 k, int64_t d, int& past) {
   const s128 top = (s128) (((unsigned __int128) 1 << 127) - 1), bottom = -top - 1;
   past = d > 0 && k > top - d ? 1 : d < 0 && k < bottom - d ? -1 : 0;
   return past ? k : k + d;
}
// the first position of [l, r) not before the target: keys run ascending there (desc: descending), and a key is before the target when
// ASC k < target (strict: k <= target), DESC k > target (strict: k >= target), so the test is monotone
template <class K>
__device__ __forceinline__ int64_t winSearch(const K* key, int64_t l, int64_t r, s128 target, int past, bool desc, bool strict) {
   if (past) return (past > 0) != desc ? r : l; // a target beyond every key: every key before it, or none
   while (l < r) {
      const int64_t m = (l + r) >> 1;
      const s128 k = (s128) key[m];
      const bool before = desc ? (strict ? k >= target : k > target) : (strict ? k <= target : k < target);
      if (before) l = m + 1;
      else r = m;
   }
   return l;
}
// per row its frame by the RANGE rules: UNBOUNDED = the partition end, CURRENT ROW = the peer bound, an offset the rows of the
// partition's non-NULL keys in [key + from, key + to] (DESC: [key - to, key - from] read downwards); a NULL-key row takes its peers
template <class K>
__global__ void __launch_bounds__(kWinThreads) winRangeKernel(const __grid_constant__ WinRangeParams p, const K* key) {
   for (int64_t i = (int64_t) blockIdx.x * kWinThreads + threadIdx.x; i < p.n; i += (int64_t) gridDim.x * kWinThreads) {
      const int64_t s = p.start[i], e = p.end[i];
      int64_t lo = s, hiEx = e + 1;
      if (p.fromKind == kWinPeer || (p.fromKind == kWinOffset && p.null[i])) lo = p.peerStart[i];
      if (p.toKind == kWinPeer || (p.toKind == kWinOffset && p.null[i])) hiEx = (int64_t) p.peerEnd[i] + 1;
      if ((p.fromKind == kWinOffset || p.toKind == kWinOffset) && !p.null[i]) {
         // the partition's non-NULL keys: NULLs sort last under ASC, first under DESC, and are peers of one another
         const int64_t ns = p.desc && p.null[s] ? (int64_t) p.peerEnd[s] + 1 : s;
         const int64_t ne = !p.desc && p.null[e] ? (int64_t) p.peerStart[e] : e + 1;
         const s128 k = (s128) key[i];
         int past;
         if (p.fromKind == kWinOffset) {
            const s128 t = winTarget(k, p.desc ? -p.from : p.from, past);
            lo = winSearch(key, ns, ne, t, past, p.desc != 0, false);
         }
         if (p.toKind == kWinOffset) {
            const s128 t = winTarget(k, p.desc ? -p.to : p.to, past);
            hiEx = winSearch(key, ns, ne, t, past, p.desc != 0, true);
         }
      }
      p.lo[i] = (uint32_t) lo;
      p.hiEx[i] = (uint32_t) hiEx;
   }
}

// ---------------------------------------------------------------- frames and function values
constexpr uint32_t kWinNone = 0xffffffffu; // permuteRows' id of a row of NULL cells: no source row
struct WinFunc {
   int32_t kind, width, wide, pad; // width: output cell bytes (MIN / MAX); wide: the tree holds i128 nodes
   uint8_t* out;
   uint8_t* valid;                  // SUM, MIN, MAX
   const unsigned long long* sums;  // SUM: the scan's i128 prefix sums
   const unsigned long long* counts; // SUM, COUNT: the scan's prefix counts
   const void* tree;                 // MIN, MAX
   const uint8_t* any;
   int64_t n;                        // LAG / LEAD offset, NTILE buckets, NTH_VALUE position
   uint32_t* src;                    // LAG, LEAD and the value functions: per row the source row to gather, kWinNone for NULL
};
struct WinFrameParams {
   const uint32_t* start;
   const uint32_t* end;
   int64_t n, from, to; // offsets already limited to +-2^40 (|j| < 2^32, so the clamp gives the same bounds)
   int32_t fromUnbounded, toUnbounded, nFuncs, range;
   uint64_t leaves;
   // the extended kernel only
   const uint32_t* ids;       // the sort's row ids (null: source order)
   const uint32_t* lo;        // RANGE frames with a bounded end: winRangeKernel's frames (null: the clamp, or both ends unbounded)
   const uint32_t* hiEx;
   const uint32_t* peerStart; // RANK, PERCENT_RANK, CUME_DIST
   const uint32_t* peerEnd;
   const uint32_t* dense;     // DENSE_RANK
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
// MIN / MAX of the frame [lo, hi] (not empty)
__device__ __forceinline__ void winMinMax(const WinFunc& f, uint64_t leaves, int64_t lo, int64_t hi, s128& v, bool& has) {
   const int isMax = f.kind == LDB_WIN_MAX;
   if (f.wide) {
      winTreeQuery((const s128*) f.tree, f.any, leaves, (uint64_t) lo, (uint64_t) hi, isMax, v, has);
   } else {
      long long w;
      winTreeQuery((const long long*) f.tree, f.any, leaves, (uint64_t) lo, (uint64_t) hi, isMax, w, has);
      v = w;
   }
}
// SUM of the frame [lo, hi]: the prefix difference, NULL when it holds no value (an empty frame, lo = hi + 1, holds none)
__device__ __forceinline__ void winSum(const WinFunc& f, int64_t lo, int64_t hi, int64_t i) {
   const unsigned long long c = f.counts[hi] - (lo ? f.counts[lo - 1] : 0ull);
   const ulonglong2 a = *(const ulonglong2*) (f.sums + 2 * hi);
   const ulonglong2 b = lo ? *(const ulonglong2*) (f.sums + 2 * (lo - 1)) : make_ulonglong2(0, 0);
   const unsigned long long dlo = a.x - b.x, dhi = a.y - b.y - (a.x < b.x ? 1ull : 0ull);
   *(ulonglong2*) (f.out + (size_t) i * 16) = c ? make_ulonglong2(dlo, dhi) : make_ulonglong2(0, 0);
   f.valid[i] = c ? 1 : 0;
}
// kEx = false: the six kinds of ldb_gpu_table_window over ROWS frames, the instance every call without the new features runs;
// kEx = true: RANGE frames (possibly empty) and the ranking, offset and value functions too
template <bool kEx>
__global__ void __launch_bounds__(kWinThreads) winFramesKernel(const __grid_constant__ WinFrameParams p) {
   for (int64_t i = (int64_t) blockIdx.x * kWinThreads + threadIdx.x; i < p.n; i += (int64_t) gridDim.x * kWinThreads) {
      const int64_t s = p.start[i], len = (int64_t) p.end[i] - s + 1, j = i - s;
      int64_t lo, hi;
      if (kEx && p.lo) {
         lo = p.lo[i];
         hi = (int64_t) p.hiEx[i] - 1;
      } else {
         lo = s + (p.fromUnbounded ? 0 : min(len - 1, max((int64_t) 0, j + p.from)));
         hi = p.toUnbounded ? s + len - 1 : s + min(len - 1, max((int64_t) 0, j + p.to));
      }
      const bool empty = kEx && lo > hi;
      for (int q = 0; q < p.nFuncs; q++) {
         const WinFunc& f = p.f[q];
         if (!kEx) {
            switch (f.kind) {
               case LDB_WIN_ROW_NUMBER: ((int64_t*) f.out)[i] = i - lo + 1; break;
               case LDB_WIN_COUNT_STAR: ((int64_t*) f.out)[i] = hi - lo + 1; break;
               case LDB_WIN_COUNT: ((int64_t*) f.out)[i] = (int64_t) (f.counts[hi] - (lo ? f.counts[lo - 1] : 0ull)); break;
               case LDB_WIN_SUM: winSum(f, lo, hi, i); break;
               default: { // MIN, MAX
                  bool has;
                  s128 v;
                  winMinMax(f, p.leaves, lo, hi, v, has);
                  winStoreCell(f.out, f.width, i, has ? v : (s128) 0);
                  f.valid[i] = has ? 1 : 0;
               }
            }
            continue;
         }
         int64_t pos = -1; // the value functions' frame or partition position
         switch (f.kind) {
            case LDB_WIN_ROW_NUMBER: ((int64_t*) f.out)[i] = p.range ? j + 1 : i - lo + 1; break;
            case LDB_WIN_COUNT_STAR: ((int64_t*) f.out)[i] = empty ? 0 : hi - lo + 1; break;
            case LDB_WIN_COUNT: ((int64_t*) f.out)[i] = empty ? 0 : (int64_t) (f.counts[hi] - (lo ? f.counts[lo - 1] : 0ull)); break;
            case LDB_WIN_SUM:
               if (empty) {
                  *(ulonglong2*) (f.out + (size_t) i * 16) = make_ulonglong2(0, 0);
                  f.valid[i] = 0;
               } else {
                  winSum(f, lo, hi, i);
               }
               break;
            case LDB_WIN_MIN:
            case LDB_WIN_MAX: {
               bool has = false;
               s128 v = 0;
               if (!empty) winMinMax(f, p.leaves, lo, hi, v, has);
               winStoreCell(f.out, f.width, i, has ? v : (s128) 0);
               f.valid[i] = has ? 1 : 0;
               break;
            }
            case LDB_WIN_RANK: ((int64_t*) f.out)[i] = (int64_t) p.peerStart[i] - s + 1; break;
            case LDB_WIN_DENSE_RANK: ((int64_t*) f.out)[i] = (int64_t) (p.dense[i] - p.dense[s]) + 1; break;
            case LDB_WIN_PERCENT_RANK: ((double*) f.out)[i] = len > 1 ? (double) ((int64_t) p.peerStart[i] - s) / (double) (len - 1) : 0.0; break;
            case LDB_WIN_CUME_DIST: ((double*) f.out)[i] = (double) ((int64_t) p.peerEnd[i] - s + 1) / (double) len; break;
            case LDB_WIN_NTILE: { // the first len % n buckets hold len / n + 1 rows, the others len / n
               const int64_t q0 = len / f.n, r = len % f.n, big = r * (q0 + 1);
               ((int64_t*) f.out)[i] = j < big ? j / (q0 + 1) + 1 : r + (j - big) / q0 + 1;
               break;
            }
            case LDB_WIN_LAG: pos = j >= f.n ? i - f.n : -1; break;
            case LDB_WIN_LEAD: pos = f.n <= len - 1 - j ? i + f.n : -1; break;
            case LDB_WIN_FIRST_VALUE: pos = empty ? -1 : lo; break;
            case LDB_WIN_LAST_VALUE: pos = empty ? -1 : hi; break;
            default: pos = !empty && f.n - 1 <= hi - lo ? lo + f.n - 1 : -1; // NTH_VALUE
         }
         if (f.src) f.src[i] = pos < 0 ? kWinNone : (uint32_t) winRow(p.ids, pos);
      }
   }
}
// LAG / LEAD with a default: the default's cell (its low `width` bytes) and validity 1 where there was no offset row
__global__ void __launch_bounds__(kWinThreads) winDefaultKernel(const uint32_t* src, int64_t n, int width, ulonglong2 cell, uint8_t* out, uint8_t* valid) {
   for (int64_t i = (int64_t) blockIdx.x * kWinThreads + threadIdx.x; i < n; i += (int64_t) gridDim.x * kWinThreads) {
      if (src[i] != kWinNone) continue;
      for (int b = 0; b < width; b++) out[(size_t) i * width + b] = (uint8_t) ((b < 8 ? cell.x >> (8 * b) : cell.y >> (8 * (b - 8))) & 0xff);
      valid[i] = 1;
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
static bool winValueKind(int kind) { return kind >= LDB_WIN_LAG; } // LAG, LEAD, FIRST_VALUE, LAST_VALUE, NTH_VALUE: a gather of the argument
static bool winPeerKind(int kind) { return kind == LDB_WIN_RANK || kind == LDB_WIN_DENSE_RANK || kind == LDB_WIN_PERCENT_RANK || kind == LDB_WIN_CUME_DIST; }
static bool winNoArgKind(int kind) { return kind == LDB_WIN_ROW_NUMBER || kind == LDB_WIN_COUNT_STAR || (kind >= LDB_WIN_RANK && kind <= LDB_WIN_NTILE); }
static WinBound winBound(int64_t b, int64_t unbounded) { return b == unbounded ? kWinUnbounded : b == 0 ? kWinPeer : kWinOffset; }

// LAG / LEAD's default as the argument's cell (its low `width` bytes), after the LdbJoinCond rule: a float argument reads fvalue, any
// other value, and the field not read is 0 or the same number
static ulonglong2 winDefaultCell(const LdbWindowFuncEx& f, const LdbColumn& a, int q) {
   const std::string what = "window function " + std::to_string(q) + " (" + a.name + "): the default";
   if (a.type == LDB_UTF8) fail(LDB_ERR_UNSUPPORTED, what + " of a utf8 argument is not supported");
   const bool isFloat = a.type == LDB_FLOAT32 || a.type == LDB_FLOAT64;
   const __int128 v = (__int128) ((unsigned __int128) (uint64_t) f.value.hi << 64 | (uint64_t) f.value.lo);
   if (isFloat ? (v != 0 && (double) v != f.fvalue) : (f.fvalue != 0.0 && f.fvalue != (double) v))
      fail(LDB_ERR_INVALID, what + "'s value and fvalue differ; the argument reads " + (isFloat ? "fvalue" : "value") + " (set the other to 0 or to the same number)");
   if (a.type == LDB_FLOAT64) {
      uint64_t bits;
      memcpy(&bits, &f.fvalue, 8);
      return make_ulonglong2(bits, 0);
   }
   if (a.type == LDB_FLOAT32) {
      if (std::isfinite(f.fvalue) && std::fabs(f.fvalue) > (double) FLT_MAX) fail(LDB_ERR_INVALID, what + " is outside float32's range");
      const float x = (float) f.fvalue;
      uint32_t bits;
      memcpy(&bits, &x, 4);
      return make_ulonglong2(bits, 0);
   }
   __int128 lo, hi;
   switch (a.type) {
      case LDB_INT8: lo = INT8_MIN, hi = INT8_MAX; break;
      case LDB_INT16: lo = INT16_MIN, hi = INT16_MAX; break;
      case LDB_INT64: lo = INT64_MIN, hi = INT64_MAX; break;
      case LDB_DECIMAL128: {
         hi = 1;
         for (int d = 0; d < std::min(std::max(a.precision, 1), 38); d++) hi *= 10;
         hi -= 1;
         lo = -hi;
         break;
      }
      default: lo = INT32_MIN, hi = INT32_MAX; // int32, date32, char(1)
   }
   if (v < lo || v > hi) fail(LDB_ERR_INVALID, what + " does not fit the argument's type");
   return make_ulonglong2((unsigned long long) v, (unsigned long long) ((unsigned __int128) v >> 64));
}

// both entry points: ldb_gpu_table_window passes a ROWS frame and maxKind = LDB_WIN_MAX
static void tableWindow(LdbTable* src, int32_t n_partition, const char* const* partition_columns, int32_t n_order, const char* const* order_columns,
                        const int32_t* descending, const LdbWindowFrame* frame, int32_t n_funcs, const LdbWindowFuncEx* funcs, int32_t n_columns,
                        const char* const* columns, const char* name, LdbTable** out, int maxKind) {
   // everything is checked before the first launch
   if (!src || !out || (n_partition > 0 && !partition_columns) || (n_order > 0 && (!order_columns || !descending)) || (n_funcs > 0 && !funcs) || !frame)
      fail(LDB_ERR_INVALID, "null argument");
   if (n_partition < 0 || n_partition > kProgMaxKeys || n_order < 0 || n_order > kProgMaxKeys) fail(LDB_ERR_INVALID, "a window takes 0..4 partition keys and 0..4 order keys");
   if (n_funcs < 1 || n_funcs > kWinMaxFuncs) fail(LDB_ERR_INVALID, "a window computes 1..8 functions");
   if (n_columns < 0 || (columns && n_columns > kWinMaxCarried)) fail(LDB_ERR_INVALID, "a window carries 0..16 columns");
   const int64_t frame_from = frame->from, frame_to = frame->to;
   if (frame_from > frame_to || frame_from == INT64_MAX || frame_to == INT64_MIN)
      fail(LDB_ERR_INVALID, "bad frame: from must be <= to, from may not be UNBOUNDED FOLLOWING (INT64_MAX) nor to UNBOUNDED PRECEDING (INT64_MIN)");
   if (frame->mode != LDB_FRAME_ROWS && frame->mode != LDB_FRAME_RANGE) fail(LDB_ERR_INVALID, "unknown frame mode " + std::to_string(frame->mode));
   const bool range = frame->mode == LDB_FRAME_RANGE;
   const WinBound fromKind = range ? winBound(frame_from, INT64_MIN) : kWinUnbounded, toKind = range ? winBound(frame_to, INT64_MAX) : kWinUnbounded;
   const bool rangeOffset = fromKind == kWinOffset || toKind == kWinOffset;
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
   if (rangeOffset) {
      if (n_order != 1) fail(LDB_ERR_UNSUPPORTED, "a RANGE frame with an offset bound takes exactly one order key (the call has " + std::to_string(n_order) + ")");
      const LdbColumn& k = src->columns[keys[n_partition].first];
      if (k.type != LDB_INT32 && k.type != LDB_INT64 && k.type != LDB_DATE32 && k.type != LDB_DECIMAL128)
         fail(LDB_ERR_UNSUPPORTED, "a RANGE frame with an offset bound orders by an int32, int64, date32 or decimal key (column " + k.name + ")");
   }
   std::vector<int> argCol(n_funcs, -1);
   std::vector<ulonglong2> defaults(n_funcs, make_ulonglong2(0, 0));
   for (int q = 0; q < n_funcs; q++) {
      const int kind = funcs[q].kind;
      if (kind < LDB_WIN_ROW_NUMBER || kind > maxKind) fail(LDB_ERR_INVALID, "unknown window function kind " + std::to_string(kind));
      if (!funcs[q].name) fail(LDB_ERR_INVALID, "a window function needs an output column name");
      const int64_t n = funcs[q].n;
      if ((kind == LDB_WIN_LAG || kind == LDB_WIN_LEAD) && n < 0) fail(LDB_ERR_INVALID, "window function " + std::to_string(q) + ": LAG / LEAD take an offset >= 0");
      if ((kind == LDB_WIN_NTILE || kind == LDB_WIN_NTH_VALUE) && n < 1) fail(LDB_ERR_INVALID, "window function " + std::to_string(q) + ": NTILE / NTH_VALUE take n >= 1");
      if (funcs[q].has_default && kind != LDB_WIN_LAG && kind != LDB_WIN_LEAD) fail(LDB_ERR_INVALID, "window function " + std::to_string(q) + ": only LAG and LEAD take a default");
      if (winNoArgKind(kind)) continue;
      const int ci = argCol[q] = column(funcs[q].column, "argument");
      const int type = src->columns[ci].type;
      if (kind == LDB_WIN_SUM && !winSumType(type))
         fail(LDB_ERR_UNSUPPORTED, "window SUM takes int8..int64 or decimal columns (column " + src->columns[ci].name + ")");
      if ((kind == LDB_WIN_MIN || kind == LDB_WIN_MAX) && !winSumType(type) && type != LDB_DATE32 && type != LDB_FSB4)
         fail(LDB_ERR_UNSUPPORTED, "window MIN / MAX take int8..int64, decimal, date32 or char(1) columns (column " + src->columns[ci].name + ")");
      if (funcs[q].has_default) defaults[q] = winDefaultCell(funcs[q], src->columns[ci], q);
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

   // the extended frame kernel runs only for the new features: a call without them launches what ldb_gpu_table_window always did
   bool ex = range, peers = fromKind == kWinPeer || toKind == kWinPeer || rangeOffset, dense = false;
   for (int q = 0; q < n_funcs; q++) {
      ex |= funcs[q].kind > LDB_WIN_MAX;
      peers |= winPeerKind(funcs[q].kind);
      dense |= funcs[q].kind == LDB_WIN_DENSE_RANK;
   }

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
   fp.range = range ? 1 : 0;
   fp.leaves = nextPow2((uint64_t) std::max<int64_t>(n, 1));
   fp.ids = ids;
   const size_t firstFunc = ob.data.size();
   for (int q = 0; q < n_funcs; q++) {
      const int kind = funcs[q].kind;
      WinFunc& f = fp.f[q];
      f.kind = kind;
      f.n = funcs[q].n;
      const LdbColumn* a = argCol[q] >= 0 ? &src->columns[argCol[q]] : nullptr;
      if (winValueKind(kind)) { // gathered by permuteRows after the frame kernel has written the source rows
         f.src = tmp.alloc<uint32_t>(rows * 4);
         outCols.push_back({funcs[q].name, a->type, a->precision, a->scale});
         ob.data.push_back(nullptr);
         ob.bytes.push_back(nullptr);
         ob.elemBytes.push_back(shipCellBytes(a->type));
         ob.validBytes.push_back(nullptr);
         continue;
      }
      const int32_t argBytes = argCol[q] >= 0 && !src->batches.empty() ? src->batches[0].elemBytes[argCol[q]] : (a ? shipCellBytes(a->type) : 8);
      if (kind == LDB_WIN_SUM) {
         f.width = 16;
         outCols.push_back({funcs[q].name, LDB_DECIMAL128, 38, a->type == LDB_DECIMAL128 ? a->scale : 0});
      } else if (kind == LDB_WIN_MIN || kind == LDB_WIN_MAX) {
         f.width = argBytes;
         f.wide = argBytes == 16;
         outCols.push_back({funcs[q].name, a->type, a->precision, a->scale});
      } else if (kind == LDB_WIN_PERCENT_RANK || kind == LDB_WIN_CUME_DIST) {
         f.width = 8;
         outCols.push_back({funcs[q].name, LDB_FLOAT64, 0, 0});
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
      ctx->launch("window_partition", [&] { winHeadsKernel<<<winGrid(ctx, (uint64_t) n), kWinThreads, 0, ctx->compute>>>(wk, ids, n, nullptr, head); });
      tileScan(ctx, tmp, WinStartOp{head, start}, n, "window_scan");
      tileScan(ctx, tmp, WinEndOp{head, end, n}, n, "window_scan");
      fp.start = start;
      fp.end = end;
      // peer groups: the partition heads or a change of the order key tuple (without order keys a partition is one peer group)
      if (peers) {
         uint8_t* peerHead = head;
         if (n_order > 0) {
            peerHead = tmp.alloc<uint8_t>(rows);
            WinKeys ok{};
            ok.n = n_order;
            for (int k = 0; k < n_order; k++) {
               bindColumn(ok.col[k], src->batches[0], keys[n_partition + k].first);
               ok.col[k].type = src->columns[keys[n_partition + k].first].type;
            }
            ctx->launch("window_peers", [&] { winHeadsKernel<<<winGrid(ctx, (uint64_t) n), kWinThreads, 0, ctx->compute>>>(ok, ids, n, head, peerHead); });
         }
         uint32_t* peerStart = tmp.alloc<uint32_t>(rows * 4);
         uint32_t* peerEnd = tmp.alloc<uint32_t>(rows * 4);
         tileScan(ctx, tmp, WinStartOp{peerHead, peerStart}, n, "window_peers");
         tileScan(ctx, tmp, WinEndOp{peerHead, peerEnd, n}, n, "window_peers");
         fp.peerStart = peerStart;
         fp.peerEnd = peerEnd;
         if (dense) {
            uint32_t* d = tmp.alloc<uint32_t>(rows * 4);
            tileScan(ctx, tmp, WinCountOp{peerHead, d}, n, "window_peers");
            fp.dense = d;
         }
      }
      // RANGE frames with a bounded end: per row [lo, hiEx) from the peer bounds and the key words' binary searches
      if (range && (fromKind != kWinUnbounded || toKind != kWinUnbounded)) {
         WinRangeParams rp{};
         rp.start = start;
         rp.end = end;
         rp.peerStart = fp.peerStart;
         rp.peerEnd = fp.peerEnd;
         rp.lo = tmp.alloc<uint32_t>(rows * 4);
         rp.hiEx = tmp.alloc<uint32_t>(rows * 4);
         rp.n = n;
         rp.from = frame_from;
         rp.to = frame_to;
         rp.fromKind = fromKind;
         rp.toKind = toKind;
         rp.desc = n_order > 0 && keys[n_partition].second;
         if (rangeOffset) {
            ProgCol key{};
            bindColumn(key, src->batches[0], keys[n_partition].first);
            key.type = src->columns[keys[n_partition].first].type;
            uint8_t* null = tmp.alloc<uint8_t>(rows);
            rp.null = null;
            if (key.elemBytes == 16) {
               s128* words = tmp.alloc<s128>(rows * 16);
               ctx->launch("window_range", [&] {
                  winKeyWordsKernel<s128><<<winGrid(ctx, (uint64_t) n), kWinThreads, 0, ctx->compute>>>(key, ids, n, words, null);
                  winRangeKernel<s128><<<winGrid(ctx, (uint64_t) n), kWinThreads, 0, ctx->compute>>>(rp, words);
               });
            } else {
               long long* words = tmp.alloc<long long>(rows * 8);
               ctx->launch("window_range", [&] {
                  winKeyWordsKernel<long long><<<winGrid(ctx, (uint64_t) n), kWinThreads, 0, ctx->compute>>>(key, ids, n, words, null);
                  winRangeKernel<long long><<<winGrid(ctx, (uint64_t) n), kWinThreads, 0, ctx->compute>>>(rp, words);
               });
            }
         } else {
            ctx->launch("window_range", [&] { winRangeKernel<long long><<<winGrid(ctx, (uint64_t) n), kWinThreads, 0, ctx->compute>>>(rp, nullptr); });
         }
         fp.lo = rp.lo;
         fp.hiEx = rp.hiEx;
      }
      // per function its scan or its tree
      for (int q = 0; q < n_funcs; q++) {
         WinFunc& f = fp.f[q];
         if (argCol[q] < 0 || winValueKind(f.kind)) continue;
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
      ctx->launch("window_frames", [&] {
         if (ex) winFramesKernel<true><<<winGrid(ctx, (uint64_t) n), kWinThreads, 0, ctx->compute>>>(fp);
         else winFramesKernel<false><<<winGrid(ctx, (uint64_t) n), kWinThreads, 0, ctx->compute>>>(fp);
      });
   }
   // the value functions: one gather of the argument's cells per function (an id of kWinNone gives a NULL cell), then LAG / LEAD's
   // default where the offset row was outside the partition
   for (int q = 0; q < n_funcs; q++) {
      const WinFunc& f = fp.f[q];
      if (!winValueKind(f.kind)) continue;
      const LdbBatch g = permuteRows(src, {argCol[q]}, &ob.elemBytes[firstFunc + q], n > 0 ? f.src : nullptr, n, cols, "window");
      ob.data[firstFunc + q] = g.data[0];
      ob.bytes[firstFunc + q] = g.bytes[0];
      ob.validBytes[firstFunc + q] = g.validBytes[0];
      if (funcs[q].has_default && n > 0) {
         ctx->launch("window_frames", [&] {
            winDefaultKernel<<<winGrid(ctx, (uint64_t) n), kWinThreads, 0, ctx->compute>>>(f.src, n, g.elemBytes[0], defaults[q], (uint8_t*) g.data[0], g.validBytes[0]);
         });
      }
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
      // the same call with a ROWS frame and kinds 1..6; only the counted functions are read (a bad count fails before they are)
      const LdbWindowFrame frame{LDB_FRAME_ROWS, 0, frame_from, frame_to};
      const bool counted = funcs && n_funcs >= 1 && n_funcs <= ldb::kWinMaxFuncs;
      std::vector<LdbWindowFuncEx> ex(counted ? n_funcs : 1, LdbWindowFuncEx{});
      for (int q = 0; counted && q < n_funcs; q++) {
         ex[q].kind = funcs[q].kind;
         ex[q].column = funcs[q].column;
         ex[q].name = funcs[q].name;
      }
      ldb::tableWindow(src, n_partition, partition_columns, n_order, order_columns, descending, &frame, n_funcs, funcs ? ex.data() : nullptr, n_columns, columns,
                       name, out, LDB_WIN_MAX);
   });
}

extern "C" int ldb_gpu_table_window_ex(LdbTable* src, int32_t n_partition, const char* const* partition_columns, int32_t n_order, const char* const* order_columns,
                                       const int32_t* descending, const LdbWindowFrame* frame, int32_t n_funcs, const LdbWindowFuncEx* funcs, int32_t n_columns,
                                       const char* const* columns, const char* name, LdbTable** out, LdbError* err) {
   return ldb::guarded(err, [&] {
      ldb::tableWindow(src, n_partition, partition_columns, n_order, order_columns, descending, frame, n_funcs, funcs, n_columns, columns, name, out, LDB_WIN_NTH_VALUE);
   });
}
