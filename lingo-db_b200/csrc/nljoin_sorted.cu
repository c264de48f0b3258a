// nljoin_sorted.cu — the sorted-ranges path of ldb_gpu_table_nl_join (nljoin.cu): the same rows, cells, order and errors as the loop,
// in O((n + m) log + candidates) instead of O(n m).
//
// Rules:
//   Key: the column that appears, on one side, in the most range conditions (<, <=, >, >=) is K and its side is S (a tie between the
//     sides: the smaller side); only equality conditions: S is the smaller side and there is no K.  S's rows that can match (the
//     words kernel's "can match" byte) are sorted by (equality words..., K's word, row id); every range condition on K bounds K from
//     below or above, so each row of the other side, the probe side P, matches one contiguous range of sorted positions, found by
//     binary searches: several lower bounds take the largest start, several upper bounds the smallest end.  <> and range conditions
//     on another column of S are residuals, checked for every candidate of a range.
//   Counts: without residuals a range's length is its count; when P is the left side it is the left row's count and a coverage scan
//     over the sorted positions marks the right rows, when S is the left side the coverage is each left row's count and a non-empty
//     range marks its right row.  With residuals one load-balanced walk over the candidates counts and marks.
//   Order: pairs are written at their left row's offset; the walk's pairs then go through a stable radix sort on (left id, right id)
//     unless they provably are in order already (S is the right side, no residuals and no range holds a descent of the sorted ids).
//   Selection (nljoin.cu): the loop runs when no condition keys a sort, when n m < kNljSortMinPairs, when this path's scratch would
//     not fit where the loop's would, and when the candidates exceed n m / kNljCandidateRatio (then the loop's write costs no more
//     than enumerating them).
#include "nljoin.cuh"
#include "program.h"
#include "tilescan.cuh"

namespace ldb {

constexpr int kNljMaxKeyWords = 2 * kNljMaxPairs;  // equality words and K's, two per 16-byte operand
constexpr int kNljSampleWords = 4096;               // the sorted key's shared-memory samples: 32 KB
constexpr int kNljSamples = 1024;                   // samples per key word at most
constexpr unsigned long long kNljSign = 0x8000000000000000ull;

// ---------------------------------------------------------------- the sorted side's key
// key word w of a row as an unsigned number in the key's order: part 0 a narrow word (signed), 1 a 16-byte operand's high word
// (signed), 2 its low word (unsigned)
__device__ __forceinline__ unsigned long long nljKeyWord(const int64_t* lo, const int64_t* hi, int64_t n, int pair, int part, int64_t row) {
   if (part == 2) return (unsigned long long) lo[(size_t) pair * n + row];
   return (unsigned long long) (part == 1 ? hi : lo)[(size_t) pair * n + row] ^ kNljSign;
}
// the rows that can match, ascending: ids[k] for k < *total
struct NljOkOp {
   using T = uint32_t;
   const uint8_t* ok;
   uint32_t* ids;
   unsigned long long* total;
   int64_t n;
   __device__ T identity() const { return 0; }
   __device__ T combine(T a, T b) const { return a + b; }
   __device__ T load(int64_t k) const { return ok[k]; }
   __device__ void store(int64_t k, T v) const {
      if (ok[k]) ids[v - 1] = (uint32_t) k;
      if (k == n - 1) *total = v;
   }
};
// blockIdx.y = key word: its minimum and maximum over the rows that can match
__global__ void __launch_bounds__(256) nljMinMaxKernel(const int64_t* lo, const int64_t* hi, int64_t n, const int* pair, const int* part, const uint8_t* ok,
                                                       unsigned long long* mm) {
   const int w = blockIdx.y;
   unsigned long long mn = ~0ull, mx = 0;
   for (int64_t i = (int64_t) blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t) gridDim.x * 256) {
      if (!ok[i]) continue;
      const unsigned long long k = nljKeyWord(lo, hi, n, pair[w], part[w], i);
      mn = min(mn, k);
      mx = max(mx, k);
   }
   for (int o = 16; o > 0; o >>= 1) {
      mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
   }
   if ((threadIdx.x & 31) == 0) {
      atomicMin(mm + 2 * w, mn);
      atomicMax(mm + 2 * w + 1, mx);
   }
}
// keys[i] = key word (pair, part) of row ids[i]
__global__ void __launch_bounds__(256) nljGatherKernel(const int64_t* lo, const int64_t* hi, int64_t nRows, int pair, int part, const uint32_t* ids, int64_t n,
                                                       unsigned long long* keys) {
   for (int64_t i = (int64_t) blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t) gridDim.x * 256) keys[i] = nljKeyWord(lo, hi, nRows, pair, part, ids[i]);
}
// desc[k] = the positions j <= k whose id is below the one before (a descent), inclusive
struct NljDescentOp {
   using T = uint32_t;
   const uint32_t* ids;
   uint32_t* desc;
   __device__ T identity() const { return 0; }
   __device__ T combine(T a, T b) const { return a + b; }
   __device__ T load(int64_t k) const { return k > 0 && ids[k - 1] > ids[k]; }
   __device__ void store(int64_t k, T v) const { desc[k] = v; }
};

// ---------------------------------------------------------------- the searches
struct NljSearchParams {
   const unsigned long long* skey; // [nw][nS]: the sorted key's words
   int64_t nS, stride;             // stride: sorted positions between shared samples
   int32_t nw, nEqWords, nSamp, nBound;
   const int64_t *lo, *hi;         // the probe side's words
   const uint8_t* ok;
   int64_t nP;
   int32_t wordPair[kNljMaxKeyWords], wordPart[kNljMaxKeyWords]; // the probe's operand of each equality word; K's part per K word
   int32_t boundPair[kNljMaxPairs], boundKind[kNljMaxPairs];    // bit 0: search for the first key > (else >=) the bound; bit 1: an upper bound
   uint32_t *rlo, *rlen;           // per probe row: its range's start and length
   uint32_t* cnt;                  // or null: cnt[p] = the length (P is the left side, no residuals)
   uint8_t* mark;                  // or null: mark[p] = 1 when the range is not empty (P is the right side, no residuals)
   const uint32_t* desc;           // or null: NljDescentOp's prefix, then *descents = 1 when some range holds a descent
   int32_t* descents;
};
// -1 / 0 / 1: the first `ncmp` key words at `pos` (words `stride` apart) against key
__device__ __forceinline__ int nljKeyCmp(const unsigned long long* words, int64_t stride, int64_t pos, const unsigned long long (&key)[kNljMaxKeyWords], int ncmp) {
#pragma unroll
   for (int w = 0; w < kNljMaxKeyWords; w++) {
      if (w < ncmp) {
         const unsigned long long a = words[(size_t) w * stride + pos];
         if (a != key[w]) return a < key[w] ? -1 : 1;
      }
   }
   return 0;
}
// the first sorted position whose key (first ncmp words) is > key (upper) or >= key: the samples first, then the one gap between two
__device__ __forceinline__ int64_t nljFind(const NljSearchParams& p, const unsigned long long* samp, const unsigned long long (&key)[kNljMaxKeyWords], int ncmp, bool upper) {
   int a = 0, b = p.nSamp;
   while (a < b) {
      const int m = (a + b) >> 1;
      const int c = nljKeyCmp(samp, p.nSamp, m, key, ncmp);
      if (upper ? c > 0 : c >= 0) b = m;
      else a = m + 1;
   }
   int64_t lo = a == 0 ? 0 : (int64_t) (a - 1) * p.stride + 1, hi = a == p.nSamp ? p.nS : (int64_t) a * p.stride;
   while (lo < hi) {
      const int64_t m = (lo + hi) >> 1;
      const int c = nljKeyCmp(p.skey, p.nS, m, key, ncmp);
      if (upper ? c > 0 : c >= 0) hi = m;
      else lo = m + 1;
   }
   return lo;
}
__global__ void __launch_bounds__(256) nljSearchKernel(const __grid_constant__ NljSearchParams p) {
   __shared__ unsigned long long samp[kNljSampleWords]; // [nw][nSamp]
   for (int i = threadIdx.x; i < p.nSamp * p.nw; i += 256) {
      const int w = i / p.nSamp, k = i - w * p.nSamp;
      samp[i] = p.skey[(size_t) w * p.nS + (int64_t) k * p.stride];
   }
   __syncthreads();
   for (int64_t r = (int64_t) blockIdx.x * 256 + threadIdx.x; r < p.nP; r += (int64_t) gridDim.x * 256) {
      int64_t lo = 0, hi = 0;
      if (p.ok[r]) {
         unsigned long long key[kNljMaxKeyWords];
#pragma unroll
         for (int w = 0; w < kNljMaxKeyWords; w++) key[w] = w < p.nEqWords ? nljKeyWord(p.lo, p.hi, p.nP, p.wordPair[w], p.wordPart[w], r) : 0;
         hi = p.nS;
         if (p.nEqWords) {
            lo = nljFind(p, samp, key, p.nEqWords, false);
            hi = nljFind(p, samp, key, p.nEqWords, true);
         }
#pragma unroll
         for (int b = 0; b < kNljMaxPairs; b++) {
            if (b < p.nBound) {
#pragma unroll
               for (int w = 0; w < kNljMaxKeyWords; w++)
                  if (w >= p.nEqWords && w < p.nw) key[w] = nljKeyWord(p.lo, p.hi, p.nP, p.boundPair[b], p.wordPart[w], r);
               const int64_t at = nljFind(p, samp, key, p.nw, p.boundKind[b] & 1);
               if (p.boundKind[b] & 2) hi = min(hi, at);
               else lo = max(lo, at);
            }
         }
         if (hi < lo) hi = lo;
      }
      const uint32_t len = (uint32_t) (hi - lo);
      p.rlo[r] = (uint32_t) lo;
      p.rlen[r] = len;
      if (p.cnt) p.cnt[r] = len;
      if (p.mark && len) p.mark[r] = 1;
      if (p.desc && len > 1 && p.desc[hi - 1] != p.desc[lo]) *p.descents = 1;
   }
}
// candOffs[p] = the candidates before probe row p; *total = all of them
struct NljCandOp {
   using T = unsigned long long;
   const uint32_t* len;
   unsigned long long* offs;
   unsigned long long* total;
   int64_t n;
   __device__ T identity() const { return 0; }
   __device__ T combine(T a, T b) const { return a + b; }
   __device__ T load(int64_t k) const { return len[k]; }
   __device__ void store(int64_t k, T v) const {
      offs[k] = v - len[k];
      if (k == n - 1) *total = v;
   }
};

// ---------------------------------------------------------------- coverage: per sorted position, the ranges that hold it
// diff[lo] += 1, diff[lo + len] -= 1 (modulo 2^32: coverage is below 2^32, so the wrapped sums are exact)
__global__ void __launch_bounds__(256) nljCoverKernel(const uint32_t* rlo, const uint32_t* rlen, int64_t nP, uint32_t* diff) {
   for (int64_t r = (int64_t) blockIdx.x * 256 + threadIdx.x; r < nP; r += (int64_t) gridDim.x * 256) {
      if (!rlen[r]) continue;
      atomicAdd(diff + rlo[r], 1u);
      atomicAdd(diff + rlo[r] + rlen[r], 0xffffffffu);
   }
}
// the scan of diff scattered back to row ids: cnt[ids[k]] = coverage (S is the left side), mark[ids[k]] = coverage > 0 (the right)
struct NljCoverOp {
   using T = uint32_t;
   const uint32_t* diff;
   const uint32_t* ids;
   uint32_t* cnt;
   uint8_t* mark;
   __device__ T identity() const { return 0; }
   __device__ T combine(T a, T b) const { return a + b; }
   __device__ T load(int64_t k) const { return diff[k]; }
   __device__ void store(int64_t k, T v) const {
      if (cnt) cnt[ids[k]] = v;
      else if (v) mark[ids[k]] = 1;
   }
};

// ---------------------------------------------------------------- the walk over the candidates
struct NljExpandParams {
   const unsigned long long* candOffs; // per probe row: its first candidate
   const uint32_t *rlo, *ids;
   int64_t nP;
   unsigned long long nCand;
   int32_t leftIsProbe, nRes;
   const int64_t *lLo, *lHi, *rLo, *rHi; // the sides' words (hi only when wide)
   int64_t nL, nR;
   int32_t resPair[kNljMaxPairs];
   uint32_t resMask[kNljMaxPairs];
   uint32_t* cnt;                     // count pass: per left row its matches, or null
   uint8_t* mark;                     // count pass: per right row 1 once matched, or null
   const unsigned long long* offs;    // write pass: per left row where its rows start (direct: a candidate's place follows from it)
   unsigned long long* cursor;        // write pass, not direct: per left row its next free place
   uint32_t *outL, *outR;
};
template <bool Wide>
__device__ __forceinline__ bool nljResidual(const NljExpandParams& p, int c, int64_t l, int64_t r) {
   const int64_t a = p.lLo[(size_t) p.resPair[c] * p.nL + l], b = p.rLo[(size_t) p.resPair[c] * p.nR + r];
   bool lt, eq;
   if constexpr (Wide) {
      const int64_t ah = p.lHi[(size_t) p.resPair[c] * p.nL + l], bh = p.rHi[(size_t) p.resPair[c] * p.nR + r];
      lt = ah < bh || (ah == bh && (uint64_t) a < (uint64_t) b);
      eq = ah == bh && a == b;
   } else {
      lt = a < b;
      eq = a == b;
   }
   return (p.resMask[c] >> (lt ? 0 : eq ? 1 : 2)) & 1u;
}
// every lane runs the same number of rounds (the warp-aggregated atomics need the whole warp); a thread's candidates ascend, so its
// probe row is searched from the last one onwards
template <bool Wide, bool Write>
__global__ void __launch_bounds__(256) nljExpandKernel(const __grid_constant__ NljExpandParams p) {
   const unsigned long long step = (unsigned long long) gridDim.x * 256;
   const int lane = threadIdx.x & 31;
   int64_t prev = 0;
   for (unsigned long long base = (unsigned long long) blockIdx.x * 256; base < p.nCand; base += step) {
      const unsigned long long q = base + threadIdx.x;
      const bool valid = q < p.nCand;
      int64_t l = 0, r = 0;
      unsigned long long within = 0;
      bool hit = false;
      if (valid) {
         int64_t a = prev, b = p.nP - 1; // the last probe row whose first candidate is <= q
         while (a < b) {
            const int64_t m = (a + b + 1) >> 1;
            if (p.candOffs[m] <= q) a = m;
            else b = m - 1;
         }
         prev = a;
         within = q - p.candOffs[a];
         const int64_t s = p.ids[p.rlo[a] + within];
         l = p.leftIsProbe ? a : s;
         r = p.leftIsProbe ? s : a;
         hit = true;
#pragma unroll
         for (int c = 0; c < kNljMaxPairs; c++)
            if (c < p.nRes) hit = hit && nljResidual<Wide>(p, c, l, r);
      }
      if constexpr (Write) {
         if (p.cursor) {
            const unsigned same = __match_any_sync(0xffffffffu, hit ? l : -1ll);
            const int leader = __ffs(same) - 1;
            unsigned long long at = 0;
            if (hit && lane == leader) at = atomicAdd(p.cursor + l, (unsigned long long) __popc(same));
            at = __shfl_sync(0xffffffffu, at, leader) + __popc(same & ((1u << lane) - 1));
            if (hit) {
               p.outL[at] = (uint32_t) l;
               p.outR[at] = (uint32_t) r;
            }
         } else if (hit) {
            const unsigned long long at = p.offs[l] + within;
            p.outL[at] = (uint32_t) l;
            p.outR[at] = (uint32_t) r;
         }
      } else {
         if (p.cnt) {
            const unsigned same = __match_any_sync(0xffffffffu, hit ? l : -1ll);
            if (hit && lane == __ffs(same) - 1) atomicAdd(p.cnt + l, (uint32_t) __popc(same));
         }
         if (p.mark && hit) p.mark[r] = 1;
      }
   }
}

// ---------------------------------------------------------------- the order
// keys[i] = (left id << bitsR) | right id, an absent right id all ones
__global__ void __launch_bounds__(256) nljOrderKeysKernel(const uint32_t* outL, const uint32_t* outR, int64_t n, int bitsR, unsigned long long* keys) {
   const unsigned long long none = (1ull << bitsR) - 1;
   for (int64_t i = (int64_t) blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t) gridDim.x * 256)
      keys[i] = ((unsigned long long) outL[i] << bitsR) | (outR[i] == kNljNone ? none : (unsigned long long) outR[i]);
}
__global__ void __launch_bounds__(256) nljOrderSplitKernel(const unsigned long long* keys, int64_t n, int bitsR, uint32_t* outL, uint32_t* outR) {
   const unsigned long long none = (1ull << bitsR) - 1;
   for (int64_t i = (int64_t) blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t) gridDim.x * 256) {
      const unsigned long long k = keys[i], r = k & none;
      outL[i] = (uint32_t) (k >> bitsR);
      outR[i] = r == none ? kNljNone : (uint32_t) r;
   }
}

// ---------------------------------------------------------------- host side
static int nljBits(unsigned long long x) { return x ? 64 - __builtin_clzll(x) : 0; }
static uint32_t nljMirror(uint32_t m) { return ((m & 1u) << 2) | (m & 2u) | ((m >> 2) & 1u); }

bool nljSortedPlan(int nc, const uint32_t* masks, const int* lCols, const int* rCols, int64_t nL, int64_t nR, NljSortedPlan* plan) {
   auto isRange = [](uint32_t m) { return m == 1 || m == 3 || m == 4 || m == 6; };
   // the column in the most range conditions: (side, column) with side 0 left, 1 right
   int best = 0, bestSide = -1, bestCol = -1;
   bool tie = false;
   for (int side = 0; side < 2; side++)
      for (int c = 0; c < nc; c++) {
         if (!isRange(masks[c])) continue;
         const int col = side ? rCols[c] : lCols[c];
         int k = 0;
         for (int d = 0; d < nc; d++)
            if (isRange(masks[d]) && (side ? rCols[d] : lCols[d]) == col) k++;
         if (k > best) best = k, bestSide = side, bestCol = col, tie = false;
         else if (k == best && side != bestSide) tie = true; // the same count on the other side
      }
   int nEq = 0;
   for (int c = 0; c < nc; c++) nEq += masks[c] == 2;
   if (!best && !nEq) return false;
   NljSortedPlan p;
   if (!best || tie) p.sLeft = nL < nR;
   else p.sLeft = bestSide == 0;
   if (best && tie) { // the tie's column on the chosen side
      bestCol = -1;
      for (int c = 0; c < nc && bestCol < 0; c++) {
         if (!isRange(masks[c])) continue;
         const int col = p.sLeft ? lCols[c] : rCols[c];
         int k = 0;
         for (int d = 0; d < nc; d++)
            if (isRange(masks[d]) && (p.sLeft ? lCols[d] : rCols[d]) == col) k++;
         if (k == best) bestCol = col;
      }
   }
   p.hasK = best > 0;
   for (int c = 0; c < nc; c++) {
      const int sCol = p.sLeft ? lCols[c] : rCols[c];
      if (masks[c] == 2) {
         p.eqPair[p.nEq++] = c;
      } else if (p.hasK && isRange(masks[c]) && sCol == bestCol) {
         if (p.kPair < 0) p.kPair = c;
         p.boundPair[p.nBound] = c;
         p.boundMask[p.nBound++] = p.sLeft ? masks[c] : nljMirror(masks[c]); // K against the probe's operand
      } else {
         p.resPair[p.nRes] = c;
         p.resMask[p.nRes++] = masks[c];
      }
   }
   *plan = p;
   return true;
}

// the sort key's words, most significant first: (pair, part) per word
static int nljKeyWords(const NljSortedPlan& p, bool wide, int* pair, int* part, int* nEqWords) {
   int nw = 0;
   auto add = [&](int c) {
      if (wide) {
         pair[nw] = c, part[nw++] = 1;
         pair[nw] = c, part[nw++] = 2;
      } else {
         pair[nw] = c, part[nw++] = 0;
      }
   };
   for (int e = 0; e < p.nEq; e++) add(p.eqPair[e]);
   *nEqWords = nw;
   if (p.hasK) add(p.kPair);
   return nw;
}

bool nljSortedCount(LdbContext* ctx, Scratch& tmp, NljSortedRun& run) {
   const NljSortedPlan& pl = run.plan;
   const NljWordsRef& S = pl.sLeft ? run.left : run.right;
   const NljWordsRef& P = pl.sLeft ? run.right : run.left;
   const int64_t nL = run.left.n, nR = run.right.n;
   int pair[kNljMaxKeyWords], part[kNljMaxKeyWords], nEqWords = 0;
   const int nw = nljKeyWords(pl, run.wide, pair, part, &nEqWords);
   const bool pairs = run.kind < LDB_NLJ_SEMI;
   const bool markRight = run.kind == LDB_NLJ_RIGHT_OUTER || run.kind == LDB_NLJ_FULL_OUTER;

   // 1. S's rows that can match, and each key word's range (the radix passes it needs)
   unsigned long long* ctr = tmp.alloc<unsigned long long>(256); // [0] sorted rows, [1] candidates, [2, 18) min / max per key word, [18] a flag
   LDB_CUDA(cudaMemsetAsync(ctr, 0, 16, ctx->compute));
   std::vector<unsigned long long> init(2 * kNljMaxKeyWords);
   for (int w = 0; w < kNljMaxKeyWords; w++) init[2 * w] = ~0ull, init[2 * w + 1] = 0;
   LDB_CUDA(cudaMemcpyAsync(ctr + 2, init.data(), init.size() * 8, cudaMemcpyHostToDevice, ctx->compute));
   int* dPairPart = tmp.alloc<int>(2 * kNljMaxKeyWords * 4);
   std::vector<int> pp(pair, pair + kNljMaxKeyWords);
   pp.insert(pp.end(), part, part + kNljMaxKeyWords);
   LDB_CUDA(cudaMemcpyAsync(dPairPart, pp.data(), pp.size() * 4, cudaMemcpyHostToDevice, ctx->compute));
   uint32_t* ids = run.keep.alloc<uint32_t>(std::max<size_t>((size_t) S.n * 4, 16));
   uint32_t* idsTmp = run.keep.alloc<uint32_t>(std::max<size_t>((size_t) S.n * 4, 16));
   unsigned long long* keys = run.sortOnly.alloc<unsigned long long>(std::max<size_t>((size_t) S.n * 8, 16));
   unsigned long long* keysTmp = run.sortOnly.alloc<unsigned long long>(std::max<size_t>((size_t) S.n * 8, 16));
   tileScan(ctx, tmp, NljOkOp{S.ok, ids, ctr, S.n}, S.n, "nljoin_sort");
   ctx->launch("nljoin_sort", [&] {
      nljMinMaxKernel<<<dim3(nljGrid(ctx, (uint64_t) S.n), (unsigned) nw), 256, 0, ctx->compute>>>(S.lo, S.hi, S.n, dPairPart, dPairPart + kNljMaxKeyWords, S.ok, ctr + 2);
   });
   unsigned long long* host = (unsigned long long*) ctx->scratch();
   LDB_CUDA(cudaMemcpyAsync(host, ctr, (2 + 2 * nw) * 8, cudaMemcpyDeviceToHost, ctx->compute));
   ctx->syncStream(ctx->compute);
   const int64_t nS = (int64_t) host[0];
   std::vector<int> digits(nw);
   for (int w = 0; w < nw; w++) digits[w] = (nljBits(host[2 + 2 * w] ^ host[3 + 2 * w]) + 7) / 8;

   // 2. the LSD sort: the least significant key word first; the ids start ascending, so equal keys keep row order
   const int64_t ctas = (nS + 256 * 16 - 1) / (256 * 16);
   unsigned int* hist = run.sortOnly.alloc<unsigned int>(std::max<size_t>((size_t) ctas * 256 * 4, 16));
   for (int w = nw - 1; w >= 0 && nS > 1; w--) {
      if (!digits[w]) continue;
      ctx->launch("nljoin_sort", [&] {
         nljGatherKernel<<<nljGrid(ctx, (uint64_t) nS), 256, 0, ctx->compute>>>(S.lo, S.hi, S.n, pair[w], part[w], ids, nS, keys);
         launchRadixSortPairs(keys, ids, keysTmp, idsTmp, nS, hist, ctx->smCount, ctx->compute, digits[w]);
      });
      if (digits[w] & 1) std::swap(ids, idsTmp);
   }
   // the sorted key's words, contiguous per word
   unsigned long long* skey = run.sortOnly.alloc<unsigned long long>(std::max<size_t>((size_t) nS * nw * 8, 16));
   if (nS > 0)
      for (int w = 0; w < nw; w++)
         ctx->launch("nljoin_sort", [&] {
            nljGatherKernel<<<nljGrid(ctx, (uint64_t) nS), 256, 0, ctx->compute>>>(S.lo, S.hi, S.n, pair[w], part[w], ids, nS, skey + (size_t) w * nS);
         });
   run.ids = ids;

   // 3. the searches
   const bool residuals = pl.nRes > 0;
   const bool direct = !pl.sLeft && !residuals; // pairs fall at offs[l] + their place in the range
   int32_t* flag = (int32_t*) (ctr + 2 + 2 * kNljMaxKeyWords);
   LDB_CUDA(cudaMemsetAsync(flag, 0, 4, ctx->compute));
   uint32_t* desc = nullptr;
   if (pairs && direct && nS > 1) {
      desc = run.sortOnly.alloc<uint32_t>((size_t) nS * 4);
      tileScan(ctx, tmp, NljDescentOp{ids, desc}, nS, "nljoin_search");
   }
   NljSearchParams sp{};
   sp.skey = skey;
   sp.nS = nS;
   sp.nw = nw;
   sp.nEqWords = nEqWords;
   const int64_t maxSamp = std::min<int64_t>(kNljSamples, kNljSampleWords / std::max(nw, 1));
   sp.stride = std::max<int64_t>(1, (nS + maxSamp - 1) / maxSamp);
   sp.nSamp = (int32_t) ((nS + sp.stride - 1) / sp.stride);
   sp.nBound = pl.nBound;
   sp.lo = P.lo;
   sp.hi = P.hi;
   sp.ok = P.ok;
   sp.nP = P.n;
   for (int w = 0; w < nw; w++) sp.wordPair[w] = pair[w], sp.wordPart[w] = part[w];
   for (int b = 0; b < pl.nBound; b++) {
      const uint32_t m = pl.boundMask[b]; // K m v: 1 <, 3 <=, 4 >, 6 >=
      sp.boundPair[b] = pl.boundPair[b];
      sp.boundKind[b] = m == 1 ? 2 : m == 3 ? 3 : m == 4 ? 1 : 0;
   }
   run.rlo = sp.rlo = run.keep.alloc<uint32_t>(std::max<size_t>((size_t) P.n * 4, 16));
   run.rlen = sp.rlen = run.keep.alloc<uint32_t>(std::max<size_t>((size_t) P.n * 4, 16));
   run.counts = run.keep.alloc<uint32_t>(std::max<size_t>((size_t) nL * 4, 16));
   if (markRight) {
      run.rightMark = run.keep.alloc<uint8_t>(std::max<size_t>((size_t) nR, 16));
      LDB_CUDA(cudaMemsetAsync(run.rightMark, 0, (size_t) nR, ctx->compute));
   }
   if (!residuals && !pl.sLeft) sp.cnt = run.counts;
   if (!residuals && pl.sLeft && markRight) sp.mark = run.rightMark;
   sp.desc = desc;
   sp.descents = flag;
   ctx->launch("nljoin_search", [&] { nljSearchKernel<<<nljGrid(ctx, (uint64_t) P.n), 256, 0, ctx->compute>>>(sp); });

   // 4. the candidates: read on the host when pairs are written or residuals checked
   if (pairs || residuals) {
      run.candOffs = run.keep.alloc<unsigned long long>((size_t) P.n * 8);
      tileScan(ctx, tmp, NljCandOp{sp.rlen, run.candOffs, ctr + 1, P.n}, P.n, "nljoin_search");
      LDB_CUDA(cudaMemcpyAsync(host, ctr + 1, 8, cudaMemcpyDeviceToHost, ctx->compute));
      LDB_CUDA(cudaMemcpyAsync(host + 1, flag, 4, cudaMemcpyDeviceToHost, ctx->compute));
      ctx->syncStream(ctx->compute);
      run.nCand = host[0];
      run.descents = *(int32_t*) (host + 1);
      // past n m / kNljCandidateRatio candidates the loop is as fast; without residuals a result that cannot fit stays here, so the
      // capacity check refuses it after this O(n log m) count rather than after the loop's
      size_t freeB = 0, totalB = 0;
      LDB_CUDA(cudaMemGetInfo(&freeB, &totalB));
      const bool refused = !residuals && (double) run.nCand * run.resultRowBytes > (double) freeB;
      const bool orderFits = (double) run.nCand * 24 + (double) run.nCand * run.resultRowBytes <= (double) freeB;
      if (!refused && ((double) run.nCand * kNljCandidateRatio > (double) nL * (double) nR || (pairs && !orderFits))) return false;
   }

   // 5. counts and markers
   if (residuals) {
      LDB_CUDA(cudaMemsetAsync(run.counts, 0, (size_t) nL * 4, ctx->compute));
      if (run.nCand > 0) {
         NljExpandParams e{};
         e.candOffs = run.candOffs;
         e.rlo = run.rlo;
         e.ids = ids;
         e.nP = P.n;
         e.nCand = run.nCand;
         e.leftIsProbe = !pl.sLeft;
         e.nRes = pl.nRes;
         e.lLo = run.left.lo, e.lHi = run.left.hi, e.rLo = run.right.lo, e.rHi = run.right.hi;
         e.nL = nL, e.nR = nR;
         for (int c = 0; c < pl.nRes; c++) e.resPair[c] = pl.resPair[c], e.resMask[c] = pl.resMask[c];
         e.cnt = run.counts;
         e.mark = run.rightMark;
         const unsigned grid = nljGrid(ctx, run.nCand);
         ctx->launch("nljoin_expand", [&] {
            if (run.wide) nljExpandKernel<true, false><<<grid, 256, 0, ctx->compute>>>(e);
            else nljExpandKernel<false, false><<<grid, 256, 0, ctx->compute>>>(e);
         });
      }
   } else if (pl.sLeft || markRight) {
      // S is the left side: the coverage is each left row's count; S is the right side: it marks the right rows
      if (pl.sLeft) LDB_CUDA(cudaMemsetAsync(run.counts, 0, (size_t) nL * 4, ctx->compute));
      if (nS > 0) {
         uint32_t* diff = run.sortOnly.alloc<uint32_t>((size_t) (nS + 1) * 4);
         LDB_CUDA(cudaMemsetAsync(diff, 0, (size_t) (nS + 1) * 4, ctx->compute));
         ctx->launch("nljoin_cover", [&] { nljCoverKernel<<<nljGrid(ctx, (uint64_t) P.n), 256, 0, ctx->compute>>>(run.rlo, run.rlen, P.n, diff); });
         tileScan(ctx, tmp, NljCoverOp{diff, ids, pl.sLeft ? run.counts : nullptr, pl.sLeft ? nullptr : run.rightMark}, nS, "nljoin_cover");
      }
   }
   return true;
}

void nljSortedWrite(LdbContext* ctx, Scratch& tmp, NljSortedRun& run, const unsigned long long* offs, uint32_t* outL, uint32_t* outR) {
   if (run.nCand == 0) return;
   const NljSortedPlan& pl = run.plan;
   const int64_t nL = run.left.n;
   NljExpandParams e{};
   e.candOffs = run.candOffs;
   e.rlo = run.rlo;
   e.ids = run.ids;
   e.nP = pl.sLeft ? run.right.n : nL;
   e.nCand = run.nCand;
   e.leftIsProbe = !pl.sLeft;
   e.nRes = pl.nRes;
   e.lLo = run.left.lo, e.lHi = run.left.hi, e.rLo = run.right.lo, e.rHi = run.right.hi;
   e.nL = nL, e.nR = run.right.n;
   for (int c = 0; c < pl.nRes; c++) e.resPair[c] = pl.resPair[c], e.resMask[c] = pl.resMask[c];
   e.offs = offs;
   if (pl.sLeft || pl.nRes) { // places taken in any order, then sorted
      e.cursor = tmp.alloc<unsigned long long>((size_t) nL * 8);
      LDB_CUDA(cudaMemcpyAsync(e.cursor, offs, (size_t) nL * 8, cudaMemcpyDeviceToDevice, ctx->compute));
   }
   e.outL = outL;
   e.outR = outR;
   const unsigned grid = nljGrid(ctx, run.nCand);
   ctx->launch("nljoin_expand", [&] {
      if (run.wide) nljExpandKernel<true, true><<<grid, 256, 0, ctx->compute>>>(e);
      else nljExpandKernel<false, true><<<grid, 256, 0, ctx->compute>>>(e);
   });
}

void nljSortedOrder(LdbContext* ctx, Scratch& tmp, NljSortedRun& run, int64_t nOrdered, uint32_t* outL, uint32_t* outR) {
   const NljSortedPlan& pl = run.plan;
   // in order already: every pair sits at its left row's offset plus its place in a range of ascending right ids
   if (nOrdered < 2 || (!pl.sLeft && !pl.nRes && !run.descents)) return;
   const int bitsR = nljBits((unsigned long long) run.right.n);
   const int digits = (nljBits((unsigned long long) (run.left.n - 1)) + bitsR + 7) / 8;
   unsigned long long* keys = tmp.alloc<unsigned long long>((size_t) nOrdered * 8);
   unsigned long long* keysTmp = tmp.alloc<unsigned long long>((size_t) nOrdered * 8);
   const int64_t ctas = (nOrdered + 256 * 16 - 1) / (256 * 16);
   unsigned int* hist = tmp.alloc<unsigned int>((size_t) ctas * 256 * 4);
   ctx->launch("nljoin_order", [&] {
      nljOrderKeysKernel<<<nljGrid(ctx, (uint64_t) nOrdered), 256, 0, ctx->compute>>>(outL, outR, nOrdered, bitsR, keys);
      // the ids ride along as the sort's values and are rewritten from the keys afterwards
      launchRadixSortPairs(keys, outL, keysTmp, outR, nOrdered, hist, ctx->smCount, ctx->compute, digits);
      nljOrderSplitKernel<<<nljGrid(ctx, (uint64_t) nOrdered), 256, 0, ctx->compute>>>(digits & 1 ? keysTmp : keys, nOrdered, bitsR, outL, outR);
   });
}

} // namespace ldb

static_assert(sizeof(ldb::NljSearchParams) <= 4096, "the sorted nested-loop join's search parameters");
static_assert(sizeof(ldb::NljExpandParams) <= 4096, "the sorted nested-loop join's walk parameters");
