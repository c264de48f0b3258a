// nljoin.cuh — what the nested-loop join's two paths share: the loop (nljoin.cu) and the sorted ranges (nljoin_sorted.cu).
#pragma once
#include "context.h"

#include <algorithm>

namespace ldb {

constexpr int kNljMaxConds = 8, kNljMaxPairs = 4, kNljMaxCols = 16;
constexpr uint32_t kNljNone = 0xffffffffu; // permuteRows' id of a row of NULL cells
// The choice between the paths (DESIGN §7, "Sorted ranges"): below kNljSortMinPairs pairs the loop finishes before the sorted path's
// launches and host reads do; past n m / kNljCandidateRatio candidates the loop's count and ordered write cost no more than the walk.
constexpr double kNljSortMinPairs = 16777216.0; // 2^24
constexpr double kNljCandidateRatio = 256.0;

inline unsigned nljGrid(const LdbContext* ctx, uint64_t items) {
   return (unsigned) std::max<uint64_t>(1, std::min<uint64_t>((items + 255) / 256, (uint64_t) ctx->smCount * 16));
}

// one side's words (nljWordsKernel): per column-to-column condition c, lo[c n + row] (and hi[c n + row] when wide) is the row's
// order-preserving operand; ok[row] = 1 when the row can match at all
struct NljWordsRef {
   const int64_t* lo;
   const int64_t* hi;
   const uint8_t* ok;
   int64_t n;
};

// Buffers from the context's pool, like Scratch's, that can also be given back to the device itself: the sorted path's buffers, freed
// before a fallback to the loop and before a capacity check that would otherwise refuse, so that neither sees less free memory than
// the loop alone would leave
class NljScratch {
   LdbContext* ctx;
   std::vector<void*> bufs;
   const int uncaught = std::uncaught_exceptions();

   public:
   explicit NljScratch(LdbContext* c) : ctx(c) {}
   NljScratch(const NljScratch&) = delete;
   NljScratch& operator=(const NljScratch&) = delete;
   ~NljScratch() {
      if (bufs.empty()) return;
      if (std::uncaught_exceptions() > uncaught) {
         cudaStreamSynchronize(ctx->compute);
         cudaGetLastError();
      }
      for (void* p : bufs) ctx->stagingRelease(p);
   }
   template <class T>
   T* alloc(size_t bytes) {
      bufs.reserve(bufs.size() + 1);
      void* p = ctx->stagingAlloc(bytes);
      bufs.push_back(p);
      return (T*) p;
   }
   bool empty() const { return bufs.empty(); }
   // once the compute stream is done with them, the buffers go back to the device (cudaFree), not to the pool
   void toDevice() {
      if (bufs.empty()) return;
      ctx->syncStream(ctx->compute);
      for (void* p : bufs) {
         ctx->stagingSize.erase(p);
         LDB_CUDA(cudaFree(p));
      }
      bufs.clear();
   }
};

// the sorted-ranges path (nljoin_sorted.cu): the side S it sorts, its range column K and what each condition becomes
struct NljSortedPlan {
   bool sLeft = false;                 // S is the left side (else the right side)
   bool hasK = false;                  // some range condition bounds K
   int nEq = 0, eqPair[kNljMaxPairs]{}; // equality conditions: the sort key's prefix, in condition order
   int kPair = -1;                     // a condition whose S operand is K (its S words are K's words)
   int nBound = 0, boundPair[kNljMaxPairs]{};
   uint32_t boundMask[kNljMaxPairs]{}; // {lt, eq, gt} of K against the probe's operand
   int nRes = 0, resPair[kNljMaxPairs]{};
   uint32_t resMask[kNljMaxPairs]{};   // {lt, eq, gt} of left against right, as the loop reads it
};
// the plan for these column-to-column conditions (masks: the loop's, of left against right; lCols / rCols: the operands' column
// indices), or false when no condition can key a sort (only <>, or none)
bool nljSortedPlan(int nc, const uint32_t* masks, const int* lCols, const int* rCols, int64_t nL, int64_t nR, NljSortedPlan* plan);

struct NljSortedRun {
   explicit NljSortedRun(LdbContext* ctx) : keep(ctx), sortOnly(ctx) {}
   // in
   NljSortedPlan plan;
   NljWordsRef left, right;
   bool wide = false;
   int kind = 0;
   double resultRowBytes = 0; // bytes per result row (the capacity check's)
   // the count: counts[l] = left row l's matches, rightMark[r] = 1 when right row r matched (null: not asked)
   uint32_t* counts = nullptr;
   uint8_t* rightMark = nullptr;
   // kept for the write
   uint32_t *ids = nullptr, *rlo = nullptr, *rlen = nullptr;
   unsigned long long* candOffs = nullptr;
   unsigned long long nCand = 0;
   int descents = 0; // some probe row's range holds a descent of S's sorted row ids
   NljScratch keep;     // what the write reads: sorted ids (two buffers, 8 B per S row), ranges and candidate offsets (16 B per P row),
                        // counts (4 B per left row) and markers (1 B per right row)
   NljScratch sortOnly; // the sort's and the searches' buffers: keys and sorted key words (16 B + 8 B per key word per S row),
                        // histograms, descents and coverage
};
// sorts S, searches every probe row's range and fills counts / rightMark; false: the candidates are too many for this path (the
// loop runs instead, over the same words)
bool nljSortedCount(LdbContext* ctx, Scratch& tmp, NljSortedRun& run);
// writes the matching pairs at offs (the scan of counts) and, once nljFillKernel has written the NULL-extended left rows, puts the
// first nOrdered rows in (left id, right id) order
void nljSortedWrite(LdbContext* ctx, Scratch& tmp, NljSortedRun& run, const unsigned long long* offs, uint32_t* outL, uint32_t* outR);
void nljSortedOrder(LdbContext* ctx, Scratch& tmp, NljSortedRun& run, int64_t nOrdered, uint32_t* outL, uint32_t* outR);

} // namespace ldb
