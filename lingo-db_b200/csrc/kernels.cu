// kernels.cu — hand-written sm_90a pipeline kernels for LingoDB's three hot paths.
//
// Design (DESIGN.md §3): every pipeline is ONE persistent, HBM-bound streaming kernel:
//   grid = SMs × resident CTAs; each CTA strides over tiles of 256 or 512 rows of every distinct fixed-width column the
//   pipeline reads, brought to shared memory by TMA bulk copies (2 stages, L2 evict_first), so each column byte crosses
//   HBM→SM once.  decimal(p<19) is computed from the low 8 bytes of its 16-byte cell — the reference truncates to i64 the
//   same way, LowerToStd.cpp:111-209.  No tensor cores: the path is integer/hash work.  Aggregates are exact wrapping
//   i64/i128 like the JIT's LLVM code.  Rows that survive a selective probe are either handled in place (warp-specialised
//   driver: K4, K5, K8) or copied to a CTA-wide survivor queue and handled by full warps (K3 with a probe, K9).
//   K1/K2  scanGroupByKernel          scan → filters → (group-by | keyless) SUMs                       Q6, Q1
//   K3     scanBuild[Pair]Kernel      scan → filters → [probe] → join-table insert (hash | composite key | direct address)
//   K4     scanProbe2GroupByKernel    scan → probe A → probe B → tiny group-by                         Q5
//   K5     scanProbeAggKernel         scan → filters → probe group-join map → atomic i128 SUM          Q3
//   K6     partition*Kernel           radix partition by h64(key) for the NVLink all-to-all
//   K7     groupMerge*Kernel          fold other GPUs' group-table images into the local table
//   K8     scanMaterializeKernel      scan → filters → [probe | Bloom-only] → compacted columns (repartition input)
//   K9     scanStarProbeGroupByKernel scan → composite-key probe → two foreign-key probes → 2-key group-by   Q9
#include "device_utils.cuh"
#include "kernels.h"
#include "../../include/ldb_gpu.h"

#include <map>
#include <mutex>
#include <string>
#include <type_traits>

namespace ldb {

constexpr int kBlock = kBlockThreads;

// =================================================================================== tiles
// A tile = kTileRows consecutive rows of every staged column.  Full tiles arrive in shared memory
// through TMA bulk copies (one elected thread issues `n` cp.async.bulk per tile; completion is
// counted in bytes on an mbarrier; 2 stages so the copy of tile t+2 overlaps the arithmetic on
// tile t+1).  The last partial tile — and tables whose column bases are not 16-byte aligned —
// are read with plain coalesced loads through the same accessor interface.
// DB = bytes per decimal128 cell as staged: 16 (Arrow layout) or 8 (narrowed HOST batch) — a compile-time constant so the
// issue-bound group-by kernel keeps immediate strides (a run-time stride made Q1 measurably slower)
template <int DB>
struct SmemTile {
   uint32_t stage; // shared-space address of the stage
   const StagedCols* sc;
   __device__ __forceinline__ int32_t i32(int col, int lr) const { return ldShared32(stage + sc->smemOffset[col] + lr * 4); }
   __device__ __forceinline__ int64_t lo64(int col, int lr) const { return ldShared64(stage + sc->smemOffset[col] + lr * DB); }
   __device__ __forceinline__ int64_t hi64(int col, int lr) const {
      if constexpr (DB == 16) return ldShared64(stage + sc->smemOffset[col] + lr * 16 + 8);
      else return lo64(col, lr) >> 63;
   }
};
template <int DB>
struct GlobalTile {
   int64_t rowBase;
   const StagedCols* sc;
   __device__ __forceinline__ int32_t i32(int col, int lr) const { return ldStream32((const int32_t*) sc->base[col] + rowBase + lr); }
   __device__ __forceinline__ int64_t lo64(int col, int lr) const { return ldStream64((const int64_t*) (sc->base[col] + (size_t) (rowBase + lr) * DB)); }
   __device__ __forceinline__ int64_t hi64(int col, int lr) const {
      if constexpr (DB == 16) return ldStream64((const int64_t*) (sc->base[col] + (size_t) (rowBase + lr) * 16 + 8));
      else return lo64(col, lr) >> 63;
   }
};
// Encoded layout (kernels.h kEncodeTileHeader): a column tile is {base of its block, max - base} followed by the tile's values packed in W
// bytes each.  A value is base + the zero-extended field; width and base are uniform per column and tile, so the decode is a
// shared load of the 32-bit word holding the field, a shift, a mask and an add.  Values come back exactly, so filters, group ids
// and aggregates run unchanged on them.
template <>
struct SmemTile<kDecEncoded> {
   uint32_t stage;
   const StagedCols* sc;
   // the W-byte field of row lr (W <= 4): a field never straddles an aligned 32-bit word
   __device__ __forceinline__ uint32_t field32(int col, int lr) const {
      const uint32_t a = stage + (uint32_t) sc->smemOffset[col] + kEncodeTileHeader + ((uint32_t) lr << sc->encShift[col]);
      return ((uint32_t) ldShared32(a & ~3u) >> ((a & 3u) * 8)) & sc->encMask[col];
   }
   __device__ __forceinline__ int32_t i32(int col, int lr) const { // int32 columns are encoded in at most 4 bytes
      return (int32_t) ((uint32_t) ldShared32(stage + sc->smemOffset[col]) + field32(col, lr));
   }
   // the zero-extended field of row lr, any W
   __device__ __forceinline__ uint64_t field(int col, int lr) const {
      if (sc->encShift[col] == 3) return (uint64_t) ldShared64(stage + (uint32_t) sc->smemOffset[col] + kEncodeTileHeader + (uint32_t) lr * 8);
      return field32(col, lr);
   }
   __device__ __forceinline__ int64_t lo64(int col, int lr) const { return (int64_t) ((uint64_t) ldShared64(stage + (uint32_t) sc->smemOffset[col]) + field(col, lr)); }
   __device__ __forceinline__ int64_t hi64(int col, int lr) const { return lo64(col, lr) >> 63; }
};
template <>
struct GlobalTile<kDecEncoded> {
   int64_t rowBase; // first row of a tile
   const StagedCols* sc;
   __device__ __forceinline__ const uint8_t* tileStart(int col) const {
      return sc->base[col] + (rowBase / sc->tileRows) * ((int64_t) kEncodeTileHeader + (int64_t) sc->tileRows * sc->elemBytes[col]);
   }
   __device__ __forceinline__ uint64_t field(int col, int lr) const {
      const uint8_t* p = tileStart(col) + kEncodeTileHeader;
      switch (sc->elemBytes[col]) {
         case 1: return __ldg(p + lr);
         case 2: return __ldg((const uint16_t*) p + lr);
         case 4: return __ldg((const uint32_t*) p + lr);
         default: return __ldg((const unsigned long long*) p + lr);
      }
   }
   __device__ __forceinline__ uint64_t base(int col) const { return (uint64_t) __ldg((const long long*) tileStart(col)); }
   __device__ __forceinline__ int32_t i32(int col, int lr) const { return (int32_t) (uint32_t) (base(col) + field(col, lr)); }
   __device__ __forceinline__ int64_t lo64(int col, int lr) const { return (int64_t) (base(col) + field(col, lr)); }
   __device__ __forceinline__ int64_t hi64(int col, int lr) const { return lo64(col, lr) >> 63; }
};
// A stage holds F consecutive tiles (stage `stage` = tiles stage * F ..): the F tiles of a column are contiguous in HBM and in shared
// memory (column c from F * smemOffset[c]), so each column still takes one bulk copy.
template <int F = 1>
__device__ __forceinline__ void issueTile(const StagedCols& sc, uint8_t* smem, uint64_t* bars /* full[] */, int64_t stage, int s) {
   const uint64_t policy = evictFirstPolicy();
   mbarExpectTx(&bars[s], (uint32_t) (F * sc.stageBytes));
   const uint32_t dst = smemAddr(smem) + (uint32_t) (s * F * sc.stageBytes);
   for (int c = 0; c < sc.n; c++) {
      const uint32_t bytes = F * ((uint32_t) sc.elemBytes[c] * (uint32_t) sc.tileRows + (uint32_t) sc.tileHeader);
      bulkLoad(dst + F * sc.smemOffset[c], sc.base[c] + (size_t) stage * bytes, bytes, &bars[s], policy);
   }
}
// fnTile(tile, rowBase, rowsInTile) is called once per tile by every CONSUMER thread (threadIdx.x < kBlock), warps converged.
// Warp-specialised: the CTA has kBlock consumer threads plus one producer warp (kThreads = kBlock + 32).  The producer's
// lane 0 refills a stage as soon as all consumer warps released it (`empty` mbarrier, one arrive per warp), so a warp
// that finished its rows moves on to the next stage instead of idling at a CTA-wide barrier behind the slowest warp
// (with __syncthreads() about half of the probe kernel's stall samples were `stall_barrier`).
constexpr int kWarps = kBlock / 32;
constexpr int kThreads = kBlock + 32;
struct TileBarriers {
   uint64_t full[kMaxStages];
   uint64_t empty[kMaxStages];
};
template <int kRowsPerThread, int DB, int kStages = ldb::kStages, class Fn>
__device__ __forceinline__ void forEachTile(const StagedCols& sc, int64_t n, uint8_t* smem, TileBarriers* bars, const Fn& fnTile) {
   constexpr int kTileRows = kRowsPerThread * kBlock; // == sc.tileRows (host binds the same constant)
   const int64_t nFull = n / kTileRows;
   const bool producer = threadIdx.x >= kBlock;
   if (sc.useTma) {
      if (threadIdx.x == 0) {
         for (int s = 0; s < kStages; s++) {
            mbarInit(&bars->full[s], 1);
            mbarInit(&bars->empty[s], kWarps);
         }
         mbarInitFence();
      }
      __syncthreads();
      if (producer) {
         if (threadIdx.x == kBlock) {
            int it = 0;
            for (int64_t t = blockIdx.x; t < nFull; t += gridDim.x, it++) {
               const int s = it % kStages;
               if (it >= kStages) mbarWaitPaused(&bars->empty[s], (uint32_t) (it / kStages - 1) & 1u, (uint32_t) sc.producerSleepNs);
               issueTile(sc, smem, bars->full, t, s);
            }
         }
      } else {
         int it = 0;
         for (int64_t t = blockIdx.x; t < nFull; t += gridDim.x, it++) {
            const int s = it % kStages;
            if (sc.consumerSleepNs) mbarWaitPaused(&bars->full[s], (uint32_t) (it / kStages) & 1u, (uint32_t) sc.consumerSleepNs);
            else mbarWait(&bars->full[s], (uint32_t) (it / kStages) & 1u);
            SmemTile<DB> tile{smemAddr(smem) + (uint32_t) s * sc.stageBytes, &sc};
            fnTile(tile, t * kTileRows, kTileRows);
            __syncwarp();
            if ((threadIdx.x & 31) == 0) mbarArrive(&bars->empty[s]); // this warp is done with stage s
         }
      }
   } else if (!producer) {
      for (int64_t t = blockIdx.x; t < nFull; t += gridDim.x) {
         __syncwarp();
         GlobalTile<DB> tile{t * kTileRows, &sc};
         fnTile(tile, t * kTileRows, kTileRows);
      }
   }
   // the partial tail tile goes to the CTA that would have been next in the round robin
   if (!producer && nFull * kTileRows < n && (int64_t) blockIdx.x == nFull % gridDim.x) {
      __syncwarp();
      GlobalTile<DB> tile{nFull * kTileRows, &sc};
      fnTile(tile, nFull * kTileRows, (int) (n - nFull * kTileRows));
   }
}
// Non-specialised variant for the arithmetic-bound group-by kernel (K1/K2): every row costs the same, so the CTA-wide
// barrier is cheap (stall_barrier 0.1 per issue) and a 9th warp would only cost registers (2 CTAs x 288 threads
// cap the kernel at 112 registers → spills).  One elected thread issues the copies, __syncthreads() recycles a stage.
// With F > 1 a TMA stage is F tiles (fnTile gets F * kTileRows rows); the full tiles after the last full stage and the partial
// tail tile are read tile by tile through GlobalTile, one CTA each, continuing the round robin of the stages.
template <int kRowsPerThread, int DB, int kStages = ldb::kStages, int F = 1, class Fn>
__device__ __forceinline__ void forEachTileUniform(const StagedCols& sc, int64_t n, uint8_t* smem, TileBarriers* bars, const Fn& fnTile) {
   constexpr int kTileRows = kRowsPerThread * kBlock;
   const int64_t nFull = n / kTileRows;
   int64_t done = nFull, turns = nFull; // tiles read by the loops below, and the round-robin turns they took
   if (sc.useTma) {
      const int64_t nStages = nFull / F;
      done = nStages * F;
      turns = nStages;
      if (threadIdx.x == 0) {
         for (int s = 0; s < kStages; s++) mbarInit(&bars->full[s], 1);
         mbarInitFence();
      }
      __syncthreads();
      if (threadIdx.x == 0) {
         for (int s = 0; s < kStages; s++) {
            int64_t t = (int64_t) blockIdx.x + (int64_t) s * gridDim.x;
            if (t < nStages) issueTile<F>(sc, smem, bars->full, t, s);
         }
      }
      int it = 0;
      for (int64_t t = blockIdx.x; t < nStages; t += gridDim.x, it++) {
         const int s = it % kStages;
         mbarWait(&bars->full[s], (uint32_t) (it / kStages) & 1u);
         SmemTile<DB> tile{smemAddr(smem) + (uint32_t) (s * F * sc.stageBytes), &sc};
         fnTile(tile, t * F * kTileRows, F * kTileRows);
         __syncthreads(); // every thread is done with stage s → refill it
         const int64_t nt = t + (int64_t) kStages * gridDim.x;
         if (threadIdx.x == 0 && nt < nStages) issueTile<F>(sc, smem, bars->full, nt, s);
      }
   } else {
      for (int64_t t = blockIdx.x; t < nFull; t += gridDim.x) {
         GlobalTile<DB> tile{t * kTileRows, &sc};
         fnTile(tile, t * kTileRows, kTileRows);
         __syncthreads(); // same contract as the TMA path: no thread starts the next tile before all finished this one
      }
   }
   const int64_t nTiles = (n + kTileRows - 1) / kTileRows;
   for (int64_t t = done + ((int64_t) blockIdx.x + gridDim.x - turns % gridDim.x) % gridDim.x; t < nTiles; t += gridDim.x) {
      __syncthreads();
      GlobalTile<DB> tile{t * kTileRows, &sc};
      fnTile(tile, t * kTileRows, (int) min(n - t * kTileRows, (int64_t) kTileRows));
   }
}
template <int kRowsPerThread, int DB, class Fn>
__device__ __forceinline__ void forEachRowUniform(const StagedCols& sc, int64_t n, uint8_t* smem, TileBarriers* bars, const Fn& fn) {
   forEachTileUniform<kRowsPerThread, DB>(sc, n, smem, bars, [&](const auto& tile, int64_t rowBase, int rows) {
#pragma unroll
      for (int j = 0; j < kRowsPerThread; j++) {
         const int lr = j * kBlock + threadIdx.x;
         const bool valid = lr < rows;
         fn(tile, valid ? lr : 0, rowBase + (valid ? lr : 0), valid);
      }
   });
}
// fn(tile, localRow, globalRow, valid) is called for every row with all 32 lanes of a warp converged
// (lanes beyond the end of the table come with valid == false), so fn may use warp collectives.
template <int kRowsPerThread, int DB, class Fn>
__device__ __forceinline__ void forEachRow(const StagedCols& sc, int64_t n, uint8_t* smem, TileBarriers* bars, const Fn& fn) {
   forEachTile<kRowsPerThread, DB>(sc, n, smem, bars, [&](const auto& tile, int64_t rowBase, int rows) {
#pragma unroll
      for (int j = 0; j < kRowsPerThread; j++) {
         const int lr = j * kBlock + threadIdx.x;
         const bool valid = lr < rows;
         fn(tile, valid ? lr : 0, rowBase + (valid ? lr : 0), valid);
      }
   });
}

// late-materialised operand: low 8 bytes of the cell of `row` (decimal(p<19) computes from them, LowerToStd.cpp:111-209)
__device__ __forceinline__ int64_t lazyLo64(const LazyCols& lc, int c, int64_t row) { return ldStream64((const int64_t*) (lc.base[c] + (size_t) row * lc.elemBytes[c])); }

// =================================================================================== filters
// Conjunction of column-vs-constant predicates (Restrictions::applyFilters, Restrictions.cpp:365-390):
// instead of one compaction pass per filter over a uint16 selection vector, every predicate is
// evaluated in registers on the staged tile and the row is simply skipped.
// IN list: linear search like the reference does for <= 10 values (Restrictions.cpp:207-218)
__device__ __noinline__ bool inListContains(const FilterCol& f, int64_t v) {
   bool any = false;
   for (int k = 0; k < f.nIn; k++) any |= v == f.inVals[k];
   return any;
}
// `x like '%needle%'` (ConstLike → StringRuntime::findMatch, RuntimeFunctions.cpp:60-170, StringRuntime.cpp:337-345): the
// reference evaluates it in the JIT'd selection above the scan; here it is one more predicate of the scan itself.
__device__ __noinline__ bool utf8Contains(const FilterCol& f, int64_t row) {
   const int32_t* off = (const int32_t*) f.base + row;
   const int32_t b = __ldg(off), e = __ldg(off + 1), n = f.strLen;
   if (e - b < n) return false;
   if (n == 0) return true;
   const uint8_t* str = f.bytes + b;
   const uint8_t first = f.str[0];
   for (int i = 0, last = e - b - n; i <= last; i++) {
      if (__ldg(str + i) != first) continue;
      int k = 1;
      while (k < n && __ldg(str + i + k) == f.str[k]) k++;
      if (k == n) return true;
   }
   return false;
}
// Filter SHAPES the join pipelines are instantiated for besides the descriptor-driven form.  The generic loop spends ≈40 issue
// slots per row on interpreting the descriptor (count, kind, IN, two 64-bit three-way compares per column;
// K3/K5 were issue-bound, not DRAM-bound), the reference's JIT emits ONE compare for the same predicate
// (SimpleTypeFilter<T, CMP>, Restrictions.cpp:163-193).  The host picks the shape (filterShape below); everything else stays generic.
enum FilterShape : int {
   FS_GENERIC = -1,
   FS_NONE = 0,      // no pushed-down filter
   FS_I32_ONE = 1,   // one int32/date32/char(1) column against one constant
   FS_I32_RANGE = 2, // one int32/date32 column against two constants (lower and upper bound)
};
__device__ __forceinline__ bool cmpMask32(int32_t a, int32_t b, uint32_t mask) {
   const uint32_t rel = a < b ? 1u : (a == b ? 2u : 4u);
   return (rel & mask) != 0;
}
// IN = the pipeline has at least one rare filter — IN list or LIKE-contains (host decides); pipelines without one carry no trace of it
template <bool IN, int FS = FS_GENERIC, class Tile>
__device__ __forceinline__ bool evalFilters(const FilterSet& F, const Tile& tile, int lr, int64_t row) {
   if constexpr (FS == FS_NONE) return true;
   if constexpr (FS == FS_I32_ONE || FS == FS_I32_RANGE) {
      const int32_t v = tile.i32(F.c[0].staged, lr);
      bool ok = cmpMask32(v, (int32_t) F.c[0].valA, F.c[0].maskA);
      if constexpr (FS == FS_I32_RANGE) ok &= cmpMask32(v, (int32_t) F.c[0].valB, F.c[0].maskB);
      return ok;
   }
   bool pass = true;
#pragma unroll
   for (int i = 0; i < kMaxFilterCols; i++) {
      if (i < F.n) {
         const FilterCol& f = F.c[i];
         int64_t v;
         if (f.kind == COL_I32) {
            v = tile.i32(f.staged, lr);
         } else if (f.kind == COL_DEC128_LO64) {
            v = tile.lo64(f.staged, lr);
         } else if (IN && f.kind == COL_UTF8_CONTAINS) {
            v = utf8Contains(f, row) ? 1 : 0;
         } else { // COL_UTF8_EQ: 1 if the string equals the constant (VarLen32Filter<Eq>, Restrictions.cpp:279-325)
            const int32_t* off = (const int32_t*) f.base + row;
            int32_t b = __ldg(off), e = __ldg(off + 1);
            bool eq = e - b == f.strLen;
            if (eq)
               for (int k = 0; k < f.strLen; k++) eq &= __ldg(f.bytes + b + k) == f.str[k];
            v = eq ? 1 : 0;
         }
         if (IN && f.nIn > 0) { // IN list (rare): out of line, so the hot kernels do not carry its code
            pass &= inListContains(f, v);
         } else {
            pass &= cmpMask(v, f.valA, f.maskA);
            if (f.maskB != 7u) pass &= cmpMask(v, f.valB, f.maskB);
         }
      }
   }
   return pass;
}

// host: the shape a filter set can run under (constants must survive the narrowing to int32)
static int filterShape(const FilterSet& F) {
   if (!tuning().specialise) return FS_GENERIC;
   if (F.n == 0) return FS_NONE;
   if (F.n != 1) return FS_GENERIC;
   const FilterCol& f = F.c[0];
   auto fits = [](int64_t v) { return v >= INT32_MIN && v <= INT32_MAX; };
   if (f.kind != COL_I32 || f.nIn > 0 || f.staged < 0 || !fits(f.valA)) return FS_GENERIC;
   if (f.maskB == 7u) return FS_I32_ONE;
   return fits(f.valB) ? FS_I32_RANGE : FS_GENERIC;
}

// =================================================================================== group table (HBM)
__device__ __forceinline__ uint64_t groupHash(const int32_t* k, int nKeys) {
   // db.hash over the key tuple: first key starts the hash, further keys are combined in
   // (LowerToStd.cpp:1139-1150); identical to the oracle's HashBuilder
   uint64_t h = hashI32(k[0]);
   if (nKeys > 1) h = hashCombine(hashI32(k[1]), h);
   return h;
}
// lookup-or-insert (lowering of subop.lookup_or_insert, SubOpToControlFlow.cpp:3065-3157, as open addressing)
__device__ __forceinline__ int32_t ldAcquire32(const int32_t* p) {
   int32_t v;
   asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
   return v;
}
__device__ int groupLookupOrInsert(const GroupTableDev& t, const int32_t* k) {
   if (t.nKeys == 0) return 0;
   uint32_t mask = (uint32_t) t.capacity - 1;
   uint32_t s = (uint32_t) groupHash(k, t.nKeys) & mask;
   for (int probes = 0; probes < t.capacity; probes++) {
      // fast path: the group exists (every row after the first of its group) — one acquire load, no CAS, no fence
      if (ldAcquire32(&t.state[s]) == 2) {
         if (t.keys[s * kMaxKeys] == k[0] && (t.nKeys < 2 || t.keys[s * kMaxKeys + 1] == k[1])) return (int) s;
         s = (s + 1) & mask;
         continue;
      }
      int st = atomicCAS(&t.state[s], 0, 1);
      if (st == 0) {
         t.keys[s * kMaxKeys + 0] = k[0];
         t.keys[s * kMaxKeys + 1] = t.nKeys > 1 ? k[1] : 0;
         __threadfence();
         atomicExch(&t.state[s], 2);
         return (int) s;
      }
      while (st == 1) st = *((volatile int32_t*) &t.state[s]);
      __threadfence();
      const volatile int32_t* tk = t.keys + s * kMaxKeys;
      if (tk[0] == k[0] && (t.nKeys < 2 || tk[1] == k[1])) return (int) s;
      s = (s + 1) & mask;
   }
   atomicExch(t.error, 1);
   return -1;
}
__device__ __forceinline__ void groupAtomicAdd(const GroupTableDev& t, int slot, int agg, i128 v, bool is64) {
   unsigned long long* p = t.acc + ((size_t) slot * kMaxAggs + agg) * 2;
   if (is64) atomicAdd(p, (unsigned long long) v.lo);
   else atomicAdd128(p, p + 1, v);
}

// =================================================================================== join table (HBM)
constexpr unsigned long long kEmptySlot = ~0ull;
constexpr uint64_t kMaxProbe = 16384; // insert reports "table full" beyond this displacement; the host regrows
// Blocked Bloom filter in front of the directory: the reference rejects most non-matching probes with a 16-bit
// tag in the bucket pointer (helpers.h:325-346) — but only after it loaded the bucket.  Here the filter is a
// separate array small enough to live in L2 (1 byte per directory slot), so a rejected probe never goes to HBM.
__device__ __forceinline__ unsigned long long packSlot(int32_t key, int32_t payload) { return ((unsigned long long) (uint32_t) payload << 32) | (uint32_t) key; }
// HashIndexedView::build's CAS push-front (LazyJoinHashtable.cpp:20-31) becomes a CAS into an open-addressing
// slot.  The caller counts successful inserts (one atomic per warp at kernel end, not one per tuple).
__device__ __forceinline__ unsigned long long* slotPtr(const JoinTableDev& t, uint64_t s) { return (unsigned long long*) (t.base + s * t.stride); }
__device__ int64_t joinInsert(const JoinTableDev& t, int32_t key, int32_t payload) {
   unsigned long long packed = packSlot(key, payload);
   if (packed == kEmptySlot) { // (-1,-1) is the empty marker and cannot be stored
      atomicExch(t.error, 3);
      return -1;
   }
   if (t.stride == 32 && payload < 0) { // bit 31 of the payload word is the group-join marker
      atomicExch(t.error, 4);
      return -1;
   }
   const uint64_t h = hashI32(key);
   uint64_t s = h & t.mask;
   const uint64_t limit = t.mask < kMaxProbe ? t.mask + 1 : kMaxProbe; // a sanely loaded table never probes this far
   for (uint64_t probes = 0; probes < limit; probes++) {
      unsigned long long old = atomicCAS(slotPtr(t, s), kEmptySlot, packed);
      if (old == kEmptySlot) {
         if (t.bloom) atomicOr(&t.bloom[(uint32_t) (h >> 32) & t.bloomMask], bloomBits(h));
         return (int64_t) s;
      }
      if (t.unique && (int32_t) (uint32_t) old == key) {
         atomicExch(t.error, 2);
         return -1;
      }
      s = (s + 1) & t.mask;
   }
   atomicExch(t.error, 1);
   return -1;
}
// direct-address table (dense integer keys): slot = key - keyMin holds the payload
__device__ __forceinline__ int64_t directInsert(const JoinTableDev& t, int32_t key, int32_t payload) {
   const uint32_t idx = (uint32_t) key - (uint32_t) t.keyMin;
   if (idx >= t.range) {
      atomicExch(t.error, 5);
      return -1;
   }
   if (payload == kDirectEmpty) {
      atomicExch(t.error, 3);
      return -1;
   }
   const int32_t old = atomicExch((int32_t*) t.base + idx, payload); // consecutive keys: consecutive addresses, one sector per 8 rows
   if (old != kDirectEmpty) { // primary keys are unique; a second row with the key is a plan error, not a multimap
      atomicExch(t.error, 2);
      return -1;
   }
   return (int64_t) idx;
}
__device__ __forceinline__ int32_t directLoad(const JoinTableDev& t, int32_t key) {
   const uint32_t idx = (uint32_t) key - (uint32_t) t.keyMin;
   return idx < t.range ? __ldg((const int32_t*) t.base + idx) : kDirectEmpty;
}
// probe (SubOpToControlFlow.cpp:2558-2586 + chain walk :2254-2313): visit every entry with the key.
// Split in two so a thread can put the Bloom loads of ALL its rows in flight before it consumes the first one.
// Bloom words are read through the read-only path with the default L1 policy: an experiment with L1::no_allocate for large filters
// (to protect small ones in L1) slowed every probe kernel down — the words of hot blocks do get reused.
__device__ __forceinline__ uint32_t ldBloom(const JoinTableDev& t, uint32_t idx) { return __ldg(t.bloom + idx); }
struct BloomProbe {
   uint64_t h;
   uint32_t word, bits;
   __device__ __forceinline__ bool mayContain() const { return (word & bits) == bits; }
};
__device__ __forceinline__ BloomProbe bloomPrefetch(const JoinTableDev& t, int32_t key, bool wanted) {
   BloomProbe b;
   b.h = hashI32(key);
   b.bits = t.bloom ? bloomBits(b.h) : 0u;
   b.word = (t.bloom && wanted) ? ldBloom(t, (uint32_t) (b.h >> 32) & t.bloomMask) : (wanted ? ~0u : 0u);
   if (!wanted) b.bits = 1u; // word == 0 → mayContain() false
   return b;
}
// COHERENT: the probed entries are written by the same kernel (K5 sets the marker bit in the payload word) → plain loads, not
// the read-only (ld.global.nc) path
template <bool COHERENT = false, class Fn>
__device__ __forceinline__ void joinProbeSlots(const JoinTableDev& t, int32_t key, uint64_t h, const Fn& fn) {
   uint64_t s = h & t.mask;
   const uint64_t limit = t.mask < kMaxProbe ? t.mask + 1 : kMaxProbe;
   for (uint64_t probes = 0; probes < limit; probes++) {
      unsigned long long e = COHERENT ? *((const volatile unsigned long long*) slotPtr(t, s)) : __ldg(slotPtr(t, s));
      if (e == kEmptySlot) return;
      if ((int32_t) (uint32_t) e == key) {
         fn((int64_t) s, (int32_t) (uint32_t) (e >> 32));
         if (t.unique) return;
      }
      s = (s + 1) & t.mask;
   }
}
template <class Fn>
__device__ __forceinline__ void joinProbe(const JoinTableDev& t, int32_t key, const Fn& fn) {
   const uint64_t h = hashI32(key);
   if (t.bloom) {
      const uint32_t bits = bloomBits(h);
      if ((ldBloom(t, (uint32_t) (h >> 32) & t.bloomMask) & bits) != bits) return;
   }
   uint64_t s = h & t.mask;
   const uint64_t limit = t.mask < kMaxProbe ? t.mask + 1 : kMaxProbe;
   for (uint64_t probes = 0; probes < limit; probes++) {
      unsigned long long e = __ldg(slotPtr(t, s));
      if (e == kEmptySlot) return;
      if ((int32_t) (uint32_t) e == key) {
         fn((int64_t) s, (int32_t) ((uint32_t) (e >> 32) & (t.stride == 32 ? 0x7fffffffu : 0xffffffffu))); // wide tables keep the marker in bit 31
         if (t.unique) return;
      }
      s = (s + 1) & t.mask;
   }
}

// ---- composite-key table (stride 16): {key0, key1} → int64 payload.
// NOT hashed like db.hash over the key tuple: h64 is bswap-symmetric (bswap(h64(x)) == h64(x)), so the reference's
// combine h64(k1) ^ bswap(h64(k0)) degenerates to h64(k1) ^ h64(k0) = f(k0*C ^ k1*C), and for correlated keys
// (ps_suppkey is ps_partkey plus a small multiple, modulo S) the low bits cluster: with open addressing the P probe of
// Q9 walked several slots per lookup at SF100 and thousands at SF300.  The reference's chained buckets
// only lose a constant factor there; a linear-probing table needs avalanche, so the pair is mixed as ONE 64-bit word
// (MurmurHash3's fmix64 finaliser).  Placement inside the table is an internal matter — results do not depend on it.
__device__ __forceinline__ uint64_t hashPair(int32_t k0, int32_t k1) {
   uint64_t x = ((uint64_t) (uint32_t) k1 << 32) | (uint32_t) k0;
   x ^= x >> 33;
   x *= 0xff51afd7ed558ccdull;
   x ^= x >> 33;
   x *= 0xc4ceb9fe1a85ec53ull;
   x ^= x >> 33;
   return x;
}
__device__ int64_t pairInsert(const JoinTableDev& t, int32_t k0, int32_t k1, int64_t payload) {
   const unsigned long long packed = packSlot(k0, k1);
   if (packed == kEmptySlot) {
      atomicExch(t.error, 3);
      return -1;
   }
   const uint64_t h = hashPair(k0, k1);
   uint64_t s = h & t.mask;
   const uint64_t limit = t.mask < kMaxProbe ? t.mask + 1 : kMaxProbe;
   for (uint64_t probes = 0; probes < limit; probes++) {
      unsigned long long old = atomicCAS(slotPtr(t, s), kEmptySlot, packed);
      if (old == kEmptySlot) {
         ((long long*) slotPtr(t, s))[1] = payload; // probes run in a later kernel
         if (t.bloom) atomicOr(&t.bloom[(uint32_t) (h >> 32) & t.bloomMask], bloomBits(h));
         return (int64_t) s;
      }
      if (t.unique && old == packed) {
         atomicExch(t.error, 2);
         return -1;
      }
      s = (s + 1) & t.mask;
   }
   atomicExch(t.error, 1);
   return -1;
}
__device__ __forceinline__ BloomProbe pairBloomPrefetch(const JoinTableDev& t, int32_t k0, int32_t k1, bool wanted) {
   BloomProbe b;
   b.h = hashPair(k0, k1);
   b.bits = t.bloom ? bloomBits(b.h) : 0u;
   b.word = (t.bloom && wanted) ? ldBloom(t, (uint32_t) (b.h >> 32) & t.bloomMask) : (wanted ? ~0u : 0u);
   if (!wanted) b.bits = 1u;
   return b;
}
template <class Fn>
__device__ __forceinline__ void pairProbeSlots(const JoinTableDev& t, int32_t k0, int32_t k1, uint64_t h, const Fn& fn) {
   const unsigned long long packed = packSlot(k0, k1);
   uint64_t s = h & t.mask;
   const uint64_t limit = t.mask < kMaxProbe ? t.mask + 1 : kMaxProbe;
   for (uint64_t probes = 0; probes < limit; probes++) {
      const ulonglong2 e = __ldg((const ulonglong2*) slotPtr(t, s)); // key pair + payload: one 16-byte load
      if (e.x == kEmptySlot) return;
      if (e.x == packed) {
         fn((int64_t) s, (int64_t) e.y);
         if (t.unique) return;
      }
      s = (s + 1) & t.mask;
   }
}

// Probe walks that start from an already loaded first slot (the caller issued the loads of several tables together)
template <class Fn>
__device__ __forceinline__ void joinProbeFrom(const JoinTableDev& t, int32_t key, uint64_t h, unsigned long long e, const Fn& fn) {
   uint64_t s = h & t.mask;
   const uint64_t limit = t.mask < kMaxProbe ? t.mask + 1 : kMaxProbe;
   for (uint64_t probes = 0; probes < limit; probes++) {
      if (e == kEmptySlot) return;
      if ((int32_t) (uint32_t) e == key) {
         fn((int32_t) ((uint32_t) (e >> 32) & (t.stride == 32 ? 0x7fffffffu : 0xffffffffu)));
         if (t.unique) return;
      }
      s = (s + 1) & t.mask;
      e = __ldg(slotPtr(t, s));
   }
}
template <class Fn>
__device__ __forceinline__ void pairProbeFrom(const JoinTableDev& t, int32_t k0, int32_t k1, uint64_t h, ulonglong2 e, const Fn& fn) {
   const unsigned long long packed = packSlot(k0, k1);
   uint64_t s = h & t.mask;
   const uint64_t limit = t.mask < kMaxProbe ? t.mask + 1 : kMaxProbe;
   for (uint64_t probes = 0; probes < limit; probes++) {
      if (e.x == kEmptySlot) return;
      if (e.x == packed) {
         fn((int64_t) e.y);
         if (t.unique) return;
      }
      s = (s + 1) & t.mask;
      e = __ldg((const ulonglong2*) slotPtr(t, s));
   }
}

// foreign-key side of a star probe: a hash directory (first slot pre-loaded) or a direct-address table (the payload itself)
__device__ __forceinline__ unsigned long long fkFirstSlot(const JoinTableDev& t, int32_t key, uint64_t h) {
   if (t.direct) return (unsigned long long) (uint32_t) directLoad(t, key);
   return __ldg(slotPtr(t, h & t.mask));
}
template <class Fn>
__device__ __forceinline__ void fkProbeFrom(const JoinTableDev& t, int32_t key, uint64_t h, unsigned long long e, const Fn& fn) {
   if (t.direct) {
      if ((int32_t) (uint32_t) e != kDirectEmpty) fn((int32_t) (uint32_t) e);
      return;
   }
   joinProbeFrom(t, key, h, e, fn);
}

// =================================================================================== aggregate expressions
template <int E, int A = 0, int B = 0, int C = 0>
struct Agg {
   static constexpr int expr = E, a = A, b = B, c = C;
   static constexpr bool is64 = (E == LDB_EXPR_COL || E == LDB_EXPR_ONE);
};

// typed like the db dialect types them (DBOps.cpp:98-107): `1` is 10^scale of the decimal operand.
// FAST = every lane of the warp has operands that fit int32 (TPC-H money does): 32-bit multiplies.
template <class A, bool FAST>
__device__ __forceinline__ i128 evalAgg(const int64_t* v, int64_t one) {
   if constexpr (A::expr == LDB_EXPR_COL) {
      return i128{(uint64_t) v[A::a], 0};
   } else if constexpr (A::expr == LDB_EXPR_MUL) {
      return FAST ? mul32x32((int32_t) v[A::a], (int32_t) v[A::b]) : mul64x64(v[A::a], v[A::b]);
   } else if constexpr (A::expr == LDB_EXPR_MUL_1MINUS) {
      return FAST ? mul32x32((int32_t) v[A::a], (int32_t) (one - v[A::b])) : mul64x64(v[A::a], one - v[A::b]);
   } else if constexpr (A::expr == LDB_EXPR_MUL_1MINUS_1PLUS) {
      if (FAST) return mul64x32pos((int64_t) (int32_t) v[A::a] * (int64_t) (int32_t) (one - v[A::b]), (int32_t) (one + v[A::c]));
      return mul128x64(mul64x64(v[A::a], one - v[A::b]), one + v[A::c]);
   } else {
      return i128{1, 0};
   }
}
// operands of one aggregate qualify for the 32-bit path
// OR of the operands as unsigned: zero above bit 30 ⇔ every operand is in [0, 2^31) (TPC-H money is);
// negative or wide operands simply take the general path
template <class A>
__device__ __forceinline__ uint64_t aggOperandBits(const int64_t* v, int64_t one) {
   if constexpr (A::expr == LDB_EXPR_MUL) return (uint64_t) v[A::a] | (uint64_t) v[A::b];
   else if constexpr (A::expr == LDB_EXPR_MUL_1MINUS) return (uint64_t) v[A::a] | (uint64_t) (one - v[A::b]);
   else if constexpr (A::expr == LDB_EXPR_MUL_1MINUS_1PLUS) return (uint64_t) v[A::a] | (uint64_t) (one - v[A::b]) | (uint64_t) (one + v[A::c]);
   else return 0;
}
__device__ __forceinline__ i128 evalAggDyn(const AggSpec& a, const int64_t* v, int64_t one) {
   switch (a.expr) {
      case LDB_EXPR_COL: return i128{(uint64_t) v[0], 0};
      case LDB_EXPR_MUL: return mul64x64(v[0], v[1]);
      case LDB_EXPR_MUL_1MINUS: return mul64x64(v[0], one - v[1]);
      case LDB_EXPR_MUL_1MINUS_1PLUS: return mul128x64(mul64x64(v[0], one - v[1]), one + v[2]);
      default: return i128{1, 0};
   }
}

// Per-stage 64-bit path of the encoded scan.  Value column c of a stage lies in [lo[c], hi[c]] (its block's min and max, from the
// tile header).  A product aggregate qualifies when each of its operands lies in [0, 2^31) and the largest product of the bounds is
// below 2^63 / R (R = rows a thread adds per stage): every row's product is then an exact non-negative int64, R of them still sum
// below 2^63, and maxRow grows to that bound.
template <class A, int R>
__device__ __forceinline__ bool aggBound64(const int64_t* lo, const int64_t* hi, int64_t one, uint64_t& maxRow) {
   if constexpr (A::is64) {
      return true; // a column sum or a count wraps at 64 bits on every path
   } else {
      constexpr int64_t k31 = 1ll << 31;
      const int64_t xl = lo[A::a], xh = hi[A::a];
      const int64_t yl = A::expr == LDB_EXPR_MUL ? lo[A::b] : one - hi[A::b], yh = A::expr == LDB_EXPR_MUL ? hi[A::b] : one - lo[A::b];
      bool ok = xl >= 0 && xh < k31 && yl >= 0 && yh < k31;
      uint64_t m = (uint64_t) xh * (uint64_t) yh; // < 2^62 when ok
      if constexpr (A::expr == LDB_EXPR_MUL_1MINUS_1PLUS) {
         const int64_t zl = one + lo[A::c], zh = one + hi[A::c];
         ok &= zl >= 0 && zh < k31;
         ok &= __umul64hi(m, (uint64_t) zh) == 0;
         m *= (uint64_t) zh;
      }
      ok &= m < (1ull << 63) / R;
      if (m > maxRow) maxRow = m;
      return ok;
   }
}
// the aggregate's value for one row of a tile that aggBound64 admitted
template <class A>
__device__ __forceinline__ int64_t evalAgg64(const int64_t* v, int64_t one) {
   auto u32 = [](int64_t x) { return (uint64_t) (uint32_t) x; };
   if constexpr (A::expr == LDB_EXPR_COL) return v[A::a];
   else if constexpr (A::expr == LDB_EXPR_MUL) return (int64_t) (u32(v[A::a]) * u32(v[A::b]));
   else if constexpr (A::expr == LDB_EXPR_MUL_1MINUS) return (int64_t) (u32(v[A::a]) * u32(one - v[A::b]));
   else if constexpr (A::expr == LDB_EXPR_MUL_1MINUS_1PLUS) return (int64_t) (u32(v[A::a]) * u32(one - v[A::b]) * u32(one + v[A::c]));
   else return 1;
}

// compile-time aggregate list: every index below is a constant after inlining, so v[]/acc[] live in registers
template <int... Is>
struct Seq {};
template <int N, int... Is>
struct MakeSeq : MakeSeq<N - 1, N - 1, Is...> {};
template <int... Is>
struct MakeSeq<0, Is...> {
   using type = Seq<Is...>;
};
template <class... As>
struct Aggs {
   static constexpr int N = sizeof...(As);
   using S = typename MakeSeq<N>::type;
   template <bool FAST, int... Is>
   static __device__ __forceinline__ void eval(i128* v, const int64_t* vals, int64_t one, Seq<Is...>) {
      ((v[Is] = evalAgg<As, FAST>(vals, one)), ...);
   }
   static __device__ __forceinline__ bool fits32(const int64_t* vals, int64_t one) { return ((aggOperandBits<As>(vals, one) | ...) >> 31) == 0; }
   template <int R>
   static __device__ __forceinline__ bool bound64(const int64_t* lo, const int64_t* hi, int64_t one, uint64_t& maxRow) {
      return (aggBound64<As, R>(lo, hi, one, maxRow) & ...);
   }
   template <int... Is>
   static __device__ __forceinline__ void eval64(int64_t* q, const int64_t* vals, int64_t one, Seq<Is...>) {
      ((q[Is] = evalAgg64<As>(vals, one)), ...);
   }
   // 64-bit aggregates add into acc as always, the products of the i128 ones into acc64 (folded into acc by fold64)
   template <int... Is>
   static __device__ __forceinline__ void accumulate64(i128* acc, int64_t* acc64, const int64_t* q, Seq<Is...>) {
      ((As::is64 ? (void) (acc[Is].lo += (uint64_t) q[Is]) : (void) (acc64[Is] += q[Is])), ...);
   }
   template <int... Is>
   static __device__ __forceinline__ void fold64(i128* acc, int64_t* acc64, Seq<Is...>) {
      ((As::is64 ? (void) 0 : (void) (acc[Is] = add128(acc[Is], i128{(uint64_t) acc64[Is], 0}), acc64[Is] = 0)), ...);
   }
   template <int... Is>
   static __device__ __forceinline__ void accumulate(i128* acc, const i128* v, Seq<Is...>) {
      ((As::is64 ? (void) (acc[Is].lo += v[Is].lo) : (void) (acc[Is] = add128(acc[Is], v[Is]))), ...);
   }
   template <int... Is>
   static __device__ __forceinline__ void sharedAdd(unsigned long long (*sAcc)[2], const i128* v, Seq<Is...>) {
      ((As::is64 ? (void) atomicAdd(&sAcc[Is][0], (unsigned long long) v[Is].lo) : atomicAdd128(&sAcc[Is][0], &sAcc[Is][1], v[Is])), ...);
   }
   template <int... Is>
   static __device__ __forceinline__ void globalAdd(const GroupTableDev& t, int slot, const i128* v, Seq<Is...>) {
      (groupAtomicAdd(t, slot, Is, v[Is], As::is64), ...);
   }
   template <class A, int I>
   static __device__ __forceinline__ void warpFlushOne(unsigned long long (*sAcc)[2], const i128* acc, int lane) {
      i128 s = A::is64 ? i128{warpSum64(acc[I].lo), 0} : warpSum128(acc[I]);
      if (lane == 0 && (s.lo | (uint64_t) s.hi)) {
         if (A::is64) atomicAdd(&sAcc[I][0], (unsigned long long) s.lo);
         else atomicAdd128(&sAcc[I][0], &sAcc[I][1], s);
      }
   }
   template <int... Is>
   static __device__ __forceinline__ void warpFlush(unsigned long long (*sAcc)[2], const i128* acc, int lane, Seq<Is...>) {
      (warpFlushOne<As, Is>(sAcc, acc, lane), ...);
   }
};

static int envInt(const char* name, int dflt, int lo, int hi) {
   const char* e = getenv(name);
   if (!e) return dflt;
   int v = atoi(e);
   return v < lo ? lo : (v > hi ? hi : v);
}
static Tuning& tuningStorage() {
   static Tuning t = [] {
      Tuning x;
      // chosen by sweeps at SF100.  With every operand staged (60 B/row tiles) deeper pipelines cost resident CTAs and lost; with
      // late-materialised operands the tiles are 8-16 B/row and K4 / K5 gain from a third stage; K9 is best with 2 rows per thread
      // and 2 stages
      x.stagesBuild = envInt("LDB_STAGES_BUILD", 3, 2, kMaxStages);
      x.stagesProbeAgg = envInt("LDB_STAGES_PROBE_AGG", 3, 2, kMaxStages);
      x.stagesProbe2 = envInt("LDB_STAGES_PROBE2", 3, 2, kMaxStages);
      x.stagesStar = envInt("LDB_STAGES_STAR", 2, 2, kMaxStages);
      x.rptBuild = envInt("LDB_RPT_BUILD", 2, 1, 4);
      x.rptStar = envInt("LDB_RPT_STAR", 2, 1, 4);
      x.specialise = envInt("LDB_SPECIALISE", 1, 0, 1);
      x.encodedScan = envInt("LDB_ENCODED_SCAN", 1, 0, 1);
      x.producerSleepNs = envInt("LDB_PRODUCER_SLEEP_NS", 0, 0, 2000);
      x.consumerSleepNs = envInt("LDB_CONSUMER_SLEEP_NS", 0, 0, 2000);
      if (x.rptStar == 3) x.rptStar = 2;
      if (x.rptBuild == 3) x.rptBuild = 2;
      return x;
   }();
   return t;
}
const Tuning& tuning() { return tuningStorage(); }
void setTuning(const Tuning& t) {
   Tuning x = t;
   auto clampStages = [](int v) { return v < 2 ? 2 : (v > kMaxStages ? kMaxStages : v); };
   x.stagesBuild = clampStages(x.stagesBuild);
   x.stagesProbeAgg = clampStages(x.stagesProbeAgg);
   x.stagesProbe2 = clampStages(x.stagesProbe2);
   x.stagesStar = clampStages(x.stagesStar);
   x.rptBuild = x.rptBuild >= 4 ? 4 : (x.rptBuild >= 2 ? 2 : 1);
   x.rptStar = x.rptStar >= 4 ? 4 : (x.rptStar >= 2 ? 2 : 1);
   x.specialise = x.specialise ? 1 : 0;
   x.encodedScan = x.encodedScan ? 1 : 0;
   x.producerSleepNs = x.producerSleepNs < 0 ? 0 : (x.producerSleepNs > 2000 ? 2000 : x.producerSleepNs);
   x.consumerSleepNs = x.consumerSleepNs < 0 ? 0 : (x.consumerSleepNs > 2000 ? 2000 : x.consumerSleepNs);
   tuningStorage() = x;
}

extern __shared__ __align__(128) uint8_t dynSmem[];

// =================================================================================== K1 / K2
// scan → filters → group by NK int32 keys → SUMs.  NK == 0 is the keyless form (Q6, SimpleState).
// Hot groups (the first GREG a CTA meets) accumulate in REGISTERS with predicated adds — the
// reference's 1024-slot per-worker pre-aggregation cache (PreAggregationHashtable.cpp:46-60) collapses to
// this for small domains; further groups use shared-memory atomics, and only a CTA that meets
// more than LG groups touches the HBM table per row.  One flush per CTA at the end.
// Encoded batches with the one-int32-constant filter (Q1) take their own STAGE path (encodedStages): the launcher stages value columns
// first, then the keys, then the filter's column (launchGB), so their layout is read from the parameter block at constant offsets.  A TMA
// stage holds kEncFrames consecutive 512-row tiles, which share one header per column (kernels.h), so the headers are read and the
// 64-bit proof runs once per stage; each thread takes 2 * kEncFrames rows of one tile in runs of 2 adjacent rows, whose fields come from one
// shared load per column (runs of 4 spilled under the 128-register cap); the filter and the key compares run on the raw fields (constant
// and keys rebased once per stage); and a stage whose header bounds prove every product a non-negative int64 below
// 2^63 / rows-per-thread (aggBound64) skips the per-row 32-bit vote and sums those products in 64-bit registers (acc64).  The per-stage
// cost, paid per 512 rows before, is paid per 512 * kEncFrames rows, and kEncStages - 1 stages stay in flight per CTA while it works on one.
constexpr int kEncFrames = 4, kEncStages = 3;
template <int DB, int FS>
constexpr bool encodedStages = DB == kDecEncoded && FS == FS_I32_ONE;
using C0 = Agg<LDB_EXPR_COL, 0>;
using C1 = Agg<LDB_EXPR_COL, 1>;
using C2 = Agg<LDB_EXPR_COL, 2>;
using ONE = Agg<LDB_EXPR_ONE>;
// Q1: sum(qty) sum(ep) sum(ep*(1-d)) sum(ep*(1-d)*(1+t)) sum(d) count over value columns qty, ep, d, t
using Q1Aggs = Aggs<C0, C1, Agg<LDB_EXPR_MUL_1MINUS, 1, 2>, Agg<LDB_EXPR_MUL_1MINUS_1PLUS, 1, 2, 3>, C2, ONE>;
constexpr int kQty = 0, kEp = 1, kDisc = 2, kTax = 3;
// Factored Q1 (scanQ1FactoredKernel).  Discount and tax take few values (TPC-H: 11 and 9), so per register group g
//   sum(ep*(1-d)*(1+t)) = sum over (d, t) of (1-d)(1+t) * S[g][d][t],   S[g][d][t] = sum of ep over g's rows with that (d, t),
// and likewise sum(ep*(1-d)), sum(d) = sum of d * count[g][d][t], sum(ep), sum(qty) and count: identities of the integers, so they
// hold modulo 2^64 and 2^128 too.  A row then costs three 32-bit shared atomics into its cell g*Dd*Dt + (d-min_d)*Dt + (t-min_t)
// (64-bit shared atomics are CAS loops on sm_90a) and the products run once per cell and CTA at the end.  The summed columns enter
// as offsets from their batch minimum (ep - min_ep, qty - min_qty; min * count is added back at the end, so negative values stay
// exact), in four 32-bit words per cell, with a split s of ep_off chosen per batch (factoredFold):
//   L = ep_off & (2^s - 1),   H = ep_off >> s,   Q = qty_off,   N = 1  (the count).
// A frame (a stage of 2 * kBlock * kEncFrames = 2048 rows, or one tile) adds at most 2048 rows to a cell, so K frames add at most
// n = 2048 K, and the words cannot overflow while n (2^s - 1), n (range_ep >> s), n range_qty and n stay below 2^32.  The launcher
// takes the s that allows the largest K (TPC-H: s = 12, K = 427; the worst batch factoredFits admits, ep_off < 2^28 and qty_off <
// 2^21, still gets K = 1), and every K-th frame each thread folds the cells it owns (cell mod kBlock) into 64-bit sums in registers
// and zeroes them.  A batch has fewer than 2^36 rows (factoredFits), so those sums stay below 2^64.
constexpr int kCells = 512;
constexpr int kCellWords = 4;
constexpr uint32_t kFacFrameRows = 2048;
static_assert(kEncFrames * kRowsPerThreadScan * kBlock <= (int) kFacFrameRows && kCells % kBlock == 0, "factored cell words overflow");
// the W-byte fields (W = 1 << sh <= 4) of 2 adjacent rows from shared address a (2W-byte aligned), zero-extended: one shared load
__device__ __forceinline__ void encodedFields2(uint32_t a, int sh, uint32_t (&x)[2]) {
   if (sh == 0) {
      uint16_t v;
      asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(a));
      x[0] = v & 0xffu;
      x[1] = v >> 8;
   } else if (sh == 1) {
      const uint32_t v = (uint32_t) ldShared32(a);
      x[0] = v & 0xffffu;
      x[1] = v >> 16;
   } else {
      ldShared32x2(a, x[0], x[1]);
   }
}
// the same for 4 adjacent rows from shared address a (4W-byte aligned): a u32, u64 or u128 load
__device__ __forceinline__ void encodedFields4(uint32_t a, int sh, uint32_t (&x)[4]) {
   if (sh == 0) {
      const uint32_t v = (uint32_t) ldShared32(a);
#pragma unroll
      for (int i = 0; i < 4; i++) x[i] = (v >> (8 * i)) & 0xffu;
   } else if (sh == 1) {
      uint32_t v0, v1;
      ldShared32x2(a, v0, v1);
      x[0] = v0 & 0xffffu;
      x[1] = v0 >> 16;
      x[2] = v1 & 0xffffu;
      x[3] = v1 >> 16;
   } else {
      asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(x[0]), "=r"(x[1]), "=r"(x[2]), "=r"(x[3]) : "r"(a));
   }
}
// CTA-local id of the keys of the lanes that `need` one (their register keys did not hold them; warp-collective: every lane calls it):
// the CTA's shared key list first, then at the first sight of a key one elected lane registers it under the CTA lock (with its HBM
// slot).  Keys are append-only, so ids never change.  A lane gets -1 when the CTA tracks LG groups already (its row goes straight to
// HBM); lanes without `need` keep `id`.
template <int LG>
__device__ __forceinline__ int ctaGroupLookup(const GroupTableDev& table, int32_t (*sKeys)[kMaxKeys], int32_t* sSlot, int32_t* sCount, int32_t* sLock,
                                              int32_t k0, int32_t k1, bool need, int id) {
   if (need) {
      const int cnt = *((volatile int32_t*) sCount);
      for (int g = 0; g < cnt; g++)
         if (sKeys[g][0] == k0 && sKeys[g][1] == k1) id = g;
      need = id < 0;
   }
   unsigned pending = __ballot_sync(0xffffffffu, need);
   while (pending) {
      const int leader = __ffs(pending) - 1;
      const int32_t lk0 = __shfl_sync(0xffffffffu, k0, leader), lk1 = __shfl_sync(0xffffffffu, k1, leader);
      int newId = -1;
      if ((threadIdx.x & 31) == leader) {
         while (atomicCAS(sLock, 0, 1) != 0) {}
         __threadfence_block();
         const int c2 = *((volatile int32_t*) sCount);
         for (int g = 0; g < c2; g++)
            if (((volatile int32_t*) sKeys[g])[0] == lk0 && ((volatile int32_t*) sKeys[g])[1] == lk1) newId = g;
         if (newId < 0 && c2 < LG) {
            int32_t kk[2] = {lk0, lk1};
            sSlot[c2] = groupLookupOrInsert(table, kk);
            sKeys[c2][0] = lk0;
            sKeys[c2][1] = lk1;
            __threadfence_block();
            *((volatile int32_t*) sCount) = c2 + 1;
            newId = c2;
         }
         __threadfence_block();
         atomicExch(sLock, 0);
      }
      newId = __shfl_sync(0xffffffffu, newId, leader);
      if (need && k0 == lk0 && k1 == lk1) {
         id = newId;
         need = false;
      }
      pending = __ballot_sync(0xffffffffu, need);
   }
   return id;
}
// self-timing (two words behind the table's error word): max(~start), max(end) of %globaltimer over the CTAs — the kernel's
// duration without event nodes, so that a captured query (CUDA graph) still reports its kernel time (runtime.cpp groupby_read)
__device__ __forceinline__ unsigned long long* selfTimeStart(const GroupTableDev& t) {
   unsigned long long* const selfTime = (unsigned long long*) (t.error) + 1;
   if (threadIdx.x == 0) {
      unsigned long long t0;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
      atomicMax(selfTime, ~t0);
   }
   return selfTime;
}
// the CTA's shared sums → one HBM atomic per (group, aggregate), then the end of the self-timing (after a barrier behind every sum)
template <int N>
__device__ __forceinline__ void flushCtaGroups(const GroupTableDev& t, const unsigned long long (*sAcc)[N][2], const int32_t* sSlot, int cnt,
                                               unsigned long long* selfTime) {
   for (int i = threadIdx.x; i < cnt * N; i += kBlock) {
      int g = i / N, a = i % N;
      int slot = sSlot[g];
      if (slot < 0) continue;
      i128 s{sAcc[g][a][0], (int64_t) sAcc[g][a][1]};
      if (s.lo | (uint64_t) s.hi) {
         unsigned long long* dst = t.acc + ((size_t) slot * kMaxAggs + a) * 2;
         atomicAdd128(dst, dst + 1, s); // 64-bit aggregates keep hi == 0 and are read back as i64
      }
   }
   __syncthreads();
   if (threadIdx.x == 0) {
      unsigned long long t1;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      atomicMax(selfTime + 1, t1);
   }
}
template <int DB, bool IN, int FS, int NK, int NV, class... As>
__global__ void __launch_bounds__(kBlock, 2) scanGroupByKernel(const __grid_constant__ GroupByParams p) {
   using AL = Aggs<As...>;
   constexpr int N = AL::N;
   constexpr bool kStaged = encodedStages<DB, FS>;
   constexpr int F = kStaged ? kEncFrames : 1;
   constexpr int GREG = NK == 0 ? 1 : 4; // register-resident groups
   constexpr int LG = 16;                // CTA-local groups (registers + shared)
   __shared__ int32_t sKeys[LG][kMaxKeys];
   __shared__ int32_t sSlot[LG];
   __shared__ int32_t sCount, sLock;
   __shared__ unsigned long long sAcc[LG][N][2];
   __shared__ __align__(8) TileBarriers barsStorage;
   TileBarriers* bars = &barsStorage;

   unsigned long long* const selfTime = selfTimeStart(p.table);
   for (int i = threadIdx.x; i < LG * N * 2; i += kBlock) (&sAcc[0][0][0])[i] = 0;
   if (threadIdx.x == 0) {
      sCount = NK == 0 ? 1 : 0;
      sLock = 0;
      if (NK == 0) sSlot[0] = 0;
   }
   __syncthreads();

   i128 acc[GREG][N];
   // products of the i128 aggregates from proven stages; `room` is what every acc64 can still take (the same in every thread: a thread
   // adds at most 2 * F rows of a stage, each at most the stage's maxRow), so acc64 never exceeds INT64_MAX
   int64_t acc64[GREG][N];
   int64_t room = INT64_MAX;
#pragma unroll
   for (int g = 0; g < GREG; g++)
#pragma unroll
      for (int a = 0; a < N; a++) {
         acc[g][a] = i128{0, 0};
         acc64[g][a] = 0;
      }
   const int64_t one = 100; // 10^scale of decimal(12,2); checked on the host
   // keys of the register-resident groups live in registers too (refreshed when the CTA registers a new key)
   int32_t rk0[GREG], rk1[GREG];
   int rcnt = 0;
#pragma unroll
   for (int g = 0; g < GREG; g++) rk0[g] = rk1[g] = 0;

   // CTA-local group id of a row's keys (warp-collective: every lane calls it)
   auto groupOf = [&](int32_t k0, int32_t k1, bool pass) {
      int id = 0;
      if constexpr (NK > 0) {
         // Resolve the CTA-local group id under WARP-UNIFORM control flow.  (A per-lane spin lock
         // here once left the warps permanently diverged: 1 active thread per instruction, many
         // times the instructions and the DRAM traffic.)
         // Fast path: branch-free compare against the register copies of the first GREG keys.
         id = -1;
#pragma unroll
         for (int g = 0; g < GREG; g++)
            if (g < rcnt && k0 == rk0[g] && k1 == rk1[g]) id = g;
         const bool need = pass && id < 0;
         if (__ballot_sync(0xffffffffu, need)) { // rare after the first tiles: a key outside the register-resident set
            id = ctaGroupLookup<LG>(p.table, sKeys, sSlot, &sCount, &sLock, k0, k1, need, id);
            // refresh the register copies (keys are append-only, so ids never change)
            const int cnt = *((volatile int32_t*) &sCount);
            rcnt = cnt < GREG ? cnt : GREG;
#pragma unroll
            for (int g = 0; g < GREG; g++) {
               if (g < rcnt) {
                  rk0[g] = ((volatile int32_t*) sKeys[g])[0];
                  rk1[g] = ((volatile int32_t*) sKeys[g])[1];
               }
            }
         }
      }
      return id;
   };
   auto add = [&](int id, const i128* v, int32_t k0, int32_t k1) {
      if (id >= 0 && id < GREG) {
#pragma unroll
         for (int g = 0; g < GREG; g++)
            if (id == g) AL::accumulate(acc[g], v, typename AL::S{});
      } else if (id >= 0) { // CTA-local but not register resident: shared-memory atomics
         AL::sharedAdd(sAcc[id], v, typename AL::S{});
      } else { // more groups than a CTA tracks: straight to the HBM table
         int32_t kk[2] = {k0, k1};
         int slot = groupLookupOrInsert(p.table, kk);
         if (slot >= 0) AL::globalAdd(p.table, slot, v, typename AL::S{});
      }
   };
   auto generalRow = [&](const auto& tile, int lr, int64_t row, bool valid) {
      int64_t vals[NV];
#pragma unroll
      for (int c = 0; c < NV; c++) vals[c] = tile.lo64(p.valueStage[c], lr);
      int32_t k0 = 0, k1 = 0;
      if constexpr (NK > 0) k0 = tile.i32(p.keyStage[0], lr);
      if constexpr (NK > 1) k1 = tile.i32(p.keyStage[1], lr);
      const bool pass = valid & evalFilters<IN, FS>(p.src.filters, tile, lr, row);
      const int id = groupOf(k0, k1, pass);
      // expressions: 32-bit multiplies when every lane's operands allow it, else the general i128 path
      i128 v[N];
      if (__all_sync(0xffffffffu, !pass || AL::fits32(vals, one))) AL::template eval<true>(v, vals, one, typename AL::S{});
      else AL::template eval<false>(v, vals, one, typename AL::S{});
      if (pass) add(id, v, k0, k1);
   };
   auto encodedStage = [&](uint32_t stage) {
      const StagedCols& sc = p.src.cols;
      constexpr int FC = NV + NK;                  // staged index of the filter's column
      constexpr int R = kRowsPerThreadScan * F;    // rows of a thread
      constexpr int kTileRows = kRowsPerThreadScan * kBlock;
      constexpr int kFrameThreads = kBlock / F;    // threads per tile of the stage
      constexpr int kRun = 2;                      // adjacent rows decoded together
      // column c's F tiles lie from stage + F * smemOffset[c]; their headers are equal (kernels.h), tile 0's stands for all
      auto col = [&](int c) { return stage + (uint32_t) (F * sc.smemOffset[c]); };
      int64_t vb[NV], lo[NV], hi[NV], range[NV];
#pragma unroll
      for (int c = 0; c < NV; c++) {
         ldShared64x2(col(c), vb[c], range[c]);
         // a column with a wide range or base gets bounds no operand test passes (and no bound arithmetic overflows)
         const bool small = (uint64_t) range[c] < (1ull << 31) && vb[c] > -(1ll << 40) && vb[c] < (1ll << 40);
         lo[c] = small ? vb[c] : -(1ll << 62);
         hi[c] = small ? vb[c] + range[c] : (1ll << 62);
      }
      uint32_t kb[2] = {0, 0};
#pragma unroll
      for (int k = 0; k < NK; k++) kb[k] = (uint32_t) ldShared32(col(NV + k));
      uint64_t maxRow = 0;
      const bool proven = AL::template bound64<R>(lo, hi, one, maxRow);
      if (proven) {
         const int64_t need = (int64_t) maxRow * R;
         if (need > room) {
#pragma unroll
            for (int g = 0; g < GREG; g++) AL::fold64(acc[g], acc64[g], typename AL::S{});
            room = INT64_MAX;
         }
         room -= need;
      }
      // `v cmp C` on the raw field x = v - base in [0, 2^32) is `flo <= x <= fhi`, negated for != (mask 5)
      uint32_t flo, fhi;
      bool finv;
      {
         const FilterCol& f = p.src.filters.c[0];
         const int64_t t = (int64_t) (int32_t) f.valA - (int64_t) ldShared32(col(FC));
         finv = f.maskA == 5u;
         const uint32_t m = finv ? 2u : f.maskA;
         const int64_t l = (m & 1u) ? 0 : (m & 2u) ? t : t + 1, h = (m & 4u) ? 0xffffffffll : (m & 2u) ? t : t - 1;
         const int64_t lc = l < 0 ? 0 : l, hc = h > 0xffffffffll ? 0xffffffffll : h;
         flo = lc > hc ? 1u : (uint32_t) lc;
         fhi = lc > hc ? 0u : (uint32_t) hc;
      }
      // the register-resident keys, rebased like the key fields (exact: the decode is base + field modulo 2^32); absolute again
      // around the general lookup and at the end of the stage
      auto rebase = [&](uint32_t sign) {
#pragma unroll
         for (int g = 0; g < GREG; g++) {
            rk0[g] = (int32_t) ((uint32_t) rk0[g] + sign * kb[0]);
            rk1[g] = (int32_t) ((uint32_t) rk1[g] + sign * kb[1]);
         }
      };
      rebase(~0u);
      const uint32_t frame = threadIdx.x / kFrameThreads, ft = threadIdx.x % kFrameThreads;
#pragma unroll 1
      for (int run = 0; run < R / kRun; run++) {
         // rows r0 .. r0 + kRun - 1 of tile `frame`: the lanes of a warp read consecutive kRun * W bytes, conflict-free at any W
         const uint32_t r0 = (run * kFrameThreads + ft) * kRun;
         auto fields = [&](int c, uint32_t (&x)[kRun]) {
            const int sh = sc.encShift[c];
            encodedFields2(col(c) + frame * (kEncodeTileHeader + ((uint32_t) kTileRows << sh)) + kEncodeTileHeader + (r0 << sh), sh, x);
         };
         // filter and keys first: only the values stay live while the rows are summed
         uint32_t xk[2][kRun], xf[kRun];
#pragma unroll
         for (int i = 0; i < kRun; i++) xk[0][i] = xk[1][i] = 0;
#pragma unroll
         for (int k = 0; k < NK; k++) fields(NV + k, xk[k]);
         fields(FC, xf);
         bool pass[kRun];
         int id[kRun];
#pragma unroll
         for (int i = 0; i < kRun; i++) {
            pass[i] = ((xf[i] >= flo) & (xf[i] <= fhi)) != finv;
            id[i] = NK > 0 ? -1 : 0;
            if constexpr (NK > 0) {
#pragma unroll
               for (int g = 0; g < GREG; g++)
                  if (g < rcnt && xk[0][i] == (uint32_t) rk0[g] && xk[1][i] == (uint32_t) rk1[g]) id[i] = g;
               if (__any_sync(0xffffffffu, pass[i] && id[i] < 0)) { // a key outside the register-resident set: look it up as absolute keys
                  rebase(1u);
                  id[i] = groupOf((int32_t) (kb[0] + xk[0][i]), (int32_t) (kb[1] + xk[1][i]), pass[i]);
                  rebase(~0u);
               }
            }
         }
         uint32_t xv[NV][kRun];
#pragma unroll
         for (int c = 0; c < NV; c++) fields(c, xv[c]);
#pragma unroll
         for (int i = 0; i < kRun; i++) {
            const int32_t k0 = (int32_t) (kb[0] + xk[0][i]), k1 = (int32_t) (kb[1] + xk[1][i]);
            int64_t vals[NV];
#pragma unroll
            for (int c = 0; c < NV; c++) vals[c] = (int64_t) ((uint64_t) vb[c] + xv[c][i]);
            if (proven) {
               int64_t q[N];
               AL::eval64(q, vals, one, typename AL::S{});
               // a one-hot test per group: an `id == g` test here was folded into a dynamically indexed acc[id], which lives in local memory
               const uint32_t hot = pass[i] && id[i] >= 0 && id[i] < GREG ? 1u << id[i] : 0u;
#pragma unroll
               for (int g = 0; g < GREG; g++)
                  if (hot >> g & 1u) AL::accumulate64(acc[g], acc64[g], q, typename AL::S{});
               if (pass[i] && !hot) {
                  i128 v[N];
#pragma unroll
                  for (int a = 0; a < N; a++) v[a] = i128{(uint64_t) q[a], 0}; // what evalAgg gives: products are >= 0 here
                  add(id[i], v, k0, k1);
               }
            } else {
               i128 v[N];
               if (__all_sync(0xffffffffu, !pass[i] || AL::fits32(vals, one))) AL::template eval<true>(v, vals, one, typename AL::S{});
               else AL::template eval<false>(v, vals, one, typename AL::S{});
               if (pass[i]) add(id[i], v, k0, k1);
            }
         }
      }
      rebase(1u);
   };
   forEachTileUniform<kRowsPerThreadScan, DB, kStaged ? kEncStages : kStages, F>(p.src.cols, p.src.nRows, dynSmem, bars, [&](const auto& tile, int64_t rowBase, int rows) {
      // the descriptor-driven filter costs more per row than the stage path saves (Q6 measured slower), so it keeps the row path
      if constexpr (std::is_same_v<std::decay_t<decltype(tile)>, SmemTile<kDecEncoded>> && kStaged) {
         encodedStage(tile.stage);
      } else {
#pragma unroll
         for (int j = 0; j < kRowsPerThreadScan; j++) {
            const int lr = j * kBlock + threadIdx.x;
            const bool valid = lr < rows;
            generalRow(tile, valid ? lr : 0, rowBase + (valid ? lr : 0), valid);
         }
      }
   });
   // ---- flush: registers → warp sums → shared → one HBM atomic per (CTA, group, aggregate)
   __syncthreads();
#pragma unroll
   for (int g = 0; g < GREG; g++) AL::fold64(acc[g], acc64[g], typename AL::S{});
   const int lane = threadIdx.x & 31;
#pragma unroll
   for (int g = 0; g < GREG; g++) AL::warpFlush(sAcc[g], acc[g], lane, typename AL::S{});
   __syncthreads();
   flushCtaGroups<N>(p.table, sAcc, sSlot, sCount, selfTime);
}

// The factored Q1 kernel: Q1's signature over an encoded batch with the one-int32-constant filter, when factoredFits admits the batch.  Its
// columns are in signature order (qty, ep, d, t, the two keys, the filter's column; toSignatureOrder).  Invariant: factoredFits proves
// on the host, from the batch's minima and ranges, that every value lies in [encMin, encMin + encRange] with ep - min_ep < 2^28,
// qty - min_qty < 2^21, 4 * Dd * Dt <= kCells and every Q1 product a non-negative int64 (aggBound64 over the batch), and that both key
// fields are 1 byte wide.  Every stage or tile header's block lies inside the batch, so each of its rows has its cell and word budgets
// and the 64-bit products of the fallback without a check in the kernel.
// A frame is one TMA stage of kFacTiles tiles or one tile read with plain loads (the tail, or a batch without TMA), and every frame ends
// at a CTA barrier.  The cell words hold p.facFoldFrames frames (K, from the batch bounds): at the start of every K-th frame of a loop,
// counted from the loop's index, and once before the tail tiles, each thread folds the cells it owns into 64-bit sums and zeroes them,
// and a second barrier lets that frame's atomics in; the other frames pay neither.  The stage ring
// holds kFacStages stages of kFacTiles tiles (50 KB at TPC-H widths; deeper rings of fewer tiles measured slower) and with about 8 KB of
// static shared memory three CTAs fit an SM, which hide the latency of each warp's dependent run (loads → compare → vote → loads →
// atomics).  A thread decodes its rows of a stage in runs of 4 adjacent rows, one shared load per column per run, so each chain
// carries 4 independent rows.
constexpr int kFacTiles = 4, kFacStages = 2;
__global__ void __launch_bounds__(kBlock, 3) scanQ1FactoredKernel(const __grid_constant__ GroupByParams p) {
   constexpr int F = kFacTiles, S = kFacStages;
   using AL = Q1Aggs;
   constexpr int N = AL::N, NV = 4, NK = 2;
   constexpr int FC = NV + NK; // staged index of the filter's column
   constexpr int GREG = 4;     // register groups (factored in the cells)
   constexpr int LG = 16;      // CTA-local groups (registers + shared)
   constexpr int RUN = 4;      // adjacent rows of a stage decoded together (encodedFields4)
   constexpr int kOwned = kCells / kBlock;
   constexpr int kTileRows = kRowsPerThreadScan * kBlock;
   static_assert(F * kTileRows <= 2048 && (2 * F) % RUN == 0 && 128 % F == 0, "a stage is one frame of whole runs in one block");
   __shared__ int32_t sKeys[LG][kMaxKeys];
   __shared__ int32_t sSlot[LG];
   __shared__ int32_t sCount, sLock;
   __shared__ unsigned long long sAcc[LG][N][2];
   __shared__ uint32_t sCell[kCellWords][kCells]; // {L, H, Q, N} words per cell
   __shared__ __align__(8) uint64_t sFull[S];        // stage s holds its tiles

   unsigned long long* const selfTime = selfTimeStart(p.table);
   for (int i = threadIdx.x; i < LG * N * 2; i += kBlock) (&sAcc[0][0][0])[i] = 0;
   for (int i = threadIdx.x; i < kCellWords * kCells; i += kBlock) (&sCell[0][0])[i] = 0;
   if (threadIdx.x == 0) sCount = sLock = 0;
   __syncthreads();

   const int64_t one = 100; // 10^scale of decimal(12,2); checked on the host
   const uint32_t fDt = (uint32_t) p.encRange[kTax] + 1u, fDdDt = ((uint32_t) p.encRange[kDisc] + 1u) * fDt;
   // 64-bit sums of the cells this thread owns (cell j * kBlock + threadIdx.x)
   uint64_t cEp[kOwned], cCnt[kOwned], cQty[kOwned];
#pragma unroll
   for (int j = 0; j < kOwned; j++) cEp[j] = cCnt[j] = cQty[j] = 0;
   auto foldCells = [&]() {
#pragma unroll
      for (int j = 0; j < kOwned; j++) {
         const int cell = j * kBlock + threadIdx.x;
         const uint32_t n = sCell[3][cell];
         if (n != 0) {
            cEp[j] += sCell[0][cell] + ((uint64_t) sCell[1][cell] << p.facShift);
            cCnt[j] += n;
            cQty[j] += sCell[2][cell];
            sCell[0][cell] = sCell[1][cell] = sCell[2][cell] = sCell[3][cell] = 0;
         }
      }
   };
   // every thread passed the barrier behind the previous frame's atomics (or the set-up); folding cells nothing added to is a no-op
   auto beginFrame = [&](bool fold) {
      if (fold) {
         foldCells();
         __syncthreads();
      }
   };

   // the frame's header bases and what follows from them: the offsets of its value fields from the batch minima (a value is
   // encMin + off + field), the key bases, and the filter as a range of the raw field
   uint32_t off[NV], cellOff = 0, kb0 = 0, kb1 = 0, flo = 0, fhi = 0;
   bool finv = false;
   // the register groups' keys as packed raw key fields of the frame (k0 - kb0 | (k1 - kb1) << 16); a group not registered yet, or whose
   // keys lie outside the frame's 1-byte fields, holds ~0u, which no packed pair of 1-byte fields equals
   uint32_t rk[GREG];
   auto registerKeys = [&]() {
      const int cnt = *((volatile int32_t*) &sCount);
#pragma unroll
      for (int g = 0; g < GREG; g++) {
         rk[g] = ~0u;
         if (g < cnt) {
            const uint32_t a = (uint32_t) ((volatile int32_t*) sKeys[g])[0] - kb0, b = (uint32_t) ((volatile int32_t*) sKeys[g])[1] - kb1;
            if ((a | b) < 256u) rk[g] = a | b << 16;
         }
      }
   };
   auto setFrame = [&](const int64_t (&base)[NV], uint32_t k0, uint32_t k1, int32_t filterBase) {
#pragma unroll
      for (int c = 0; c < NV; c++) off[c] = (uint32_t) (base[c] - p.encMin[c]);
      cellOff = off[kDisc] * fDt + off[kTax];
      kb0 = k0;
      kb1 = k1;
      // `v cmp C` on the raw field x = v - base in [0, 2^32) is `flo <= x <= fhi`, negated for != (mask 5)
      const FilterCol& f = p.src.filters.c[0];
      const int64_t t = (int64_t) (int32_t) f.valA - (int64_t) filterBase;
      finv = f.maskA == 5u;
      const uint32_t m = finv ? 2u : f.maskA;
      const int64_t l = (m & 1u) ? 0 : (m & 2u) ? t : t + 1, h = (m & 4u) ? 0xffffffffll : (m & 2u) ? t : t - 1;
      const int64_t lc = l < 0 ? 0 : l, hc = h > 0xffffffffll ? 0xffffffffll : h;
      flo = lc > hc ? 1u : (uint32_t) lc;
      fhi = lc > hc ? 0u : (uint32_t) hc;
      registerKeys();
   };
   // K adjacent rows of the frame (warp-collective): their raw key and filter fields, whether they exist, and a loader of their value fields
   auto rows = [&](const auto& xk0, const auto& xk1, const auto& xf, const auto& valid, const auto& values) {
      constexpr int K = std::extent_v<std::remove_reference_t<decltype(xk0)>>;
      bool pass[K], miss = false;
      int id[K];
#pragma unroll
      for (int i = 0; i < K; i++) {
         pass[i] = valid[i] & (((xf[i] >= flo) & (xf[i] <= fhi)) != finv);
         const uint32_t pk = xk0[i] | xk1[i] << 16;
         id[i] = -1;
#pragma unroll
         for (int g = 0; g < GREG; g++)
            if (pk == rk[g]) id[i] = g;
         miss |= pass[i] & (id[i] < 0);
      }
      if (__any_sync(0xffffffffu, miss)) { // a key outside the register groups: the CTA's shared list, then registration
#pragma unroll
         for (int i = 0; i < K; i++)
            id[i] = ctaGroupLookup<LG>(p.table, sKeys, sSlot, &sCount, &sLock, (int32_t) (kb0 + xk0[i]), (int32_t) (kb1 + xk1[i]), pass[i] && id[i] < 0, id[i]);
         registerKeys();
      }
      uint32_t xv[NV][K];
      values(xv);
#pragma unroll
      for (int i = 0; i < K; i++) {
         if (pass[i] && (uint32_t) id[i] < (uint32_t) GREG) {
            const uint32_t c = (uint32_t) id[i] * fDdDt + xv[kDisc][i] * fDt + xv[kTax][i] + cellOff;
            const uint32_t ep = xv[kEp][i] + off[kEp], epHi = ep >> p.facShift;
            atomicAdd(&sCell[0][c], ep - (epHi << p.facShift));
            atomicAdd(&sCell[1][c], epHi);
            atomicAdd(&sCell[2][c], xv[kQty][i] + off[kQty]);
            atomicAdd(&sCell[3][c], 1u);
         } else if (pass[i]) { // a group past the register set: its products in 64 bits (proven), shared sums or the HBM table
            int64_t vals[NV], q[N];
#pragma unroll
            for (int c = 0; c < NV; c++) vals[c] = p.encMin[c] + (int64_t) (off[c] + xv[c][i]);
            AL::eval64(q, vals, one, typename AL::S{});
            i128 v[N];
#pragma unroll
            for (int a = 0; a < N; a++) v[a] = i128{(uint64_t) q[a], 0};
            if (id[i] >= 0) {
               AL::sharedAdd(sAcc[id[i]], v, typename AL::S{});
            } else {
               int32_t kk[2] = {(int32_t) (kb0 + xk0[i]), (int32_t) (kb1 + xk1[i])};
               const int slot = groupLookupOrInsert(p.table, kk);
               if (slot >= 0) AL::globalAdd(p.table, slot, v, typename AL::S{});
            }
         }
      }
   };
   const StagedCols& sc = p.src.cols;
   // one stage in shared memory: its F tiles of column c lie from stage + F * smemOffset[c] with equal headers (kernels.h), tile 0's
   // stands for all; thread t takes 2F rows of tile t / (kBlock / F) in runs of RUN adjacent rows, the lanes of a warp reading
   // consecutive RUN * W bytes per column, conflict-free at any W
   auto stageFrame = [&](uint32_t stage, bool fold) {
      beginFrame(fold);
      auto col = [&](int c) { return stage + (uint32_t) (F * sc.smemOffset[c]); };
      int64_t base[NV];
#pragma unroll
      for (int c = 0; c < NV; c++) base[c] = ldShared64(col(c));
      setFrame(base, (uint32_t) ldShared32(col(NV)), (uint32_t) ldShared32(col(NV + 1)), ldShared32(col(FC)));
      constexpr int kFrameThreads = kBlock / F; // threads per tile of the stage
      const uint32_t frame = threadIdx.x / kFrameThreads, ft = threadIdx.x % kFrameThreads;
#pragma unroll 1
      for (int run = 0; run < 2 * F / RUN; run++) {
         const uint32_t r0 = (run * kFrameThreads + ft) * RUN;
         auto fields = [&](int c, uint32_t (&x)[RUN]) {
            const int sh = sc.encShift[c];
            const uint32_t a = col(c) + frame * (kEncodeTileHeader + ((uint32_t) kTileRows << sh)) + kEncodeTileHeader + (r0 << sh);
            encodedFields4(a, sh, x);
         };
         uint32_t xk0[RUN], xk1[RUN], xf[RUN];
         fields(NV, xk0);
         fields(NV + 1, xk1);
         fields(FC, xf);
         bool valid[RUN];
#pragma unroll
         for (int i = 0; i < RUN; i++) valid[i] = true;
         rows(xk0, xk1, xf, valid, [&](uint32_t (&xv)[NV][RUN]) {
#pragma unroll
            for (int c = 0; c < NV; c++) fields(c, xv[c]);
         });
      }
   };
   // one tile through plain loads: thread t takes rows t and kBlock + t
   auto tileFrame = [&](int64_t t, bool fold) {
      beginFrame(fold);
      GlobalTile<kDecEncoded> tile{t * kTileRows, &sc};
      const int nRows = (int) min(p.src.nRows - t * kTileRows, (int64_t) kTileRows);
      int64_t base[NV];
#pragma unroll
      for (int c = 0; c < NV; c++) base[c] = (int64_t) tile.base(c);
      setFrame(base, (uint32_t) tile.base(NV), (uint32_t) tile.base(NV + 1), (int32_t) tile.base(FC));
      constexpr int K = kRowsPerThreadScan;
      int lr[K];
      bool valid[K];
      uint32_t xk0[K], xk1[K], xf[K];
#pragma unroll
      for (int i = 0; i < K; i++) {
         lr[i] = i * kBlock + threadIdx.x;
         valid[i] = lr[i] < nRows;
         if (!valid[i]) lr[i] = 0;
         xk0[i] = (uint32_t) tile.field(NV, lr[i]);
         xk1[i] = (uint32_t) tile.field(NV + 1, lr[i]);
         xf[i] = (uint32_t) tile.field(FC, lr[i]);
      }
      rows(xk0, xk1, xf, valid, [&](uint32_t (&xv)[NV][K]) {
#pragma unroll
         for (int c = 0; c < NV; c++)
#pragma unroll
            for (int i = 0; i < K; i++) xv[c][i] = (uint32_t) tile.field(c, lr[i]);
      });
   };

   // CTA b takes stages b, b + grid, ..; the full tiles after the last full stage and the partial tail tile go tile by tile through
   // plain loads, continuing that round robin.  Each loop folds the cell words at its frames 0, K, 2K, .. (frame 0 of the tail loop
   // folds what the stages left)
   const uint32_t K = p.facFoldFrames;
   const int64_t nFull = p.src.nRows / kTileRows;
   int64_t done = nFull, turns = nFull; // tiles read by the loops below, and the round-robin turns they took
   if (sc.useTma) {
      const int64_t nStages = nFull / F;
      done = nStages * F;
      turns = nStages;
      if (threadIdx.x == 0) {
         for (int s = 0; s < S; s++) mbarInit(&sFull[s], 1);
         mbarInitFence();
      }
      __syncthreads();
      if (threadIdx.x == 0) {
         for (int s = 0; s < S; s++) {
            const int64_t t = (int64_t) blockIdx.x + (int64_t) s * gridDim.x;
            if (t < nStages) issueTile<F>(sc, dynSmem, sFull, t, s);
         }
      }
      for (int64_t t = blockIdx.x; t < nStages; t += gridDim.x) {
         const uint32_t it = (uint32_t) (t - blockIdx.x) / gridDim.x; // this CTA's stage count (a batch has < 2^36 rows), not kept live
         const int s = it % S;
         mbarWait(&sFull[s], (uint32_t) (it / S) & 1u);
         stageFrame(smemAddr(dynSmem) + (uint32_t) (s * F * sc.stageBytes), it % K == 0);
         __syncthreads(); // every thread is done with stage s → refill it
         const int64_t nt = t + (int64_t) S * gridDim.x;
         if (threadIdx.x == 0 && nt < nStages) issueTile<F>(sc, dynSmem, sFull, nt, s);
      }
   } else {
      for (int64_t t = blockIdx.x; t < nFull; t += gridDim.x) {
         tileFrame(t, (uint32_t) (t - blockIdx.x) / gridDim.x % K == 0);
         __syncthreads();
      }
   }
   const int64_t nTiles = (p.src.nRows + kTileRows - 1) / kTileRows;
   const int64_t t0 = done + ((int64_t) blockIdx.x + gridDim.x - turns % gridDim.x) % gridDim.x;
   for (int64_t t = t0; t < nTiles; t += gridDim.x) {
      tileFrame(t, (uint32_t) (t - t0) / gridDim.x % K == 0);
      __syncthreads();
   }
   // ---- flush: the last frame's cells, then each owned cell's six aggregates, exact modulo 2^64 / 2^128 like the per-row sums; per
   // register group this thread's owned cells of the group, summed over the warp, one shared atomic per warp and aggregate
   foldCells();
   const int lane = threadIdx.x & 31;
#pragma unroll 1
   for (int g = 0; g < GREG; g++) {
      i128 s[N];
#pragma unroll
      for (int a = 0; a < N; a++) s[a] = i128{0, 0};
#pragma unroll
      for (int j = 0; j < kOwned; j++) {
         const uint32_t cell = j * kBlock + threadIdx.x, dt = cell % fDdDt;
         if (cCnt[j] == 0 || cell / fDdDt != (uint32_t) g) continue;
         const int64_t d = p.encMin[kDisc] + (int64_t) (dt / fDt), t = p.encMin[kTax] + (int64_t) (dt % fDt);
         const uint64_t n = cCnt[j];
         const i128 ep = add128(i128{cEp[j], 0}, mul64x64(p.encMin[kEp], (int64_t) n));
         const i128 epd = mul128x64(ep, one - d);
         i128 v[N];
         v[0] = i128{cQty[j] + (uint64_t) p.encMin[kQty] * n, 0};
         v[1] = i128{ep.lo, 0};
         v[2] = epd;
         v[3] = mul128x64(epd, one + t);
         v[4] = i128{(uint64_t) d * n, 0};
         v[5] = i128{n, 0};
         AL::accumulate(s, v, typename AL::S{});
      }
      AL::warpFlush(sAcc[g], s, lane, typename AL::S{});
   }
   __syncthreads();
   flushCtaGroups<N>(p.table, sAcc, sSlot, sCount, selfTime);
}

// ---- signature registry
static std::string signature(const GroupByParams& p) {
   std::string s = "k" + std::to_string(p.nKeys) + "v" + std::to_string(p.nValueCols);
   for (int i = 0; i < p.nAggs; i++) {
      const AggSpec& a = p.aggs[i];
      int used = a.expr == LDB_EXPR_COL ? 1 : a.expr == LDB_EXPR_MUL || a.expr == LDB_EXPR_MUL_1MINUS ? 2 : a.expr == LDB_EXPR_MUL_1MINUS_1PLUS ? 3 : 0;
      s += "|" + std::to_string(a.expr);
      for (int k = 0; k < used; k++) s += (k ? "," : ":") + std::to_string(a.col[k]);
   }
   return s;
}
// persistent grid: SMs x resident CTAs of this instantiation (occupancy API), never more than the tiles
template <class K>
static int persistentGrid(K kernel, const StagedCols& sc, int64_t nRows, int smCount, size_t* dynBytes, int threads = kThreads, int stages = kStages) {
   *dynBytes = sc.useTma ? (size_t) stages * sc.stageBytes : 0;
   // static + dynamic shared memory beyond 48 KB needs the opt-in (K9 carries 12 KB of static group slots), so always ask — but only
   // ever RAISE a kernel's limit: several contexts of one process (threads) launch the same kernel with different tile sizes, and
   // lowering the attribute between another thread's query and its launch made that launch fail with "invalid argument"
   if (*dynBytes > 0) {
      static std::mutex m;
      static std::map<const void*, size_t> granted;
      std::lock_guard<std::mutex> lock(m);
      size_t& g = granted[(const void*) kernel];
      if (*dynBytes > g) {
         cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) *dynBytes);
         g = *dynBytes;
      }
   }
   int perSm = 1;
   cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, kernel, threads, *dynBytes);
   if (perSm < 1) perSm = 1;
   int64_t tiles = (nRows + sc.tileRows - 1) / sc.tileRows;
   return (int) std::min<int64_t>(std::max<int64_t>(tiles, 1), (int64_t) smCount * perSm);
}
static bool hasInList(const FilterSet& f) { // "rare" filters: IN lists and LIKE-contains
   for (int i = 0; i < f.n; i++)
      if (f.c[i].nIn > 0 || f.c[i].kind == COL_UTF8_CONTAINS) return true;
   return false;
}
template <int DB, bool IN, int FS, int NK, int NV, class... As>
static void launchGBd(const GroupByParams& p, int smCount, cudaStream_t s) {
   size_t dyn;
   constexpr int tiles = encodedStages<DB, FS> ? kEncStages * kEncFrames : kStages; // tiles held in shared memory
   int grid = persistentGrid(scanGroupByKernel<DB, IN, FS, NK, NV, As...>, p.src.cols, p.src.nRows, smCount, &dyn, kBlock, tiles);
   scanGroupByKernel<DB, IN, FS, NK, NV, As...><<<grid, kBlock, dyn, s>>>(p);
}
// The stage path reads fields of at most 4 bytes (an 8-byte field is a value column no product proof admits) and must fit its stages in
// one CTA's shared memory; other encoded batches take the instance with the descriptor-driven filter.
template <class K>
static bool encodedStagesFit(K kernel, const StagedCols& sc) {
   for (int c = 0; c < sc.n; c++)
      if (sc.elemBytes[c] > 4) return false;
   int dev = 0, optin = 0;
   cudaFuncAttributes fa{};
   cudaGetDevice(&dev);
   cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
   cudaFuncGetAttributes(&fa, kernel);
   return (int64_t) kEncStages * kEncFrames * sc.stageBytes + (int64_t) fa.sharedSizeBytes <= optin;
}
// The factored kernel (Q1Aggs, kCells) runs when the batch's discount and tax domains give every register group its cells, and the
// batch's own bounds (encMin, encRange) prove what each stage header would: ep - min_ep < 2^28 and qty - min_qty < 2^21 (the word
// budgets) and the 64-bit product bound of the per-row stage path (aggBound64 on the batch range), so every row of a register group
// factors and only rows of groups past the register set take the fallback.  The batch must also be short enough for the 64-bit cell
// sums (2^36 rows of ep_off < 2^28), its key fields 1 byte wide (the kernel compares both keys as one packed word), and its stages and
// shared memory must leave three CTAs per SM (one fewer resident CTA costs more than the factoring saves).  Any other batch takes the
// per-row stage instance, which keeps its sums in registers.
static bool factoredFits(const GroupByParams& p) {
   const uint64_t dd = p.encRange[kDisc], dt = p.encRange[kTax];
   if (dd >= kCells || dt >= kCells || 4 * (dd + 1) * (dt + 1) > (uint64_t) kCells || p.src.nRows >= (1ll << 36)) return false;
   if (p.encRange[kEp] >= (1ull << 28) || p.encRange[kQty] >= (1ull << 21)) return false;
   // aggBound64 of ep * (1 - d) * (1 + t) over the batch: operands in [0, 2^31), largest product below 2^63 / (2 * kEncFrames)
   const int64_t one = 100, k31 = 1ll << 31;
   const int64_t epLo = p.encMin[kEp], epHi = epLo + (int64_t) p.encRange[kEp];
   const int64_t dLo = one - (p.encMin[kDisc] + (int64_t) dd), dHi = one - p.encMin[kDisc];
   const int64_t tLo = one + p.encMin[kTax], tHi = one + p.encMin[kTax] + (int64_t) dt;
   if (p.encMin[kDisc] < -k31 || p.encMin[kDisc] > k31 || p.encMin[kTax] < -k31 || p.encMin[kTax] > k31) return false;
   if (epLo < 0 || epHi >= k31 || dLo < 0 || dHi >= k31 || tLo < 0 || tHi >= k31) return false;
   if ((unsigned __int128) epHi * (uint64_t) dHi * (uint64_t) tHi >= (unsigned __int128) ((1ull << 63) / (kRowsPerThreadScan * kEncFrames))) return false;
   const StagedCols& sc = p.src.cols;
   for (int c = 0; c < sc.n; c++)
      if (sc.elemBytes[c] > 4) return false;
   if (sc.elemBytes[4] != 1 || sc.elemBytes[5] != 1) return false; // the keys (signature order)
   int dev = 0, perSm = 0, reserved = 0;
   cudaFuncAttributes fa{};
   cudaGetDevice(&dev);
   cudaDeviceGetAttribute(&perSm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
   cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev);
   cudaFuncGetAttributes(&fa, (const void*) scanQ1FactoredKernel);
   return 3 * ((int64_t) kFacStages * kFacTiles * sc.stageBytes + (int64_t) fa.sharedSizeBytes + reserved) <= perSm;
}
// The factored kernel's cell-word split s and fold interval K (kernels.cu, Factored Q1): the s in [0, 28] that allows the largest K
// with n = kFacFrameRows * K rows per cell between folds keeping n (2^s - 1), n (range_ep >> s), n range_qty and n below 2^32.  The
// last bound caps K below 2^21.  Every batch factoredFits admits (range_ep < 2^28, range_qty < 2^21) gets K >= 1 at s = 20.
static void factoredFold(GroupByParams& p) {
   constexpr uint64_t kMaxN = 0xffffffffull;
   const uint64_t rq = p.encRange[kQty];
   p.facShift = 20;
   p.facFoldFrames = 0;
   for (uint32_t sh = 0; sh <= 28; sh++) {
      const uint64_t top = std::max<uint64_t>(std::max<uint64_t>((1ull << sh) - 1, p.encRange[kEp] >> sh), std::max<uint64_t>(rq, 1));
      const uint64_t k = kMaxN / (top * kFacFrameRows);
      if (k > p.facFoldFrames) {
         p.facShift = sh;
         p.facFoldFrames = (uint32_t) k;
      }
   }
}
static void launchQ1Factored(GroupByParams p, int smCount, cudaStream_t s) {
   factoredFold(p);
   size_t dyn;
   int grid = persistentGrid(scanQ1FactoredKernel, p.src.cols, p.src.nRows, smCount, &dyn, kBlock, kFacStages * kFacTiles);
   scanQ1FactoredKernel<<<grid, kBlock, dyn, s>>>(p);
}
// The encoded instance reads its columns' layout at constant indices: value column c is staged column c, key k is NV + k, and a
// shaped filter's column is NV + NK.  Permutes the staged columns (and every index into them) into that order; returns the filter
// shape the permuted parameters can run under.  Keys and values are distinct staged columns (scanGroupByEncodable).
static int toSignatureOrder(GroupByParams& p) {
   const StagedCols src = p.src.cols;
   int order[kMaxStagedCols], pos[kMaxStagedCols], n = 0;
   auto place = [&](int c) {
      for (int i = 0; i < n; i++)
         if (order[i] == c) return;
      order[n++] = c;
   };
   for (int v = 0; v < p.nValueCols; v++) place(p.valueStage[v]);
   for (int k = 0; k < p.nKeys; k++) place(p.keyStage[k]);
   if (p.src.filters.n > 0 && p.src.filters.c[0].staged >= 0) place(p.src.filters.c[0].staged);
   for (int c = 0; c < src.n; c++) place(c);
   StagedCols& sc = p.src.cols;
   for (int i = 0; i < n; i++) {
      pos[order[i]] = i;
      sc.base[i] = src.base[order[i]];
      sc.elemBytes[i] = src.elemBytes[order[i]];
      sc.smemOffset[i] = src.smemOffset[order[i]];
      sc.encShift[i] = src.encShift[order[i]];
      sc.encMask[i] = src.encMask[order[i]];
   }
   for (int v = 0; v < p.nValueCols; v++) p.valueStage[v] = pos[p.valueStage[v]];
   for (int k = 0; k < p.nKeys; k++) p.keyStage[k] = pos[p.keyStage[k]];
   for (int f = 0; f < p.src.filters.n; f++)
      if (p.src.filters.c[f].staged >= 0) p.src.filters.c[f].staged = pos[p.src.filters.c[f].staged];
   const int fs = filterShape(p.src.filters);
   if ((fs == FS_I32_ONE || fs == FS_I32_RANGE) && p.src.filters.c[0].staged != p.nValueCols + p.nKeys) return FS_GENERIC; // e.g. a filter on a key
   return fs;
}
// ENC: the signature is also compiled for the encoded layout (only without IN lists; scanGroupByEncodable says which); ENC_ONE: and
// for the one-int32-constant filter shape (Q1's l_shipdate <= date), otherwise the encoded instance evaluates the filter descriptor
template <bool ENC, bool ENC_ONE, int NK, int NV, class... As>
static void launchGB(const GroupByParams& p, int smCount, cudaStream_t s) {
   const bool in = hasInList(p.src.filters);
   if constexpr (ENC) {
      if (p.src.cols.decBytes == kDecEncoded) {
         GroupByParams q = p;
         const int fs = toSignatureOrder(q);
         if constexpr (ENC_ONE) {
            if (fs == FS_I32_ONE) {
               if constexpr (NK == 2 && NV == 4 && std::is_same_v<Aggs<As...>, Q1Aggs>) {
                  if (factoredFits(q)) {
                     launchQ1Factored(q, smCount, s);
                     return;
                  }
               }
               if (encodedStagesFit(scanGroupByKernel<kDecEncoded, false, FS_I32_ONE, NK, NV, As...>, q.src.cols)) {
                  launchGBd<kDecEncoded, false, FS_I32_ONE, NK, NV, As...>(q, smCount, s);
                  return;
               }
            }
         }
         launchGBd<kDecEncoded, false, FS_GENERIC, NK, NV, As...>(q, smCount, s);
         return;
      }
   }
   if (p.src.cols.decBytes == 8) {
      if (in) launchGBd<8, true, FS_GENERIC, NK, NV, As...>(p, smCount, s);
      else launchGBd<8, false, FS_GENERIC, NK, NV, As...>(p, smCount, s);
   } else {
      if (in) launchGBd<16, true, FS_GENERIC, NK, NV, As...>(p, smCount, s);
      else launchGBd<16, false, FS_GENERIC, NK, NV, As...>(p, smCount, s);
   }
}
// the signatures compiled for the encoded layout as well: Q1 and Q6, the two the encoded column copy exists for
static const char* const kSigQ1 = "k2v4|0:0|0:1|2:1,2|3:1,2,3|0:2|4";
static const char* const kSigQ6 = "k0v2|1:0,1";
bool scanGroupByEncodable(const GroupByParams& p) {
   const std::string sig = signature(p);
   if ((sig != kSigQ1 && sig != kSigQ6) || hasInList(p.src.filters)) return false;
   // the encoded instance stages every key and value column once (toSignatureOrder)
   int stage[kMaxKeys + kMaxValueCols], n = 0;
   for (int k = 0; k < p.nKeys; k++) stage[n++] = p.keyStage[k];
   for (int v = 0; v < p.nValueCols; v++) stage[n++] = p.valueStage[v];
   for (int i = 0; i < n; i++)
      for (int j = 0; j < i; j++)
         if (stage[i] == stage[j]) return false;
   return true;
}
bool scanGroupByFactored(const GroupByParams& p) {
   if (p.src.cols.decBytes != kDecEncoded || signature(p) != kSigQ1 || hasInList(p.src.filters)) return false;
   GroupByParams q = p;
   return toSignatureOrder(q) == FS_I32_ONE && factoredFits(q);
}
bool launchScanGroupBy(const GroupByParams& p, int smCount, cudaStream_t s, const char** why) {
   std::string sig = signature(p);
   if (p.src.cols.decBytes == kDecEncoded && !scanGroupByEncodable(p)) {
      *why = "group-by pipeline bound to the encoded layout has no encoded instantiation";
      return false;
   }
   // Q1 pricing summary: sum(a) sum(b) sum(b*(1-c)) sum(b*(1-c)*(1+d)) sum(c) count   (resources/sql/tpch/1.sql)
   if (sig == kSigQ1) {
      launchGB<true, true, 2, 4, C0, C1, Agg<LDB_EXPR_MUL_1MINUS, 1, 2>, Agg<LDB_EXPR_MUL_1MINUS_1PLUS, 1, 2, 3>, C2, ONE>(p, smCount, s);
   } else if (sig == "k1v4|0:0|0:1|2:1,2|3:1,2,3|0:2|4") {
      launchGB<false, false, 1, 4, C0, C1, Agg<LDB_EXPR_MUL_1MINUS, 1, 2>, Agg<LDB_EXPR_MUL_1MINUS_1PLUS, 1, 2, 3>, C2, ONE>(p, smCount, s);
   } else if (sig == kSigQ6) { // Q6 forecast revenue: sum(a*b)
      launchGB<true, false, 0, 2, Agg<LDB_EXPR_MUL, 0, 1>>(p, smCount, s);
   } else if (sig == "k0v2|2:0,1") { // keyless sum(a*(1-b))
      launchGB<false, false, 0, 2, Agg<LDB_EXPR_MUL_1MINUS, 0, 1>>(p, smCount, s);
   } else if (sig == "k0v1|0:0|4") { // keyless sum(a), count
      launchGB<false, false, 0, 1, C0, ONE>(p, smCount, s);
   } else if (sig == "k1v2|2:0,1") { // group by k: sum(a*(1-b))
      launchGB<false, false, 1, 2, Agg<LDB_EXPR_MUL_1MINUS, 0, 1>>(p, smCount, s);
   } else if (sig == "k2v2|2:0,1") {
      launchGB<false, false, 2, 2, Agg<LDB_EXPR_MUL_1MINUS, 0, 1>>(p, smCount, s);
   } else if (sig == "k1v1|0:0|4") { // group by k: sum(a), count
      launchGB<false, false, 1, 1, C0, ONE>(p, smCount, s);
   } else if (sig == "k2v1|0:0|4") {
      launchGB<false, false, 2, 1, C0, ONE>(p, smCount, s);
   } else {
      static thread_local std::string msg;
      msg = "no compiled group-by pipeline for aggregate signature '" + sig + "' (register it in kernels.cu:launchScanGroupBy)";
      *why = msg.c_str();
      return false;
   }
   return true;
}

// =================================================================================== survivor queue
// The probe kernels (K3 with a parent probe, K4, K5, K9) keep only a few percent of the scanned rows after the Bloom filter
// of the first table.  Handling those in place leaves ~2 active lanes per warp on the dependent part (directory walks,
// i128 arithmetic, atomics) and holds the tile's stage until the slowest chain is done (the
// probe ran several times longer than the scan alone).  Instead the scan COPIES each survivor's operands (NW 32-bit words) into a CTA-wide queue in shared memory;
// whenever the queue holds a CTA's worth, every thread takes one entry: kBlock independent chains in flight, all lanes busy.
template <int NW, int RPT = kRowsPerThreadStar>
struct SurvivorQueue {
   static constexpr int kCap = kBlock + RPT * kBlock; // a drain leaves < kBlock entries; one tile adds <= its rows
   int32_t w[NW][kCap];
   int count;
   __device__ __forceinline__ int claim() { return atomicAdd(&count, 1); }
   __device__ __forceinline__ void put64(int word, int q, int64_t v) {
      w[word][q] = (int32_t) (uint32_t) (uint64_t) v;
      w[word + 1][q] = (int32_t) (uint32_t) ((uint64_t) v >> 32);
   }
   __device__ __forceinline__ int64_t get64(int word, int q) const { return (int64_t) (((uint64_t) (uint32_t) w[word + 1][q] << 32) | (uint32_t) w[word][q]); }
};
// Called by every thread of the CTA after a barrier that published the pushes.  Processes entries kBlock at a time until
// fewer than kBlock are left (all == false) or none (all == true, at the end of the kernel).
template <class Q, class Fn>
__device__ __forceinline__ void drainQueue(Q& q, bool all, const Fn& process) {
   int count = q.count < Q::kCap ? q.count : Q::kCap; // claims beyond the capacity were handled in place by their owners
   if (!(count >= kBlock || (all && count > 0))) return;
   while (count >= kBlock || (all && count > 0)) {
      const int n = count < kBlock ? count : kBlock;
      if ((int) threadIdx.x < n) process(count - n + (int) threadIdx.x);
      count -= n;
   }
   __syncthreads(); // every thread read q.count and finished its entries
   if (threadIdx.x == 0) q.count = count;
   __syncthreads();
}
// CTA-local group table for the kernels that aggregate matched rows into a handful of groups (K4: 5 nations, K9: 175
// nation-years): the reference's per-worker pre-aggregation cache (PreAggregationHashtable.cpp:46-60) as shared-memory
// slots flushed once per CTA — 10^8 matched rows over 175 groups would otherwise serialise on 175 HBM addresses.
constexpr int kLocalGroups = 256; // power of two; further groups go straight to the HBM table
struct LocalGroups {
   unsigned long long key[kLocalGroups];
   unsigned long long acc[kLocalGroups][2];
   __device__ __forceinline__ void init() {
      for (int i = threadIdx.x; i < kLocalGroups; i += blockDim.x) {
         key[i] = ~0ull;
         acc[i][0] = acc[i][1] = 0;
      }
   }
   // is64: the aggregate is a 64-bit SUM (wraps at 64 bits, hi stays 0) — LdbExprKind COL / ONE
   __device__ __forceinline__ void add(const GroupTableDev& global, int32_t g0, int32_t g1, i128 v, bool is64);
   __device__ __forceinline__ void flush(const GroupTableDev& global, bool is64);
};

__device__ __forceinline__ void LocalGroups::add(const GroupTableDev& global, int32_t g0, int32_t g1, i128 v, bool is64) {
   const unsigned long long packed = packSlot(g0, g1);
   if (packed != kEmptySlot) {
      uint32_t s = (uint32_t) hashPair(g0, g1) & (kLocalGroups - 1);
      for (int probes = 0; probes < kLocalGroups; probes++) {
         unsigned long long cur = *((volatile unsigned long long*) &key[s]);
         if (cur == kEmptySlot) cur = atomicCAS(&key[s], kEmptySlot, packed);
         if (cur == kEmptySlot || cur == packed) {
            if (is64) atomicAdd(&acc[s][0], (unsigned long long) v.lo);
            else atomicAdd128(&acc[s][0], &acc[s][1], v);
            return;
         }
         s = (s + 1) & (kLocalGroups - 1);
      }
   }
   int32_t kk[2] = {g0, g1};
   int slot = groupLookupOrInsert(global, kk);
   if (slot >= 0) groupAtomicAdd(global, slot, 0, v, is64);
}
__device__ __forceinline__ void LocalGroups::flush(const GroupTableDev& global, bool is64) {
   for (int i = threadIdx.x; i < kLocalGroups; i += blockDim.x) {
      const unsigned long long k = key[i];
      if (k == kEmptySlot) continue;
      const i128 v{acc[i][0], (int64_t) acc[i][1]};
      int32_t kk[2] = {(int32_t) (uint32_t) k, (int32_t) (uint32_t) (k >> 32)};
      int slot = groupLookupOrInsert(global, kk);
      if (slot >= 0) groupAtomicAdd(global, slot, 0, v, is64);
   }
}

// one atomic per warp for the build-side entry count
__device__ __forceinline__ void flushInsertCount(const JoinTableDev& t, unsigned long long local) {
   __syncwarp();
   unsigned long long total = warpSum64(local);
   if ((threadIdx.x & 31) == 0 && total) atomicAdd(t.count, total);
}

// =================================================================================== K3 build
// scan → filters → [probe parent table] → insert {key, payload, side…}
// (subop.materialize + rt::GrowingBuffer::insert + rt::HashIndexedView::build; for the group-join
//  the lookup_or_insert of the left input, RelAlgToSubOp.cpp:2682-2950)
template <int DB, int RPT, int NS, int FS = FS_GENERIC>
__global__ void __launch_bounds__(kBlock, 4) scanBuildKernel(const __grid_constant__ BuildParams p) {
   constexpr bool IN = true; // latency-bound kernels keep the IN path in
   __shared__ __align__(8) TileBarriers barsStorage;
   __shared__ SurvivorQueue<5, RPT> queue; // {probe key, build key, own payload, side0, side1}
   TileBarriers* bars = &barsStorage;
   if (threadIdx.x == 0) queue.count = 0;
   __syncthreads();
   unsigned long long inserted = 0;
   auto insert = [&](int32_t key, int32_t payload, int32_t side0, int32_t side1) {
      if (p.sink.direct) {
         if (directInsert(p.sink, key, payload) >= 0) inserted++;
         return;
      }
      int64_t slot = joinInsert(p.sink, key, payload);
      if (slot >= 0) {
         inserted++;
         int32_t* lanes = (int32_t*) (p.sink.base + (uint64_t) slot * 32 + 8); // side0, side1 of the 32-byte entry
         if (p.nSide > 0) lanes[0] = side0;
         if (p.nSide > 1) lanes[1] = side1;
      }
   };
   auto process = [&](int q) { // a queued row: walk the parent's directory, insert once per match
      const int32_t probeKey = queue.w[0][q];
      if (p.probe.unique) {
         // at most one match: finish the walk first, then insert with the warp converged again — inside the walk the insert's CAS
         // retries ran once per (walk step x retry) group of lanes, ~8 dependent HBM round trips per warp with 5 lanes active on
         // average (a large share of K3's stall samples sat behind that CAS)
         bool found = false;
         int32_t parent = 0;
         joinProbeSlots(p.probe, probeKey, hashI32(probeKey), [&](int64_t, int32_t parentPayload) {
            found = true;
            parent = parentPayload;
         });
         if (found) insert(queue.w[1][q], p.payloadStage >= 0 ? queue.w[2][q] : (int32_t) (parent & (p.probe.stride == 32 ? 0x7fffffff : -1)), queue.w[3][q], queue.w[4][q]);
         return;
      }
      joinProbeSlots(p.probe, probeKey, hashI32(probeKey), [&](int64_t, int32_t parentPayload) {
         insert(queue.w[1][q], p.payloadStage >= 0 ? queue.w[2][q] : (int32_t) (parentPayload & (p.probe.stride == 32 ? 0x7fffffff : -1)), queue.w[3][q], queue.w[4][q]);
      });
   };
   forEachTileUniform<RPT, DB, NS>(p.src.cols, p.src.nRows, dynSmem, bars, [&](const auto& tile, int64_t rowBase, int rows) {
#pragma unroll
      for (int j = 0; j < RPT; j++) {
         const int lrRaw = j * kBlock + threadIdx.x;
         const bool valid = lrRaw < rows;
         const int lr = valid ? lrRaw : 0;
         const bool ok = valid && evalFilters<IN, FS>(p.src.filters, tile, lr, rowBase + lr);
         const int32_t key = tile.i32(p.keyStage, lr);
         int32_t ownPayload = p.payloadStage >= 0 ? tile.i32(p.payloadStage, lr) : 0;
         if (p.payloadKind == PAYLOAD_YEAR_OF_DATE32) ownPayload = yearOfDays(ownPayload); // extract(year from <date32 column>)
         const int32_t side0 = p.nSide > 0 ? tile.i32(p.sideStage[0], lr) : 0, side1 = p.nSide > 1 ? tile.i32(p.sideStage[1], lr) : 0;
         if (!p.hasProbe) { // plain build: every row that passed the filters inserts — nothing to compact
            if (ok) insert(key, ownPayload, side0, side1);
            continue;
         }
         const int32_t probeKey = tile.i32(p.probeKeyStage, lr);
         if (bloomPrefetch(p.probe, probeKey, ok).mayContain()) {
            const int q = queue.claim();
            queue.w[0][q] = probeKey;
            queue.w[1][q] = key;
            queue.w[2][q] = ownPayload;
            queue.w[3][q] = side0;
            queue.w[4][q] = side1;
         }
      }
      if (p.hasProbe) {
         __syncthreads();
         drainQueue(queue, false, process);
      }
   });
   __syncthreads();
   drainQueue(queue, true, process);
   flushInsertCount(p.sink, inserted);
}
// composite-key build: {key, key2} → int64 payload (a decimal(p<19) column's value or an int32 column), optionally
// restricted to rows whose probe key exists in a parent table (Q9: partsupp ⋈ part(p_name like '%green%'))
template <int DB>
__global__ void __launch_bounds__(kThreads, 4) scanBuildPairKernel(const __grid_constant__ BuildParams p) {
   constexpr bool IN = true;
   __shared__ __align__(8) TileBarriers barsStorage;
   TileBarriers* bars = &barsStorage;
   unsigned long long inserted = 0;
   forEachRow<kRowsPerThreadStar, DB>(p.src.cols, p.src.nRows, dynSmem, bars, [&](const auto& tile, int lr, int64_t row, bool valid) {
      if (!(valid && evalFilters<IN>(p.src.filters, tile, lr, row))) return;
      const int32_t k0 = tile.i32(p.keyStage, lr), k1 = tile.i32(p.keyStage2, lr);
      int64_t payload = 0;
      if (p.payloadStage >= 0) payload = p.payloadKind == PAYLOAD_DEC_LO64 ? tile.lo64(p.payloadStage, lr) : (int64_t) tile.i32(p.payloadStage, lr);
      if (p.hasProbe) {
         joinProbe(p.probe, tile.i32(p.probeKeyStage, lr), [&](int64_t, int32_t) {
            if (pairInsert(p.sink, k0, k1, payload) >= 0) inserted++;
         });
      } else if (pairInsert(p.sink, k0, k1, payload) >= 0) {
         inserted++;
      }
   });
   flushInsertCount(p.sink, inserted);
}
void launchScanBuild(const BuildParams& p, int smCount, cudaStream_t s) {
   size_t dyn;
   if (p.sink.stride == 16) {
      if (p.src.cols.decBytes == 8) {
         int grid = persistentGrid(scanBuildPairKernel<8>, p.src.cols, p.src.nRows, smCount, &dyn);
         scanBuildPairKernel<8><<<grid, kThreads, dyn, s>>>(p);
      } else {
         int grid = persistentGrid(scanBuildPairKernel<16>, p.src.cols, p.src.nRows, smCount, &dyn);
         scanBuildPairKernel<16><<<grid, kThreads, dyn, s>>>(p);
      }
      return;
   }
   // (RPT, NS) from tuning(): the host bound the tiles with the same rows-per-thread (runtime.cpp)
   const int rpt = tuning().rptBuild, ns = tuning().stagesBuild;
#define LDB_BUILD_CASE(DBV, RPTV, NSV)                                                                                          \
   if (rpt == RPTV && ns == NSV) {                                                                                              \
      int grid = persistentGrid(scanBuildKernel<DBV, RPTV, NSV>, p.src.cols, p.src.nRows, smCount, &dyn, kBlock, NSV);          \
      scanBuildKernel<DBV, RPTV, NSV><<<grid, kBlock, dyn, s>>>(p);                                                             \
      return;                                                                                                                   \
   }
   // filter-shape instantiations: tuned tile shape (2 rows per thread, 3 stages) only
   const int fs = rpt == 2 && ns == 3 ? filterShape(p.src.filters) : FS_GENERIC;
#define LDB_BUILD_FS(DBV, FSV)                                                                                                  \
   if (p.src.cols.decBytes == DBV && fs == FSV) {                                                                               \
      int grid = persistentGrid(scanBuildKernel<DBV, 2, 3, FSV>, p.src.cols, p.src.nRows, smCount, &dyn, kBlock, 3);            \
      scanBuildKernel<DBV, 2, 3, FSV><<<grid, kBlock, dyn, s>>>(p);                                                             \
      return;                                                                                                                   \
   }
   LDB_BUILD_FS(16, FS_NONE) LDB_BUILD_FS(16, FS_I32_ONE) LDB_BUILD_FS(16, FS_I32_RANGE) LDB_BUILD_FS(8, FS_NONE) LDB_BUILD_FS(8, FS_I32_ONE) LDB_BUILD_FS(8, FS_I32_RANGE)
#undef LDB_BUILD_FS
   if (p.src.cols.decBytes == 8) {
      LDB_BUILD_CASE(8, 1, 2) LDB_BUILD_CASE(8, 2, 2) LDB_BUILD_CASE(8, 4, 2) LDB_BUILD_CASE(8, 1, 3) LDB_BUILD_CASE(8, 2, 3) LDB_BUILD_CASE(8, 4, 3)
      LDB_BUILD_CASE(8, 1, 4) LDB_BUILD_CASE(8, 2, 4) LDB_BUILD_CASE(8, 4, 4)
   } else {
      LDB_BUILD_CASE(16, 1, 2) LDB_BUILD_CASE(16, 2, 2) LDB_BUILD_CASE(16, 4, 2) LDB_BUILD_CASE(16, 1, 3) LDB_BUILD_CASE(16, 2, 3) LDB_BUILD_CASE(16, 4, 3)
      LDB_BUILD_CASE(16, 1, 4) LDB_BUILD_CASE(16, 2, 4) LDB_BUILD_CASE(16, 4, 4)
   }
#undef LDB_BUILD_CASE
}

// =================================================================================== K8 materialize
// scan → filters → [probe / Bloom-only semi-join] → append the selected columns, compacted, to dense buffers
// (subop.materialize; the reference appends row tuples to per-worker GrowingBuffers, GrowingBuffer.cpp:44 —
//  here one warp-aggregated atomic claims the output range of all emitting lanes).
__device__ __forceinline__ bool bloomMayContain(const JoinTableDev& t, int32_t key) {
   if (!t.bloom) return true;
   const uint64_t h = hashI32(key);
   const uint32_t bits = bloomBits(h);
   return (ldBloom(t, (uint32_t) (h >> 32) & t.bloomMask) & bits) == bits;
}
// Two instantiations: MULTI = false (no probe, Bloom-only semi-join, or a unique-key probe: at most one output per row) claims
// the output range of a whole TILE with one global atomic (CTA-wide prefix sum of the emit flags) — with a single counter,
// one atomic per warp-row cost 11.8 ms on the 600 M-row lineitem scan, 2.3x the scan itself; MULTI = true (non-unique build
// keys, any number of matches per row) keeps the warp-aggregated claim.
template <int DB, bool MULTI>
__global__ void __launch_bounds__(MULTI ? kThreads : kBlock, 4) scanMaterializeKernel(const __grid_constant__ MaterializeParams p) {
   constexpr bool IN = true;
   __shared__ __align__(8) TileBarriers barsStorage;
   TileBarriers* bars = &barsStorage;
   auto writeRow = [&](const auto& tile, int lr, unsigned long long pos, int32_t payload) {
      if (pos >= (unsigned long long) p.capacity) return;
      for (int c = 0; c < p.nOut; c++) {
         if (p.outStage[c] < 0) {
            ((int32_t*) p.out[c])[pos] = payload;
         } else if (p.outElem[c] == 4) {
            ((int32_t*) p.out[c])[pos] = tile.i32(p.outStage[c], lr);
         } else {
            longlong2 v;
            v.x = tile.lo64(p.outStage[c], lr);
            v.y = tile.hi64(p.outStage[c], lr);
            ((longlong2*) p.out[c])[pos] = v;
         }
      }
   };
   if constexpr (MULTI) {
      forEachRow<kRowsPerThreadProbe, DB>(p.src.cols, p.src.nRows, dynSmem, bars, [&](const auto& tile, int lr, int64_t row, bool valid) {
         if (!(valid && evalFilters<IN>(p.src.filters, tile, lr, row))) return;
         joinProbe(p.probe, tile.i32(p.probeKeyStage, lr), [&](int64_t, int32_t payload) {
            const unsigned active = __activemask();
            const int lane = threadIdx.x & 31, leader = __ffs(active) - 1;
            unsigned long long base = 0;
            if (lane == leader) base = atomicAdd(p.count, (unsigned long long) __popc(active));
            base = __shfl_sync(active, base, leader);
            writeRow(tile, lr, base + __popc(active & ((1u << lane) - 1)), payload);
         });
      });
   } else {
      __shared__ unsigned int warpTotals[kWarps];
      __shared__ unsigned long long tileBase;
      forEachTileUniform<kRowsPerThreadProbe, DB>(p.src.cols, p.src.nRows, dynSmem, bars, [&](const auto& tile, int64_t rowBase, int rows) {
         const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
         bool emit[kRowsPerThreadProbe];
         int32_t payload[kRowsPerThreadProbe];
         int lrs[kRowsPerThreadProbe];
         unsigned ballots[kRowsPerThreadProbe];
         unsigned total = 0;
#pragma unroll
         for (int j = 0; j < kRowsPerThreadProbe; j++) {
            const int lr = j * kBlock + threadIdx.x;
            const bool valid = lr < rows;
            lrs[j] = valid ? lr : 0;
            bool ok = valid && evalFilters<IN>(p.src.filters, tile, lrs[j], rowBase + lrs[j]);
            payload[j] = 0;
            if (ok && p.hasProbe) {
               const int32_t key = tile.i32(p.probeKeyStage, lrs[j]);
               if (p.bloomOnly) {
                  ok = bloomMayContain(p.probe, key);
               } else {
                  bool found = false;
                  joinProbe(p.probe, key, [&](int64_t, int32_t pay) {
                     found = true;
                     payload[j] = pay;
                  });
                  ok = found;
               }
            }
            emit[j] = ok;
            ballots[j] = __ballot_sync(0xffffffffu, ok);
            total += __popc(ballots[j]);
         }
         if (lane == 0) warpTotals[warp] = total;
         __syncthreads();
         if (threadIdx.x == 0) {
            unsigned sum = 0;
            for (int w = 0; w < kWarps; w++) sum += warpTotals[w];
            tileBase = sum ? atomicAdd(p.count, (unsigned long long) sum) : 0ull; // ONE global atomic per tile
         }
         __syncthreads();
         unsigned long long pos = tileBase;
         for (int w = 0; w < warp; w++) pos += warpTotals[w];
#pragma unroll
         for (int j = 0; j < kRowsPerThreadProbe; j++) {
            if (emit[j]) writeRow(tile, lrs[j], pos + __popc(ballots[j] & ((1u << lane) - 1)), payload[j]);
            pos += __popc(ballots[j]);
         }
         __syncthreads(); // warpTotals / tileBase are reused by the next tile
      });
   }
}
template <int DB>
static void launchMat(const MaterializeParams& p, int smCount, cudaStream_t s) {
   size_t dyn;
   const bool multi = p.hasProbe && !p.bloomOnly && !p.probe.unique;
   if (multi) {
      int grid = persistentGrid(scanMaterializeKernel<DB, true>, p.src.cols, p.src.nRows, smCount, &dyn);
      scanMaterializeKernel<DB, true><<<grid, kThreads, dyn, s>>>(p);
   } else {
      int grid = persistentGrid(scanMaterializeKernel<DB, false>, p.src.cols, p.src.nRows, smCount, &dyn, kBlock);
      scanMaterializeKernel<DB, false><<<grid, kBlock, dyn, s>>>(p);
   }
}
void launchScanMaterialize(const MaterializeParams& p, int smCount, cudaStream_t s) {
   if (p.src.cols.decBytes == 8) launchMat<8>(p, smCount, s);
   else launchMat<16>(p, smCount, s);
}

// =================================================================================== K5 probe + aggregate
// (K4 and K5 handle their survivors IN PLACE under the warp-specialised driver: measured against the survivor-queue form
//  at SF100, K5 4.27 vs 5.13 ms and K4 5.2 vs 5.9 ms — their dependent part is one directory walk plus an atomic, too short
//  to pay for a CTA barrier per 256-row tile; K3-with-probe and K9, whose chains are long, gain 1.8x / 2.9x from the queue.)
// scan → filters → pure lookup in the group-join map → SUM into the shared entry.  The reference
// takes a per-entry spin lock (SubOpToControlFlow.cpp:4218-4251, EntryLock.cpp:9-25) or an
// atomic_rmw; here the i128 SUM is two 64-bit atomics with carry (exact, order independent).
template <int NV, int DB, int NS, int FS = FS_GENERIC>
__global__ void __launch_bounds__(kThreads, FS == FS_GENERIC ? 4 : 5) scanProbeAggKernel(const __grid_constant__ ProbeAggParams p) {
   constexpr bool IN = true;
   __shared__ __align__(8) TileBarriers barsStorage;
   TileBarriers* bars = &barsStorage;
   const int64_t one = 100;
   forEachTile<kRowsPerThreadProbe, DB, NS>(p.src.cols, p.src.nRows, dynSmem, bars, [&](const auto& tile, int64_t rowBase, int rows) {
      int32_t key[kRowsPerThreadProbe];
      int lrs[kRowsPerThreadProbe];
      BloomProbe bp[kRowsPerThreadProbe];
      // phase A: filters + hash + Bloom load of every row of this thread (all loads in flight together)
#pragma unroll
      for (int j = 0; j < kRowsPerThreadProbe; j++) {
         const int lr = j * kBlock + threadIdx.x;
         const bool valid = lr < rows;
         lrs[j] = valid ? lr : 0;
         const bool ok = valid && evalFilters<IN, FS>(p.src.filters, tile, lrs[j], rowBase + lrs[j]);
         key[j] = tile.i32(p.probeKeyStage, lrs[j]);
         bp[j] = bloomPrefetch(p.table, key[j], ok);
      }
      // phase B: the few survivors walk the directory and add into the shared entry
#pragma unroll
      for (int j = 0; j < kRowsPerThreadProbe; j++) {
         if (!bp[j].mayContain()) continue;
         auto add = [&](int64_t slot, int32_t payloadWord) {
            int64_t vals[NV];
#pragma unroll
            for (int c = 0; c < NV; c++) vals[c] = lazyLo64(p.values, c, rowBase + lrs[j]);
            i128 v = evalAggDyn(p.agg, vals, one);
            uint8_t* entry = p.table.base + (uint64_t) slot * 32;
            atomicAdd128((unsigned long long*) (entry + 16), (unsigned long long*) (entry + 24), v);
            if (payloadWord >= 0) ((int32_t*) entry)[1] = payloadWord | (int32_t) 0x80000000; // marker: idempotent plain store, same sector
         };
         if (p.table.unique) { // one match at most: finish the directory walk, then fetch the operands and add with the lanes converged
            int64_t slot = -1;
            int32_t word = 0;
            joinProbeSlots<true>(p.table, key[j], bp[j].h, [&](int64_t s, int32_t payloadWord) {
               slot = s;
               word = payloadWord;
            });
            if (slot >= 0) add(slot, word);
         } else {
            joinProbeSlots<true>(p.table, key[j], bp[j].h, add);
         }
      }
   });
}
bool launchScanProbeAgg(const ProbeAggParams& p, int smCount, cudaStream_t s, const char** why) {
   int nv = p.agg.expr == LDB_EXPR_COL ? 1 : p.agg.expr == LDB_EXPR_MUL_1MINUS_1PLUS ? 3 : 2;
   if (p.agg.col[0] != 0 || (nv > 1 && p.agg.col[1] != 1) || (nv > 2 && p.agg.col[2] != 2)) {
      *why = "probe-aggregate pipeline expects value columns in expression order";
      return false;
   }
   size_t dyn;
   const int ns = tuning().stagesProbeAgg;
#define LDB_PA_CASE(NVV, DBV, NSV)                                                                                   \
   if (nv == NVV && p.src.cols.decBytes == DBV && ns == NSV) {                                                       \
      int grid = persistentGrid(scanProbeAggKernel<NVV, DBV, NSV>, p.src.cols, p.src.nRows, smCount, &dyn, kThreads, NSV); \
      scanProbeAggKernel<NVV, DBV, NSV><<<grid, kThreads, dyn, s>>>(p);                                              \
      return true;                                                                                                   \
   }
   // filter-shape instantiations exist for the tuned pipeline depth only; everything else runs descriptor-driven
   const int fs = ns == 3 ? filterShape(p.src.filters) : FS_GENERIC;
#define LDB_PA_FS(NVV, DBV, FSV)                                                                                             \
   if (nv == NVV && p.src.cols.decBytes == DBV && fs == FSV) {                                                               \
      int grid = persistentGrid(scanProbeAggKernel<NVV, DBV, 3, FSV>, p.src.cols, p.src.nRows, smCount, &dyn, kThreads, 3); \
      scanProbeAggKernel<NVV, DBV, 3, FSV><<<grid, kThreads, dyn, s>>>(p);                                                   \
      return true;                                                                                                           \
   }
#define LDB_PA_FS_ALL(NVV, DBV) LDB_PA_FS(NVV, DBV, FS_NONE) LDB_PA_FS(NVV, DBV, FS_I32_ONE) LDB_PA_FS(NVV, DBV, FS_I32_RANGE)
   LDB_PA_FS_ALL(1, 8) LDB_PA_FS_ALL(1, 16) LDB_PA_FS_ALL(2, 8) LDB_PA_FS_ALL(2, 16) LDB_PA_FS_ALL(3, 8) LDB_PA_FS_ALL(3, 16)
#undef LDB_PA_FS_ALL
#undef LDB_PA_FS
#define LDB_PA_ALL(NVV, DBV) LDB_PA_CASE(NVV, DBV, 2) LDB_PA_CASE(NVV, DBV, 3) LDB_PA_CASE(NVV, DBV, 4)
   LDB_PA_ALL(1, 8) LDB_PA_ALL(1, 16) LDB_PA_ALL(2, 8) LDB_PA_ALL(2, 16) LDB_PA_ALL(3, 8) LDB_PA_ALL(3, 16)
#undef LDB_PA_ALL
#undef LDB_PA_CASE
   *why = "no probe-aggregate instantiation for this shape";
   return false;
}

// =================================================================================== K4 probe, probe, group
// scan → probe A on keyA → probe B on keyB → keep rows whose payloads agree (the composite join key
// (l_suppkey, c_nationkey) = (s_suppkey, s_nationkey) of Q5) → group by that payload → SUM.
template <int NV, int DB, int NS, int FS = FS_GENERIC>
__global__ void __launch_bounds__(kThreads, FS == FS_GENERIC ? 4 : 5) scanProbe2GroupByKernel(const __grid_constant__ Probe2GroupByParams p) {
   constexpr bool IN = true;
   __shared__ __align__(8) TileBarriers barsStorage;
   TileBarriers* bars = &barsStorage;
   const int64_t one = 100;
   forEachTile<kRowsPerThreadProbe, DB, NS>(p.src.cols, p.src.nRows, dynSmem, bars, [&](const auto& tile, int64_t rowBase, int rows) {
      int32_t key[kRowsPerThreadProbe];
      int lrs[kRowsPerThreadProbe];
      BloomProbe bp[kRowsPerThreadProbe];
#pragma unroll
      for (int j = 0; j < kRowsPerThreadProbe; j++) { // phase A: Bloom filter of table A for every row (loads in flight together)
         const int lr = j * kBlock + threadIdx.x;
         const bool valid = lr < rows;
         lrs[j] = valid ? lr : 0;
         const bool ok = valid && evalFilters<IN, FS>(p.src.filters, tile, lrs[j], rowBase + lrs[j]);
         key[j] = tile.i32(p.keyStageA, lrs[j]);
         bp[j] = bloomPrefetch(p.tableA, key[j], ok);
      }
      int32_t keyB[kRowsPerThreadProbe];
      BloomProbe bpB[kRowsPerThreadProbe];
#pragma unroll
      for (int j = 0; j < kRowsPerThreadProbe; j++) { // phase B: survivors consult table B's filter (the plan puts the smaller table first)
         keyB[j] = tile.i32(p.keyStageB, lrs[j]);
         bpB[j] = bloomPrefetch(p.tableB, keyB[j], bp[j].mayContain());
      }
#pragma unroll
      for (int j = 0; j < kRowsPerThreadProbe; j++) { // phase C: the few rows both filters let through walk the directories
         if (!bpB[j].mayContain()) continue;
         joinProbeSlots(p.tableA, key[j], bp[j].h, [&](int64_t, int32_t payA) {
            joinProbeSlots(p.tableB, keyB[j], bpB[j].h, [&](int64_t, int32_t payB) {
               // bit 31 of a wide entry is the group-join marker, not payload: each side drops its own marker before the compare
               const int32_t a = p.tableA.stride == 32 ? (payA & 0x7fffffff) : payA, b = p.tableB.stride == 32 ? (payB & 0x7fffffff) : payB;
               if (a != b) return;
               int64_t vals[NV];
#pragma unroll
               for (int c = 0; c < NV; c++) vals[c] = lazyLo64(p.values, c, rowBase + lrs[j]);
               int32_t kk[2] = {b, 0};
               int slot = groupLookupOrInsert(p.groups, kk);
               if (slot >= 0) groupAtomicAdd(p.groups, slot, 0, evalAggDyn(p.agg, vals, one), p.agg.expr == LDB_EXPR_COL || p.agg.expr == LDB_EXPR_ONE);
            });
         });
      }
   });
}
bool launchScanProbe2GroupBy(const Probe2GroupByParams& p, int smCount, cudaStream_t s, const char** why) {
   int nv = p.agg.expr == LDB_EXPR_COL ? 1 : p.agg.expr == LDB_EXPR_MUL_1MINUS_1PLUS ? 3 : 2;
   if (p.agg.col[0] != 0 || (nv > 1 && p.agg.col[1] != 1) || (nv > 2 && p.agg.col[2] != 2)) {
      *why = "probe-probe-group pipeline expects value columns in expression order";
      return false;
   }
   size_t dyn;
   const int ns = tuning().stagesProbe2;
#define LDB_P2_CASE(NVV, DBV, NSV)                                                                                        \
   if (nv == NVV && p.src.cols.decBytes == DBV && ns == NSV) {                                                            \
      int grid = persistentGrid(scanProbe2GroupByKernel<NVV, DBV, NSV>, p.src.cols, p.src.nRows, smCount, &dyn, kThreads, NSV); \
      scanProbe2GroupByKernel<NVV, DBV, NSV><<<grid, kThreads, dyn, s>>>(p);                                              \
      return true;                                                                                                        \
   }
   const int fs = ns == 3 ? filterShape(p.src.filters) : FS_GENERIC; // shape instantiations: tuned depth only
#define LDB_P2_FS(NVV, DBV, FSV)                                                                                                  \
   if (nv == NVV && p.src.cols.decBytes == DBV && fs == FSV) {                                                                    \
      int grid = persistentGrid(scanProbe2GroupByKernel<NVV, DBV, 3, FSV>, p.src.cols, p.src.nRows, smCount, &dyn, kThreads, 3); \
      scanProbe2GroupByKernel<NVV, DBV, 3, FSV><<<grid, kThreads, dyn, s>>>(p);                                                   \
      return true;                                                                                                                \
   }
#define LDB_P2_FS_ALL(NVV, DBV) LDB_P2_FS(NVV, DBV, FS_NONE) LDB_P2_FS(NVV, DBV, FS_I32_ONE) LDB_P2_FS(NVV, DBV, FS_I32_RANGE)
   LDB_P2_FS_ALL(1, 8) LDB_P2_FS_ALL(1, 16) LDB_P2_FS_ALL(2, 8) LDB_P2_FS_ALL(2, 16) LDB_P2_FS_ALL(3, 8) LDB_P2_FS_ALL(3, 16)
#undef LDB_P2_FS_ALL
#undef LDB_P2_FS
#define LDB_P2_ALL(NVV, DBV) LDB_P2_CASE(NVV, DBV, 2) LDB_P2_CASE(NVV, DBV, 3) LDB_P2_CASE(NVV, DBV, 4)
   LDB_P2_ALL(1, 8) LDB_P2_ALL(1, 16) LDB_P2_ALL(2, 8) LDB_P2_ALL(2, 16) LDB_P2_ALL(3, 8) LDB_P2_ALL(3, 16)
#undef LDB_P2_ALL
#undef LDB_P2_CASE
   *why = "no probe-probe-group instantiation for this shape";
   return false;
}

// =================================================================================== K9 star probe, group
// scan → probe P on the composite key (Bloom first: Q9 keeps 5 % of lineitem) → probe S → probe O → group by the two
// int32 payloads → SUM(a * (1 - b) - c * d), c = P's int64 payload.  The reference's per-worker pre-aggregation
// cache (PreAggregationHashtable.cpp:46-60) becomes a per-CTA shared-memory table flushed once per CTA: ~10^8 matched
// rows over 175 groups would otherwise serialise on 175 HBM addresses.
// Survivor queue of bounded size: a claim beyond the capacity is handled in place by its owner (only non-selective inputs get
// there), so the queue — and with it the CTA's shared memory — stays small and more CTAs are resident.
struct StarQueue {
   static constexpr int kCap = 3 * kBlock;
   int32_t w[6][kCap]; // k0, k1, kS, kO, row lo, row hi
   int count;
};
template <int DB, int RPT, int NS, int FS = FS_GENERIC>
__global__ void __launch_bounds__(kBlock, 4) scanStarProbeGroupByKernel(const __grid_constant__ StarProbeParams p) {
   constexpr bool IN = true;
   __shared__ __align__(8) TileBarriers barsStorage;
   __shared__ StarQueue queue;
   __shared__ LocalGroups groups;
   TileBarriers* bars = &barsStorage;
   groups.init();
   if (threadIdx.x == 0) queue.count = 0;
   __syncthreads();
   const int64_t one = 100;
   // the three probes of a row and its three operand loads are independent of each other: all first loads are issued together
   // (S and O are foreign-key probes that always hit, so their Bloom filters are not consulted)
   auto handle = [&](int32_t k0, int32_t k1, int32_t kS, int32_t kO, int64_t row) {
      // (the third probe's key rides in the tiles although only P's survivors need it: fetching it per survivor — one sector instead of
      //  4 B of every row — measured 5.42 vs 5.40 ms at SF100, the dependent load costs what the smaller tile saves)
      const uint64_t hP = hashPair(k0, k1), hS = p.tableS.direct ? 0 : hashI32(kS), hO = p.tableO.direct ? 0 : hashI32(kO);
      const ulonglong2 eP = __ldg((const ulonglong2*) slotPtr(p.tableP, hP & p.tableP.mask));
      const unsigned long long eS = fkFirstSlot(p.tableS, kS, hS), eO = fkFirstSlot(p.tableO, kO, hO);
      const int64_t a = lazyLo64(p.values, 0, row), b = lazyLo64(p.values, 1, row), d = lazyLo64(p.values, 2, row);
      pairProbeFrom(p.tableP, k0, k1, hP, eP, [&](int64_t c) {
         fkProbeFrom(p.tableS, kS, hS, eS, [&](int32_t g0) {
            fkProbeFrom(p.tableO, kO, hO, eO, [&](int32_t g1) { groups.add(p.groups, g0, g1, sub128(mul64x64(a, one - b), mul64x64(c, d)), false); });
         });
      });
   };
   auto process = [&](int q) {
      handle(queue.w[0][q], queue.w[1][q], queue.w[2][q], queue.w[3][q], (int64_t) (((uint64_t) (uint32_t) queue.w[5][q] << 32) | (uint32_t) queue.w[4][q]));
   };
   forEachTileUniform<RPT, DB, NS>(p.src.cols, p.src.nRows, dynSmem, bars, [&](const auto& tile, int64_t rowBase, int rows) {
      int32_t k0[RPT], k1[RPT];
      int lrs[RPT];
      BloomProbe bp[RPT];
#pragma unroll
      for (int j = 0; j < RPT; j++) { // filters + P's Bloom word of every row of this thread: RPT loads in flight per thread
         const int lrRaw = j * kBlock + threadIdx.x;
         const bool valid = lrRaw < rows;
         lrs[j] = valid ? lrRaw : 0;
         const bool ok = valid && evalFilters<IN, FS>(p.src.filters, tile, lrs[j], rowBase + lrs[j]);
         k0[j] = tile.i32(p.keyStageP0, lrs[j]);
         k1[j] = tile.i32(p.keyStageP1, lrs[j]);
         bp[j] = pairBloomPrefetch(p.tableP, k0[j], k1[j], ok);
      }
#pragma unroll
      for (int j = 0; j < RPT; j++) { // survivors join the queue (or, if it is full, are handled in place)
         if (!bp[j].mayContain()) continue;
         const int32_t kS = tile.i32(p.keyStageS, lrs[j]), kO = tile.i32(p.keyStageO, lrs[j]);
         const int64_t row = rowBase + lrs[j];
         const int q = atomicAdd(&queue.count, 1);
         if (q < StarQueue::kCap) {
            queue.w[0][q] = k0[j];
            queue.w[1][q] = k1[j];
            queue.w[2][q] = kS;
            queue.w[3][q] = kO;
            queue.w[4][q] = (int32_t) (uint32_t) (uint64_t) row;
            queue.w[5][q] = (int32_t) (uint32_t) ((uint64_t) row >> 32);
         } else {
            handle(k0[j], k1[j], kS, kO, row);
         }
      }
      __syncthreads();
      drainQueue(queue, false, process);
   });
   __syncthreads();
   drainQueue(queue, true, process);
   __syncthreads();
   groups.flush(p.groups, false);
}
bool launchScanStarProbeGroupBy(const StarProbeParams& p, int smCount, cudaStream_t s, const char** why) {
   size_t dyn;
   const int ns = tuning().stagesStar, rpt = tuning().rptStar;
#define LDB_STAR_CASE(DBV, RPTV, NSV)                                                                                          \
   if (p.src.cols.decBytes == DBV && rpt == RPTV && ns == NSV) {                                                               \
      int grid = persistentGrid(scanStarProbeGroupByKernel<DBV, RPTV, NSV>, p.src.cols, p.src.nRows, smCount, &dyn, kBlock, NSV); \
      scanStarProbeGroupByKernel<DBV, RPTV, NSV><<<grid, kBlock, dyn, s>>>(p);                                                 \
      return true;                                                                                                             \
   }
   // filter-shape instantiations: tuned tile shape (2 rows per thread, 2 stages) only
   const int fs = rpt == 2 && ns == 2 ? filterShape(p.src.filters) : FS_GENERIC;
#define LDB_STAR_FS(DBV, FSV)                                                                                                        \
   if (p.src.cols.decBytes == DBV && fs == FSV) {                                                                                    \
      int grid = persistentGrid(scanStarProbeGroupByKernel<DBV, 2, 2, FSV>, p.src.cols, p.src.nRows, smCount, &dyn, kBlock, 2);      \
      scanStarProbeGroupByKernel<DBV, 2, 2, FSV><<<grid, kBlock, dyn, s>>>(p);                                                       \
      return true;                                                                                                                   \
   }
   LDB_STAR_FS(16, FS_NONE) LDB_STAR_FS(16, FS_I32_ONE) LDB_STAR_FS(16, FS_I32_RANGE) LDB_STAR_FS(8, FS_NONE) LDB_STAR_FS(8, FS_I32_ONE) LDB_STAR_FS(8, FS_I32_RANGE)
#undef LDB_STAR_FS
   // the staged columns of a star probe are int32 keys only (the operands are late-materialised): decBytes stays at its default
   LDB_STAR_CASE(16, 1, 2) LDB_STAR_CASE(16, 2, 2) LDB_STAR_CASE(16, 4, 2) LDB_STAR_CASE(16, 1, 3) LDB_STAR_CASE(16, 2, 3) LDB_STAR_CASE(16, 4, 3)
   LDB_STAR_CASE(16, 1, 4) LDB_STAR_CASE(16, 2, 4) LDB_STAR_CASE(16, 4, 4)
   LDB_STAR_CASE(8, 1, 2) LDB_STAR_CASE(8, 2, 2) LDB_STAR_CASE(8, 4, 2) LDB_STAR_CASE(8, 1, 3) LDB_STAR_CASE(8, 2, 3) LDB_STAR_CASE(8, 4, 3)
   LDB_STAR_CASE(8, 1, 4) LDB_STAR_CASE(8, 2, 4) LDB_STAR_CASE(8, 4, 4)
#undef LDB_STAR_CASE
   *why = "no star-probe instantiation for this tile shape"; // a missing instantiation must not leave the group-by silently empty
   return false;
}

// =================================================================================== top-k over the group-join map
// Final scan of the map (marker == true) + Heap (include/lingodb/runtime/Heap.h): order by
// (agg desc, side0 asc, key asc).  Each CTA keeps its own top-k in shared memory; the host merges.
__device__ __forceinline__ bool topkBefore(const TopKRowDev& a, const TopKRowDev& b) {
   if (a.aggHi != b.aggHi) return a.aggHi > b.aggHi;
   if (a.aggLo != b.aggLo) return a.aggLo > b.aggLo;
   if (a.side0 != b.side0) return a.side0 < b.side0;
   return a.key < b.key;
}
constexpr int kTopKMax = 64;
// agg64: the aggregate lane holds a 64-bit SUM (LdbExprKind COL / ONE): its value is the low word, sign-extended — the high word only
// collected the carries of the two-word atomics.  It is normalised here, before the ranking and the threshold see it.
__global__ void __launch_bounds__(kBlock) joinTopKKernel(JoinTableDev t, int k, bool agg64, TopKRowDev* out) {
   __shared__ TopKRowDev best[kTopKMax];
   // Lock-free reject: once the CTA holds k rows, sThreshold is the k-th row's aggregate when that fits 64 unsigned bits (0 otherwise).
   // The k-th only ever improves, so a stale value is merely a weaker filter, and a single 64-bit shared word cannot be read torn: a
   // candidate with a non-negative 64-bit aggregate STRICTLY below it can never enter the top k, whatever the tie-breakers say.
   __shared__ unsigned long long sThreshold;
   __shared__ int sCount, sLock;
   if (threadIdx.x == 0) {
      sCount = 0;
      sLock = 0;
      sThreshold = 0;
   }
   __syncthreads();
   const uint64_t cap = t.mask + 1;
   auto consider = [&](const TopKRowDev& c) {
      if (c.aggHi == 0 && c.aggLo < *((volatile unsigned long long*) &sThreshold)) return;
      bool done = false;
      while (!done) {
         if (atomicCAS(&sLock, 0, 1) == 0) {
            __threadfence_block();
            int n = *((volatile int*) &sCount);
            int pos = n;
            while (pos > 0 && topkBefore(c, best[pos - 1])) pos--;
            if (pos < k) {
               int end = n < k ? n : k - 1;
               for (int i = end; i > pos; i--) best[i] = best[i - 1];
               best[pos] = c;
               const int n2 = n < k ? n + 1 : k;
               if (n2 == k) *((volatile unsigned long long*) &sThreshold) = best[k - 1].aggHi == 0 ? best[k - 1].aggLo : 0ull;
               if (n < k) *((volatile int*) &sCount) = n + 1;
            }
            __threadfence_block();
            atomicExch(&sLock, 0);
            done = true;
         }
      }
   };
   // The map is read once, after the probe kernel finished: kTopKUnroll whole entries (one 32-byte sector each, two 16-byte loads) are
   // in flight per thread — with one 8-byte load per thread per iteration the scan of the 1 GB Q3 map ran at 2.9 TB/s (0.37 ms at SF100)
   constexpr int kTopKUnroll = 8;
   for (uint64_t sBase = (uint64_t) blockIdx.x * kBlock * kTopKUnroll; sBase < cap; sBase += (uint64_t) gridDim.x * kBlock * kTopKUnroll) {
      uint4 lo[kTopKUnroll], hi[kTopKUnroll];
#pragma unroll
      for (int u = 0; u < kTopKUnroll; u++) {
         const uint64_t s = sBase + (uint64_t) u * kBlock + threadIdx.x;
         if (s < cap) {
            const uint4* entry = (const uint4*) (t.base + s * 32);
            lo[u] = __ldg(entry);
            hi[u] = __ldg(entry + 1);
         } else {
            lo[u] = make_uint4(0xffffffffu, 0xffffffffu, 0, 0); // kEmptySlot
            hi[u] = make_uint4(0, 0, 0, 0);
         }
      }
#pragma unroll
      for (int u = 0; u < kTopKUnroll; u++) {
         __syncwarp(); // re-converge after the previous candidate's try-lock
         if (lo[u].x == 0xffffffffu && lo[u].y == 0xffffffffu) continue;
         if (!(lo[u].y & 0x80000000u)) continue; // marker bit: the group saw at least one probe-side row
         TopKRowDev c;
         c.key = (int32_t) lo[u].x;
         c.side0 = (int32_t) lo[u].z;
         c.side1 = (int32_t) lo[u].w;
         c.valid = 1;
         c.aggLo = ((unsigned long long) hi[u].y << 32) | hi[u].x;
         c.aggHi = agg64 ? (long long) c.aggLo >> 63 : (long long) (((unsigned long long) hi[u].w << 32) | hi[u].z);
         consider(c);
      }
   }
   __syncthreads();
   for (int i = threadIdx.x; i < k; i += kBlock) {
      TopKRowDev r = best[i < sCount ? i : 0];
      if (i >= sCount) r.valid = 0;
      out[(size_t) blockIdx.x * k + i] = r;
   }
}
void launchJoinTopK(const JoinTableDev& t, int k, bool agg64, TopKRowDev* out, int* outBlocks, int smCount, cudaStream_t s) {
   int grid = smCount * 2;
   *outBlocks = grid;
   joinTopKKernel<<<grid, kBlock, 0, s>>>(t, k, agg64, out);
}

// 32-byte entries start as {empty marker, zero side lanes, zero aggregate}
__global__ void initWideTableKernel(uint8_t* base, uint64_t capacity) {
   for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < capacity; i += (uint64_t) gridDim.x * blockDim.x) {
      ulonglong4 v;
      v.x = kEmptySlot;
      v.y = v.z = v.w = 0;
      *(ulonglong4*) (base + i * 32) = v;
   }
}
void launchInitWideTable(uint8_t* base, uint64_t capacity, int smCount, cudaStream_t s) {
   int grid = (int) std::min<uint64_t>((capacity + 255) / 256, (uint64_t) smCount * 16);
   initWideTableKernel<<<grid < 1 ? 1 : grid, 256, 0, s>>>(base, capacity);
}

// =================================================================================== small helpers
__global__ void fill64Kernel(unsigned long long* p, unsigned long long v, int64_t n) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) p[i] = v;
}
void launchFill64(unsigned long long* p, unsigned long long v, int64_t n, int smCount, cudaStream_t s) {
   int grid = (int) std::min<int64_t>((n + 255) / 256, (int64_t) smCount * 8);
   if (grid < 1) grid = 1;
   fill64Kernel<<<grid, 256, 0, s>>>(p, v, n);
}
__global__ void insertTuplesKernel(JoinTableDev t, const int32_t* keys, const int32_t* payloads, const int32_t* side0, const int32_t* side1, int64_t n) {
   unsigned long long inserted = 0;
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      int64_t slot = joinInsert(t, keys[i], payloads ? payloads[i] : 0);
      if (slot >= 0) {
         inserted++;
         if (side0) ((int32_t*) (t.base + (uint64_t) slot * 32))[2] = side0[i];
         if (side1) ((int32_t*) (t.base + (uint64_t) slot * 32))[3] = side1[i];
      }
   }
   flushInsertCount(t, inserted);
}
void launchInsertTuples(const JoinTableDev& t, const int32_t* keys, const int32_t* payloads, const int32_t* side0, const int32_t* side1, int64_t n, int smCount, cudaStream_t s) {
   int grid = (int) std::min<int64_t>(std::max<int64_t>((n + 255) / 256, 1), (int64_t) smCount * 8);
   insertTuplesKernel<<<grid, 256, 0, s>>>(t, keys, payloads, side0, side1, n);
}
// min/max of an int32 column (the plan's density test for a direct-address table)
__global__ void columnRangeKernel(const int32_t* col, int64_t n, int32_t* minMax) {
   int32_t lo = INT32_MAX, hi = INT32_MIN;
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      const int32_t v = ldStream32(col + i);
      lo = v < lo ? v : lo;
      hi = v > hi ? v : hi;
   }
   for (int o = 16; o > 0; o >>= 1) {
      const int32_t l2 = __shfl_xor_sync(0xffffffffu, lo, o), h2 = __shfl_xor_sync(0xffffffffu, hi, o);
      lo = l2 < lo ? l2 : lo;
      hi = h2 > hi ? h2 : hi;
   }
   if ((threadIdx.x & 31) == 0) {
      atomicMin(&minMax[0], lo);
      atomicMax(&minMax[1], hi);
   }
}
void launchColumnRange(const int32_t* col, int64_t n, int32_t* minMax, int smCount, cudaStream_t s) {
   int grid = (int) std::min<int64_t>(std::max<int64_t>((n + 1023) / 1024, 1), (int64_t) smCount * 8);
   columnRangeKernel<<<grid, 256, 0, s>>>(col, n, minMax);
}
__global__ void hashI64Kernel(const int64_t* a, const int64_t* b, int64_t n, uint64_t* out) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      uint64_t h = hash64((uint64_t) a[i]);
      if (b) h = hashCombine(hash64((uint64_t) b[i]), h);
      out[i] = h;
   }
}
void launchHashI64(const int64_t* a, const int64_t* b, int64_t n, uint64_t* out, cudaStream_t s) {
   int grid = (int) std::min<int64_t>(std::max<int64_t>((n + 255) / 256, 1), 1024);
   hashI64Kernel<<<grid, 256, 0, s>>>(a, b, n, out);
}
// K7: fold partial groups (e.g. gathered from the other GPUs) into the table
__global__ void groupMergeRowsKernel(GroupTableDev t, const int32_t* keys, const unsigned long long* acc, int32_t nRows) {
   const int64_t total = (int64_t) nRows * t.nAggs;
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t) gridDim.x * blockDim.x) {
      const int64_t r = i / t.nAggs;
      const int a = (int) (i % t.nAggs);
      int32_t kk[2] = {keys[r * kMaxKeys], keys[r * kMaxKeys + 1]};
      int slot = groupLookupOrInsert(t, kk);
      if (slot < 0) continue;
      i128 v{acc[((size_t) r * kMaxAggs + a) * 2], (int64_t) acc[((size_t) r * kMaxAggs + a) * 2 + 1]};
      unsigned long long* dst = t.acc + ((size_t) slot * kMaxAggs + a) * 2;
      atomicAdd128(dst, dst + 1, v);
   }
}
void launchGroupMergeRows(const GroupTableDev& t, const int32_t* keys, const unsigned long long* acc, int32_t nRows, cudaStream_t s) {
   const int64_t total = (int64_t) nRows * t.nAggs;
   int grid = (int) std::max<int64_t>(1, std::min<int64_t>((total + 127) / 128, 256));
   groupMergeRowsKernel<<<grid, 128, 0, s>>>(t, keys, acc, nRows);
}

// K7 (multi-GPU): fold the all-gathered table images of the other ranks into this rank's table
__global__ void groupMergeImagesKernel(GroupTableDev t, const uint8_t* images, int nTables, int skip) {
   const size_t cap = (size_t) t.capacity;
   const size_t imageBytes = groupImageBytes(t.capacity);
   const int64_t total = (int64_t) nTables * t.capacity * t.nAggs;
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t) gridDim.x * blockDim.x) {
      const int a = (int) (i % t.nAggs);
      const int64_t slotIdx = (i / t.nAggs) % t.capacity;
      const int tab = (int) (i / ((int64_t) t.nAggs * t.capacity));
      if (tab == skip) continue;
      const uint8_t* img = images + (size_t) tab * imageBytes;
      const int32_t* st = (const int32_t*) img;
      if (t.nKeys != 0 && st[slotIdx] != 2) continue; // a keyless SimpleState has one always-occupied slot (its state word is never written)
      const int32_t* keys = (const int32_t*) (img + cap * 4) + (size_t) slotIdx * kMaxKeys;
      const unsigned long long* acc = (const unsigned long long*) (img + cap * 4 + cap * kMaxKeys * 4) + ((size_t) slotIdx * kMaxAggs + a) * 2;
      int32_t kk[2] = {keys[0], keys[1]};
      int slot = groupLookupOrInsert(t, kk);
      if (slot < 0) continue;
      unsigned long long* dst = t.acc + ((size_t) slot * kMaxAggs + a) * 2;
      atomicAdd128(dst, dst + 1, i128{acc[0], (int64_t) acc[1]});
   }
}
void launchGroupMergeImages(const GroupTableDev& t, const uint8_t* images, int nTables, int skip, cudaStream_t s) {
   const int64_t total = (int64_t) nTables * t.capacity * t.nAggs;
   int grid = (int) std::max<int64_t>(1, std::min<int64_t>((total + 127) / 128, 296));
   groupMergeImagesKernel<<<grid, 128, 0, s>>>(t, images, nTables, skip);
}

// =================================================================================== K6 radix partition
// dest = top bits of the reference hash (the low bits stay for the local directory, mirroring the
// reference's use of hash & 63 for its 64 partitions, PreAggregationHashtable.cpp:47-51)
// (explicit __umulhi: nvcc 12.9 folded `((h >> 32) * (uint64_t) n) >> 32` feeding a shared-memory index into a
//  32-bit IMAD that kept the LOW half — out-of-bounds shared atomics under compute-sanitizer)
__device__ __forceinline__ int partOf(int32_t key, int nParts) { return (int) __umulhi((uint32_t) (hashI32(key) >> 32), (uint32_t) nParts); }
__global__ void __launch_bounds__(kBlock) partitionHistogramKernel(const int32_t* keys, int64_t n, int nParts, unsigned long long* counts) {
   __shared__ unsigned int sCnt[64];
   for (int i = threadIdx.x; i < 64; i += kBlock) sCnt[i] = 0;
   __syncthreads();
   // lanes of a warp that go to the same partition share one shared-memory atomic (with 1..8 partitions a per-lane atomic is a
   // 4..32-way bank conflict: 22 ms for 20 M tuples)
   for (int64_t base = (int64_t) blockIdx.x * kBlock; base < n; base += (int64_t) gridDim.x * kBlock) {
      const int64_t i = base + threadIdx.x;
      const bool valid = i < n;
      const int part = valid ? partOf(ldStream32(keys + i), nParts) : -1;
      const unsigned active = __ballot_sync(0xffffffffu, valid);
      if (!valid) continue;
      const unsigned peers = __match_any_sync(active, part);
      if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&sCnt[part], (unsigned) __popc(peers));
   }
   __syncthreads();
   for (int i = threadIdx.x; i < nParts; i += kBlock)
      if (sCnt[i]) atomicAdd(&counts[i], (unsigned long long) sCnt[i]);
}
void launchPartitionHistogram(const int32_t* keys, int64_t n, int nParts, unsigned long long* counts, int smCount, cudaStream_t s) {
   int grid = (int) std::min<int64_t>(std::max<int64_t>((n + kBlock - 1) / kBlock, 1), (int64_t) smCount * 8);
   partitionHistogramKernel<<<grid, kBlock, 0, s>>>(keys, n, nParts, counts);
}
struct PartitionCols {
   const void* in[4];
   void* out[4];
   int32_t width[4];
   int32_t n;
};
__global__ void __launch_bounds__(kBlock) partitionScatterKernel(const int32_t* keys, PartitionCols cols, int64_t n, int nParts, unsigned long long* cursors, int32_t* outKeys) {
   // warp-aggregated claims: lanes going to the same partition share one atomic (__match_any_sync)
   for (int64_t base = (int64_t) blockIdx.x * kBlock; base < n; base += (int64_t) gridDim.x * kBlock) {
      int64_t i = base + threadIdx.x;
      bool valid = i < n;
      int32_t key = valid ? ldStream32(keys + i) : 0;
      int part = valid ? partOf(key, nParts) : -1;
      unsigned active = __ballot_sync(0xffffffffu, valid);
      if (!valid) continue;
      unsigned peers = __match_any_sync(active, part);
      int leader = __ffs(peers) - 1;
      int lane = threadIdx.x & 31;
      unsigned long long pos = 0;
      if (lane == leader) pos = atomicAdd(&cursors[part], (unsigned long long) __popc(peers));
      pos = __shfl_sync(peers, pos, leader) + __popc(peers & ((1u << lane) - 1));
      outKeys[pos] = key;
      for (int c = 0; c < cols.n; c++) {
         if (cols.width[c] == 4) ((int32_t*) cols.out[c])[pos] = ((const int32_t*) cols.in[c])[i];
         else if (cols.width[c] == 8) ((int64_t*) cols.out[c])[pos] = ((const int64_t*) cols.in[c])[i];
         else ((int4*) cols.out[c])[pos] = ((const int4*) cols.in[c])[i];
      }
   }
}
void launchPartitionScatter(const int32_t* keys, const void* const* payloadCols, const int32_t* widths, int nPayload, int64_t n, int nParts, unsigned long long* cursors, int32_t* outKeys, void* const* outPayload, int smCount, cudaStream_t s) {
   PartitionCols cols{};
   cols.n = nPayload;
   for (int c = 0; c < nPayload; c++) {
      cols.in[c] = payloadCols[c];
      cols.out[c] = outPayload[c];
      cols.width[c] = widths[c];
   }
   int grid = (int) std::min<int64_t>(std::max<int64_t>((n + kBlock - 1) / kBlock, 1), (int64_t) smCount * 8);
   partitionScatterKernel<<<grid, kBlock, 0, s>>>(keys, cols, n, nParts, cursors, outKeys);
}

// =================================================================================== K10 fused scan → partition → peer store
// (multi-GPU repartition step of a join: subop.materialize + the exchange the reference does not have, SURVEY §8e)
template <int DB>
__global__ void __launch_bounds__(kBlock, 4) scanPartitionSendKernel(const __grid_constant__ SendParams p) {
   constexpr bool IN = true;
   __shared__ __align__(8) TileBarriers barsStorage;
   __shared__ unsigned int sCnt[kMaxRanks];
   __shared__ unsigned long long sBase[kMaxRanks];
   TileBarriers* bars = &barsStorage;
   if (threadIdx.x < kMaxRanks) sCnt[threadIdx.x] = 0;
   __syncthreads();
   const int words = 1 + p.nDec;
   forEachTileUniform<kRowsPerThreadProbe, DB>(p.src.cols, p.src.nRows, dynSmem, bars, [&](const auto& tile, int64_t rowBase, int rows) {
      bool emit[kRowsPerThreadProbe];
      int lrs[kRowsPerThreadProbe], dest[kRowsPerThreadProbe];
      int32_t key[kRowsPerThreadProbe], second[kRowsPerThreadProbe];
      unsigned pos[kRowsPerThreadProbe];
#pragma unroll
      for (int j = 0; j < kRowsPerThreadProbe; j++) {
         const int lr = j * kBlock + threadIdx.x;
         const bool valid = lr < rows;
         lrs[j] = valid ? lr : 0;
         bool ok = valid && evalFilters<IN>(p.src.filters, tile, lrs[j], rowBase + lrs[j]);
         key[j] = tile.i32(p.keyStage, lrs[j]);
         second[j] = p.secondStage >= 0 ? tile.i32(p.secondStage, lrs[j]) : 0;
         if (p.secondYear) second[j] = yearOfDays(second[j]);
         if (ok && p.hasProbe) {
            const int32_t pk = tile.i32(p.probeKeyStage, lrs[j]);
            if (p.bloomOnly) {
               ok = bloomMayContain(p.probe, pk);
            } else {
               bool found = false;
               joinProbe(p.probe, pk, [&](int64_t, int32_t pay) {
                  found = true;
                  if (p.secondStage < 0) second[j] = pay;
               });
               ok = found;
            }
         }
         emit[j] = ok;
         dest[j] = ok ? partOf(key[j], p.world) : 0;
         pos[j] = ok ? atomicAdd(&sCnt[dest[j]], 1u) : 0u; // few percent of the rows get here: a shared atomic each is cheap
      }
      __syncthreads();
      if (threadIdx.x < p.world) { // ONE global atomic per destination per tile claims the range of all its tuples
         const unsigned n = sCnt[threadIdx.x];
         sBase[threadIdx.x] = n ? atomicAdd(&p.cursors[threadIdx.x], (unsigned long long) n) : 0ull;
      }
      __syncthreads();
#pragma unroll
      for (int j = 0; j < kRowsPerThreadProbe; j++) {
         if (!emit[j]) continue;
         const unsigned long long at = sBase[dest[j]] + pos[j];
         if (at >= (unsigned long long) p.capacity) {
            atomicExch(p.error, 6);
            continue;
         }
         unsigned long long* out = (unsigned long long*) p.dest[dest[j]] + at * words; // peer HBM over NVLink (or local for dest == rank)
         out[0] = packSlot(key[j], second[j]);
         for (int d = 0; d < p.nDec; d++) out[1 + d] = (unsigned long long) lazyLo64(p.dec, d, rowBase + lrs[j]);
      }
      if (threadIdx.x < kMaxRanks) sCnt[threadIdx.x] = 0;
      __syncthreads();
   });
}
void launchScanPartitionSend(const SendParams& p, int smCount, cudaStream_t s) {
   size_t dyn;
   if (p.src.cols.decBytes == 8) {
      int grid = persistentGrid(scanPartitionSendKernel<8>, p.src.cols, p.src.nRows, smCount, &dyn, kBlock);
      scanPartitionSendKernel<8><<<grid, kBlock, dyn, s>>>(p);
   } else {
      int grid = persistentGrid(scanPartitionSendKernel<16>, p.src.cols, p.src.nRows, smCount, &dyn, kBlock);
      scanPartitionSendKernel<16><<<grid, kBlock, dyn, s>>>(p);
   }
}
// =================================================================================== K11 star probe → peer store
template <int DB, int RPT>
__global__ void __launch_bounds__(kBlock, 4) scanStarProbeSendKernel(const __grid_constant__ StarSendParams p) {
   constexpr bool IN = true;
   __shared__ __align__(8) TileBarriers barsStorage;
   __shared__ StarQueue queue;
   TileBarriers* bars = &barsStorage;
   if (threadIdx.x == 0) queue.count = 0;
   __syncthreads();
   const int64_t one = 100;
   auto handle = [&](int32_t k0, int32_t k1, int32_t kS, int32_t kO, int64_t row) {
      const uint64_t hP = hashPair(k0, k1), hS = p.tableS.direct ? 0 : hashI32(kS);
      const ulonglong2 eP = __ldg((const ulonglong2*) slotPtr(p.tableP, hP & p.tableP.mask));
      const unsigned long long eS = fkFirstSlot(p.tableS, kS, hS);
      const int64_t a = lazyLo64(p.values, 0, row), b = lazyLo64(p.values, 1, row), d = lazyLo64(p.values, 2, row);
      const int dest = partOf(kO, p.world);
      pairProbeFrom(p.tableP, k0, k1, hP, eP, [&](int64_t c) {
         fkProbeFrom(p.tableS, kS, hS, eS, [&](int32_t g0) {
            const i128 v = sub128(mul64x64(a, one - b), mul64x64(c, d));
            // lanes of the warp that ship to the same rank share one claim of the (device-local) cursor
            const unsigned peers = __match_any_sync(__activemask(), dest);
            const int lane = threadIdx.x & 31, leader = __ffs(peers) - 1;
            unsigned long long at = 0;
            if (lane == leader) at = atomicAdd(&p.cursors[dest], (unsigned long long) __popc(peers));
            at = __shfl_sync(peers, at, leader) + __popc(peers & ((1u << lane) - 1));
            if (at >= (unsigned long long) p.capacity) {
               atomicExch(p.error, 6);
               return;
            }
            unsigned long long* out = (unsigned long long*) p.dest[dest] + at * 3;
            out[0] = packSlot(kO, g0);
            out[1] = (unsigned long long) v.lo;
            out[2] = (unsigned long long) v.hi;
         });
      });
   };
   auto process = [&](int q) {
      handle(queue.w[0][q], queue.w[1][q], queue.w[2][q], queue.w[3][q], (int64_t) (((uint64_t) (uint32_t) queue.w[5][q] << 32) | (uint32_t) queue.w[4][q]));
   };
   forEachTileUniform<RPT, DB, 2>(p.src.cols, p.src.nRows, dynSmem, bars, [&](const auto& tile, int64_t rowBase, int rows) {
      int32_t k0[RPT], k1[RPT];
      int lrs[RPT];
      BloomProbe bp[RPT];
#pragma unroll
      for (int j = 0; j < RPT; j++) {
         const int lrRaw = j * kBlock + threadIdx.x;
         const bool valid = lrRaw < rows;
         lrs[j] = valid ? lrRaw : 0;
         const bool ok = valid && evalFilters<IN>(p.src.filters, tile, lrs[j], rowBase + lrs[j]);
         k0[j] = tile.i32(p.keyStageP0, lrs[j]);
         k1[j] = tile.i32(p.keyStageP1, lrs[j]);
         bp[j] = pairBloomPrefetch(p.tableP, k0[j], k1[j], ok);
      }
#pragma unroll
      for (int j = 0; j < RPT; j++) {
         if (!bp[j].mayContain()) continue;
         const int32_t kS = tile.i32(p.keyStageS, lrs[j]), kO = tile.i32(p.keyStageO, lrs[j]);
         const int64_t row = rowBase + lrs[j];
         const int q = atomicAdd(&queue.count, 1);
         if (q < StarQueue::kCap) {
            queue.w[0][q] = k0[j];
            queue.w[1][q] = k1[j];
            queue.w[2][q] = kS;
            queue.w[3][q] = kO;
            queue.w[4][q] = (int32_t) (uint32_t) (uint64_t) row;
            queue.w[5][q] = (int32_t) (uint32_t) ((uint64_t) row >> 32);
         } else {
            handle(k0[j], k1[j], kS, kO, row);
         }
      }
      __syncthreads();
      drainQueue(queue, false, process);
   });
   __syncthreads();
   drainQueue(queue, true, process);
}
void launchScanStarProbeSend(const StarSendParams& p, int smCount, cudaStream_t s) {
   size_t dyn;
   if (p.src.cols.decBytes == 8) {
      int grid = persistentGrid(scanStarProbeSendKernel<8, 2>, p.src.cols, p.src.nRows, smCount, &dyn, kBlock, 2);
      scanStarProbeSendKernel<8, 2><<<grid, kBlock, dyn, s>>>(p);
   } else {
      int grid = persistentGrid(scanStarProbeSendKernel<16, 2>, p.src.cols, p.src.nRows, smCount, &dyn, kBlock, 2);
      scanStarProbeSendKernel<16, 2><<<grid, kBlock, dyn, s>>>(p);
   }
}
__global__ void __launch_bounds__(kBlock) probeReceivedGroupBy2Kernel(JoinTableDev table, GroupTableDev groupsOut, const uint8_t* recv, int world, int64_t capacity, const unsigned long long* counts) {
   __shared__ LocalGroups groups;
   groups.init();
   __syncthreads();
   const int64_t total = (int64_t) world * capacity;
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t) gridDim.x * blockDim.x) {
      const int src = (int) (i / capacity);
      const int64_t idx = i - (int64_t) src * capacity;
      if ((unsigned long long) idx >= counts[src]) continue;
      const unsigned long long* tup = (const unsigned long long*) recv + i * 3;
      const unsigned long long w0 = tup[0];
      const int32_t key = (int32_t) (uint32_t) w0, g0 = (int32_t) (uint32_t) (w0 >> 32);
      const i128 v{tup[1], (int64_t) tup[2]};
      joinProbe(table, key, [&](int64_t, int32_t g1) { groups.add(groupsOut, g0, g1, v, false); });
   }
   __syncthreads();
   groups.flush(groupsOut, false);
}
void launchProbeReceivedGroupBy2(const JoinTableDev& table, const GroupTableDev& groups, const uint8_t* recv, int world, int64_t capacity, const unsigned long long* counts, int smCount, cudaStream_t s) {
   const int64_t total = (int64_t) world * capacity;
   int grid = (int) std::min<int64_t>(std::max<int64_t>((total + kBlock - 1) / kBlock, 1), (int64_t) smCount * 4);
   probeReceivedGroupBy2Kernel<<<grid, kBlock, 0, s>>>(table, groups, recv, world, capacity, counts);
}

// tuples received from `world` sources: sub-region s holds counts[s] tuples (count read from device memory: no host round trip)
__global__ void __launch_bounds__(kBlock) insertReceivedKernel(JoinTableDev t, const uint8_t* recv, int world, int64_t capacity, const unsigned long long* counts) {
   unsigned long long inserted = 0;
   const int64_t total = (int64_t) world * capacity;
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t) gridDim.x * blockDim.x) {
      const int src = (int) (i / capacity);
      const int64_t idx = i - (int64_t) src * capacity;
      if ((unsigned long long) idx >= counts[src]) continue;
      const unsigned long long e = ((const unsigned long long*) recv)[i];
      if (joinInsert(t, (int32_t) (uint32_t) e, (int32_t) (uint32_t) (e >> 32)) >= 0) inserted++;
   }
   flushInsertCount(t, inserted);
}
void launchInsertReceived(const JoinTableDev& t, const uint8_t* recv, int world, int64_t capacity, const unsigned long long* counts, int smCount, cudaStream_t s) {
   const int64_t total = (int64_t) world * capacity;
   int grid = (int) std::min<int64_t>(std::max<int64_t>((total + kBlock - 1) / kBlock, 1), (int64_t) smCount * 8);
   insertReceivedKernel<<<grid, kBlock, 0, s>>>(t, recv, world, capacity, counts);
}
__global__ void __launch_bounds__(kBlock) probeReceivedGroupByKernel(JoinTableDev tableA, JoinTableDev tableB, GroupTableDev groupsOut, const uint8_t* recv, int world, int64_t capacity,
                                                                     const unsigned long long* counts, int64_t one) {
   __shared__ LocalGroups groups;
   groups.init();
   __syncthreads();
   const int64_t total = (int64_t) world * capacity;
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t) gridDim.x * blockDim.x) {
      const int src = (int) (i / capacity);
      const int64_t idx = i - (int64_t) src * capacity;
      if ((unsigned long long) idx >= counts[src]) continue;
      const unsigned long long* tup = (const unsigned long long*) recv + i * 3;
      const unsigned long long w0 = tup[0];
      const int32_t keyA = (int32_t) (uint32_t) w0, keyB = (int32_t) (uint32_t) (w0 >> 32);
      const int64_t a = (int64_t) tup[1], b = (int64_t) tup[2];
      joinProbe(tableA, keyA, [&](int64_t, int32_t payA) {
         joinProbe(tableB, keyB, [&](int64_t, int32_t payB) {
            if (payA == payB) groups.add(groupsOut, payB, 0, mul64x64(a, one - b), false);
         });
      });
   }
   __syncthreads();
   groups.flush(groupsOut, false);
}
void launchProbeReceivedGroupBy(const JoinTableDev& tableA, const JoinTableDev& tableB, const GroupTableDev& groups, const uint8_t* recv, int world, int64_t capacity,
                                const unsigned long long* counts, int64_t one, int smCount, cudaStream_t s) {
   const int64_t total = (int64_t) world * capacity;
   int grid = (int) std::min<int64_t>(std::max<int64_t>((total + kBlock - 1) / kBlock, 1), (int64_t) smCount * 4);
   probeReceivedGroupByKernel<<<grid, kBlock, 0, s>>>(tableA, tableB, groups, recv, world, capacity, counts, one);
}

} // namespace ldb
