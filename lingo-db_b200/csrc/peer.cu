// peer.cu — multi-GPU exchange over peer-mapped HBM (NVLink 5 / NVSwitch), one process per GPU.
//
// No reference counterpart: the reference is single-process (SURVEY §2 "Parallelism strategies").  Every rank owns a
// SYMMETRIC HEAP (one cudaMalloc, same layout everywhere) that its peers map through CUDA IPC; a transfer is a kernel
// that STORES into the peer's heap over NVLink and then publishes a flag (fence.sys + st.release.sys), the receiver's
// kernel spins on the flag in its own memory (ld.acquire.sys).  No NCCL call, no host round trip, no proxy thread on the
// data path — the partial aggregates of Q1/Q6/Q9 (≈9–140 KB) cost one small kernel instead of export + all-gather + merge,
// and the repartition step of a join writes its tuples straight into the receiver's buffer from the partition kernel.
//
//   heap: | barrier flags [world] | gather flags [2][world] | mailbox [2][world][kSlotBytes] | user region … |
//
// Flags are monotonic epoch counters, so nothing is ever reset; the mailbox is double-buffered by epoch parity: a writer
// can be at most one collective ahead of any reader (its next collective waits for that reader's push), so parity p is
// never overwritten while a peer still reads it.
#include "context.h"
#include "device_utils.cuh"
#include "keyhash.cuh"
#include "peer.h"
#include "progcol.cuh"
#include "program.h"
#include "sortkey.cuh"
#include "tilescan.cuh"

#include <algorithm>
#include <cstring>

namespace ldb {

// ---------------------------------------------------------------- device side
__device__ __forceinline__ void stReleaseSys(unsigned long long* p, unsigned long long v) { asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ unsigned long long ldAcquireSys(const unsigned long long* p) {
   unsigned long long v;
   asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
   return v;
}
__device__ __forceinline__ unsigned long long globalTimerNs() {
   unsigned long long t;
   asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
   return t;
}
// Spin until *flag >= epoch.  Bounded (a peer that died must not hang this GPU): on timeout the comm's error word is set
// and the caller's data is garbage — the host reports LDB_ERR_CUDA at the next check.
__device__ __forceinline__ bool waitFlag(const unsigned long long* flag, unsigned long long epoch, int32_t* error, unsigned long long timeoutNs) {
   const unsigned long long t0 = globalTimerNs();
   unsigned spins = 0;
   while (ldAcquireSys(flag) < epoch) {
      if ((++spins & 1023u) == 0) {
         if (globalTimerNs() - t0 > timeoutNs) {
            atomicExch(error, 1);
            return false;
         }
         __nanosleep(200);
      }
   }
   return true;
}

// all-to-all "I am here": CTA p tells peer p and waits for peer p
enum EpochKind { EPOCH_BARRIER = 0, EPOCH_GATHER = 1, EPOCH_MERGE = 2 };
__device__ __forceinline__ unsigned long long nextEpoch(const PeerView& v, int kind) { return ((const volatile unsigned long long*) (v.heap[v.rank] + kEpochsOff))[kind] + 1; }
// runs behind every collective kernel (stream order): the epoch a kernel reads is stable for all its CTAs
__global__ void peerBumpKernel(PeerView v, int kindA, int kindB) {
   unsigned long long* e = (unsigned long long*) (v.heap[v.rank] + kEpochsOff);
   e[kindA]++;
   if (kindB >= 0) e[kindB]++;
}
__global__ void peerBarrierKernel(PeerView v) {
   const unsigned long long epoch = nextEpoch(v, EPOCH_BARRIER);
   const int p = blockIdx.x;
   if (p == v.rank || threadIdx.x != 0) return;
   __threadfence_system(); // everything this GPU wrote into peer memory before the barrier (earlier kernels of the stream included)
   stReleaseSys((unsigned long long*) (v.heap[p] + kBarrierFlagsOff) + v.rank, epoch);
   waitFlag((const unsigned long long*) (v.heap[v.rank] + kBarrierFlagsOff) + p, epoch, v.error, v.timeoutNs);
}

// all-gather of one small block (<= kSlotBytes, multiple of 16): CTA p copies `src` into peer p's mailbox slot [parity][rank]
// with 128-bit stores, publishes the flag, then waits for peer p's block.  Afterwards mailbox[parity][*] of the own heap is
// complete (the own slot is filled locally by CTA `rank`).
__device__ __forceinline__ void pushBlock(const PeerView& v, int p, const uint8_t* src, size_t bytes, unsigned long long epoch) {
   const int parity = (int) (epoch & 1);
   uint8_t* dst = v.heap[p] + kMailboxOff + ((size_t) parity * v.world + v.rank) * kSlotBytes;
   const int4* s4 = (const int4*) src;
   int4* d4 = (int4*) dst;
   for (size_t i = threadIdx.x; i < bytes / 16; i += blockDim.x) d4[i] = s4[i];
   __syncthreads();
   if (threadIdx.x == 0 && p != v.rank) {
      __threadfence_system();
      stReleaseSys((unsigned long long*) (v.heap[p] + kGatherFlagsOff) + (size_t) parity * v.world + v.rank, epoch);
   }
}
__device__ __forceinline__ bool waitBlock(const PeerView& v, int p, unsigned long long epoch) {
   const int parity = (int) (epoch & 1);
   __shared__ int ok;
   if (threadIdx.x == 0) ok = p == v.rank ? 1 : (waitFlag((const unsigned long long*) (v.heap[v.rank] + kGatherFlagsOff) + (size_t) parity * v.world + p, epoch, v.error, v.timeoutNs) ? 1 : 0);
   __syncthreads();
   return ok != 0;
}
__global__ void __launch_bounds__(256) peerAllGatherKernel(PeerView v, const uint8_t* src, size_t bytes) {
   const unsigned long long epoch = nextEpoch(v, EPOCH_GATHER);
   const int p = blockIdx.x;
   pushBlock(v, p, src, bytes, epoch);
   waitBlock(v, p, epoch);
}

// K7 over NVLink: all-gather of the group-table image fused with the merge.  CTA p pushes this rank's table (the table IS
// the image: state | keys | acc) to peer p, waits for peer p's image and folds it into the local table with the same
// lookup-or-insert + two-word atomic adds the single-GPU flush uses (rt::PreAggregationHashtable::merge semantics: sums per key).
__device__ int peerGroupLookupOrInsert(const GroupTableDev& t, const int32_t* k); // kernels.cu twin, defined below
__global__ void __launch_bounds__(256) peerGroupAllMergeKernel(PeerView v, GroupTableDev t, size_t imageBytes) {
   const unsigned long long epoch = nextEpoch(v, EPOCH_GATHER);
   const unsigned long long localTarget = nextEpoch(v, EPOCH_MERGE) * (unsigned long long) (v.world - 1);
   const int p = blockIdx.x;
   if (p == v.rank) return; // the own table is merged into, not from
   pushBlock(v, p, (const uint8_t*) t.state, imageBytes, epoch);
   // every CTA must have READ the table (its push) before any CTA starts folding a peer's image INTO it: rendezvous of the
   // world-1 co-resident CTAs on a monotonic counter in this GPU's own memory
   if (threadIdx.x == 0) {
      unsigned long long* sync = (unsigned long long*) (v.heap[v.rank] + kLocalSyncOff);
      __threadfence();
      atomicAdd(sync, 1ull);
      while (*((volatile unsigned long long*) sync) < localTarget) {}
   }
   __syncthreads();
   if (!waitBlock(v, p, epoch)) return;
   const int parity = (int) (epoch & 1);
   const uint8_t* img = v.heap[v.rank] + kMailboxOff + ((size_t) parity * v.world + p) * kSlotBytes;
   const size_t cap = (size_t) t.capacity;
   const int32_t* st = (const int32_t*) img;
   const int32_t* keys = (const int32_t*) (img + cap * 4);
   const unsigned long long* acc = (const unsigned long long*) (img + cap * 4 + cap * kMaxKeys * 4);
   const int total = t.capacity * t.nAggs; // <= 2048 * 8
   for (int i = threadIdx.x; i < total; i += blockDim.x) {
      const int slotIdx = i / t.nAggs, a = i % t.nAggs;
      if (t.nKeys == 0 ? slotIdx != 0 : st[slotIdx] != 2) continue;
      int32_t kk[2] = {keys[(size_t) slotIdx * kMaxKeys], keys[(size_t) slotIdx * kMaxKeys + 1]};
      const int slot = peerGroupLookupOrInsert(t, kk);
      if (slot < 0) continue;
      const unsigned long long* src = acc + ((size_t) slotIdx * kMaxAggs + a) * 2;
      unsigned long long* dst = t.acc + ((size_t) slot * kMaxAggs + a) * 2;
      atomicAdd128(dst, dst + 1, i128{src[0], (int64_t) src[1]});
   }
}
// same open-addressing protocol as kernels.cu groupLookupOrInsert (state 0 empty / 1 being written / 2 ready)
__device__ int peerGroupLookupOrInsert(const GroupTableDev& t, const int32_t* k) {
   if (t.nKeys == 0) return 0;
   const uint32_t mask = (uint32_t) t.capacity - 1;
   uint64_t h = hashI32(k[0]);
   if (t.nKeys > 1) h = hashCombine(hashI32(k[1]), h);
   uint32_t s = (uint32_t) h & mask;
   for (int probes = 0; probes < t.capacity; probes++) {
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

// OR-all-reduce of a bit array that every rank keeps at the SAME heap offset (the Bloom filters of the hash partitions of one
// logical build side): every rank reads its peers' words over NVLink (P2P loads) and ORs them into its own copy.  A peer that
// already folded some ranks in only contributes bits the result contains anyway, so no second buffer is needed; barriers
// before (all builds done) and after (nobody is still reading) are the caller's.
__global__ void __launch_bounds__(256) peerOrReduceKernel(PeerView v, size_t heapOff, size_t words4 /* number of uint4 */) {
   uint4* own = (uint4*) (v.heap[v.rank] + heapOff);
   for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < words4; i += (size_t) gridDim.x * blockDim.x) {
      uint4 a = own[i];
      for (int p = 0; p < v.world; p++) {
         if (p == v.rank) continue;
         uint4 b; // peer words change while they are read (the peer ORs too): a coherent (non-nc) 128-bit load
         asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w) : "l"((const uint4*) (v.heap[p] + heapOff) + i) : "memory");
         a.x |= b.x;
         a.y |= b.y;
         a.z |= b.z;
         a.w |= b.w;
      }
      own[i] = a;
   }
}

__global__ void peerPublishCountsKernel(PeerView v, size_t cursorsOff, size_t countsOff) {
   const int d = threadIdx.x;
   if (d >= v.world) return;
   const unsigned long long n = *((const unsigned long long*) (v.heap[v.rank] + cursorsOff) + d);
   *((unsigned long long*) (v.heap[d] + countsOff) + v.rank) = n; // plain store into the peer; the barrier that follows publishes it
}

// ---------------------------------------------------------------- table exchange (ldb_gpu_table_exchange, include/ldb_gpu.h)
// A stable multi-way partition of a table's rows by owner rank, as the radix sort's hist / scan / scatter: the count kernel gives every
// CTA (a fixed tile of one batch) a per-destination histogram, a scan turns the histograms into each CTA's offset per destination, and
// the send kernel ranks the rows of each tile per destination (match_any + per-warp counts) and stores their cells straight into the
// owner's receive region.  Receive region of a rank with n rows (column-major, every array 16-byte aligned):
//   cells of column 0 (n x outBytes[0]) | … | cells of column m-1 | validity bytes of column 0 (n) | … | validity bytes of column m-1
// Source s's rows start at row Σ_{s' < s} M[s'][d] of receiver d, M[s][d] = the rows source s sends rank d.
// With utf8 columns (ldb_gpu_table_exchange_varlen) a utf8 column's "cells" are its n + 1 int32 offsets, and its bytes follow every
// column's cells: … cells / offsets of column m-1 | bytes of utf8 column 0 (B_0) | … | validity bytes …; source s's bytes of utf8 column
// j start at byte Σ_{s' < s} Bytes[s'][d][j].  The count kernel then also histograms the bytes per (destination, utf8 column, CTA).
constexpr int kShipMaxCols = 16;
constexpr int kShipThreads = 256;
constexpr int64_t kShipTile = 16 * kShipThreads; // rows per CTA; tiles never span batches
struct TableShipBatch {
   ProgCol cols[kShipMaxCols];  // shipped columns of this batch (bindColumn)
   ProgCol keys[kProgMaxKeys];  // key columns of this batch
   int32_t outBytes[kShipMaxCols];
   int32_t nCols, nKeys, world;
   int32_t broadcast;           // every row to every rank (no keys)
   int64_t nRows, firstRow;     // this batch's rows and the source row number of its row 0
   int64_t ctaBase, nCtas;      // this batch's first CTA in the histograms, and the CTAs of all batches
   uint8_t* owners;             // per source row: its owner (count writes, send reads)
   unsigned long long* hist;    // [world][nCtas]: count: rows per (destination, CTA); after the scan: the CTA's offset in the destination
   uint8_t* recv[kMaxPeers];    // every rank's receive region (peer-mapped)
   unsigned long long rows[kMaxPeers]; // the rows every rank receives (its N_d)
   unsigned long long base[kMaxPeers]; // the row of receiver d where this source's rows start
   // utf8 columns
   int32_t nStr;                       // shipped utf8 columns
   int8_t strCol[kShipMaxCols];        // utf8 column j: its index among the shipped columns
   int8_t strOf[kShipMaxCols];         // shipped column c: its utf8 index j, or -1
   uint32_t strBytes[kMaxPeers][kShipMaxCols]; // B_j of every receiver (<= 2^31 - 1: decided before the send)
   uint32_t byteBase[kMaxPeers][kShipMaxCols]; // the byte of receiver d's column j where this source's bytes start
};
static_assert(sizeof(TableShipBatch) <= 4096, "TableShipBatch is a __grid_constant__ kernel parameter (4 KiB at most)");
// hist rows of the count kernel: rows of destination d at row d, bytes of (destination d, utf8 column j) at row world + d nStr + j;
// the scan turns row r into totals[r], which the matrix all-gather carries (kShipBlockU64 u64 per rank at most)
constexpr int kShipBlockU64 = kMaxPeers * (1 + kShipMaxCols);
// byte offsets of the arrays of a receive region of n rows; returns its size.  strOf[c] >= 0 marks a utf8 column (n + 1 int32 offsets)
// whose bytes, strBytes[strOf[c]], follow the cells of every column; bytesOff[j] = where utf8 column j's bytes start.
__host__ __device__ inline uint64_t shipLayout(uint64_t n, const int32_t* outBytes, int nCols, const int8_t* strOf, int nStr, const uint32_t* strBytes,
                                               uint64_t* colOff, uint64_t* validOff, uint64_t* bytesOff) {
   uint64_t off = 0;
   for (int c = 0; c < nCols; c++) {
      colOff[c] = off;
      off += ((strOf[c] >= 0 ? (n + 1) * 4 : n * (uint64_t) outBytes[c]) + 15) & ~uint64_t(15);
   }
   for (int j = 0; j < nStr; j++) {
      bytesOff[j] = off;
      off += ((uint64_t) strBytes[j] + 15) & ~uint64_t(15);
   }
   for (int c = 0; c < nCols; c++) {
      validOff[c] = off;
      off += (n + 15) & ~uint64_t(15);
   }
   return off;
}
__device__ __forceinline__ int shipOwnerOf(const TableShipBatch& p, int64_t row) {
   int64_t keys[kProgMaxKeys];
   uint32_t nulls = 0;
#pragma unroll
   for (int k = 0; k < kProgMaxKeys; k++) {
      if (k >= p.nKeys) break;
      const Val kv = loadCol(p.keys[k], row); // the value the aggregation sink groups by: int64 of an integer, a decimal's low 8 bytes
      keys[k] = kv.null ? 0 : (int64_t) kv.v;
      nulls |= (kv.null ? 1u : 0u) << k;
   }
   return keyOwner(keyTupleHash(keys, p.nKeys, nulls), p.world);
}
// a utf8 cell's byte count: bytes[off[i] .. off[i+1]) as strCompare (program.cu) reads them; a NULL string ships none.  A warp's 32 cells
// come from one batch, whose offsets are int32, so their sum fits 32 bits.
__device__ __forceinline__ uint32_t shipStrLen(const ProgCol& c, int64_t row) {
   if (colIsNull(c, row)) return 0;
   const int32_t* off = (const int32_t*) c.data + row;
   return (uint32_t) (off[1] - off[0]);
}
// the count kernel's body for an owner rule ownerOf(row): tableShipCountKernel (key hash) and tableShipCountRangeKernel (sort splitters).
// Per CTA the rows per destination, in hist row d, and with utf8 columns the bytes per (destination, utf8 column), in hist row
// world + d nStr + j.  A broadcast counts every row for destination 0 (the other destinations' rows stay 0) and writes no owners.
template <class OwnerOf>
__device__ __forceinline__ void shipCountRows(const TableShipBatch& p, const OwnerOf& ownerOf) {
   __shared__ unsigned int cnt[kMaxPeers];
   __shared__ unsigned long long bytes[kMaxPeers * kShipMaxCols];
   if (threadIdx.x < kMaxPeers) cnt[threadIdx.x] = 0;
   for (int x = threadIdx.x; x < kMaxPeers * kShipMaxCols; x += kShipThreads) bytes[x] = 0;
   __syncthreads();
   const int lane = threadIdx.x & 31;
   const int64_t begin = (int64_t) blockIdx.x * kShipTile, end = min(begin + kShipTile, p.nRows);
   for (int64_t t = begin; t < end; t += kShipThreads) {
      const int64_t i = t + threadIdx.x;
      const bool valid = i < end;
      const int d = !valid ? -1 : p.broadcast ? 0 : ownerOf(i);
      if (valid && !p.broadcast) p.owners[p.firstRow + i] = (uint8_t) d;
      const unsigned same = __match_any_sync(0xffffffffu, d);
      const bool leader = valid && lane == __ffs(same) - 1;
      if (leader) atomicAdd(&cnt[d], (unsigned) __popc(same));
      for (int j = 0; j < p.nStr; j++) {
         const unsigned sum = __reduce_add_sync(same, valid ? shipStrLen(p.cols[p.strCol[j]], i) : 0u);
         if (leader) atomicAdd(&bytes[d * p.nStr + j], (unsigned long long) sum);
      }
   }
   __syncthreads();
   const size_t at = (size_t) p.ctaBase + blockIdx.x;
   if (threadIdx.x < p.world) p.hist[(size_t) threadIdx.x * p.nCtas + at] = cnt[threadIdx.x];
   for (int x = threadIdx.x; x < p.world * p.nStr; x += kShipThreads) p.hist[(size_t) (p.world + x) * p.nCtas + at] = bytes[x];
}
__global__ void __launch_bounds__(kShipThreads) tableShipCountKernel(const __grid_constant__ TableShipBatch p) {
   shipCountRows(p, [&](int64_t i) { return shipOwnerOf(p, i); });
}
// one cell into the receive region: the low outBytes bytes of the source cell; a narrowed 8-byte decimal sign-extended to 16
__device__ __forceinline__ void shipCell(const ProgCol& c, int w, int64_t row, uint8_t* dst) {
   const uint8_t* s = c.data + (size_t) row * c.elemBytes;
   switch (w) {
      case 16:
         if (c.elemBytes == 16) {
            *(int4*) dst = *(const int4*) s;
         } else {
            const long long v = *(const long long*) s;
            *(longlong2*) dst = make_longlong2(v, v >> 63);
         }
         break;
      case 8: *(uint64_t*) dst = *(const uint64_t*) s; break;
      case 4: *(uint32_t*) dst = *(const uint32_t*) s; break;
      case 2: *(uint16_t*) dst = *(const uint16_t*) s; break;
      default: *dst = *s;
   }
}
// The send kernel: a row's thread stores its fixed-width cells, its validity bytes and, per utf8 column, the offset of its string in the
// receiver: this source's byte base + the CTA's scanned bytes + the bytes of earlier passes, of earlier warps and of the earlier lanes of
// its warp with the same destination.  So the strings of one warp's rows for one destination are adjacent in the receiver, and the whole
// warp copies that range: lanes take consecutive bytes, each walking the warp's rows in (destination, lane) order.  A broadcast ranks
// every row for destination 0 and stores it into every rank; one without utf8 columns is not counted (hist is null), and its CTA's rows
// start at firstRow + begin, where the scan would have put them.
// kStrings = false, for shipments without utf8 columns, drops the string work and arrays (the string instance sent one int64 column 1.5x slower).
constexpr int kShipWarps = kShipThreads / 32;
template <bool kStrings>
__global__ void __launch_bounds__(kShipThreads) tableShipSendKernel(const __grid_constant__ TableShipBatch p) {
   constexpr int kS = kStrings ? kShipMaxCols : 1, kSlots = kStrings ? 32 : 1; // the string arrays' extents
   __shared__ uint64_t colOff[kMaxPeers][kShipMaxCols], validOff[kMaxPeers][kShipMaxCols], bytesOff[kMaxPeers][kS];
   __shared__ unsigned long long running[kMaxPeers];        // this CTA's rows for destination d before the pass (from base[d])
   __shared__ unsigned long long byteRunning[kMaxPeers][kS]; // its bytes of utf8 column j for d before the pass (from byteBase)
   __shared__ unsigned int warpCnt[kShipWarps][kMaxPeers];
   __shared__ unsigned int warpBytes[kShipWarps][kMaxPeers][kS];
   __shared__ uint32_t slotEnd[kShipWarps][kSlots + 1]; // the warp's lanes in (destination, lane) order: slot k's string is [slotEnd[k], slotEnd[k+1])
   __shared__ int32_t slotSrc[kShipWarps][kSlots];      // and starts at source byte slotSrc[k]
   const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
   const int world = p.world, nStr = kStrings ? p.nStr : 0;
   const int64_t begin = (int64_t) blockIdx.x * kShipTile, end = min(begin + kShipTile, p.nRows);
   const size_t at = (size_t) p.ctaBase + blockIdx.x;
   if (threadIdx.x < world) {
      const int d = threadIdx.x;
      shipLayout(p.rows[d], p.outBytes, p.nCols, p.strOf, nStr, p.strBytes[d], colOff[d], validOff[d], bytesOff[d]);
      running[d] = p.hist ? p.hist[(size_t) d * p.nCtas + at] : (unsigned long long) (p.firstRow + begin);
   }
   for (int x = threadIdx.x; x < world * nStr; x += kShipThreads) byteRunning[x / nStr][x % nStr] = p.hist[(size_t) (world + x) * p.nCtas + at];
   __syncthreads();
   for (int64_t t = begin; t < end; t += kShipThreads) {
      for (int x = threadIdx.x; x < kShipWarps * kMaxPeers; x += kShipThreads) (&warpCnt[0][0])[x] = 0;
      if constexpr (kStrings)
         for (int x = threadIdx.x; x < kShipWarps * kMaxPeers * kShipMaxCols; x += kShipThreads) (&warpBytes[0][0][0])[x] = 0;
      __syncthreads();
      const int64_t i = t + threadIdx.x;
      const bool valid = i < end;
      const int d = !valid ? kMaxPeers : p.broadcast ? 0 : p.owners[p.firstRow + i];
      const unsigned same = __match_any_sync(0xffffffffu, d);
      const unsigned rankInWarp = __popc(same & ((1u << lane) - 1));
      const bool leader = valid && rankInWarp == 0;
      if (leader) warpCnt[warp][d] = __popc(same);
      for (int j = 0; j < nStr; j++) {
         const unsigned sum = __reduce_add_sync(same, valid ? shipStrLen(p.cols[p.strCol[j]], i) : 0u);
         if (leader) warpBytes[warp][d][j] = sum;
      }
      __syncthreads();
      // the row's slot (invalid lanes take the last ones) and its position relative to the source's first row in a receiver
      unsigned slot = kStrings ? __popc(__ballot_sync(0xffffffffu, valid)) + rankInWarp : 0, first = 0;
      unsigned long long rel = 0;
      if (valid) {
         unsigned before = 0;
         for (int w = 0; w < warp; w++) before += warpCnt[w][d];
         for (int e = 0; e < d; e++) first += warpCnt[warp][e];
         slot = first + rankInWarp;
         rel = running[d] + before + rankInWarp;
         for (int r = p.broadcast ? 0 : d; r < (p.broadcast ? world : d + 1); r++) {
            uint8_t* dst = p.recv[r];
            const unsigned long long pos = p.base[r] + rel;
            for (int c = 0; c < p.nCols; c++) {
               const bool null = colIsNull(p.cols[c], i);
               if (!kStrings || p.strOf[c] < 0) shipCell(p.cols[c], p.outBytes[c], i, dst + colOff[r][c] + pos * (uint64_t) p.outBytes[c]);
               dst[validOff[r][c] + pos] = null ? 0 : 1;
            }
         }
      }
      for (int j = 0; j < nStr; j++) {
         const int c = p.strCol[j];
         const ProgCol& sc = p.cols[c];
         uint32_t len = 0;
         int32_t from = 0;
         if (valid && !colIsNull(sc, i)) {
            const int32_t* o = (const int32_t*) sc.data + i;
            from = o[0];
            len = (uint32_t) (o[1] - o[0]);
         }
         __syncwarp(); // the previous column's copy is done with the slots
         slotSrc[warp][slot] = from;
         slotEnd[warp][slot + 1] = len;
         __syncwarp();
         uint32_t x = slotEnd[warp][lane + 1]; // inclusive scan of the lengths in slot order
         for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
         }
         slotEnd[warp][lane + 1] = x;
         if (lane == 0) slotEnd[warp][0] = 0;
         __syncwarp();
         if (valid) { // the row's offset: where its string starts in the receiver's column
            unsigned long long relB = byteRunning[d][j] + (slotEnd[warp][slot] - slotEnd[warp][first]);
            for (int w = 0; w < warp; w++) relB += warpBytes[w][d][j];
            for (int r = p.broadcast ? 0 : d; r < (p.broadcast ? world : d + 1); r++)
               *(int32_t*) (p.recv[r] + colOff[r][c] + (p.base[r] + rel) * 4) = (int32_t) (p.byteBase[r][j] + relB);
         }
         // the strings: per destination of the warp, one contiguous range of the receiver's bytes
         unsigned gs = 0;
         for (int g = 0; g < world; g++) {
            const unsigned n = warpCnt[warp][g];
            if (n == 0) continue;
            const uint32_t e0 = slotEnd[warp][gs], total = slotEnd[warp][gs + n] - e0;
            unsigned long long relB = byteRunning[g][j];
            for (int w = 0; w < warp; w++) relB += warpBytes[w][g][j];
            unsigned k = gs;
            for (uint32_t b = lane; b < total; b += 32) {
               const uint32_t a = e0 + b;
               while (slotEnd[warp][k + 1] <= a) k++;
               const uint8_t v = sc.bytes[(int64_t) slotSrc[warp][k] + (a - slotEnd[warp][k])];
               for (int r = p.broadcast ? 0 : g; r < (p.broadcast ? world : g + 1); r++) p.recv[r][bytesOff[r][j] + p.byteBase[r][j] + relB + b] = v;
            }
            gs += n;
         }
      }
      __syncthreads();
      if (threadIdx.x < world) {
         unsigned tot = 0;
         for (int w = 0; w < kShipWarps; w++) tot += warpCnt[w][threadIdx.x];
         running[threadIdx.x] += tot;
      }
      for (int x = threadIdx.x; x < world * nStr; x += kShipThreads) {
         unsigned long long tot = 0;
         for (int w = 0; w < kShipWarps; w++) tot += warpBytes[w][x / nStr][x % nStr];
         byteRunning[x / nStr][x % nStr] += tot;
      }
      __syncthreads();
   }
}

// ---------------------------------------------------------------- sort exchange (ldb_gpu_table_sort_exchange, include/ldb_gpu.h)
// A row's place in the global order is its canonical tuple: per key its NULL flag and its value sign-extended to 128 bits (sortCell,
// sortkey.cuh: the cell read buildSortWordsKernel makes), both inverted for DESC, then (source rank, source row).  Word 0 holds the NULL
// flags in bits 56.. and rank << 48 | row below them; words 1 + 2k and 2 + 2k the high word (sign bit flipped) and the low word of key k,
// so unsigned word comparisons give the order of ldb_gpu_table_order_by_keys whatever width a shard staged a decimal key at.  Every tuple
// is distinct, so splitters taken from samples cut even a table of equal keys into balanced ranges.
constexpr int kSortSamples = 1024;                     // samples per rank (S)
constexpr int kSortTupleWords = 1 + 2 * kProgMaxKeys;  // 72 bytes
constexpr size_t kSortBlockBytes = 16 + (size_t) kSortSamples * kSortTupleWords * 8; // {n_r, S_r}, then S_r tuples
static_assert(kSortBlockBytes % 16 == 0 && kSortBlockBytes <= kSlotBytes, "a rank's samples are one all-gather block");
constexpr unsigned long long kSortRowMask = (1ull << 56) - 1; // (rank, row) of word 0
struct SortSplit {
   int32_t nKeys, nSplit, rank, pad;
   int32_t desc[kProgMaxKeys];
   unsigned long long split[kMaxPeers - 1][kSortTupleWords]; // ascending; rank d owns the tuples t with split[d-1] < t <= split[d]
};
__host__ __device__ __forceinline__ bool sortTupleLess(const unsigned long long* a, const unsigned long long* b, int nKeys) {
#pragma unroll
   for (int k = 0; k < kProgMaxKeys; k++) {
      if (k >= nKeys) break;
      const unsigned long long na = (a[0] >> (56 + k)) & 1, nb = (b[0] >> (56 + k)) & 1;
      if (na != nb) return na < nb;
      if (a[1 + 2 * k] != b[1 + 2 * k]) return a[1 + 2 * k] < b[1 + 2 * k];
      if (a[2 + 2 * k] != b[2 + 2 * k]) return a[2 + 2 * k] < b[2 + 2 * k];
   }
   return (a[0] & kSortRowMask) < (b[0] & kSortRowMask);
}
__device__ __forceinline__ void sortTupleOf(const TableShipBatch& p, const SortSplit& s, int64_t i, unsigned long long (&w)[kSortTupleWords]) {
   unsigned long long nulls = 0;
#pragma unroll
   for (int k = 0; k < kProgMaxKeys; k++) {
      w[1 + 2 * k] = w[2 + 2 * k] = 0;
      if (k >= s.nKeys) continue;
      const ProgCol& c = p.keys[k];
      const bool null = colIsNull(c, i);
      const SortCell v = null ? SortCell{0, 0} : sortCell(c.data, c.elemBytes, i);
      const unsigned long long inv = s.desc[k] ? ~0ull : 0ull;
      w[1 + 2 * k] = v.hi ^ 0x8000000000000000ull ^ inv;
      w[2 + 2 * k] = v.lo ^ inv;
      nulls |= (unsigned long long) ((null ? 1 : 0) ^ (s.desc[k] ? 1 : 0)) << k;
   }
   w[0] = nulls << 56 | (unsigned long long) s.rank << 48 | (unsigned long long) (p.firstRow + i);
}
// the range owner: the number of splitters below the row's tuple (binary search over <= 7 splitters in the parameter space)
__device__ __forceinline__ int sortRangeOwner(const TableShipBatch& p, const SortSplit& s, int64_t i) {
   unsigned long long w[kSortTupleWords];
   sortTupleOf(p, s, i, w);
   int lo = 0, hi = s.nSplit;
   while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (sortTupleLess(s.split[mid], w, s.nKeys)) lo = mid + 1;
      else hi = mid;
   }
   return lo;
}
__global__ void __launch_bounds__(kShipThreads) tableShipCountRangeKernel(const __grid_constant__ TableShipBatch p, const __grid_constant__ SortSplit s) {
   shipCountRows(p, [&](int64_t i) { return sortRangeOwner(p, s, i); });
}
// sample j of a table of `total` rows is row mix64(j + c) mod total (a hash of the index, not a stride: a periodic input cannot alias
// it); the launch over one batch writes the samples that fall into it, as tuples at out[j]
__global__ void __launch_bounds__(256) sortSampleKernel(const __grid_constant__ TableShipBatch p, const __grid_constant__ SortSplit s, int64_t total, unsigned long long* out) {
   const int j = blockIdx.x * blockDim.x + threadIdx.x;
   if (j >= kSortSamples) return;
   const int64_t row = (int64_t) (mix64(0x9E3779B97F4A7C15ull + (unsigned long long) j) % (unsigned long long) total) - p.firstRow;
   if (row < 0 || row >= p.nRows) return;
   unsigned long long w[kSortTupleWords];
   sortTupleOf(p, s, row, w);
#pragma unroll
   for (int x = 0; x < kSortTupleWords; x++) out[(size_t) j * kSortTupleWords + x] = w[x];
}

// Permute: rows ids[0..n) (ids null: rows 0..n-1) of a table of one or more batches into new single-batch columns: fixed-width cells at
// outBytes (a narrowed decimal sign-extended, as the exchange ships it) and validity bytes by row id; a utf8 column's lengths by row id
// (permuteCellsKernel, which also sums each CTA's bytes), the exclusive scan of the CTA sums (rowScanKernel), then its offsets and
// bytes (permuteStringsKernel: each warp copies its 32 rows' strings, one contiguous range of the output, together).
constexpr uint32_t kPermuteNone = 0xffffffffu; // the id of a row of NULL cells (no caller has 2^32 - 1 rows)
struct PermuteBatch {
   ProgCol cols[kShipMaxCols];
   int64_t firstRow, nRows;
};
struct PermuteParams {
   const PermuteBatch* dir; // device, sorted by firstRow
   int32_t nBatches, nCols, nStr, pad;
   int32_t outBytes[kShipMaxCols];
   int8_t strOf[kShipMaxCols], strCol[kShipMaxCols];
   const uint32_t* ids;
   int64_t n, nCtas;
   uint8_t* data[kShipMaxCols]; // cells, or n + 1 int32 offsets (lengths until permuteStringsKernel)
   uint8_t* valid[kShipMaxCols];
   uint8_t* chars[kShipMaxCols];
   unsigned long long* hist; // [nStr][nCtas]: a CTA's bytes, then (scanned) where they start
};
// the batch holding row `row`, as the program kernel's side-column directory is searched
__device__ __forceinline__ const PermuteBatch& permuteBatchOf(const PermuteParams& q, int64_t row) {
   int lo = 0, hi = q.nBatches - 1;
   while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (q.dir[mid].firstRow <= row) lo = mid;
      else hi = mid - 1;
   }
   return q.dir[lo];
}
__global__ void __launch_bounds__(kShipThreads) permuteCellsKernel(const __grid_constant__ PermuteParams q) {
   __shared__ unsigned long long bytes[kShipMaxCols];
   for (int j = threadIdx.x; j < kShipMaxCols; j += kShipThreads) bytes[j] = 0;
   __syncthreads();
   const int64_t begin = (int64_t) blockIdx.x * kShipTile, end = min(begin + kShipTile, q.n);
   for (int64_t t = begin; t < end; t += kShipThreads) {
      const int64_t i = t + threadIdx.x;
      const bool ok = i < end;
      const uint32_t id = ok && q.ids ? q.ids[i] : 0u;
      const bool none = id == kPermuteNone; // a NULL row: NULL cells (the nested-loop join's unmatched side)
      const int64_t row = !ok || none ? 0 : q.ids ? (int64_t) id : i;
      const PermuteBatch& b = permuteBatchOf(q, row);
      const int64_t r = none ? 0 : row - b.firstRow;
      for (int c = 0; c < q.nCols; c++) {
         const ProgCol& col = b.cols[c];
         uint32_t len = 0;
         if (ok && none) {
            q.valid[c][i] = 0;
            if (q.strOf[c] < 0) {
               for (int x = 0; x < q.outBytes[c]; x++) q.data[c][(size_t) i * q.outBytes[c] + x] = 0;
            } else {
               ((uint32_t*) q.data[c])[i] = 0;
            }
         } else if (ok) {
            const bool null = colIsNull(col, r);
            q.valid[c][i] = null ? 0 : 1;
            if (q.strOf[c] < 0) {
               shipCell(col, q.outBytes[c], r, q.data[c] + (size_t) i * q.outBytes[c]);
            } else {
               if (!null) len = (uint32_t) (((const int32_t*) col.data)[r + 1] - ((const int32_t*) col.data)[r]);
               ((uint32_t*) q.data[c])[i] = len;
            }
         }
         if (q.strOf[c] >= 0) {
            const unsigned sum = __reduce_add_sync(0xffffffffu, len);
            if ((threadIdx.x & 31) == 0 && sum) atomicAdd(&bytes[q.strOf[c]], (unsigned long long) sum);
         }
      }
   }
   __syncthreads();
   for (int j = threadIdx.x; j < q.nStr; j += kShipThreads) q.hist[(size_t) j * q.nCtas + blockIdx.x] = bytes[j];
}
__global__ void __launch_bounds__(kShipThreads) permuteStringsKernel(const __grid_constant__ PermuteParams q) {
   __shared__ unsigned long long warpSums[kShipWarps];
   __shared__ unsigned long long running;
   __shared__ uint32_t slotEnd[kShipWarps][33]; // the warp's strings: slot k at [slotEnd[k], slotEnd[k+1]) of the warp's range
   __shared__ const uint8_t* slotSrc[kShipWarps][32];
   const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
   const int64_t begin = (int64_t) blockIdx.x * kShipTile, end = min(begin + kShipTile, q.n);
   for (int j = 0; j < q.nStr; j++) {
      const int c = q.strCol[j];
      int32_t* off = (int32_t*) q.data[c];
      uint8_t* out = q.chars[c];
      if (threadIdx.x == 0) running = q.hist[(size_t) j * q.nCtas + blockIdx.x];
      __syncthreads();
      for (int64_t t = begin; t < end; t += kShipThreads) {
         const int64_t i = t + threadIdx.x;
         const bool ok = i < end;
         const uint32_t len = ok ? (uint32_t) off[i] : 0u;
         const uint8_t* src = nullptr;
         if (ok && len) {
            const int64_t row = q.ids ? (int64_t) q.ids[i] : i;
            const PermuteBatch& b = permuteBatchOf(q, row);
            const ProgCol& col = b.cols[c];
            src = col.bytes + ((const int32_t*) col.data)[row - b.firstRow];
         }
         uint32_t x = len; // inclusive scan of the warp's lengths
         for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
         }
         if (lane == 31) warpSums[warp] = x;
         slotEnd[warp][lane + 1] = x;
         if (lane == 0) slotEnd[warp][0] = 0;
         slotSrc[warp][lane] = src;
         __syncthreads();
         unsigned long long warpBase = running;
         for (int w = 0; w < warp; w++) warpBase += warpSums[w];
         if (ok) {
            off[i] = (int32_t) (warpBase + x - len);
            if (i == q.n - 1) off[q.n] = (int32_t) (warpBase + x);
         }
         __syncwarp();
         const uint32_t total = slotEnd[warp][32];
         unsigned k = 0;
         for (uint32_t a = lane; a < total; a += 32) {
            while (slotEnd[warp][k + 1] <= a) k++;
            out[warpBase + a] = slotSrc[warp][k][a - slotEnd[warp][k]];
         }
         __syncthreads();
         if (threadIdx.x == 0)
            for (int w = 0; w < kShipWarps; w++) running += warpSums[w];
         __syncthreads();
      }
   }
}

// ---------------------------------------------------------------- dictionary unification (ldb_gpu_dict_unify, include/ldb_gpu.h)
// This rank's exported dictionary into its block of receiver blockIdx.y's region: the offsets array and the bytes array, each padded to
// 16 bytes, back to back, so the block is one run of 16-byte vectors.  The sources are padded the same way.
__global__ void __launch_bounds__(256) dictSendKernel(const __grid_constant__ PeerView v, size_t blockOff, const int4* offsets, size_t offVecs, const int4* bytes, size_t byteVecs) {
   int4* dst = (int4*) (v.heap[blockIdx.y] + blockOff);
   for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < offVecs + byteVecs; i += (size_t) gridDim.x * blockDim.x) dst[i] = i < offVecs ? offsets[i] : bytes[i - offVecs];
}

} // namespace ldb

using namespace ldb;

// ---------------------------------------------------------------- host side
PeerView LdbComm::view() const {
   PeerView v{};
   v.rank = rank;
   v.world = world;
   for (int i = 0; i < world; i++) v.heap[i] = peerHeap[i];
   v.error = error;
   v.timeoutNs = timeoutNs;
   return v;
}

extern "C" {

int64_t ldb_gpu_comm_reserved_bytes(void) { return (int64_t) kUserOff; }

int ldb_gpu_comm_create(LdbContext* ctx, int32_t rank, int32_t world, int64_t user_bytes, LdbComm** out, uint8_t* handle_out, LdbError* err) {
   return guarded(err, [&] {
      if (!ctx || !out || !handle_out) fail(LDB_ERR_INVALID, "null argument");
      if (world < 1 || world > kMaxPeers || rank < 0 || rank >= world) fail(LDB_ERR_INVALID, "rank/world out of range (1..8 ranks)");
      if (user_bytes < 0) fail(LDB_ERR_INVALID, "negative heap size");
      LDB_CUDA(cudaSetDevice(ctx->device));
      auto c = std::make_unique<LdbComm>();
      c->ctx = ctx;
      c->rank = rank;
      c->world = world;
      c->userBytes = ((size_t) user_bytes + 255) & ~size_t(255);
      c->heapBytes = kUserOff + c->userBytes + 256;
      LDB_CUDA(cudaMalloc((void**) &c->heap, c->heapBytes)); // plain cudaMalloc: legacy IPC handles cannot export pool / VMM allocations
      LDB_CUDA(cudaMemsetAsync(c->heap, 0, kUserOff, ctx->compute));
      c->error = (int32_t*) (c->heap + kUserOff + c->userBytes);
      LDB_CUDA(cudaMemsetAsync(c->error, 0, 256, ctx->compute));
      ctx->syncStream(ctx->compute);
      c->peerHeap[rank] = c->heap;
      if (const char* e = getenv("LDB_PEER_TIMEOUT_MS")) c->timeoutNs = (unsigned long long) std::max(1, atoi(e)) * 1000000ull;
      // CUDA loads kernels lazily, and loading one may have to wait for running kernels: a collective kernel that spins on a peer
      // while the next launch (of this or another rank in the same process) is still being loaded would stall until the
      // timeout — so every collective kernel is loaded now
      cudaFuncAttributes fa;
      LDB_CUDA(cudaFuncGetAttributes(&fa, peerBarrierKernel));
      LDB_CUDA(cudaFuncGetAttributes(&fa, peerBumpKernel));
      LDB_CUDA(cudaFuncGetAttributes(&fa, peerAllGatherKernel));
      LDB_CUDA(cudaFuncGetAttributes(&fa, peerGroupAllMergeKernel));
      LDB_CUDA(cudaFuncGetAttributes(&fa, peerOrReduceKernel));
      LDB_CUDA(cudaFuncGetAttributes(&fa, peerPublishCountsKernel));
      LDB_CUDA(cudaFuncGetAttributes(&fa, tableShipCountKernel));
      LDB_CUDA(cudaFuncGetAttributes(&fa, rowScanKernel<unsigned long long>));
      LDB_CUDA(cudaFuncGetAttributes(&fa, tableShipSendKernel<false>));
      LDB_CUDA(cudaFuncGetAttributes(&fa, tableShipSendKernel<true>));
      LDB_CUDA(cudaFuncGetAttributes(&fa, tableShipCountRangeKernel));
      LDB_CUDA(cudaFuncGetAttributes(&fa, sortSampleKernel));
      LDB_CUDA(cudaFuncGetAttributes(&fa, permuteCellsKernel));
      LDB_CUDA(cudaFuncGetAttributes(&fa, permuteStringsKernel));
      LDB_CUDA(cudaFuncGetAttributes(&fa, dictSendKernel));
      loadHashAggExchangeKernels();
      // the pinned scratch the collectives read counts into: allocating host memory can wait for running kernels, so it is taken now
      // rather than on a rank's first collective while a peer of the same process may already be waiting for it
      ctx->scratch();
      cudaIpcMemHandle_t h;
      LDB_CUDA(cudaIpcGetMemHandle(&h, c->heap));
      static_assert(sizeof(h) == LDB_IPC_HANDLE_BYTES, "cudaIpcMemHandle_t is 64 bytes");
      memcpy(handle_out, &h, sizeof(h));
      *out = c.release();
   });
}

// all_handles: world x 64 bytes in rank order (exchanged by the caller: torch.distributed all_gather, MPI, a file …)
int ldb_gpu_comm_connect(LdbComm* c, const uint8_t* all_handles, LdbError* err) {
   return guarded(err, [&] {
      if (!c || !all_handles) fail(LDB_ERR_INVALID, "null argument");
      LDB_CUDA(cudaSetDevice(c->ctx->device));
      for (int p = 0; p < c->world; p++) {
         if (p == c->rank) continue;
         cudaIpcMemHandle_t h;
         memcpy(&h, all_handles + (size_t) p * LDB_IPC_HANDLE_BYTES, sizeof(h));
         void* ptr = nullptr;
         LDB_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
         c->peerHeap[p] = (uint8_t*) ptr;
         c->ipcOpened[p] = true;
      }
      c->connected = true;
   });
}

// single-process variant (tests, one process driving several devices): peers are other LdbComm objects of this process
int ldb_gpu_comm_connect_local(LdbComm** comms, int32_t n, LdbError* err) {
   return guarded(err, [&] {
      if (!comms || n < 1 || n > kMaxPeers) fail(LDB_ERR_INVALID, "bad comm list");
      for (int i = 0; i < n; i++) {
         if (!comms[i] || comms[i]->world != n || comms[i]->rank != i) fail(LDB_ERR_INVALID, "comm list must hold ranks 0..n-1 of one world");
         LDB_CUDA(cudaSetDevice(comms[i]->ctx->device));
         for (int p = 0; p < n; p++) {
            if (p == i) continue;
            if (comms[p]->ctx->device != comms[i]->ctx->device) {
               int can = 0;
               LDB_CUDA(cudaDeviceCanAccessPeer(&can, comms[i]->ctx->device, comms[p]->ctx->device));
               if (!can) fail(LDB_ERR_UNSUPPORTED, "devices cannot access each other's memory");
               cudaError_t e = cudaDeviceEnablePeerAccess(comms[p]->ctx->device, 0);
               if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) LDB_CUDA(e);
               cudaGetLastError();
            }
            comms[i]->peerHeap[p] = comms[p]->heap;
         }
         comms[i]->connected = true;
      }
   });
}

void ldb_gpu_comm_destroy(LdbComm* c) {
   if (!c) return;
   cudaSetDevice(c->ctx->device);
   cudaStreamSynchronize(c->ctx->compute);
   for (int p = 0; p < c->world; p++)
      if (c->ipcOpened[p]) cudaIpcCloseMemHandle(c->peerHeap[p]);
   cudaFree(c->heap);
   delete c;
}

void* ldb_gpu_comm_heap(LdbComm* c, int64_t* user_bytes) {
   if (!c) return nullptr;
   if (user_bytes) *user_bytes = (int64_t) c->userBytes;
   return c->heap + kUserOff;
}
int32_t ldb_gpu_comm_rank(LdbComm* c) { return c ? c->rank : -1; }
int32_t ldb_gpu_comm_world(LdbComm* c) { return c ? c->world : 0; }

static void wantConnected(LdbComm* c) {
   if (!c) fail(LDB_ERR_INVALID, "null comm");
   if (!c->connected && c->world > 1) fail(LDB_ERR_INVALID, "comm is not connected to its peers yet");
}

// the barrier on the compute stream (the current device is the comm's)
static void commBarrier(LdbComm* c) {
   if (c->world == 1) return;
   LdbContext* ctx = c->ctx;
   ctx->launch("peer_barrier", [&] {
      peerBarrierKernel<<<c->world, 32, 0, ctx->compute>>>(c->view());
      peerBumpKernel<<<1, 1, 0, ctx->compute>>>(c->view(), EPOCH_BARRIER, -1);
   });
}
// waits for the compute stream and fails if a collective's wait timed out; the error word is read into pinned memory (a pageable copy
// could stall a peer of the same process: see ldb_gpu_hashagg_exchange)
static void checkPeers(LdbComm* c, int32_t* pinnedWord) {
   LDB_CUDA(cudaMemcpyAsync(pinnedWord, c->error, 4, cudaMemcpyDeviceToHost, c->ctx->compute));
   c->ctx->syncStream(c->ctx->compute);
   if (*pinnedWord) fail(LDB_ERR_CUDA, "a peer did not arrive at a collective within the timeout (LDB_PEER_TIMEOUT_MS)");
}

int ldb_gpu_comm_barrier(LdbComm* c, LdbError* err) {
   return guarded(err, [&] {
      wantConnected(c);
      if (c->world == 1) return;
      LDB_CUDA(cudaSetDevice(c->ctx->device));
      commBarrier(c);
   });
}

// all-gather of `bytes` (multiple of 16, <= kSlotBytes) from DEVICE memory `src`, eagerly on the compute stream (not inside a capture);
// returns this rank's mailbox half the collective fills: block of rank r at result + r * kSlotBytes, valid until the next-but-one gather
static uint8_t* allGatherSmall(LdbComm* c, const void* src, size_t bytes) {
   LdbContext* ctx = c->ctx;
   const unsigned long long epoch = ++c->gatherEpochHost; // mirror of the device counter (every rank issues the same collectives)
   ctx->launch("peer_allgather", [&] {
      peerAllGatherKernel<<<c->world, 256, 0, ctx->compute>>>(c->view(), (const uint8_t*) src, bytes);
      peerBumpKernel<<<1, 1, 0, ctx->compute>>>(c->view(), EPOCH_GATHER, -1);
   });
   return c->heap + kMailboxOff + (size_t) (epoch & 1) * c->world * kSlotBytes;
}

// all-gather of `bytes` (multiple of 16, <= slot size) from DEVICE memory `src`; returns the device address of the gathered
// blocks of this collective: block of rank r at result + r * ldb_gpu_comm_slot_bytes().  Valid until the next-but-one gather.
int64_t ldb_gpu_comm_slot_bytes(void) { return (int64_t) kSlotBytes; }
int ldb_gpu_comm_allgather_small(LdbComm* c, const void* src, int64_t bytes, void** result, LdbError* err) {
   return guarded(err, [&] {
      wantConnected(c);
      if (bytes <= 0 || bytes > (int64_t) kSlotBytes || bytes % 16) fail(LDB_ERR_INVALID, "all-gather blocks are 16..262144 bytes, multiples of 16");
      LdbContext* ctx = c->ctx;
      LDB_CUDA(cudaSetDevice(ctx->device));
      if (ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "the small all-gather returns a parity-dependent address and cannot be captured");
      uint8_t* gathered = allGatherSmall(c, src, (size_t) bytes);
      if (result) *result = gathered;
   });
}

int ldb_gpu_groupby_allmerge(LdbState* s, LdbComm* c, LdbError* err) {
   return guarded(err, [&] {
      if (!s || (s->kind != LDB_STATE_GROUPBY && s->kind != LDB_STATE_SIMPLE)) fail(LDB_ERR_INVALID, "not a group state");
      wantConnected(c);
      if (s->ctx != c->ctx) fail(LDB_ERR_INVALID, "state and comm belong to different contexts");
      ldb_gpu_want_bound_lanes_internal(s);
      if (c->world == 1) return;
      const size_t image = (groupImageBytes(s->group.capacity) + 15) & ~size_t(15); // the table allocation carries 16 spare bytes (error word)
      if (image > kSlotBytes) fail(LDB_ERR_UNSUPPORTED, "group table image larger than a mailbox slot (capacity <= 1024 groups)");
      LdbContext* ctx = c->ctx;
      LDB_CUDA(cudaSetDevice(ctx->device));
      // the mirror follows the device epoch: bumped when the kernel runs (now, or at every replay of a capture), never at capture
      if (ctx->capturing) ctx->capturing->onLaunch.push_back([c] { ++c->gatherEpochHost; });
      else ++c->gatherEpochHost;
      ctx->launch("peer_group_allmerge", [&] {
         peerGroupAllMergeKernel<<<c->world, 256, 0, ctx->compute>>>(c->view(), s->group, image);
         peerBumpKernel<<<1, 1, 0, ctx->compute>>>(c->view(), EPOCH_GATHER, EPOCH_MERGE);
      });
   });
}

int ldb_gpu_comm_or_reduce(LdbComm* c, int64_t user_offset, int64_t bytes, LdbError* err) {
   return guarded(err, [&] {
      wantConnected(c);
      if (user_offset < 0 || bytes < 0 || user_offset % 16 || bytes % 16 || (size_t) (user_offset + bytes) > c->userBytes) fail(LDB_ERR_INVALID, "OR-reduce range outside the heap or not 16-byte aligned");
      if (c->world == 1 || bytes == 0) return;
      LdbContext* ctx = c->ctx;
      LDB_CUDA(cudaSetDevice(ctx->device));
      const size_t n4 = (size_t) bytes / 16;
      const int grid = (int) std::min<size_t>((n4 + 255) / 256, (size_t) ctx->smCount * 8);
      ctx->launch("peer_or_reduce", [&] { peerOrReduceKernel<<<grid, 256, 0, ctx->compute>>>(c->view(), kUserOff + (size_t) user_offset, n4); });
   });
}

int ldb_gpu_comm_heap_zero(LdbComm* c, int64_t user_offset, int64_t bytes, LdbError* err) {
   return guarded(err, [&] {
      if (!c || user_offset < 0 || bytes < 0 || (size_t) (user_offset + bytes) > c->userBytes) fail(LDB_ERR_INVALID, "range outside the comm's user heap");
      LDB_CUDA(cudaSetDevice(c->ctx->device));
      LDB_CUDA(cudaMemsetAsync(c->heap + kUserOff + user_offset, 0, (size_t) bytes, c->ctx->compute));
   });
}
int ldb_gpu_comm_heap_read(LdbComm* c, int64_t user_offset, int64_t bytes, void* host_dst, LdbError* err) {
   return guarded(err, [&] {
      if (!c || !host_dst || user_offset < 0 || bytes < 0 || (size_t) (user_offset + bytes) > c->userBytes) fail(LDB_ERR_INVALID, "range outside the comm's user heap");
      LDB_CUDA(cudaSetDevice(c->ctx->device));
      LDB_CUDA(cudaMemcpyAsync(host_dst, c->heap + kUserOff + user_offset, (size_t) bytes, cudaMemcpyDeviceToHost, c->ctx->compute));
      c->ctx->syncStream(c->ctx->compute);
   });
}
static void wantRange(LdbComm* c, int64_t off, int64_t bytes, const char* what) {
   if (off < 0 || bytes < 0 || off % 16 || (size_t) (off + bytes) > c->userBytes) fail(LDB_ERR_CAPACITY, std::string(what) + " outside the comm's user heap (create the comm with a larger heap)");
}
int ldb_gpu_comm_publish_counts(LdbComm* c, int64_t cursors_offset, int64_t counts_offset, LdbError* err) {
   return guarded(err, [&] {
      wantConnected(c);
      wantRange(c, cursors_offset, 16 * 8, "cursors");
      wantRange(c, counts_offset, kMaxPeers * 8, "counts");
      LdbContext* ctx = c->ctx;
      LDB_CUDA(cudaSetDevice(ctx->device));
      ctx->launch("peer_publish_counts", [&] { peerPublishCountsKernel<<<1, 32, 0, ctx->compute>>>(c->view(), kUserOff + (size_t) cursors_offset, kUserOff + (size_t) counts_offset); });
   });
}
int ldb_gpu_join_table_insert_received(LdbState* table, LdbComm* c, int64_t recv_offset, int64_t capacity, int64_t counts_offset, LdbError* err) {
   return guarded(err, [&] {
      wantConnected(c);
      if (!table || table->kind != LDB_STATE_JOIN_TABLE || table->join.stride != 8 || table->join.direct) fail(LDB_ERR_INVALID, "insert target must be a plain single-key join table");
      wantRange(c, recv_offset, (int64_t) c->world * capacity * 8, "receive region");
      wantRange(c, counts_offset, kMaxPeers * 8, "counts");
      LdbContext* ctx = c->ctx;
      LDB_CUDA(cudaSetDevice(ctx->device));
      uint8_t* user = c->heap + kUserOff;
      ctx->launch("join_build", [&] { launchInsertReceived(table->join, user + recv_offset, c->world, capacity, (const unsigned long long*) (user + counts_offset), ctx->smCount, ctx->compute); });
   });
}
int ldb_gpu_probe_received_groupby(LdbState* ta, LdbState* tb, LdbState* groups, LdbComm* c, int64_t recv_offset, int64_t capacity, int64_t counts_offset, int32_t scale, LdbError* err) {
   return guarded(err, [&] {
      wantConnected(c);
      for (LdbState* t : {ta, tb})
         if (!t || t->kind != LDB_STATE_JOIN_TABLE || t->join.stride != 8 || t->join.direct) fail(LDB_ERR_INVALID, "probe tables must be plain single-key join tables");
      if (!groups || groups->kind != LDB_STATE_GROUPBY || groups->group.nKeys != 1 || groups->group.nAggs != 1) fail(LDB_ERR_INVALID, "sink must be a group-by state with one key and one aggregate");
      if (scale < 0 || scale > 18) fail(LDB_ERR_INVALID, "decimal scale out of range");
      wantRange(c, recv_offset, (int64_t) c->world * capacity * 24, "receive region");
      wantRange(c, counts_offset, kMaxPeers * 8, "counts");
      ldb_gpu_bind_lane_width_internal(groups, 0, LDB_EXPR_MUL_1MINUS); // a * (10^scale - b): a 128-bit sum
      int64_t one = 1;
      for (int i = 0; i < scale; i++) one *= 10;
      LdbContext* ctx = c->ctx;
      LDB_CUDA(cudaSetDevice(ctx->device));
      uint8_t* user = c->heap + kUserOff;
      ctx->launch("join_probe2_groupby", [&] {
         launchProbeReceivedGroupBy(ta->join, tb->join, groups->group, user + recv_offset, c->world, capacity, (const unsigned long long*) (user + counts_offset), one, ctx->smCount, ctx->compute);
      });
   });
}

int ldb_gpu_probe_received_groupby2(LdbState* table, LdbState* groups, LdbComm* c, int64_t recv_offset, int64_t capacity, int64_t counts_offset, LdbError* err) {
   return guarded(err, [&] {
      wantConnected(c);
      if (!table || table->kind != LDB_STATE_JOIN_TABLE || table->join.stride != 8 || table->join.direct) fail(LDB_ERR_INVALID, "probe table must be a plain single-key join table");
      if (!groups || groups->kind != LDB_STATE_GROUPBY || groups->group.nKeys != 2 || groups->group.nAggs != 1) fail(LDB_ERR_INVALID, "sink must be a group-by state with two keys and one aggregate");
      wantRange(c, recv_offset, (int64_t) c->world * capacity * 24, "receive region");
      wantRange(c, counts_offset, kMaxPeers * 8, "counts");
      ldb_gpu_bind_lane_width_internal(groups, 0, LDB_EXPR_MUL_1MINUS_MINUS_PAYMUL); // the shipped K11 sums are 128-bit
      LdbContext* ctx = c->ctx;
      LDB_CUDA(cudaSetDevice(ctx->device));
      uint8_t* user = c->heap + kUserOff;
      ctx->launch("join_probe_received_groupby", [&] {
         launchProbeReceivedGroupBy2(table->join, groups->group, user + recv_offset, c->world, capacity, (const unsigned long long*) (user + counts_offset), ctx->smCount, ctx->compute);
      });
   });
}

// Partitioned merge of program hash aggregations (include/ldb_gpu.h).  User-heap layout from recv_offset: the receive region (world
// sub-regions of `capacity` entries, program.h HashAggShip), then this rank's cursors u64[kMaxPeers], then its counts u64[kMaxPeers].
// barrier (nobody still merges an earlier exchange out of the region) → zero cursors → send → publish counts → barrier → host read of
// the counts (overflow check) → merge.
static_assert(kMaxPeers == sizeof(HashAggShip::recv) / sizeof(uint8_t*), "HashAggShip holds one receive region per peer");
int ldb_gpu_hashagg_exchange(LdbState* local, LdbState* owned, LdbComm* c, int64_t recv_offset, int64_t capacity, LdbError* err) {
   return guarded(err, [&] {
      if (!local || !owned || !c) fail(LDB_ERR_INVALID, "null argument");
      if (local->kind != LDB_STATE_HASHAGG || owned->kind != LDB_STATE_HASHAGG) fail(LDB_ERR_INVALID, "the exchange takes two hash aggregation states");
      if (local == owned) fail(LDB_ERR_INVALID, "local and owned must be two distinct states");
      if (local->ctx != c->ctx || owned->ctx != c->ctx) fail(LDB_ERR_INVALID, "states and comm belong to different contexts");
      const HashAggDev& lt = local->hashagg;
      const HashAggDev& ot = owned->hashagg;
      if (lt.nKeys != ot.nKeys) fail(LDB_ERR_INVALID, "local and owned have different key counts");
      if (lt.nAggs != ot.nAggs) fail(LDB_ERR_INVALID, "local and owned have different aggregate counts");
      for (int a = 0; a < lt.nAggs; a++)
         if (local->aggKinds[a] != owned->aggKinds[a]) fail(LDB_ERR_INVALID, "local and owned have different aggregate kinds");
      wantConnected(c);
      const int64_t entry = (int64_t) lt.entryBytes, tail = 2 * 8 * kMaxPeers;
      const int64_t user = (int64_t) c->userBytes;
      if (capacity < 0 || recv_offset < 0 || recv_offset % 16 || recv_offset > user || capacity > (user - recv_offset) / entry / c->world ||
          (int64_t) c->world * capacity * entry + tail > user - recv_offset)
         fail(LDB_ERR_INVALID, "receive region outside the comm's user heap or not 16-byte aligned");
      LdbContext* ctx = c->ctx;
      if (ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "the hash aggregation exchange reads the received counts on the host and cannot be captured");
      LDB_CUDA(cudaSetDevice(ctx->device));
      const size_t cursorsOff = (size_t) recv_offset + (size_t) c->world * (size_t) capacity * (size_t) entry, countsOff = cursorsOff + 8 * kMaxPeers;
      uint8_t* heap = c->heap + kUserOff;
      HashAggShip x{};
      for (int d = 0; d < c->world; d++) x.recv[d] = c->peerHeap[d] + kUserOff + recv_offset;
      x.cursors = (unsigned long long*) (heap + cursorsOff);
      x.counts = (const unsigned long long*) (heap + countsOff);
      x.capacity = capacity;
      x.rank = c->rank;
      x.world = c->world;
      for (int a = 0; a < lt.nAggs; a++) x.kinds[a] = local->aggKinds[a];
      // the counts are read into pinned memory (allocated before the first barrier): a copy into pageable memory blocks inside the driver
      // while this rank's barrier waits for the peers, and a peer of the same process could then not launch its own barrier
      unsigned long long* counts = (unsigned long long*) ctx->scratch();
      int32_t* timedOut = (int32_t*) (counts + kMaxPeers);
      commBarrier(c);
      ctx->launch("hashagg_send", [&] {
         LDB_CUDA(cudaMemsetAsync(x.cursors, 0, 8 * kMaxPeers, ctx->compute));
         launchHashAggSend(lt, x, ctx->smCount, ctx->compute);
         peerPublishCountsKernel<<<1, 32, 0, ctx->compute>>>(c->view(), kUserOff + cursorsOff, kUserOff + countsOff);
      });
      commBarrier(c);
      LDB_CUDA(cudaMemcpyAsync(counts, x.counts, 8 * (size_t) c->world, cudaMemcpyDeviceToHost, ctx->compute));
      checkPeers(c, timedOut);
      const unsigned long long most = *std::max_element(counts, counts + c->world);
      if (most > (unsigned long long) capacity)
         fail(LDB_ERR_CAPACITY, "hash aggregation exchange: a source sent this rank " + std::to_string(most) + " groups, more than the receive capacity " +
                                   std::to_string(capacity) + "; retry with capacity " + std::to_string(most));
      ctx->launch("hashagg_merge", [&] { launchHashAggMerge(ot, x, most, ctx->smCount, ctx->compute); });
   });
}

// Repartition of a table's rows (include/ldb_gpu.h).  count (per batch) → scan → all-gather of the per-destination totals → host read of
// the count matrix, capacity decision (identical on every rank) → barrier → send (per batch) → barrier → copy-out of the own region →
// host wait.  While a rank's collectives wait for its peers nothing here blocks inside the driver: the temporaries and the pinned
// scratch are taken before the first collective, the output buffers after the last, and host reads go to pinned memory.
// With utf8 columns (ldb_gpu_table_exchange_varlen) the count and send kernels also count and ship the strings' bytes, the matrix also
// carries every rank's bytes per (destination, utf8 column), and the host decides the int32 limit of the receivers' offsets before the
// capacity.  A broadcast without utf8 columns skips the count: every rank receives every source's rows, which the host knows.
// The sort exchange (ldb_gpu_table_sort_exchange) runs the same shipment with the range owner rule of its splitters; only the count
// kernel differs, and what it does with the received region (sort and permute instead of copy-out).
static_assert((size_t) kMaxPeers * kShipBlockU64 * 8 + 64 + 8 * kMaxPeers + 4 * kShipMaxCols <= LdbContext::kPinnedScratchBytes,
              "the table exchange's matrix, error word and offset ends fit the pinned scratch");
// the columns `columns` names (NULL: every column of src) as column indices of src
static std::vector<int> shipColumns(bool varlen, LdbTable* src, int32_t n_columns, const char* const* columns) {
   std::vector<int> ship;
   if (columns) {
      if (n_columns < 1) fail(LDB_ERR_INVALID, "columns names 1..16 columns (NULL: all columns of the table)");
      for (int i = 0; i < n_columns; i++) {
         const int ci = src->colIndex(columns[i]);
         if (ci < 0) fail(LDB_ERR_INVALID, std::string("unknown column ") + (columns[i] ? columns[i] : "(null)"));
         ship.push_back(ci);
      }
   } else {
      for (int ci = 0; ci < (int) src->columns.size(); ci++) ship.push_back(ci);
   }
   if (ship.size() > (size_t) kShipMaxCols) fail(LDB_ERR_INVALID, "the exchange ships up to 16 columns");
   for (int ci : ship)
      if (!varlen && src->columns[ci].type == LDB_UTF8) fail(LDB_ERR_UNSUPPORTED, "the exchange ships fixed-width columns (utf8 column " + src->columns[ci].name + ")");
   return ship;
}
static void wantRegion(LdbComm* c, int64_t recv_offset, int64_t recv_bytes) {
   if (recv_offset < 0 || recv_bytes < 0 || recv_offset % 16 || recv_offset > (int64_t) c->userBytes || recv_bytes > (int64_t) c->userBytes - recv_offset)
      fail(LDB_ERR_INVALID, "receive region outside the comm's user heap or not 16-byte aligned");
}

// One shipment of a table's rows, for arguments the caller checked.  The constructor takes what a rank needs before its first collective
// (staging waits, temporaries, pinned scratch); ship() counts under an owner rule (the key hash, or the splitters of a sort) and runs the
// protocol up to the second barrier, after which this rank's region holds its `mine` received rows at colOff / bytesOff / validOff;
// finish() waits for the work queued after it and reports a peer that timed out.
struct TableShipment {
   LdbTable* src;
   LdbComm* c;
   LdbContext* ctx;
   int world;
   std::vector<int> ship, key;
   int nCols, nStr = 0;
   int32_t outBytes[kShipMaxCols] = {};
   int8_t strCol[kShipMaxCols] = {}, strOf[kShipMaxCols] = {};
   bool broadcast, strings;
   size_t blockU64;
   int64_t nCtas = 0;
   Scratch tmp;
   unsigned long long *hist, *totals, *matrix, *upload;
   int32_t* timedOut;
   uint32_t* offEnds;
   TableShipBatch p{};
   int64_t recvOffset, regionBytes;
   unsigned long long mine = 0;
   uint64_t colOff[kShipMaxCols], validOff[kShipMaxCols], bytesOff[kShipMaxCols];
   uint8_t* region = nullptr;

   TableShipment(LdbTable* s, std::vector<int> shipped, std::vector<int> keys, LdbComm* comm, int64_t recv_offset, int64_t recv_bytes)
       : src(s), c(comm), ctx(comm->ctx), world(comm->world), ship(std::move(shipped)), key(std::move(keys)), nCols((int) ship.size()), tmp(comm->ctx),
         recvOffset(recv_offset), regionBytes(recv_bytes) {
      LDB_CUDA(cudaSetDevice(ctx->device));
      for (int j = 0; j < nCols; j++) outBytes[j] = shipCellBytes(src->columns[ship[j]].type);
      // before the first collective: staging waits, temporaries, pinned scratch
      for (auto& b : src->batches) ldb_gpu_wait_batch_internal(ctx, &b);
      for (auto& b : src->batches) nCtas += (b.nRows + kShipTile - 1) / kShipTile;
      // the utf8 columns among the shipped ones: the histograms have world (1 + nStr) rows
      for (int j = 0; j < nCols; j++) {
         strOf[j] = -1;
         if (src->columns[ship[j]].type == LDB_UTF8) {
            strOf[j] = (int8_t) nStr;
            strCol[nStr++] = (int8_t) j;
         }
      }
      strings = nStr > 0;
      blockU64 = (size_t) kMaxPeers * (1 + nStr); // this rank's totals in the all-gather: rows, then bytes per (d, column)
      broadcast = key.empty();
      uint8_t* owners = broadcast ? nullptr : tmp.alloc<uint8_t>((size_t) std::max<int64_t>(src->numRows, 1));
      hist = broadcast && !strings ? nullptr : tmp.alloc<unsigned long long>((size_t) std::max<int64_t>(nCtas, 1) * world * (1 + nStr) * 8);
      totals = tmp.alloc<unsigned long long>(8 * blockU64);
      matrix = (unsigned long long*) ctx->scratch(); // [world][blockU64]: M[s][d] at [s][d], Bytes[s][d][j] at [s][world + d nStr + j]
      timedOut = (int32_t*) (matrix + kMaxPeers * kShipBlockU64);
      upload = matrix + kMaxPeers * kShipBlockU64 + 8;
      offEnds = (uint32_t*) (upload + kMaxPeers); // B_j of this rank: the last offset of each received utf8 column
      p.nCols = nCols;
      p.nKeys = (int32_t) key.size();
      p.world = world;
      p.broadcast = broadcast ? 1 : 0;
      p.nCtas = nCtas;
      p.owners = owners;
      p.hist = hist;
      for (int j = 0; j < nCols; j++) p.outBytes[j] = outBytes[j];
      p.nStr = nStr;
      for (int j = 0; j < nCols; j++) p.strOf[j] = strOf[j];
      for (int j = 0; j < nStr; j++) p.strCol[j] = strCol[j];
   }
   TableShipBatch bindBatch(const LdbBatch& b, int64_t firstRow, int64_t ctaBase) const {
      TableShipBatch q = p;
      for (int j = 0; j < nCols; j++) {
         bindColumn(q.cols[j], b, ship[j]);
         q.cols[j].type = src->columns[ship[j]].type;
      }
      for (int k = 0; k < (int) key.size(); k++) {
         bindColumn(q.keys[k], b, key[k]);
         q.keys[k].type = src->columns[key[k]].type;
      }
      q.nRows = b.nRows;
      q.firstRow = firstRow;
      q.ctaBase = ctaBase;
      return q;
   }
   // every non-empty batch with its source row number and first CTA, in source order
   void eachBatch(const std::function<void(const TableShipBatch&, int)>& fn) const {
      int64_t first = 0, cta = 0;
      for (auto& b : src->batches) {
         if (b.nRows > 0) fn(bindBatch(b, first, cta), (int) ((b.nRows + kShipTile - 1) / kShipTile));
         first += b.nRows;
         cta += (b.nRows + kShipTile - 1) / kShipTile;
      }
   }
   // range: the owner rule of the sort exchange's splitters (null: the key hash, or every rank without keys)
   void run(const SortSplit* range) {
      if (broadcast && !strings) {
         for (int d = 0; d < kMaxPeers; d++) upload[d] = d < world ? (unsigned long long) src->numRows : 0ull;
         LDB_CUDA(cudaMemcpyAsync(totals, upload, 8 * kMaxPeers, cudaMemcpyHostToDevice, ctx->compute));
      } else {
         ctx->launch("table_exchange_count", [&] {
            LDB_CUDA(cudaMemsetAsync(totals, 0, 8 * blockU64, ctx->compute));
            eachBatch([&](const TableShipBatch& q, int grid) {
               if (range) tableShipCountRangeKernel<<<grid, kShipThreads, 0, ctx->compute>>>(q, *range);
               else tableShipCountKernel<<<grid, kShipThreads, 0, ctx->compute>>>(q);
            });
            rowScanKernel<<<world * (1 + nStr), 1024, 0, ctx->compute>>>(hist, nCtas, totals);
         });
      }
      // the count matrix on every rank
      if (world == 1) {
         LDB_CUDA(cudaMemcpyAsync(matrix, totals, 8 * blockU64, cudaMemcpyDeviceToHost, ctx->compute));
      } else {
         const uint8_t* gathered = allGatherSmall(c, totals, 8 * blockU64);
         LDB_CUDA(cudaMemcpy2DAsync(matrix, 8 * blockU64, gathered, kSlotBytes, 8 * blockU64, world, cudaMemcpyDeviceToHost, ctx->compute));
      }
      checkPeers(c, timedOut);
      // per receiver, from the same matrix on every rank: its rows and bytes, this source's bases in them, then the two decisions.  A
      // broadcast counted every row for destination 0, and every rank receives what destination 0 would.
      auto rowsOf = [&](int s, int d) { return matrix[s * blockU64 + (broadcast ? 0 : d)]; };
      auto bytesOf = [&](int s, int d, int j) { return matrix[s * blockU64 + world + (broadcast ? 0 : d) * nStr + j]; };
      uint64_t recvBytes[kMaxPeers][kShipMaxCols] = {};
      for (int d = 0; d < world; d++) {
         unsigned long long n = 0;
         for (int s = 0; s < world; s++) {
            if (s == c->rank) p.base[d] = n;
            n += rowsOf(s, d);
         }
         p.rows[d] = n;
         for (int j = 0; j < nStr; j++) {
            for (int s = 0; s < world; s++) {
               if (s == c->rank) p.byteBase[d][j] = (uint32_t) std::min<uint64_t>(recvBytes[d][j], INT32_MAX); // exact once the limit holds
               recvBytes[d][j] += bytesOf(s, d, j);
            }
         }
      }
      for (int d = 0; d < world; d++)
         for (int j = 0; j < nStr; j++)
            if (recvBytes[d][j] > (uint64_t) INT32_MAX)
               fail(LDB_ERR_UNSUPPORTED, "table exchange: rank " + std::to_string(d) + " would receive " + std::to_string(recvBytes[d][j]) + " bytes of utf8 column " +
                                            src->columns[ship[strCol[j]]].name + ", more than 2^31 - 1 (utf8 offsets are int32)");
      uint64_t need = 0;
      for (int d = 0; d < world; d++) {
         for (int j = 0; j < nStr; j++) p.strBytes[d][j] = (uint32_t) recvBytes[d][j];
         need = std::max(need, shipLayout(p.rows[d], outBytes, nCols, strOf, nStr, p.strBytes[d], colOff, validOff, bytesOff));
      }
      if (need > (uint64_t) regionBytes)
         fail(LDB_ERR_CAPACITY, "table exchange: a rank receives rows that need " + std::to_string(need) + " bytes of receive region, more than recv_bytes " +
                                   std::to_string(regionBytes) + "; retry with recv_bytes " + std::to_string(need));
      mine = p.rows[c->rank];
      for (int d = 0; d < world; d++) p.recv[d] = c->peerHeap[d] + kUserOff + recvOffset;
      commBarrier(c); // no peer still copies out of, or otherwise reads, the region it is about to receive into
      ctx->launch("table_exchange_send", [&] {
         eachBatch([&](const TableShipBatch& q, int grid) {
            TableShipBatch r = q;
            for (int d = 0; d < world; d++) {
               r.recv[d] = p.recv[d];
               r.rows[d] = p.rows[d];
               r.base[d] = p.base[d];
               for (int j = 0; j < nStr; j++) {
                  r.strBytes[d][j] = p.strBytes[d][j];
                  r.byteBase[d][j] = p.byteBase[d][j];
               }
            }
            if (strings) tableShipSendKernel<true><<<grid, kShipThreads, 0, ctx->compute>>>(r);
            else tableShipSendKernel<false><<<grid, kShipThreads, 0, ctx->compute>>>(r);
         });
      });
      commBarrier(c); // every peer's rows are in this rank's region
      shipLayout(mine, outBytes, nCols, strOf, nStr, p.strBytes[c->rank], colOff, validOff, bytesOff);
      region = c->heap + kUserOff + recvOffset;
      // a utf8 column's last offset is B_j, which the matrix gave: written into the region, its n + 1 offsets are one array
      for (int j = 0; j < nStr; j++) {
         offEnds[j] = p.strBytes[c->rank][j];
         LDB_CUDA(cudaMemcpyAsync(region + colOff[strCol[j]] + mine * 4, &offEnds[j], 4, cudaMemcpyHostToDevice, ctx->compute));
      }
   }
   // the received rows as a single-batch table over the region (valid until finish())
   void receivedView(LdbTable& v) const {
      v.ctx = ctx;
      v.numRows = (int64_t) mine;
      v.batches.resize(1);
      LdbBatch& b = v.batches[0];
      b.nRows = (int64_t) mine;
      for (int j = 0; j < nCols; j++) {
         v.columns.push_back(src->columns[ship[j]]);
         b.data.push_back(region + colOff[j]);
         b.bytes.push_back(strOf[j] >= 0 ? region + bytesOff[strOf[j]] : nullptr);
         b.elemBytes.push_back(outBytes[j]);
         b.validBytes.push_back(region + validOff[j]);
      }
   }
   void finish() { checkPeers(c, timedOut); } // the region is free for the next collective, the temporaries for the pool
};

static void tableExchange(bool varlen, LdbTable* src, int32_t n_keys, const char* const* key_columns, int32_t n_columns, const char* const* columns, LdbComm* c,
                          int64_t recv_offset, int64_t recv_bytes, const char* name, LdbTable** out) {
   if (!src || !c || !out || (n_keys > 0 && !key_columns)) fail(LDB_ERR_INVALID, "null argument");
   if (n_keys < 0 || n_keys > kProgMaxKeys) fail(LDB_ERR_INVALID, "the exchange takes 0..4 key columns");
   if (src->ctx != c->ctx) fail(LDB_ERR_INVALID, "table and comm belong to different contexts");
   std::vector<int> ship = shipColumns(varlen, src, n_columns, columns), key;
   for (int k = 0; k < n_keys; k++) {
      const int ci = src->colIndex(key_columns[k]);
      if (ci < 0) fail(LDB_ERR_INVALID, std::string("unknown key column ") + (key_columns[k] ? key_columns[k] : "(null)"));
      const int type = src->columns[ci].type;
      if (type == LDB_UTF8 || type == LDB_FLOAT32 || type == LDB_FLOAT64) fail(LDB_ERR_UNSUPPORTED, "exchange keys are integer, date, char(1) or decimal columns");
      key.push_back(ci);
   }
   wantConnected(c);
   wantRegion(c, recv_offset, recv_bytes);
   LdbContext* ctx = c->ctx;
   if (ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "the table exchange reads the row counts on the host and cannot be captured");
   TableShipment s(src, std::move(ship), std::move(key), c, recv_offset, recv_bytes);
   s.run(nullptr);
   // copy-out into buffers the new table owns: one device-to-device copy per array
   const unsigned long long mine = s.mine;
   Scratch cols(ctx);
   std::vector<LdbColumn> outCols;
   LdbBatch ob;
   ob.nRows = (int64_t) mine;
   ctx->launch("table_exchange_copy", [&] {
      for (int j = 0; j < s.nCols; j++) {
         const LdbColumn& sc = src->columns[s.ship[j]];
         outCols.push_back({sc.name, sc.type, sc.precision, sc.scale});
         const int sj = s.strOf[j];
         const size_t bytes = sj >= 0 ? ((size_t) mine + 1) * 4 : (size_t) mine * s.outBytes[j];
         uint8_t* data = cols.alloc<uint8_t>(std::max<size_t>(bytes, 16));
         uint8_t* valid = cols.alloc<uint8_t>(std::max<size_t>(mine, 16));
         uint8_t* chars = nullptr;
         if (sj >= 0) {
            const size_t nb = s.p.strBytes[c->rank][sj];
            chars = cols.alloc<uint8_t>(std::max<size_t>(nb, 16));
            LDB_CUDA(cudaMemcpyAsync(data, s.region + s.colOff[j], bytes, cudaMemcpyDeviceToDevice, ctx->compute));
            if (nb) LDB_CUDA(cudaMemcpyAsync(chars, s.region + s.bytesOff[sj], nb, cudaMemcpyDeviceToDevice, ctx->compute));
         }
         if (mine) {
            if (sj < 0) LDB_CUDA(cudaMemcpyAsync(data, s.region + s.colOff[j], bytes, cudaMemcpyDeviceToDevice, ctx->compute));
            LDB_CUDA(cudaMemcpyAsync(valid, s.region + s.validOff[j], (size_t) mine, cudaMemcpyDeviceToDevice, ctx->compute));
         }
         ob.data.push_back(data);
         ob.bytes.push_back(chars);
         ob.elemBytes.push_back(s.outBytes[j]);
         ob.validBytes.push_back(valid);
      }
   });
   s.finish();
   *out = addResultTable(ctx, name ? name : "received", std::move(outCols), std::move(ob), cols);
}
int ldb_gpu_table_exchange(LdbTable* src, int32_t n_keys, const char* const* key_columns, int32_t n_columns, const char* const* columns, LdbComm* c,
                           int64_t recv_offset, int64_t recv_bytes, const char* name, LdbTable** out, LdbError* err) {
   return guarded(err, [&] { tableExchange(false, src, n_keys, key_columns, n_columns, columns, c, recv_offset, recv_bytes, name, out); });
}
int ldb_gpu_table_exchange_varlen(LdbTable* src, int32_t n_keys, const char* const* key_columns, int32_t n_columns, const char* const* columns, LdbComm* c,
                                  int64_t recv_offset, int64_t recv_bytes, const char* name, LdbTable** out, LdbError* err) {
   return guarded(err, [&] { tableExchange(true, src, n_keys, key_columns, n_columns, columns, c, recv_offset, recv_bytes, name, out); });
}

} // extern "C"
// Rows ids[0..n) (null: 0..n-1) of columns `cols` of `t` (any number of batches) into new single-batch buffers of `bufs`, cells at
// outBytes: the permute kernels, with a host read of each utf8 column's byte total in between (it sizes the bytes array).  Returns the
// batch (nRows, data, bytes, elemBytes, validBytes); synchronises.  `what` names the caller's operation in the error for a utf8 column
// of more than 2^31 - 1 bytes.
LdbBatch ldb::permuteRows(LdbTable* t, const std::vector<int>& cols, const int32_t* outBytes, const uint32_t* ids, int64_t n, Scratch& bufs, const char* what) {
   LdbContext* ctx = t->ctx;
   Scratch tmp(ctx);
   PermuteParams q{};
   q.nCols = (int32_t) cols.size();
   q.ids = ids;
   q.n = n;
   q.nCtas = (n + kShipTile - 1) / kShipTile;
   std::vector<PermuteBatch> dir;
   int64_t first = 0;
   for (auto& b : t->batches) {
      if (b.nRows > 0) {
         PermuteBatch pb{};
         for (int j = 0; j < q.nCols; j++) {
            bindColumn(pb.cols[j], b, cols[j]);
            pb.cols[j].type = t->columns[cols[j]].type;
         }
         pb.firstRow = first;
         pb.nRows = b.nRows;
         dir.push_back(pb);
      }
      first += b.nRows;
   }
   q.nBatches = (int32_t) dir.size();
   LdbBatch ob;
   ob.nRows = n;
   for (int j = 0; j < q.nCols; j++) {
      const bool str = t->columns[cols[j]].type == LDB_UTF8;
      q.outBytes[j] = outBytes[j];
      q.strOf[j] = (int8_t) (str ? q.nStr : -1);
      if (str) q.strCol[q.nStr++] = (int8_t) j;
      q.data[j] = bufs.alloc<uint8_t>(std::max<size_t>(str ? ((size_t) n + 1) * 4 : (size_t) n * outBytes[j], 16));
      q.valid[j] = bufs.alloc<uint8_t>(std::max<size_t>((size_t) n, 16));
      if (str && n == 0) LDB_CUDA(cudaMemsetAsync(q.data[j], 0, 4, ctx->compute));
   }
   unsigned long long* totals = (unsigned long long*) ((uint8_t*) ctx->scratch() + LdbContext::kPinnedScratchBytes) - kShipMaxCols;
   if (n > 0) {
      if (dir.empty()) dir.push_back(PermuteBatch{}); // a table without rows: every id is kPermuteNone, the entry is never read for a row
      PermuteBatch* dd = tmp.alloc<PermuteBatch>(dir.size() * sizeof(PermuteBatch));
      LDB_CUDA(cudaMemcpyAsync(dd, dir.data(), dir.size() * sizeof(PermuteBatch), cudaMemcpyHostToDevice, ctx->compute));
      q.dir = dd;
      q.hist = tmp.alloc<unsigned long long>((size_t) std::max(q.nStr, 1) * (size_t) q.nCtas * 8);
      unsigned long long* devTotals = tmp.alloc<unsigned long long>(kShipMaxCols * 8);
      ctx->launch("sort_exchange_permute", [&] {
         permuteCellsKernel<<<(unsigned) q.nCtas, kShipThreads, 0, ctx->compute>>>(q);
         if (q.nStr) {
            rowScanKernel<<<q.nStr, 1024, 0, ctx->compute>>>(q.hist, q.nCtas, devTotals);
            LDB_CUDA(cudaMemcpyAsync(totals, devTotals, 8 * (size_t) q.nStr, cudaMemcpyDeviceToHost, ctx->compute));
         }
      });
      ctx->syncStream(ctx->compute);
   }
   for (int j = 0; j < q.nCols; j++) {
      const int sj = q.strOf[j];
      const uint64_t nb = sj >= 0 && n > 0 ? totals[sj] : 0;
      if (nb > (uint64_t) INT32_MAX)
         fail(LDB_ERR_UNSUPPORTED, std::string(what) + ": " + std::to_string(nb) + " bytes of utf8 column " + t->columns[cols[j]].name + " in one table, more than 2^31 - 1 (utf8 offsets are int32)");
      q.chars[j] = sj >= 0 ? bufs.alloc<uint8_t>(std::max<size_t>(nb, 16)) : nullptr;
      ob.data.push_back(q.data[j]);
      ob.bytes.push_back(q.chars[j]);
      ob.elemBytes.push_back(outBytes[j]);
      ob.validBytes.push_back(q.valid[j]);
   }
   if (n > 0 && q.nStr) ctx->launch("sort_exchange_permute", [&] { permuteStringsKernel<<<(unsigned) q.nCtas, kShipThreads, 0, ctx->compute>>>(q); });
   ctx->syncStream(ctx->compute); // the directory and the CTA sums go back to the pool
   return ob;
}
extern "C" {
// the stable sort of a table of any number of batches by its key columns (index, descending): row ids global to the table, in `scratch`.
// A single batch is sorted where it is; otherwise the keys are first permuted into one batch (16-byte decimal cells), whose order is the
// same: sortRows composes a key's words from its canonical value (sortCell).
static uint32_t* sortTableRows(Scratch& scratch, LdbTable* t, const std::vector<std::pair<int, int>>& keys) {
   if (t->batches.size() == 1) return sortRows(scratch, t, keys, t->numRows);
   std::vector<int> cols;
   std::vector<int32_t> widths;
   std::vector<std::pair<int, int>> at;
   LdbTable k{};
   k.ctx = t->ctx;
   k.numRows = t->numRows;
   for (auto& kc : keys) {
      at.push_back({(int) cols.size(), kc.second});
      cols.push_back(kc.first);
      widths.push_back(shipCellBytes(t->columns[kc.first].type));
      k.columns.push_back(t->columns[kc.first]);
   }
   k.batches.push_back(permuteRows(t, cols, widths.data(), nullptr, t->numRows, scratch, "sort exchange"));
   return sortRows(scratch, &k, at, t->numRows);
}

// Rows in global order (include/ldb_gpu.h).  Without LIMIT: samples of every rank's canonical tuples → all-gather → the same splitters
// on every rank (host) → the table shipment with the range owner rule → sort of the received rows by the keys (the received order,
// source rank then source row, breaks ties) → permute from the region into the new table.  With LIMIT: a local sort and permute of
// the rank's first `limit` rows → the shipment of those rows to rank 0 (every splitter above every tuple) → rank 0 sorts them and
// keeps the first `limit`.
static_assert((size_t) kMaxPeers * kSortBlockBytes + 8 * kShipMaxCols + 64 <= LdbContext::kPinnedScratchBytes, "every rank's samples fit the pinned scratch");
static_assert(sizeof(TableShipBatch) + sizeof(SortSplit) <= 4096, "the range count kernels' parameters");
static void sortExchange(LdbTable* src, int32_t n_keys, const char* const* key_columns, const int32_t* descending, int32_t n_columns, const char* const* columns,
                         int64_t limit, LdbComm* c, int64_t recv_offset, int64_t recv_bytes, const char* name, LdbTable** out, int64_t* first_row,
                         int64_t* total_rows) {
   int devices = 0;
   if (cudaGetDeviceCount(&devices) != cudaSuccess || devices == 0) {
      cudaGetLastError();
      fail(LDB_ERR_NO_DEVICE, "no CUDA device available: the GPU operator runtime has no CPU fallback");
   }
   if (!src || !c || !out || !key_columns || !descending || !first_row || !total_rows) fail(LDB_ERR_INVALID, "null argument");
   if (n_keys < 1 || n_keys > kProgMaxKeys) fail(LDB_ERR_INVALID, "the sort exchange takes 1..4 key columns");
   if (src->ctx != c->ctx) fail(LDB_ERR_INVALID, "table and comm belong to different contexts");
   std::vector<int> ship = shipColumns(true, src, n_columns, columns), key, keyAt;
   const int nUser = (int) ship.size();
   for (int k = 0; k < n_keys; k++) {
      const int ci = src->colIndex(key_columns[k]);
      if (ci < 0) fail(LDB_ERR_INVALID, std::string("unknown key column ") + (key_columns[k] ? key_columns[k] : "(null)"));
      const int type = src->columns[ci].type;
      if (type != LDB_INT32 && type != LDB_DATE32 && type != LDB_FSB4 && type != LDB_INT64 && type != LDB_DECIMAL128)
         fail(LDB_ERR_UNSUPPORTED, "sort exchange keys are int32, date32, char(1), int64 or decimal columns (column " + src->columns[ci].name + ")");
      key.push_back(ci);
      const int at = (int) (std::find(ship.begin(), ship.end(), ci) - ship.begin());
      if (at == (int) ship.size()) ship.push_back(ci); // a key that is not shipped travels as a hidden column
      keyAt.push_back(at);
   }
   if (ship.size() > (size_t) kShipMaxCols) fail(LDB_ERR_INVALID, "the sort exchange ships up to 16 columns, key columns not among them included");
   wantConnected(c);
   wantRegion(c, recv_offset, recv_bytes);
   LdbContext* ctx = c->ctx;
   if (ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "the sort exchange reads row counts and samples on the host and cannot be captured");
   LDB_CUDA(cudaSetDevice(ctx->device));
   if (src->numRows >= (int64_t) 1 << 32) fail(LDB_ERR_UNSUPPORTED, "the sort exchange sorts up to 2^32 - 1 rows per rank");
   for (auto& b : src->batches) ldb_gpu_wait_batch_internal(ctx, &b);
   const int world = c->world;
   std::vector<std::pair<int, int>> order; // (column of the received rows, descending)
   for (int k = 0; k < n_keys; k++) order.push_back({keyAt[k], descending[k] ? 1 : 0});
   SortSplit split{};
   split.nKeys = n_keys;
   split.nSplit = world - 1;
   split.rank = c->rank;
   for (int k = 0; k < n_keys; k++) split.desc[k] = descending[k] ? 1 : 0;
   Scratch local(ctx);
   LdbTable top{}; // LIMIT: this rank's first `limit` rows in order, the shipped columns
   LdbTable* from = src;
   std::vector<int> fromCols = ship, fromKeys = key;
   if (limit >= 0) {
      const int64_t m = std::min<int64_t>(limit, src->numRows);
      std::vector<std::pair<int, int>> keys;
      for (int k = 0; k < n_keys; k++) keys.push_back({key[k], split.desc[k]});
      const uint32_t* ids = m ? sortTableRows(local, src, keys) : nullptr;
      int32_t widths[kShipMaxCols];
      for (size_t j = 0; j < ship.size(); j++) widths[j] = shipCellBytes(src->columns[ship[j]].type);
      top.ctx = ctx;
      top.numRows = m;
      for (int ci : ship) top.columns.push_back(src->columns[ci]);
      top.batches.push_back(permuteRows(src, ship, widths, ids, m, local, "sort exchange"));
      from = &top;
      for (size_t j = 0; j < ship.size(); j++) fromCols[j] = (int) j;
      for (int k = 0; k < n_keys; k++) fromKeys[k] = keyAt[k];
      for (auto& w : split.split) // every tuple goes below every splitter: to rank 0
         for (auto& x : w) x = ~0ull;
   }
   TableShipment s(from, fromCols, fromKeys, c, recv_offset, recv_bytes);
   if (limit < 0) {
      unsigned long long* block = s.tmp.alloc<unsigned long long>(kSortBlockBytes);
      unsigned long long* pin = (unsigned long long*) ctx->scratch();
      unsigned long long* hdr = (unsigned long long*) ((uint8_t*) pin + LdbContext::kPinnedScratchBytes) - kShipMaxCols - 8;
      const int64_t n = src->numRows;
      hdr[0] = (unsigned long long) n;
      hdr[1] = n > 0 ? kSortSamples : 0;
      ctx->launch("sort_exchange_sample", [&] {
         LDB_CUDA(cudaMemcpyAsync(block, hdr, 16, cudaMemcpyHostToDevice, ctx->compute));
         s.eachBatch([&](const TableShipBatch& q, int) { sortSampleKernel<<<kSortSamples / 256, 256, 0, ctx->compute>>>(q, split, n, block + 2); });
      });
      if (world == 1) {
         LDB_CUDA(cudaMemcpyAsync(pin, block, kSortBlockBytes, cudaMemcpyDeviceToHost, ctx->compute));
      } else {
         const uint8_t* gathered = allGatherSmall(c, block, kSortBlockBytes);
         LDB_CUDA(cudaMemcpy2DAsync(pin, kSortBlockBytes, gathered, kSlotBytes, kSortBlockBytes, world, cudaMemcpyDeviceToHost, ctx->compute));
      }
      checkPeers(c, s.timedOut);
      // the splitters, the same on every rank: sample j of rank r stands for n_r / S_r rows; splitter d - 1 is the sample at which the
      // rows it and the smaller samples stand for first reach d N / world
      struct Sample {
         const unsigned long long* w;
         double rows;
      };
      std::vector<Sample> all;
      double total = 0;
      for (int r = 0; r < world; r++) {
         const unsigned long long* b = pin + r * (kSortBlockBytes / 8);
         total += (double) b[0];
         for (unsigned long long j = 0; j < b[1]; j++) all.push_back({b + 2 + j * kSortTupleWords, (double) b[0] / (double) b[1]});
      }
      std::sort(all.begin(), all.end(), [&](const Sample& a, const Sample& b) { return sortTupleLess(a.w, b.w, n_keys); });
      size_t i = 0;
      double below = 0;
      for (int d = 1; d < world; d++) {
         while (i < all.size() && below + all[i].rows < total * d / world) below += all[i++].rows;
         for (int x = 0; x < kSortTupleWords; x++) split.split[d - 1][x] = i < all.size() ? all[i].w[x] : ~0ull;
      }
   }
   s.run(&split);
   // the received rows (source rank, then source row: the tie order) sorted by the keys, permuted from the region into the new table
   LdbTable view{};
   s.receivedView(view);
   const int64_t got = (int64_t) s.mine;
   if (got >= (int64_t) 1 << 32) fail(LDB_ERR_UNSUPPORTED, "the sort exchange sorts up to 2^32 - 1 received rows per rank");
   const int64_t keep = limit >= 0 ? std::min<int64_t>(got, limit) : got;
   Scratch sorted(ctx), cols(ctx);
   const uint32_t* ids = keep ? sortRows(sorted, &view, order, got) : nullptr;
   std::vector<int> outCols;
   for (int j = 0; j < nUser; j++) outCols.push_back(j);
   LdbBatch ob = permuteRows(&view, outCols, s.outBytes, ids, keep, cols, "sort exchange");
   s.finish();
   int64_t before = 0, all = 0;
   for (int d = 0; d < world; d++) {
      const int64_t rows = limit >= 0 ? (d == 0 ? std::min<int64_t>((int64_t) s.p.rows[0], limit) : 0) : (int64_t) s.p.rows[d];
      if (d < c->rank) before += rows;
      all += rows;
   }
   std::vector<LdbColumn> outDesc;
   for (int j = 0; j < nUser; j++) outDesc.push_back(src->columns[ship[j]]);
   *out = addResultTable(ctx, name ? name : "sorted", std::move(outDesc), std::move(ob), cols);
   *first_row = before;
   *total_rows = all;
}
int ldb_gpu_table_sort_exchange(LdbTable* src, int32_t n_keys, const char* const* key_columns, const int32_t* descending, int32_t n_columns, const char* const* columns,
                                int64_t limit, LdbComm* c, int64_t recv_offset, int64_t recv_bytes, const char* name, LdbTable** out, int64_t* first_row,
                                int64_t* total_rows, LdbError* err) {
   return guarded(err, [&] { sortExchange(src, n_keys, key_columns, descending, n_columns, columns, limit, c, recv_offset, recv_bytes, name, out, first_row, total_rows); });
}

// Union of every rank's string dictionary (include/ldb_gpu.h).  Local counters → export → all-gather of {status, n, bytes} → host
// decision from the gathered counts (identical on every rank) → barrier → send → barrier → concatenation of the received blocks → sort →
// codes → ranked build.  As in the table exchange, the temporaries are taken before the first collective and the rest after the last.
static uint64_t align16(uint64_t x) { return (x + 15) & ~uint64_t(15); }
int ldb_gpu_dict_unify(LdbState* local, LdbComm* c, int64_t recv_offset, int64_t recv_bytes, LdbState** out, LdbError* err) {
   return guarded(err, [&] {
      if (!local || !c || !out) fail(LDB_ERR_INVALID, "null argument");
      if (local->kind != LDB_STATE_DICT) fail(LDB_ERR_INVALID, "not a string dictionary");
      if (local->ctx != c->ctx) fail(LDB_ERR_INVALID, "dictionary and comm belong to different contexts");
      wantConnected(c);
      wantRegion(c, recv_offset, recv_bytes);
      LdbContext* ctx = c->ctx;
      if (ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "dictionary unification reads the string counts on the host and cannot be captured");
      LDB_CUDA(cudaSetDevice(ctx->device));
      const int world = c->world;
      // pinned scratch: [0, 4) local counters, [8, 12) this rank's gathered block, [16, 16 + 4 world) every rank's, then the error word
      unsigned long long* pin = (unsigned long long*) ctx->scratch();
      unsigned long long* block = pin + 8;
      unsigned long long* blocks = pin + 16;
      int32_t* timedOut = (int32_t*) (blocks + 4 * kMaxPeers);
      LDB_CUDA(cudaMemcpyAsync(pin, local->dict.ctr, 24, cudaMemcpyDeviceToHost, ctx->compute));
      ctx->syncStream(ctx->compute);
      // a dictionary that overflowed (its contents are unspecified) or that no block could carry sends no strings, only its status
      const uint32_t status = (uint32_t) pin[2];
      const bool sends = status == 0 && pin[0] <= (unsigned long long) INT32_MAX;
      const int64_t n = sends ? (int64_t) pin[1] : 0, bytes = sends ? (int64_t) pin[0] : 0;
      block[0] = status;
      block[1] = (unsigned long long) n;
      block[2] = status == 0 ? pin[0] : 0;
      block[3] = 0;
      Scratch tmp(ctx);
      uint32_t* offs = tmp.alloc<uint32_t>(align16((uint64_t) (n + 1) * 4));
      uint8_t* data = tmp.alloc<uint8_t>(std::max<uint64_t>(align16((uint64_t) bytes), 16));
      ctx->launch("dict_export", [&] { launchDictExport(local->dict, n, offs, data, ctx->smCount, ctx->compute); });
      const uint8_t* gathered = allGatherSmall(c, block, 32);
      LDB_CUDA(cudaMemcpy2DAsync(blocks, 32, gathered, kSlotBytes, 32, world, cudaMemcpyDeviceToHost, ctx->compute));
      checkPeers(c, timedOut);
      // every rank decides from the same gathered counts
      uint64_t blockOff[kMaxPeers + 1] = {}, byteBase[kMaxPeers + 1] = {}, rowBase[kMaxPeers + 1] = {};
      for (int s = 0; s < world; s++) {
         const unsigned long long* b = blocks + 4 * s;
         if (b[0]) fail(LDB_ERR_CAPACITY, "dictionary unification: the string dictionary of rank " + std::to_string(s) + " overflowed earlier (error word " + std::to_string(b[0]) +
                                             "; recreate it larger)");
         blockOff[s + 1] = blockOff[s] + align16((b[1] + 1) * 4) + align16(b[2]);
         byteBase[s + 1] = byteBase[s] + b[2];
         rowBase[s + 1] = rowBase[s] + b[1];
      }
      if (byteBase[world] > (uint64_t) INT32_MAX) fail(LDB_ERR_UNSUPPORTED, "dictionary unification: the ranks' strings exceed 2^31 - 1 bytes (utf8 offsets are int32)");
      if (blockOff[world] > (uint64_t) recv_bytes)
         fail(LDB_ERR_CAPACITY, "dictionary unification: the ranks' strings need " + std::to_string(blockOff[world]) + " bytes of receive region, more than recv_bytes " +
                                   std::to_string(recv_bytes) + "; retry with recv_bytes " + std::to_string(blockOff[world]));
      commBarrier(c); // no peer still reads the region it is about to receive into
      const size_t offVecs = align16((uint64_t) (n + 1) * 4) / 16, byteVecs = align16((uint64_t) bytes) / 16;
      ctx->launch("dict_unify_send", [&] {
         const dim3 grid((unsigned) std::min<size_t>(std::max<size_t>((offVecs + byteVecs + 255) / 256, 1), (size_t) ctx->smCount * 2), (unsigned) world);
         dictSendKernel<<<grid, 256, 0, ctx->compute>>>(c->view(), kUserOff + (size_t) recv_offset + blockOff[c->rank], (const int4*) offs, offVecs, (const int4*) data, byteVecs);
      });
      commBarrier(c); // every peer's block is in this rank's region
      checkPeers(c, timedOut);
      // the received blocks as one utf8 column of N strings, in rank order
      const int64_t N = (int64_t) rowBase[world];
      Scratch col(ctx);
      uint32_t* allOffs = col.alloc<uint32_t>((size_t) (N + 1) * 4);
      uint8_t* allBytes = col.alloc<uint8_t>(std::max<uint64_t>(byteBase[world], 16));
      const uint8_t* region = c->heap + kUserOff + recv_offset;
      ctx->launch("dict_unify_concat", [&] {
         for (int s = 0; s < world; s++) {
            const uint64_t ns = rowBase[s + 1] - rowBase[s], bs = byteBase[s + 1] - byteBase[s];
            // n_s + 1 offsets each: the last one of source s equals the first of source s + 1
            launchDictRebase((const uint32_t*) (region + blockOff[s]), (int64_t) ns + 1, (uint32_t) byteBase[s], allOffs + rowBase[s], ctx->smCount, ctx->compute);
            if (bs) LDB_CUDA(cudaMemcpyAsync(allBytes + byteBase[s], region + blockOff[s] + align16((ns + 1) * 4), bs, cudaMemcpyDeviceToDevice, ctx->compute));
         }
      });
      LdbTable all{};
      all.ctx = ctx;
      all.columns = {{"str", LDB_UTF8, 0, 0}};
      all.numRows = N;
      all.batches.resize(1);
      all.batches[0].nRows = N;
      all.batches[0].data = {allOffs};
      all.batches[0].bytes = {allBytes};
      all.batches[0].elemBytes = {4};
      uint32_t* ids = sortRows(col, &all, {{0, 0}}, N);
      uint32_t* codes = col.alloc<uint32_t>((size_t) (N + 1) * 4);
      uint32_t* arenaOff = col.alloc<uint32_t>((size_t) (N + 1) * 4);
      ctx->launch("dict_unify_ranks", [&] { launchDictUnionRanks(allOffs, allBytes, ids, N, codes, arenaOff, ctx->smCount, ctx->compute); });
      uint32_t* totals = (uint32_t*) pin;
      LDB_CUDA(cudaMemcpyAsync(totals, codes + N, 4, cudaMemcpyDeviceToHost, ctx->compute));
      LDB_CUDA(cudaMemcpyAsync(totals + 1, arenaOff + N, 4, cudaMemcpyDeviceToHost, ctx->compute));
      ctx->syncStream(ctx->compute);
      const int64_t nu = totals[0], bu = totals[1];
      if (nu > kDictMaxStrings) fail(LDB_ERR_UNSUPPORTED, "dictionary unification: the union holds " + std::to_string(nu) + " strings, more than a dictionary's 2^30");
      LdbState* u = ldb_gpu_dict_new_internal(ctx, nu, bu);
      u->unified = true;
      try {
         ctx->launch("dict_unify_build", [&] { launchDictRankedBuild(u->dict, allOffs, allBytes, ids, N, codes, arenaOff, ctx->smCount, ctx->compute); });
         ldb_gpu_dict_counters_internal(u); // synchronises: the region is free again, the temporaries go back to the pool
      } catch (...) {
         ldb_gpu_state_destroy(u);
         throw;
      }
      *out = u;
   });
}

// surfaces a timed-out wait (dead or stuck peer); synchronises the compute stream
int ldb_gpu_comm_check(LdbComm* c, LdbError* err) {
   return guarded(err, [&] {
      if (!c) fail(LDB_ERR_INVALID, "null comm");
      LDB_CUDA(cudaSetDevice(c->ctx->device));
      int32_t e = 0;
      LDB_CUDA(cudaMemcpyAsync(&e, c->error, 4, cudaMemcpyDeviceToHost, c->ctx->compute));
      c->ctx->syncStream(c->ctx->compute);
      if (e) fail(LDB_ERR_CUDA, "a peer did not arrive at a collective within the timeout (LDB_PEER_TIMEOUT_MS)");
   });
}

} // extern "C"
