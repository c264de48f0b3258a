// program.cu — the GENERIC pipeline kernel: scan → register program → {hash aggregation | join-table build | materialize},
// the large-domain hash aggregation table, its export, and a radix sort for ORDER BY.  See program.h.
#include "device_utils.cuh"
#include "keyhash.cuh"
#include "progcol.cuh"
#include "program.h"
#include "sortkey.cuh"
#include "tilescan.cuh"
#include "../../include/ldb_gpu.h"

#include <algorithm>

namespace ldb {

// twins of the join-table primitives of kernels.cu (plain single-key tables and direct-address tables)
__device__ __forceinline__ int32_t directLoadProg(const JoinTableDev& t, int32_t key) {
   const uint32_t idx = (uint32_t) key - (uint32_t) t.keyMin;
   return idx < t.range ? __ldg((const int32_t*) t.base + idx) : kDirectEmpty;
}
__device__ bool joinInsertProg(const JoinTableDev& t, int32_t key, int32_t payload) {
   const unsigned long long packed = ((unsigned long long) (uint32_t) payload << 32) | (uint32_t) key;
   if (packed == ~0ull) {
      atomicExch(t.error, 3);
      return false;
   }
   const uint64_t h = hashI32(key);
   uint64_t s = h & t.mask;
   const uint64_t limit = t.mask < 16384 ? t.mask + 1 : 16384;
   for (uint64_t probes = 0; probes < limit; probes++) {
      const unsigned long long old = atomicCAS((unsigned long long*) (t.base + s * t.stride), ~0ull, packed);
      if (old == ~0ull) {
         if (t.bloom) atomicOr(&t.bloom[(uint32_t) (h >> 32) & t.bloomMask], bloomBits(h));
         return true;
      }
      if ((int32_t) (uint32_t) old == key && t.unique) { // a set of keys (semi-join build side): duplicates are dropped, not an error
         return false;
      }
      s = (s + 1) & t.mask;
   }
   atomicExch(t.error, 1);
   return false;
}
// the cell a program column reads: the scanned row for a column of the source table; for a side column the row its row register
// holds, located in the side table's batch directory.  nullptr: that register is NULL or outside the side table, so the value is
// NULL (outer-join semantics).
__device__ __forceinline__ const ProgCol* cellOf(const ProgCol& c, const Val* regs, int64_t row, ProgCol& tmp, int64_t& at) {
   if (c.rowReg < 0) {
      at = row;
      return &c;
   }
   const Val rv = regs[c.rowReg];
   if (rv.null || rv.v < 0 || rv.v >= (s128) c.sideRows) return nullptr;
   at = (int64_t) rv.v;
   if (!c.dir) return &c; // single-batch side table: the column's own pointers
   int lo = 0, hi = c.nBatches - 1;
   while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (c.dir[mid].firstRow <= at) lo = mid;
      else hi = mid - 1;
   }
   const ProgSideBatch& b = c.dir[lo];
   tmp = c;
   tmp.data = b.data;
   tmp.bytes = b.bytes;
   tmp.validity = b.validity;
   tmp.validBytes = b.validBytes;
   tmp.bitOffset = b.bitOffset;
   tmp.elemBytes = b.elemBytes;
   at -= b.firstRow;
   return &tmp;
}
// LDB_OP_PROBE_EACH / LDB_OP_EXISTS: the next match of `key` along its linear-probe run, resuming at slot `s` after `probes` probes.
// false: the run ended.  A run that reaches the probe bound of a table larger than the bound sets the table's error word (6 for
// PROBE_EACH, 8 for EXISTS) instead of ending early with a truncated match list.
__device__ bool probeEachNext(const JoinTableDev& t, int32_t key, uint64_t& s, uint32_t& probes, int32_t& payload, int boundError = 6) {
   if (t.direct) {
      if (probes++) return false; // one slot per key
      payload = directLoadProg(t, key);
      return payload != kDirectEmpty;
   }
   while (probes <= t.mask && probes < 16384) {
      const unsigned long long e = __ldg((const unsigned long long*) (t.base + s * t.stride));
      if (e == ~0ull) return false;
      s = (s + 1) & t.mask;
      probes++;
      if ((int32_t) (uint32_t) e == key) {
         payload = (int32_t) (uint32_t) (e >> 32);
         return true;
      }
   }
   if (probes >= 16384 && t.mask >= 16384) atomicExch(t.error, boundError);
   return false;
}
__device__ __forceinline__ bool cmpI(s128 a, s128 b, int op) {
   switch (op) {
      case LDB_EQ: return a == b;
      case LDB_NEQ: return a != b;
      case LDB_LT: return a < b;
      case LDB_LTE: return a <= b;
      case LDB_GT: return a > b;
      default: return a >= b;
   }
}
__device__ __forceinline__ bool cmpF(double a, double b, int op) {
   switch (op) {
      case LDB_EQ: return a == b;
      case LDB_NEQ: return a != b;
      case LDB_LT: return a < b;
      case LDB_LTE: return a <= b;
      case LDB_GT: return a > b;
      default: return a >= b;
   }
}
// VarLen32 ordering (VarLen32Filter<CMP>, Restrictions.cpp:234-325): bytewise, shorter string first on a common prefix
__device__ int strCompare(const ProgCol& c, int64_t row, const uint8_t* k, int klen) {
   const int32_t* off = (const int32_t*) c.data + row;
   const int32_t b = off[0], n = off[1] - off[0];
   const uint8_t* s = c.bytes + b;
   const int m = n < klen ? n : klen;
   for (int i = 0; i < m; i++)
      if (s[i] != k[i]) return s[i] < k[i] ? -1 : 1;
   return n == klen ? 0 : (n < klen ? -1 : 1);
}
__device__ bool strLike(const ProgCol& c, int64_t row, const uint8_t* k, int klen, int kind) {
   const int32_t* off = (const int32_t*) c.data + row;
   const int32_t b = off[0], n = off[1] - off[0];
   const uint8_t* s = c.bytes + b;
   if (n < klen) return false;
   if (kind == 0 || kind == 1) { // prefix% / %suffix
      const uint8_t* p = kind == 0 ? s : s + (n - klen);
      for (int i = 0; i < klen; i++)
         if (p[i] != k[i]) return false;
      return true;
   }
   for (int i = 0; i + klen <= n; i++) { // %contains%
      int j = 0;
      while (j < klen && s[i + j] == k[j]) j++;
      if (j == klen) return true;
   }
   return false;
}
// ---------------------------------------------------------------- string dictionary (DictDev, program.h)
// where a string with hash h lives in the directory: its tag (the high 32 bits of h, the upper half of its slot word), its first slot
// and the linear probe sequence from there, at most dictProbeLimit slots long.  One definition for dictCode and the ranked build of a
// unified dictionary, so that a lookup finds every string the build placed.
__device__ __forceinline__ unsigned long long dictTag(uint64_t h) { return (h >> 32) << 32; }
__device__ __forceinline__ uint64_t dictFirstSlot(uint64_t h, uint64_t mask) { return h & mask; }
__device__ __forceinline__ uint64_t dictNextSlot(uint64_t slot, uint64_t mask) { return (slot + 1) & mask; }
__device__ __forceinline__ uint64_t dictProbeLimit(uint64_t mask) { return mask + 1 < 65536 ? mask + 1 : 65536; }
__device__ __forceinline__ void dictFail(const DictDev& d, int code) { atomicCAS((unsigned int*) (d.ctr + 2), 0u, (unsigned int) code); }
// the code of string s[0..n) in dictionary d; absent: inserted when `insert`, else -1.  -2: the dictionary failed (its error word
// is set, the call reports LDB_ERR_CAPACITY).  A slot is claimed by CAS (empty → tag | kDictWriting); its claimer reserves arena
// bytes, copies the string, takes a code, writes the entry and publishes tag | code + 1 with one atomic store — or tag | kDictFailed
// when it cannot, so that no reader waits forever.  A reader that meets its tag waits for the publication, then compares the whole
// string bytewise (loads through L2: the arena is written by other SMs during the same launch).  A hit takes no atomic.
__device__ __noinline__ int32_t dictCode(const DictDev& d, const uint8_t* s, int32_t n, int insert) {
   const uint64_t h = strHash(s, n);
   const unsigned long long tag = dictTag(h);
   uint64_t slot = dictFirstSlot(h, d.mask);
   const uint64_t limit = dictProbeLimit(d.mask);
   for (uint64_t probes = 0; probes < limit; probes++) {
      unsigned long long* sp = d.slots + slot;
      unsigned long long w = *((volatile unsigned long long*) sp);
      if ((uint32_t) w == 0) {
         if (!insert) return -1;
         w = atomicCAS(sp, 0ull, tag | kDictWriting);
         if (w == 0) {
            int fail = 0;
            const unsigned long long off = atomicAdd(d.ctr, (unsigned long long) n);
            unsigned long long code = 0;
            if (off + (unsigned long long) n > (unsigned long long) d.arenaCap) {
               fail = 2;
            } else {
               for (int32_t i = 0; i < n; i++) d.arena[off + i] = s[i];
               code = atomicAdd(d.ctr + 1, 1ull);
               if (code >= (unsigned long long) d.codeCap) fail = 3;
            }
            if (fail) {
               dictFail(d, fail);
               atomicExch(sp, tag | kDictFailed);
               return -2;
            }
            d.entryOff[code] = (int64_t) off;
            d.entryLen[code] = n;
            __threadfence();
            atomicExch(sp, tag | (unsigned long long) (code + 1));
            return (int32_t) code;
         }
      }
      if ((w & 0xffffffff00000000ull) == tag) {
         while ((uint32_t) w == kDictWriting) {
            __nanosleep(64);
            w = *((volatile unsigned long long*) sp);
         }
         if ((uint32_t) w == kDictFailed) return -2;
         __threadfence();
         const int32_t code = (int32_t) ((uint32_t) w - 1);
         if (__ldcg(d.entryLen + code) == n) {
            const uint8_t* a = d.arena + __ldcg(d.entryOff + code);
            int32_t i = 0;
            while (i < n && __ldcg(a + i) == s[i]) i++;
            if (i == n) return code;
         }
      }
      slot = dictNextSlot(slot, d.mask);
   }
   dictFail(d, 1);
   return -2;
}

// ---------------------------------------------------------------- key-tuple join table (KeyJoinDev, program.h)
// Kept out of line (__noinline__), like dictCode, and called only from programKernel<true>: programs without a key-tuple table run
// programKernel<false>, which has none of this code.  The calls take the table descriptor and the key tuple by value and return their
// results by value: no pointer into the register file or into the kernel parameters escapes into them.
struct KeyTuple {
   int64_t k[kProgMaxKeys];
};
struct KeyCursor { // a probe run: the next slot, the probes taken, the tuple's tag; `live` false: the run ended (or never started)
   uint64_t slot;
   uint32_t probes, tag;
   bool live;
};
struct KeyHit {
   KeyCursor next;
   int64_t payload;
   bool hit;
};
__device__ __forceinline__ uint8_t* keyEntry(const KeyJoinDev& t, uint64_t s) { return t.base + s * t.entryBytes; }
// the entry at e holds exactly the tuple `keys`: 16-byte loads (keys start 16 bytes into an entry; an odd last key reads the entry's
// padding), through L2 (`coherent`: a build reads entries other SMs publish during the same launch) or the read-only path
__device__ __forceinline__ bool keysEqual(const KeyJoinDev& t, const uint8_t* e, const KeyTuple& keys, bool coherent) {
   const longlong2* kp = (const longlong2*) (e + 16);
   for (int k = 0; k < t.nKeys; k += 2) {
      const longlong2 w = coherent ? __ldcg(kp + k / 2) : __ldg(kp + k / 2);
      if (w.x != keys.k[k] || (k + 1 < t.nKeys && w.y != keys.k[k + 1])) return false;
   }
   return true;
}
// the tuple of registers regs[reg(0)], …, regs[reg(n - 1)]: 0, or bit 0 = a NULL component, bit 1 = a component outside int64
template <class Reg>
__device__ __forceinline__ int gatherTuple(const Val* regs, int n, Reg reg, KeyTuple& keys) {
   int bad = 0;
   for (int k = 0; k < n; k++) {
      const Val v = regs[reg(k)];
      bad |= v.null ? 1 : (v.v != (s128) (int64_t) v.v ? 2 : 0);
      keys.k[k] = (int64_t) v.v;
   }
   return bad;
}
// insert: claims an empty slot by CAS (0 → tag | kKeyJoinWriting), writes the payload and the keys, fences and publishes
// tag | kKeyJoinReady with one atomic store.  A multimap insert skips occupied slots without reading their keys.  A unique insert that
// meets its own tag waits (__nanosleep) for the publication, then compares the keys and drops a duplicate.  false: not inserted (a
// duplicate, or error word 1: no empty slot within kKeyJoinInsertBound probes — a full directory, or that many entries sharing one run,
// e.g. duplicates of one tuple in a multimap).  The bound keeps a build that overflows the table from walking the whole directory for
// every row; every 1024 probes the insert also gives up once another row has set the error word.
constexpr uint64_t kKeyJoinInsertBound = 65536;
__device__ __noinline__ bool keyJoinInsert(const KeyJoinDev t, const KeyTuple keys, int64_t payload) {
   const uint64_t h = keyTupleHash(keys.k, t.nKeys, 0);
   const unsigned long long tag = (h >> 32) << 32;
   uint64_t s = h & t.mask;
   const uint64_t limit = t.mask + 1 < kKeyJoinInsertBound ? t.mask + 1 : kKeyJoinInsertBound;
   for (uint64_t probes = 0; probes < limit; probes++) {
      if ((probes & 1023) == 1023 && *((volatile int32_t*) t.error)) return false; // the call fails already
      uint8_t* e = keyEntry(t, s);
      unsigned long long* wp = (unsigned long long*) e;
      unsigned long long w = *((volatile unsigned long long*) wp);
      if (w == 0) {
         w = atomicCAS(wp, 0ull, tag | kKeyJoinWriting);
         if (w == 0) {
            int64_t* ep = (int64_t*) e;
            ep[1] = payload;
            for (int k = 0; k < t.nKeys; k++) ep[2 + k] = keys.k[k];
            __threadfence();
            atomicExch(wp, tag | kKeyJoinReady);
            if (t.bloom) atomicOr(&t.bloom[(uint32_t) (h >> 32) & t.bloomMask], bloomBits(h));
            return true;
         }
      }
      if (t.unique && (w & 0xffffffff00000000ull) == tag) {
         while ((uint32_t) w == kKeyJoinWriting) {
            __nanosleep(64);
            w = *((volatile unsigned long long*) wp);
         }
         __threadfence();
         if (keysEqual(t, e, keys, true)) return false;
      }
      s = (s + 1) & t.mask;
   }
   atomicExch(t.error, 1);
   return false;
}
// the start of a probe run for `keys` (a tuple without NULL or out-of-range components): not live when the Bloom filter rules it out
__device__ __noinline__ KeyCursor keyJoinStart(const KeyJoinDev t, const KeyTuple keys) {
   const uint64_t h = keyTupleHash(keys.k, t.nKeys, 0);
   KeyCursor c{h & t.mask, 0, (uint32_t) (h >> 32), true};
   if (t.bloom) {
      const uint32_t bits = bloomBits(h);
      c.live = (__ldg(&t.bloom[(uint32_t) (h >> 32) & t.bloomMask]) & bits) == bits;
   }
   return c;
}
// the next entry of `keys` along its probe run from cursor c (PROBE takes the first, PROBE_EACH every one).  The state word (with the tag)
// and the payload come in one 16-byte load; the keys are loaded only on a tag match.  A program never builds and probes one table, so no
// probe shares a launch with a build: the loads take the read-only path.  A run that reaches the interpreter's bound in a directory larger
// than the bound sets the error word (6): the call fails rather than miss a match.
__device__ __noinline__ KeyHit keyJoinNext(const KeyJoinDev t, const KeyTuple keys, KeyCursor c) {
   KeyHit r{c, 0, false};
   while (r.next.probes <= t.mask && r.next.probes < 16384) {
      const uint8_t* e = keyEntry(t, r.next.slot);
      const ulonglong2 head = __ldg((const ulonglong2*) e);
      if (head.x == 0) {
         r.next.live = false;
         return r;
      }
      r.next.slot = (r.next.slot + 1) & t.mask;
      r.next.probes++;
      if ((uint32_t) (head.x >> 32) == r.next.tag && keysEqual(t, e, keys, false)) {
         r.payload = (int64_t) head.y;
         r.hit = true;
         return r;
      }
   }
   if (r.next.probes >= 16384 && t.mask >= 16384) atomicExch(t.error, 6);
   r.next.live = false;
   return r;
}

// ---------------------------------------------------------------- hash aggregation table
constexpr uint32_t kSeenBit = 1u, kClaimBit = 1u << 8, kKeyNullBit = 1u << 16;
__device__ __forceinline__ uint8_t* entryAt(const HashAggDev& t, uint64_t s) { return t.base + s * t.entryBytes; }
// lookup-or-insert by key tuple (subop.lookup_or_insert, SubOpToControlFlow.cpp:3065-3157; NULL keys form a group of their own).
// kindOf(a) is aggregate a's LdbAggKind, which gives a new group's identity values.  Shared by the interpreter's sink (hashAggFind) and
// the exchange's merge (hashAggMergeKernel); forced inline, so that each caller compiles exactly the code it had on its own.
template <class KindOf>
__device__ __forceinline__ uint8_t* hashAggFindIn(const HashAggDev& t, const KindOf& kindOf, const int64_t* keys, uint32_t keyNulls) {
   if (t.nKeys == 0) return t.base; // keyless: the table is one pre-initialised entry
   const uint64_t h = keyTupleHash(keys, t.nKeys, keyNulls);
   uint64_t s = h & t.mask;
   const uint64_t limit = t.mask + 1 < 65536 ? t.mask + 1 : 65536;
   for (uint64_t probes = 0; probes < limit; probes++) {
      uint8_t* e = entryAt(t, s);
      uint32_t* state = (uint32_t*) e;
      uint32_t st = *((volatile uint32_t*) state);
      if (st == 0) {
         st = atomicCAS(state, 0u, 1u);
         if (st == 0) { // this thread creates the group: keys, key-null bits, aggregate identities, then publish
            uint32_t* flags = state + 1;
            *flags = keyNulls * kKeyNullBit;
            int64_t* ek = (int64_t*) (e + 16);
            for (int k = 0; k < t.nKeys; k++) ek[k] = keys[k];
            unsigned long long* ea = (unsigned long long*) (e + 16 + 8 * kProgMaxKeys);
            for (int a = 0; a < t.nAggs; a++) {
               unsigned long long lo = 0, hi = 0;
               switch (kindOf(a)) {
                  case LDB_AGG_MIN: // INT128_MAX
                     lo = ~0ull;
                     hi = ~0ull >> 1;
                     break;
                  case LDB_AGG_MAX: hi = 1ull << 63; break; // INT128_MIN
                  case LDB_AGG_MIN_F64:
                  case LDB_AGG_MAX_F64: lo = kF64MinMaxIdentity; break;
                  default: break;
               }
               ea[2 * a] = lo;
               ea[2 * a + 1] = hi;
            }
            __threadfence();
            atomicExch(state, 2u);
            atomicAdd(t.count, 1ull);
            return e;
         }
      }
      while (st == 1) st = *((volatile uint32_t*) state);
      __threadfence();
      const uint32_t fl = *((volatile uint32_t*) (state + 1));
      bool eq = ((fl >> 16) & 0xfu) == keyNulls;
      const volatile int64_t* ek = (const volatile int64_t*) (e + 16);
      for (int k = 0; k < t.nKeys && eq; k++) eq = ((keyNulls >> k) & 1u) || ek[k] == keys[k];
      if (eq) return e;
      s = (s + 1) & t.mask;
   }
   atomicExch(t.error, 1);
   return nullptr;
}
__device__ uint8_t* hashAggFind(const ProgramParams& p, const int64_t* keys, uint32_t keyNulls) {
   return hashAggFindIn(p.agg, [&](int a) { return p.aggs[a].kind; }, keys, keyNulls);
}
// exact MIN / MAX of a 16-byte aggregate cell: a 16-byte compare-and-swap loop (one atomic per update when uncontended, like the
// 8-byte atomicMin it replaces).  The plain read is only the first guess of the CAS: its two 8-byte halves may come from different
// updates, so a "not better" decision taken on it alone could drop a value.  The loop ends on a CAS that either installs x or
// confirms (by rewriting the same value) that the cell already holds one at least as good.
__device__ __forceinline__ void atomicMinMax128(unsigned long long* cell, s128 x, bool isMax) {
   unsigned __int128* p = (unsigned __int128*) cell; // 16-byte aligned: entries are 48 + 16 nAggs bytes from an aligned base
   const volatile unsigned long long* vc = cell;
   unsigned __int128 cur = ((unsigned __int128) vc[1] << 64) | vc[0];
   while (true) {
      const bool better = isMax ? x > (s128) cur : x < (s128) cur;
      const unsigned __int128 prev = atomicCAS(p, cur, better ? (unsigned __int128) x : cur);
      if (prev == cur) return;
      cur = prev;
   }
}
// The order MIN_F64 / MAX_F64 keep (include/ldb_gpu.h, LdbAggKind): NaN loses to every other value, -0.0 orders below +0.0, ±inf
// are ordinary values.  So the result does not depend on the order of the updates, and a group whose non-NULL inputs are all NaN ends
// at NaN.  For non-NaN doubles the integer key b ^ ((b >> 63) & INT64_MAX) of the bits b orders like the values, with -0.0 < +0.0.
__device__ __forceinline__ long long f64OrderKey(double x) {
   const long long b = __double_as_longlong(x);
   return b ^ ((b >> 63) & 0x7fffffffffffffffll);
}
__device__ __forceinline__ bool f64Better(double d, unsigned long long cur, bool isMin) {
   const double c = __longlong_as_double((long long) cur);
   if (isnan(d)) return false;
   if (isnan(c)) return true;
   return isMin ? f64OrderKey(d) < f64OrderKey(c) : f64OrderKey(d) > f64OrderKey(c);
}
// MIN / MAX of a double cell: a CAS loop that ends once the cell holds a value at least as good as d.  The cell only ever gets
// better, so a "not better" decision on the plain 8-byte read stays true.
__device__ __forceinline__ void atomicMinMaxF64(unsigned long long* lo, double d, bool isMin) {
   unsigned long long cur = *((volatile unsigned long long*) lo);
   while (f64Better(d, cur, isMin)) {
      const unsigned long long prev = atomicCAS(lo, cur, (unsigned long long) __double_as_longlong(d));
      if (prev == cur) break;
      cur = prev;
   }
}
// the ANY claim of aggregate a: true for the one thread that sets the claim bit, which then writes the value
__device__ __forceinline__ bool claimAny(uint32_t* flags, int a) {
   if (*((volatile uint32_t*) flags) & (kClaimBit << a)) return false;
   return !(atomicOr(flags, kClaimBit << a) & (kClaimBit << a));
}
// in-place aggregate update (subop.reduce lowering + combine functions, SubOpToControlFlow.cpp:3540-3769, RelAlgToSubOp.cpp:1809-2025):
// NULL inputs are skipped, an aggregate that never saw a value stays NULL (its "seen" bit)
__device__ void hashAggUpdate(const ProgramParams& p, uint8_t* e, const Val* regs) {
   uint32_t* flags = (uint32_t*) e + 1;
   unsigned long long* ea = (unsigned long long*) (e + 16 + 8 * kProgMaxKeys);
   for (int a = 0; a < p.nAggs; a++) {
      const int kind = p.aggs[a].kind;
      unsigned long long* lo = ea + 2 * a;
      if (kind == LDB_AGG_COUNT_STAR) {
         atomicAdd(lo, 1ull);
         continue;
      }
      const Val x = regs[p.aggs[a].reg];
      if (x.null) continue;
      const uint32_t seen = kSeenBit << a;
      switch (kind) {
         case LDB_AGG_SUM: atomicAdd128(lo, lo + 1, i128{(uint64_t) x.v, (int64_t) (x.v >> 64)}); break;
         case LDB_AGG_SUM_F64: atomicAdd((double*) lo, asF64(x)); break;
         case LDB_AGG_COUNT: atomicAdd(lo, 1ull); break;
         case LDB_AGG_MIN:
         case LDB_AGG_MAX: atomicMinMax128(lo, x.v, kind == LDB_AGG_MAX); break;
         case LDB_AGG_MIN_F64:
         case LDB_AGG_MAX_F64: atomicMinMaxF64(lo, asF64(x), kind == LDB_AGG_MIN_F64); break;
         case LDB_AGG_ANY:
            if (!claimAny(flags, a)) continue; // somebody else's value is the group's "any"
            lo[0] = (unsigned long long) (uint64_t) x.v;
            lo[1] = (unsigned long long) (uint64_t) (x.v >> 64);
            __threadfence();
            break;
         default: break;
      }
      if (!(*((volatile uint32_t*) flags) & seen)) atomicOr(flags, seen);
   }
}
// combine of a partial aggregate state `r` (an entry of another table with the same aggregates) into the group's entry `e`
// (rt::PreAggregationHashtable::merge's combine): counts add; every other aggregate takes r's value only when r has seen one —
// sums add, MIN / MAX keep the better value, ANY takes r's value when e has not claimed one yet.  The seen bits are ORed in.
__device__ void hashAggCombine(const HashAggDev& t, const int32_t* kinds, uint8_t* e, const uint8_t* r) {
   uint32_t* flags = (uint32_t*) e + 1;
   const uint32_t rf = ((const uint32_t*) r)[1];
   unsigned long long* ea = (unsigned long long*) (e + 16 + 8 * kProgMaxKeys);
   const unsigned long long* ra = (const unsigned long long*) (r + 16 + 8 * kProgMaxKeys);
   for (int a = 0; a < t.nAggs; a++) {
      const int kind = kinds[a];
      unsigned long long* lo = ea + 2 * a;
      const unsigned long long xlo = ra[2 * a], xhi = ra[2 * a + 1];
      if (kind == LDB_AGG_COUNT || kind == LDB_AGG_COUNT_STAR) {
         if (xlo) atomicAdd(lo, xlo);
         continue;
      }
      if (!(rf & (kSeenBit << a))) continue;
      switch (kind) {
         case LDB_AGG_SUM: atomicAdd128(lo, lo + 1, i128{xlo, (int64_t) xhi}); break;
         case LDB_AGG_SUM_F64: atomicAdd((double*) lo, __longlong_as_double((long long) xlo)); break;
         case LDB_AGG_MIN:
         case LDB_AGG_MAX: atomicMinMax128(lo, (s128) (((unsigned __int128) xhi << 64) | xlo), kind == LDB_AGG_MAX); break;
         case LDB_AGG_MIN_F64:
         case LDB_AGG_MAX_F64: atomicMinMaxF64(lo, __longlong_as_double((long long) xlo), kind == LDB_AGG_MIN_F64); break;
         case LDB_AGG_ANY:
            if (!(rf & (kClaimBit << a)) || !claimAny(flags, a)) break;
            lo[0] = xlo;
            lo[1] = xhi;
            __threadfence();
            break;
         default: break;
      }
   }
   const uint32_t seen = rf & ((1u << t.nAggs) - 1u);
   if ((*((volatile uint32_t*) flags) & seen) != seen) atomicOr(flags, seen);
}

// ---------------------------------------------------------------- the interpreter
// One thread per scanned row.  Without LDB_OP_PROBE_EACH the program, the WHERE test and the sink run once.  With it, the
// instructions from PROBE_EACH on, the WHERE test and the sink run once per match: the warp keeps iterating together until no lane
// has a match left (the materialize sink's ballot needs all 32 lanes), and a lane without a tuple in an iteration does not pass.
// KeyTuples: the instance that also reads and builds key-tuple join tables.  Programs without one run the instance that has none of
// that code: even an untaken key-tuple build call in the sink made the plain-table build kernel four times slower (register allocation
// and scheduling of the whole loop change with it).
// Marks: the instance that also runs LDB_OP_MARK and records, per table, the slot the latest PROBE / PROBE_EACH matched.  For the
// same reason only programs with a MARK run it; with Marks false none of that code is compiled in.
// Exists: the instance that also runs LDB_OP_EXISTS, again launched only for programs that contain one.  The walk over a key's matches
// is a state machine on the program counter: EXISTS takes the first match and runs its residual block (a key without a match runs it
// once with dst NULL, so that a warp's lanes stay together); at the block's last instruction the walk either jumps back to the block's
// first instruction with the next match or writes the verdict and falls through.  Its cursor
// (ex*) is separate from PROBE_EACH's, because an EXISTS after a PROBE_EACH walks while the PROBE_EACH run is still open.
template <bool KeyTuples, bool Marks, bool Exists>
__global__ void __launch_bounds__(256) programKernel(const __grid_constant__ ProgramParams p) {
   unsigned long long inserted = 0;
   for (int64_t base = (int64_t) blockIdx.x * blockDim.x; base < p.nRows; base += (int64_t) gridDim.x * blockDim.x) {
      const int64_t row = base + threadIdx.x;
      const bool valid = row < p.nRows;
      Val regs[kProgMaxRegs] = {};
      bool pending = valid; // this row may still produce a tuple
      int start = 0;        // first instruction of the next iteration
      // PROBE_EACH cursor: 0 not started, 1 walking the run, 2 run ended
      int eachState = 0;
      bool eachEmitted = false;
      int32_t eachKey = 0;
      uint64_t eachSlot = 0;
      uint32_t eachProbes = 0;
      KeyCursor eachCur{}; // key-tuple tables
      // Marks: the directory slot of the entry the latest PROBE / PROBE_EACH of tables[k] matched for this tuple (kNoSlot: none)
      uint64_t hitSlot[Marks ? kProgMaxTables : 1];
      if (Marks)
         for (int k = 0; k < kProgMaxTables; k++) hitSlot[k] = kNoSlot;
      // Exists: the EXISTS at exPc walks its key's matches while exEnd (its block's last instruction) is >= 0
      int exPc = 0, exEnd = -1;
      bool exMiss = false; // the key has no match: the block runs once for nothing
      int32_t exKey = 0;
      uint64_t exSlot = 0;
      uint32_t exProbes = 0;
      KeyCursor exCur{};
      KeyTuple exKeys;
      // the next match of the walk: its payload in `pay`; false: the run ended
      auto exNext = [&](const ProgInstr& ex, int64_t& pay) {
         if (KeyTuples && p.keyTables[ex.arg].nKeys) {
            const KeyHit h = keyJoinNext(p.keyTables[ex.arg], exKeys, exCur);
            exCur = h.next;
            pay = h.payload;
            return h.hit;
         }
         int32_t pay32 = 0;
         const bool hit = probeEachNext(p.tables[ex.arg], exKey, exSlot, exProbes, pay32, 8);
         pay = pay32;
         return hit;
      };
      while (true) {
         bool pass = false;
         if (pending) {
            bool tuple = true;
            for (int pc = start; pc < p.nInstr; pc++) {
               const ProgInstr in = p.instr[pc];
               // EXISTS's b is its block length (up to 94), not a register: never an index into regs
               const Val a = regs[in.a], b = regs[Exists && in.op == LDB_OP_EXISTS ? 0 : in.b];
               Val r;
               r.v = 0;
               r.null = false;
               switch (in.op) {
                  case LDB_OP_LOAD: {
                     const ProgCol& c = p.cols[in.arg];
                     if (c.rowReg < 0) {
                        r = loadCol(c, row);
                     } else {
                        ProgCol tmp;
                        int64_t at;
                        const ProgCol* cc = cellOf(c, regs, row, tmp, at);
                        if (cc) r = loadCol(*cc, at);
                        else r.null = true;
                     }
                     break;
                  }
                  case LDB_OP_ROWID: r.v = (s128) (p.firstRow + row); break;
                  case LDB_OP_CONST: r.v = (s128) (((unsigned __int128) (uint64_t) p.constHi[in.arg] << 64) | p.constLo[in.arg]); break;
                  case LDB_OP_ADD: r.v = (s128) ((unsigned __int128) a.v + (unsigned __int128) b.v); r.null = a.null | b.null; break;
                  case LDB_OP_SUB: r.v = (s128) ((unsigned __int128) a.v - (unsigned __int128) b.v); r.null = a.null | b.null; break;
                  case LDB_OP_MUL: r.v = (s128) ((unsigned __int128) a.v * (unsigned __int128) b.v); r.null = a.null | b.null; break;
                  case LDB_OP_DIV:
                     r.null = a.null | b.null | (b.v == 0);
                     if (!r.null) r.v = a.v / b.v; // sdiv: truncating (DecimalDiv lowering, LowerToStd.cpp:651-700)
                     break;
                  case LDB_OP_NEG: r.v = (s128) (0 - (unsigned __int128) a.v); r.null = a.null; break;
                  case LDB_OP_CMP: r.v = cmpI(a.v, b.v, in.arg); r.null = a.null | b.null; break;
                  case LDB_OP_AND: // three-valued: false dominates NULL
                     if ((!a.null && a.v == 0) || (!b.null && b.v == 0)) r.v = 0;
                     else if (a.null | b.null) r.null = true;
                     else r.v = 1;
                     break;
                  case LDB_OP_OR: // true dominates NULL
                     if ((!a.null && a.v != 0) || (!b.null && b.v != 0)) r.v = 1;
                     else if (a.null | b.null) r.null = true;
                     else r.v = 0;
                     break;
                  case LDB_OP_NOT: r.v = a.v == 0; r.null = a.null; break;
                  case LDB_OP_ISNULL: r.v = a.null; break;
                  case LDB_OP_SELECT: {
                     const Val c = regs[in.arg];
                     r = (!c.null && c.v != 0) ? a : b;
                     break;
                  }
                  case LDB_OP_I2F: r = fromF64((double) a.v, a.null); break;
                  case LDB_OP_FADD: r = fromF64(asF64(a) + asF64(b), a.null | b.null); break;
                  case LDB_OP_FSUB: r = fromF64(asF64(a) - asF64(b), a.null | b.null); break;
                  case LDB_OP_FMUL: r = fromF64(asF64(a) * asF64(b), a.null | b.null); break;
                  case LDB_OP_FDIV: r = fromF64(asF64(a) / asF64(b), a.null | b.null); break;
                  case LDB_OP_FCMP: r.v = cmpF(asF64(a), asF64(b), in.arg); r.null = a.null | b.null; break;
                  case LDB_OP_STRCMP: {
                     ProgCol tmp;
                     int64_t at;
                     const ProgCol* c = cellOf(p.cols[in.a], regs, row, tmp, at);
                     r.null = !c || colIsNull(*c, at);
                     if (!r.null) r.v = cmpI((s128) strCompare(*c, at, p.strings[in.arg], p.stringLen[in.arg]), 0, in.b);
                     break;
                  }
                  case LDB_OP_STRLIKE: {
                     ProgCol tmp;
                     int64_t at;
                     const ProgCol* c = cellOf(p.cols[in.a], regs, row, tmp, at);
                     r.null = !c || colIsNull(*c, at);
                     if (!r.null) r.v = strLike(*c, at, p.strings[in.arg], p.stringLen[in.arg], in.b);
                     break;
                  }
                  case LDB_OP_YEAR: r.v = (s128) yearOfDays((int32_t) a.v); r.null = a.null; break;
                  case LDB_OP_STRKEY8: {
                     ProgCol tmp;
                     int64_t at;
                     const ProgCol* c = cellOf(p.cols[in.a], regs, row, tmp, at);
                     r.null = !c || colIsNull(*c, at);
                     if (!r.null) {
                        const int32_t* off = (const int32_t*) c->data + at;
                        const int32_t b0 = off[0], n = off[1] - off[0];
                        uint64_t k = 0;
                        for (int i = 0; i < 8; i++) k = (k << 8) | (i < n ? c->bytes[b0 + i] : 0);
                        r.v = (s128) (int64_t) k;
                     }
                     break;
                  }
                  case LDB_OP_STRCODE: { // string → its dictionary code; b = 1 inserts an absent string, b = 0 gives NULL for it
                     ProgCol tmp;
                     int64_t at;
                     const ProgCol* c = cellOf(p.cols[in.a], regs, row, tmp, at);
                     r.null = !c || colIsNull(*c, at);
                     if (!r.null) {
                        const int32_t* off = (const int32_t*) c->data + at;
                        const int32_t code = dictCode(p.dicts[in.arg], c->bytes + off[0], off[1] - off[0], in.b);
                        r.null = code < 0;
                        r.v = code < 0 ? 0 : code;
                     }
                     break;
                  }
                  case LDB_OP_PROBE: { // key → payload of a unique/multimap single-key table; absent key = NULL (semi / anti / mark / outer)
                     const JoinTableDev& t = p.tables[in.arg];
                     r.null = true;
                     if (Marks) hitSlot[in.arg] = kNoSlot;
                     if (KeyTuples && p.keyTables[in.arg].nKeys) { // key-tuple table: the keys are registers a .. a + nKeys - 1
                        KeyTuple keys;
                        if (!gatherTuple(regs, p.keyTables[in.arg].nKeys, [&](int k) { return in.a + k; }, keys)) { // NULL / past int64: no match
                           const KeyCursor c = keyJoinStart(p.keyTables[in.arg], keys);
                           const KeyHit h = c.live ? keyJoinNext(p.keyTables[in.arg], keys, c) : KeyHit{c, 0, false};
                           r.v = h.payload;
                           r.null = !h.hit;
                           if (Marks && h.hit) hitSlot[in.arg] = (h.next.slot - 1) & p.keyTables[in.arg].mask; // the cursor is past the hit
                        }
                     } else if (!a.null && a.v == (s128) (int32_t) a.v) {
                        const int32_t key = (int32_t) a.v;
                        if (t.direct) {
                           const int32_t pay = directLoadProg(t, key);
                           if (pay != kDirectEmpty) {
                              r.v = pay;
                              r.null = false;
                              if (Marks) hitSlot[in.arg] = (uint32_t) key - (uint32_t) t.keyMin;
                           }
                        } else {
                           const uint64_t h = hashI32(key);
                           bool maybe = true;
                           if (t.bloom) {
                              const uint32_t bits = bloomBits(h);
                              maybe = (__ldg(&t.bloom[(uint32_t) (h >> 32) & t.bloomMask]) & bits) == bits;
                           }
                           uint64_t s = h & t.mask;
                           for (uint64_t probes = 0; maybe && probes <= t.mask && probes < 16384; probes++) {
                              const unsigned long long e = __ldg((const unsigned long long*) (t.base + s * t.stride));
                              if (e == ~0ull) break;
                              if ((int32_t) (uint32_t) e == key) {
                                 r.v = (s128) (int32_t) ((uint32_t) (e >> 32) & (t.stride == 32 ? 0x7fffffffu : 0xffffffffu));
                                 r.null = false;
                                 if (Marks) hitSlot[in.arg] = s;
                                 break;
                              }
                              s = (s + 1) & t.mask;
                           }
                        }
                     }
                     break;
                  }
                  case LDB_OP_PROBE_EACH: { // the next match; b = 1: a row without any match yields one tuple with a NULL payload
                     const JoinTableDev& t = p.tables[in.arg];
                     const bool tuple64 = KeyTuples && p.keyTables[in.arg].nKeys != 0; // key-tuple table: keys in registers a .. a + nKeys - 1,
                                                                                         // its run in eachCur
                     KeyTuple eachKeys;
                     if (tuple64 && eachState != 2 && gatherTuple(regs, p.keyTables[in.arg].nKeys, [&](int k) { return in.a + k; }, eachKeys)) eachState = 2;
                     if (eachState == 0) {
                        eachState = 2; // a NULL key (or one outside int32) never matches
                        if (tuple64) {
                           eachCur = keyJoinStart(p.keyTables[in.arg], eachKeys);
                           if (eachCur.live) eachState = 1;
                        } else if (!a.null && a.v == (s128) (int32_t) a.v) {
                           eachKey = (int32_t) a.v;
                           const uint64_t h = hashI32(eachKey);
                           eachSlot = h & t.mask;
                           eachState = 1;
                           if (!t.direct && t.bloom) {
                              const uint32_t bits = bloomBits(h);
                              if ((__ldg(&t.bloom[(uint32_t) (h >> 32) & t.bloomMask]) & bits) != bits) eachState = 2;
                           }
                        }
                     }
                     int32_t pay = 0;
                     int64_t pay64 = 0;
                     auto tupleNext = [&] {
                        const KeyHit h = keyJoinNext(p.keyTables[in.arg], eachKeys, eachCur);
                        eachCur = h.next;
                        pay64 = h.payload;
                        return h.hit;
                     };
                     r.null = true;
                     if (Marks) hitSlot[in.arg] = kNoSlot;
                     if (eachState == 1 && (tuple64 ? tupleNext() : probeEachNext(t, eachKey, eachSlot, eachProbes, pay))) {
                        r.v = tuple64 ? pay64 : pay;
                        r.null = false;
                        if (Marks) // the cursors are past the hit; a direct-address table has one slot per key
                           hitSlot[in.arg] = tuple64 ? (eachCur.slot - 1) & p.keyTables[in.arg].mask
                                                     : t.direct ? (uint64_t) ((uint32_t) eachKey - (uint32_t) t.keyMin) : (eachSlot - 1) & t.mask;
                     } else {
                        eachState = 2;
                        pending = false;
                        tuple = in.b == 1 && !eachEmitted;
                     }
                     eachEmitted = true;
                     break;
                  }
                  default:
                     if (Marks && in.op == LDB_OP_MARK) { // marks the entry the latest probe of tables[arg] matched, when a is TRUE
                        const uint64_t slot = hitSlot[in.arg];
                        r.v = !a.null && a.v != 0 && slot != kNoSlot;
                        if (r.v != 0) { // check, then store: idempotent, and other threads write the byte in the same launch
                           volatile uint8_t* m = p.marks[in.arg] + slot;
                           if (*m == 0) *m = 1;
                        }
                     } else if (Exists && in.op == LDB_OP_EXISTS) { // the walk starts: the key's first match, or FALSE and past the block
                        bool live = false;
                        if (KeyTuples && p.keyTables[in.arg].nKeys) {
                           if (!gatherTuple(regs, p.keyTables[in.arg].nKeys, [&](int k) { return in.a + k; }, exKeys)) { // NULL / past int64: no match
                              exCur = keyJoinStart(p.keyTables[in.arg], exKeys);
                              live = exCur.live;
                           }
                        } else if (!a.null && a.v == (s128) (int32_t) a.v) {
                           const JoinTableDev& t = p.tables[in.arg];
                           exKey = (int32_t) a.v;
                           const uint64_t h = hashI32(exKey);
                           exSlot = h & t.mask;
                           exProbes = 0;
                           live = true;
                           if (!t.direct && t.bloom) {
                              const uint32_t bits = bloomBits(h);
                              live = (__ldg(&t.bloom[(uint32_t) (h >> 32) & t.bloomMask]) & bits) == bits;
                           }
                        }
                        int64_t pay = 0;
                        const bool hit = live && exNext(in, pay);
                        if (in.b == 0) {
                           r.v = hit; // no residual: a match is enough
                        } else { // the block runs with dst = this match's payload.  Without a match it runs once too, with dst NULL and
                                 // its residual ignored: the lanes of a warp stay on the same instructions (skipping the block made the
                                 // interpreter run the two instruction streams one after the other, 5x slower at half the rows matching)
                           r.v = pay;
                           r.null = !hit;
                           exMiss = !hit;
                           exPc = pc;
                           exEnd = pc + in.b;
                        }
                     } else {
                        r.null = true;
                     }
               }
               if (!tuple) break;
               regs[in.dst] = r;
               if (Exists && pc == exEnd) { // the last instruction of an EXISTS block wrote the residual r: TRUE ends the walk, else the next match
                  const ProgInstr ex = p.instr[exPc];
                  Val v{0, false};
                  int64_t pay = 0;
                  if (exMiss) {
                     // no match at all: FALSE
                  } else if (!r.null && r.v != 0) {
                     v.v = 1;
                  } else if (exNext(ex, pay)) {
                     v.v = pay; // back to the block's first instruction with dst = the next match's payload
                     pc = exPc;
                  }
                  if (pc != exPc) exEnd = -1;
                  regs[ex.dst] = v;
               }
            }
            pass = tuple;
            if (tuple && p.filterReg >= 0) { // WHERE: NULL is not true
               const Val f = regs[p.filterReg];
               pass = !f.null && f.v != 0;
            }
            if (p.eachPc < 0) pending = false;
            start = p.eachPc;
         }
         if (p.sinkKind == 1) {
            if (pass) {
               int64_t keys[kProgMaxKeys];
               uint32_t nulls = 0;
               for (int k = 0; k < p.nKeys; k++) {
                  const Val kv = regs[p.keyReg[k]];
                  keys[k] = kv.null ? 0 : (int64_t) kv.v;
                  nulls |= (kv.null ? 1u : 0u) << k;
               }
               uint8_t* e = hashAggFind(p, keys, nulls);
               if (e) hashAggUpdate(p, e, regs);
            }
         } else if (p.sinkKind == 2) {
            if (KeyTuples && pass && p.keyBuild.nKeys) { // a key-tuple table: keys from keyReg[], int64 keys and payloads
               KeyTuple keys;
               const int bad = gatherTuple(regs, p.nKeys, [&](int k) { return p.keyReg[k]; }, keys);
               const s128 pay = p.buildPayloadReg >= 0 && !regs[p.buildPayloadReg].null ? regs[p.buildPayloadReg].v : 0;
               if (bad & 1) {
                  // a NULL key component never matches: the row is not stored
               } else if (bad || pay != (s128) (int64_t) pay) {
                  atomicExch(p.keyBuild.error, 7); // keys and payloads are int64
               } else if (keyJoinInsert(p.keyBuild, keys, (int64_t) pay)) {
                  inserted++;
               }
            } else if (pass) {
               const Val k = regs[p.buildKeyReg];
               if (!k.null) { // NULL keys never match (SQL join semantics); a NULL payload is stored as 0
                  const s128 pay = p.buildPayloadReg >= 0 && !regs[p.buildPayloadReg].null ? regs[p.buildPayloadReg].v : 0;
                  if (k.v != (s128) (int32_t) k.v || pay != (s128) (int32_t) pay) atomicExch(p.build.error, 7); // keys and payloads are int32
                  else if (joinInsertProg(p.build, (int32_t) k.v, (int32_t) pay)) inserted++;
               }
            }
         } else if (p.sinkKind == 3) { // warp-aggregated append of the selected registers
            const unsigned m = __ballot_sync(0xffffffffu, pass);
            if (m) {
               const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
               unsigned long long pos = 0;
               if (lane == leader) pos = atomicAdd(p.outCount, (unsigned long long) __popc(m));
               pos = __shfl_sync(0xffffffffu, pos, leader) + __popc(m & ((1u << lane) - 1));
               if (pass && pos < (unsigned long long) p.outCapacity) {
                  for (int c = 0; c < p.nOut; c++) {
                     const Val x = regs[p.outReg[c]];
                     ulonglong2 cell;
                     cell.x = (unsigned long long) (uint64_t) x.v;
                     cell.y = (unsigned long long) (uint64_t) (x.v >> 64);
                     ((ulonglong2*) p.outValues[c])[pos] = cell;
                     p.outValid[c][pos] = x.null ? 0 : 1;
                  }
               }
            }
         }
         if (p.eachPc < 0 || !__any_sync(0xffffffffu, pending)) break;
      }
   }
   if (p.sinkKind == 2) {
      unsigned long long total = warpSum64(inserted);
      if ((threadIdx.x & 31) == 0 && total) atomicAdd(KeyTuples && p.keyBuild.nKeys ? p.keyBuild.count : p.build.count, total);
   }
}
void launchProgram(const ProgramParams& p, int smCount, cudaStream_t s) {
   int grid = (int) std::min<int64_t>(std::max<int64_t>((p.nRows + 255) / 256, 1), (int64_t) smCount * 8);
   bool keyTuples = p.keyBuild.nKeys != 0, marks = false;
   for (int k = 0; k < kProgMaxTables; k++) {
      keyTuples |= p.keyTables[k].nKeys != 0;
      marks |= p.marks[k] != nullptr;
   }
   bool exists = false;
   for (int i = 0; i < p.nInstr; i++) exists |= p.instr[i].op == LDB_OP_EXISTS;
   if (exists) {
      if (marks) {
         if (keyTuples) programKernel<true, true, true><<<grid, 256, 0, s>>>(p);
         else programKernel<false, true, true><<<grid, 256, 0, s>>>(p);
      } else {
         if (keyTuples) programKernel<true, false, true><<<grid, 256, 0, s>>>(p);
         else programKernel<false, false, true><<<grid, 256, 0, s>>>(p);
      }
   } else if (marks) {
      if (keyTuples) programKernel<true, true, false><<<grid, 256, 0, s>>>(p);
      else programKernel<false, true, false><<<grid, 256, 0, s>>>(p);
   } else {
      if (keyTuples) programKernel<true, false, false><<<grid, 256, 0, s>>>(p);
      else programKernel<false, false, false><<<grid, 256, 0, s>>>(p);
   }
}

// ---------------------------------------------------------------- join-table markers
// One thread per directory slot: an occupancy test for the table's kind, the marker test, then a warp-aggregated append (one atomic
// per warp), as hashAggExportKernel.  Runs after the launches that built and marked the table: plain loads.
__global__ void __launch_bounds__(256) joinMarksKernel(JoinTableDev t, KeyJoinDev k, const uint8_t* marks, int which, MarkScanOut o, unsigned long long* counter) {
   const uint64_t slots = k.nKeys ? k.mask + 1 : t.direct ? (uint64_t) t.range : t.mask + 1;
   const int nKeys = k.nKeys ? k.nKeys : 1;
   for (uint64_t base = (uint64_t) blockIdx.x * blockDim.x; base < slots; base += (uint64_t) gridDim.x * blockDim.x) {
      const uint64_t s = base + threadIdx.x;
      bool occ = false;
      int64_t key[kProgMaxKeys] = {};
      int64_t pay = 0;
      if (s < slots) {
         if (k.nKeys) {
            const uint8_t* e = k.base + s * k.entryBytes;
            const ulonglong2 head = *(const ulonglong2*) e;
            occ = (uint32_t) head.x == kKeyJoinReady;
            pay = (int64_t) head.y;
#pragma unroll
            for (int j = 0; j < kProgMaxKeys; j++)
               if (j < k.nKeys) key[j] = ((const int64_t*) (e + 16))[j];
         } else if (t.direct) {
            const int32_t v = ((const int32_t*) t.base)[s];
            occ = v != kDirectEmpty;
            key[0] = (int64_t) s + t.keyMin;
            pay = v;
         } else {
            const unsigned long long e = *(const unsigned long long*) (t.base + s * t.stride);
            occ = e != ~0ull;
            key[0] = (int32_t) (uint32_t) e;
            pay = (int32_t) (uint32_t) (e >> 32);
         }
      }
      const bool marked = occ && marks && marks[s];
      const bool take = occ && (which < 0 || (which == 1) == marked);
      const unsigned m = __ballot_sync(0xffffffffu, take);
      if (!m) continue;
      const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
      unsigned long long pos = 0;
      if (lane == leader) pos = atomicAdd(counter, (unsigned long long) __popc(m));
      pos = __shfl_sync(0xffffffffu, pos, leader) + __popc(m & ((1u << lane) - 1));
      if (!take || pos >= (unsigned long long) o.capacity) continue;
#pragma unroll
      for (int j = 0; j < kProgMaxKeys; j++)
         if (j < nKeys) o.keyCols[j][pos] = key[j];
      o.payload[pos] = pay;
      if (o.marked) o.marked[pos] = marked ? 1 : 0;
   }
}
void launchJoinMarks(const JoinTableDev& t, const KeyJoinDev& k, const uint8_t* marks, int which, const MarkScanOut& o, unsigned long long* counter, int smCount, cudaStream_t s) {
   const uint64_t slots = k.nKeys ? k.mask + 1 : t.direct ? (uint64_t) t.range : t.mask + 1;
   const int grid = (int) std::min<uint64_t>((slots + 255) / 256, (uint64_t) smCount * 8);
   joinMarksKernel<<<grid < 1 ? 1 : grid, 256, 0, s>>>(t, k, marks, which, o, counter);
}

__global__ void hashAggInitKernel(HashAggDev t) {
   const uint64_t words = (t.mask + 1) * (uint64_t) t.entryBytes / 8;
   unsigned long long* w = (unsigned long long*) t.base;
   for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (uint64_t) gridDim.x * blockDim.x) w[i] = 0;
}
void launchHashAggInit(const HashAggDev& t, int smCount, cudaStream_t s) {
   const uint64_t words = (t.mask + 1) * (uint64_t) t.entryBytes / 8;
   int grid = (int) std::min<uint64_t>((words + 255) / 256, (uint64_t) smCount * 16);
   hashAggInitKernel<<<grid < 1 ? 1 : grid, 256, 0, s>>>(t);
}
struct ExportPtrs {
   int64_t* keyCols[kProgMaxKeys];
   uint8_t* keyValid[kProgMaxKeys];
   uint8_t* aggCols[kProgMaxAggs];
   uint8_t* aggValid[kProgMaxAggs];
};
// the scan over the hash table's entries that starts the reference's next pipeline (createIterator, PreAggregationHashtable.cpp:160-170),
// as a compaction into columns
__global__ void __launch_bounds__(256) hashAggExportKernel(HashAggDev t, ExportPtrs o, unsigned long long* counter, uint32_t countAggMask) {
   const uint64_t cap = t.mask + 1;
   for (uint64_t base = (uint64_t) blockIdx.x * blockDim.x; base < cap; base += (uint64_t) gridDim.x * blockDim.x) {
      const uint64_t s = base + threadIdx.x;
      const uint8_t* e = s < cap ? entryAt(t, s) : nullptr;
      const bool occ = e && *((const uint32_t*) e) == 2u;
      const unsigned m = __ballot_sync(0xffffffffu, occ);
      if (!m) continue;
      const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
      unsigned long long pos = 0;
      if (lane == leader) pos = atomicAdd(counter, (unsigned long long) __popc(m));
      pos = __shfl_sync(0xffffffffu, pos, leader) + __popc(m & ((1u << lane) - 1));
      if (!occ) continue;
      const uint32_t fl = ((const uint32_t*) e)[1];
      const int64_t* ek = (const int64_t*) (e + 16);
      for (int k = 0; k < t.nKeys; k++) {
         o.keyCols[k][pos] = ek[k];
         o.keyValid[k][pos] = ((fl >> (16 + k)) & 1u) ? 0 : 1;
      }
      const ulonglong2* ea = (const ulonglong2*) (e + 16 + 8 * kProgMaxKeys);
      for (int a = 0; a < t.nAggs; a++) {
         ((ulonglong2*) o.aggCols[a])[pos] = ea[a];
         o.aggValid[a][pos] = (((fl >> a) & 1u) || ((countAggMask >> a) & 1u)) ? 1 : 0; // counts are never NULL
      }
   }
}
void launchHashAggExport(const HashAggDev& t, int64_t* const* keyCols, uint8_t* const* keyValid, uint8_t* const* aggCols, uint8_t* const* aggValid, unsigned long long* counter, uint32_t countAggMask, int smCount, cudaStream_t s) {
   ExportPtrs o{};
   for (int k = 0; k < t.nKeys; k++) {
      o.keyCols[k] = keyCols[k];
      o.keyValid[k] = keyValid[k];
   }
   for (int a = 0; a < t.nAggs; a++) {
      o.aggCols[a] = aggCols[a];
      o.aggValid[a] = aggValid[a];
   }
   const uint64_t cap = t.mask + 1;
   int grid = (int) std::min<uint64_t>((cap + 255) / 256, (uint64_t) smCount * 8);
   hashAggExportKernel<<<grid < 1 ? 1 : grid, 256, 0, s>>>(t, o, counter, countAggMask);
}

// ---------------------------------------------------------------- exchange of hash aggregations across ranks (HashAggShip, program.h)
// Send: one thread per slot of `local`.  A ready group goes to its owner, the rank the high 32 bits of its placement hash select; the
// warp claims its positions with one atomicAdd per (warp, destination) on this rank's cursors, and each lane stores its whole entry into
// the owner's receive region with 16-byte stores.  Positions at or past the capacity are counted but not written.  The keyless
// state's one entry goes to every rank.
__global__ void __launch_bounds__(256) hashAggSendKernel(HashAggDev t, const __grid_constant__ HashAggShip x) {
   const uint32_t n16 = t.entryBytes / 16;
   if (t.nKeys == 0) {
      const int d = threadIdx.x;
      if (blockIdx.x != 0 || d >= x.world) return;
      const unsigned long long pos = atomicAdd(x.cursors + d, 1ull);
      if (pos >= (unsigned long long) x.capacity) return;
      int4* dst = (int4*) (x.recv[d] + ((uint64_t) x.rank * x.capacity + pos) * t.entryBytes);
      for (uint32_t i = 0; i < n16; i++) dst[i] = ((const int4*) t.base)[i];
      return;
   }
   const uint64_t cap = t.mask + 1;
   for (uint64_t base = (uint64_t) blockIdx.x * blockDim.x; base < cap; base += (uint64_t) gridDim.x * blockDim.x) {
      const uint64_t s = base + threadIdx.x;
      const uint8_t* e = s < cap ? entryAt(t, s) : nullptr;
      const bool occ = e && *((const uint32_t*) e) == 2u;
      int owner = -1;
      if (occ) {
         const uint64_t h = keyTupleHash((const int64_t*) (e + 16), t.nKeys, (((const uint32_t*) e)[1] >> 16) & 0xfu);
         owner = keyOwner(h, x.world);
      }
      if (!__any_sync(0xffffffffu, occ)) continue;
      const unsigned same = __match_any_sync(0xffffffffu, owner);
      const int lane = threadIdx.x & 31, leader = __ffs(same) - 1;
      unsigned long long pos = 0;
      if (occ && lane == leader) pos = atomicAdd(x.cursors + owner, (unsigned long long) __popc(same));
      pos = __shfl_sync(0xffffffffu, pos, leader) + __popc(same & ((1u << lane) - 1));
      if (!occ || pos >= (unsigned long long) x.capacity) continue;
      const int4* src = (const int4*) e;
      int4* dst = (int4*) (x.recv[owner] + ((uint64_t) x.rank * x.capacity + pos) * t.entryBytes);
      for (uint32_t i = 0; i < n16; i++) dst[i] = src[i];
   }
}
// Merge: every entry received from source s (min(counts[s], capacity) of them) is looked up or inserted in `owned` and combined into it
__global__ void __launch_bounds__(256) hashAggMergeKernel(HashAggDev t, const __grid_constant__ HashAggShip x) {
   const uint8_t* recv = x.recv[x.rank];
   for (int s = 0; s < x.world; s++) {
      const unsigned long long n = min(x.counts[s], (unsigned long long) x.capacity);
      for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t) gridDim.x * blockDim.x) {
         const uint8_t* r = recv + ((uint64_t) s * x.capacity + i) * t.entryBytes;
         int64_t keys[kProgMaxKeys];
         for (int k = 0; k < t.nKeys; k++) keys[k] = ((const int64_t*) (r + 16))[k];
         uint8_t* e = hashAggFindIn(t, [&](int a) { return x.kinds[a]; }, keys, (((const uint32_t*) r)[1] >> 16) & 0xfu);
         if (e) hashAggCombine(t, x.kinds, e, r);
      }
   }
}
void launchHashAggSend(const HashAggDev& local, const HashAggShip& x, int smCount, cudaStream_t s) {
   const uint64_t cap = local.mask + 1;
   const int grid = (int) std::min<uint64_t>((cap + 255) / 256, (uint64_t) smCount * 8);
   hashAggSendKernel<<<grid < 1 ? 1 : grid, 256, 0, s>>>(local, x);
}
void launchHashAggMerge(const HashAggDev& owned, const HashAggShip& x, uint64_t maxReceived, int smCount, cudaStream_t s) {
   const int grid = (int) std::min<uint64_t>((maxReceived + 255) / 256, (uint64_t) smCount * 8);
   hashAggMergeKernel<<<grid < 1 ? 1 : grid, 256, 0, s>>>(owned, x);
}
void loadHashAggExchangeKernels() {
   cudaFuncAttributes fa;
   cudaFuncGetAttributes(&fa, hashAggSendKernel);
   cudaFuncGetAttributes(&fa, hashAggMergeKernel);
}

// ---------------------------------------------------------------- radix sort (64-bit keys, 32-bit values), up to 8 passes of 8 bits
// (GrowingBuffer::sort → parallel sort of the materialised tuples, GrowingBuffer.cpp:54-78, Sorting.cpp; here LSD radix on an
//  order-preserving 64-bit key the host builds from the ORDER BY columns).  Stable; HBM-bound: 2 x (12 B read + 12 B write) per pass.
constexpr int kSortThreads = 256;
constexpr int kSortItemsPerCta = 256 * 16;
__global__ void __launch_bounds__(kSortThreads) sortHistKernel(const unsigned long long* keys, int64_t n, int shift, unsigned int* hist /* [256][gridDim.x] */) {
   __shared__ unsigned int h[256];
   h[threadIdx.x] = 0;
   __syncthreads();
   const int64_t begin = (int64_t) blockIdx.x * kSortItemsPerCta, end = begin + kSortItemsPerCta < n ? begin + kSortItemsPerCta : n;
   for (int64_t i = begin + threadIdx.x; i < end; i += kSortThreads) atomicAdd(&h[(keys[i] >> shift) & 255u], 1u);
   __syncthreads();
   hist[(size_t) threadIdx.x * gridDim.x + blockIdx.x] = h[threadIdx.x];
}
__global__ void __launch_bounds__(kSortThreads) sortScatterKernel(const unsigned long long* keys, const uint32_t* vals, unsigned long long* keysOut, uint32_t* valsOut, int64_t n, int shift, const unsigned int* hist) {
   __shared__ unsigned int running[256];      // global base + items of this digit already placed by this CTA
   __shared__ unsigned int warpCnt[8][256];   // per-warp digit counts of the current tile
   running[threadIdx.x] = hist[(size_t) threadIdx.x * gridDim.x + blockIdx.x];
   const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
   const int64_t begin = (int64_t) blockIdx.x * kSortItemsPerCta, end = begin + kSortItemsPerCta < n ? begin + kSortItemsPerCta : n;
   for (int64_t tile = begin; tile < end; tile += kSortThreads) {
      for (int i = threadIdx.x; i < 8 * 256; i += kSortThreads) (&warpCnt[0][0])[i] = 0;
      __syncthreads();
      const int64_t i = tile + threadIdx.x;
      const bool valid = i < end;
      const unsigned long long k = valid ? keys[i] : 0ull;
      const unsigned d = valid ? (unsigned) ((k >> shift) & 255u) : 256u;
      const unsigned active = __ballot_sync(0xffffffffu, valid);
      unsigned rankInWarp = 0;
      if (valid) {
         const unsigned peers = __match_any_sync(active, d);
         rankInWarp = __popc(peers & ((1u << lane) - 1));
         if (rankInWarp == 0) warpCnt[warp][d] = __popc(peers);
      }
      __syncthreads();
      if (valid) {
         unsigned before = 0;
         for (int w = 0; w < warp; w++) before += warpCnt[w][d];
         const unsigned pos = running[d] + before + rankInWarp;
         keysOut[pos] = k;
         valsOut[pos] = vals[i];
      }
      __syncthreads();
      unsigned tot = 0;
      for (int w = 0; w < 8; w++) tot += warpCnt[w][threadIdx.x];
      running[threadIdx.x] += tot;
      __syncthreads();
   }
}
void launchRadixSortPairs(unsigned long long* keys, uint32_t* vals, unsigned long long* keysTmp, uint32_t* valsTmp, int64_t n, unsigned int* histScratch, int smCount, cudaStream_t s,
                          int digits) {
   if (n <= 0) return;
   const int ctas = (int) ((n + kSortItemsPerCta - 1) / kSortItemsPerCta);
   unsigned long long* kin = keys;
   unsigned long long* kout = keysTmp;
   uint32_t* vin = vals;
   uint32_t* vout = valsTmp;
   for (int pass = 0; pass < digits; pass++) {
      sortHistKernel<<<ctas, kSortThreads, 0, s>>>(kin, n, pass * 8, histScratch);
      rowScanKernel<<<1, 1024, 0, s>>>(histScratch, (int64_t) ctas * 256, nullptr); // digit-major [256][ctas]
      sortScatterKernel<<<ctas, kSortThreads, 0, s>>>(kin, vin, kout, vout, n, pass * 8, histScratch);
      std::swap(kin, kout);
      std::swap(vin, vout);
   }
}

// ---------------------------------------------------------------- multi-key ORDER BY, dictionary ranks and export
// The sort words of one key at the current permutation: an LSD composition of launchRadixSortPairs (stable) sorts by the last key
// first; a utf8 key is its length word, then its 8-byte chunks from the last to the first.  Zero padding makes a proper prefix tie
// with its extension on every chunk, and the length pass, run before them, puts the shorter one first: bytewise order with
// unsigned bytes, the order of LDB_OP_STRCMP.  A 16-byte cell (an i128) is two words the same way: chunk 0 its low word, unsigned,
// then chunk 1 its high word with the sign bit flipped.  A nullable key ends with its NULL flag (kind 3), the most significant
// word of the key: NULLs, which tie on every value word, go last, and DESC's inversion puts them first.
__global__ void buildSortWordsKernel(const uint8_t* col, const uint8_t* bytes, int elemBytes, SortValidity valid, int kind, int chunk, int64_t n, int descending,
                                     int first, uint32_t* ids, unsigned long long* keys, int32_t* maxLen) {
   int32_t longest = 0;
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      const uint32_t row = first ? (uint32_t) i : ids[i];
      if (first) ids[i] = row;
      const int64_t bit = valid.bitOffset + row;
      const bool isNull = valid.bytes ? !valid.bytes[row] : valid.bitmap ? !((valid.bitmap[bit >> 3] >> (bit & 7)) & 1) : false;
      unsigned long long k = 0;
      if (kind == 3) {
         k = isNull;
      } else if (isNull) {
         // k = 0: every NULL gets the same value word
      } else if (kind == 0 && elemBytes == 16) { // the value of sortCell (sortkey.cuh), a word at a time
         k = chunk ? sortWideWord(col, row, 1) ^ 0x8000000000000000ull : sortWideWord(col, row, 0);
      } else if (kind == 0) {
         k = (unsigned long long) sortNarrowValue(col, elemBytes, row) ^ 0x8000000000000000ull;
      } else {
         const int32_t* off = (const int32_t*) col + row;
         const int32_t b = off[0], len = off[1] - off[0];
         if (kind == 1) {
            k = (unsigned long long) (uint32_t) len;
            longest = len > longest ? len : longest;
         } else {
            for (int j = 0; j < 8; j++) {
               const int32_t at = chunk * 8 + j;
               k = (k << 8) | (at < len ? bytes[b + at] : 0u);
            }
         }
      }
      keys[i] = descending ? ~k : k;
   }
   if (kind == 1) {
      longest = (int32_t) __reduce_max_sync(0xffffffffu, (unsigned) longest);
      if ((threadIdx.x & 31) == 0 && longest) atomicMax(maxLen, longest);
   }
}
void launchBuildSortWords(const uint8_t* col, const uint8_t* bytes, int elemBytes, SortValidity valid, int kind, int chunk, int64_t n, int descending, int first,
                          uint32_t* ids, unsigned long long* keys, int32_t* maxLen, int smCount, cudaStream_t s) {
   int grid = (int) std::min<int64_t>(std::max<int64_t>((n + 255) / 256, 1), (int64_t) smCount * 8);
   buildSortWordsKernel<<<grid, 256, 0, s>>>(col, bytes, elemBytes, valid, kind, chunk, n, descending, first, ids, keys, maxLen);
}
__global__ void scatterRanksKernel(const uint32_t* ids, int64_t n, int32_t* rank) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) rank[ids[i]] = (int32_t) i;
}
void launchScatterRanks(const uint32_t* ids, int64_t n, int32_t* rank, int smCount, cudaStream_t s) {
   int grid = (int) std::min<int64_t>(std::max<int64_t>((n + 255) / 256, 1), (int64_t) smCount * 8);
   scatterRanksKernel<<<grid, 256, 0, s>>>(ids, n, rank);
}
__global__ void dictLengthsKernel(const int32_t* len, int64_t n, uint32_t* offsets) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (int64_t) gridDim.x * blockDim.x) offsets[i] = i < n ? (uint32_t) len[i] : 0u;
}
// one warp per code
__global__ void dictCopyKernel(DictDev d, int64_t n, const uint32_t* offsets, uint8_t* out) {
   const int lane = threadIdx.x & 31;
   for (int64_t c = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < n; c += ((int64_t) gridDim.x * blockDim.x) >> 5) {
      const uint8_t* src = d.arena + d.entryOff[c];
      uint8_t* dst = out + offsets[c];
      for (int32_t i = lane; i < d.entryLen[c]; i += 32) dst[i] = src[i];
   }
}
void launchDictExport(const DictDev& d, int64_t n, uint32_t* offsets, uint8_t* bytes, int smCount, cudaStream_t s) {
   int grid = (int) std::min<int64_t>(std::max<int64_t>((n + 256) / 256, 1), (int64_t) smCount * 8);
   dictLengthsKernel<<<grid, 256, 0, s>>>(d.entryLen, n, offsets);
   rowScanKernel<<<1, 1024, 0, s>>>(offsets, n + 1, nullptr); // exclusive: offsets[n] = total bytes
   if (n) dictCopyKernel<<<(int) std::min<int64_t>((n + 7) / 8, (int64_t) smCount * 16), 256, 0, s>>>(d, n, offsets, bytes);
}

// ---------------------------------------------------------------- unified dictionaries (ldb_gpu_dict_unify, peer.cu)
__global__ void dictRebaseKernel(const uint32_t* src, int64_t n, uint32_t add, uint32_t* dst) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) dst[i] = src[i] + add;
}
void launchDictRebase(const uint32_t* src, int64_t n, uint32_t add, uint32_t* dst, int smCount, cudaStream_t s) {
   int grid = (int) std::min<int64_t>(std::max<int64_t>((n + 255) / 256, 1), (int64_t) smCount * 8);
   dictRebaseKernel<<<grid, 256, 0, s>>>(src, n, add, dst);
}
// sorted position i: isNew[i] = 1 when its string differs from the one at position i - 1 (position 0 always), newLen[i] = its length
// then, else 0; both get a trailing 0 at position n for the exclusive scans that follow
__global__ void dictUnionFlagsKernel(const uint32_t* offsets, const uint8_t* bytes, const uint32_t* ids, int64_t n, uint32_t* isNew, uint32_t* newLen) {
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (int64_t) gridDim.x * blockDim.x) {
      if (i == n) {
         isNew[n] = newLen[n] = 0;
         continue;
      }
      const uint32_t r = ids[i], b = offsets[r], len = offsets[r + 1] - b;
      bool fresh = i == 0;
      if (!fresh) {
         const uint32_t q = ids[i - 1], pb = offsets[q], plen = offsets[q + 1] - pb;
         fresh = plen != len;
         for (uint32_t j = 0; j < len && !fresh; j++) fresh = bytes[b + j] != bytes[pb + j];
      }
      isNew[i] = fresh ? 1u : 0u;
      newLen[i] = fresh ? len : 0u;
   }
}
void launchDictUnionRanks(const uint32_t* offsets, const uint8_t* bytes, const uint32_t* ids, int64_t n, uint32_t* codes, uint32_t* arenaOff, int smCount, cudaStream_t s) {
   int grid = (int) std::min<int64_t>(std::max<int64_t>((n + 256) / 256, 1), (int64_t) smCount * 8);
   dictUnionFlagsKernel<<<grid, 256, 0, s>>>(offsets, bytes, ids, n, codes, arenaOff);
   rowScanKernel<<<1, 1024, 0, s>>>(codes, n + 1, nullptr);
   rowScanKernel<<<1, 1024, 0, s>>>(arenaOff, n + 1, nullptr);
}
// one thread per sorted position that starts a new string: its bytes into the arena at arenaOff[i], its entry at code codes[i], and a slot
// on its probe sequence claimed and published with code + 1 in one CAS (nothing reads the dictionary during the build).  Which of two
// strings that share a probe run takes which slot depends on timing; codes, entries and arena do not.
__global__ void dictRankedBuildKernel(DictDev d, const uint32_t* offsets, const uint8_t* bytes, const uint32_t* ids, int64_t n, const uint32_t* codes,
                                      const uint32_t* arenaOff) {
   if (blockIdx.x == 0 && threadIdx.x == 0) {
      d.ctr[0] = arenaOff[n];
      d.ctr[1] = codes[n];
   }
   for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
      const uint32_t code = codes[i];
      if (codes[i + 1] == code) continue;
      const uint32_t r = ids[i], b = offsets[r];
      const int32_t len = (int32_t) (offsets[r + 1] - b);
      const uint8_t* s = bytes + b;
      const uint32_t off = arenaOff[i];
      for (int32_t j = 0; j < len; j++) d.arena[off + j] = s[j];
      d.entryOff[code] = off;
      d.entryLen[code] = len;
      const uint64_t h = strHash(s, len);
      const unsigned long long word = dictTag(h) | (unsigned long long) (code + 1);
      uint64_t slot = dictFirstSlot(h, d.mask);
      const uint64_t limit = dictProbeLimit(d.mask);
      uint64_t probes = 0;
      while (probes < limit && atomicCAS(d.slots + slot, 0ull, word) != 0ull) {
         slot = dictNextSlot(slot, d.mask);
         probes++;
      }
      if (probes == limit) dictFail(d, 1);
   }
}
void launchDictRankedBuild(const DictDev& d, const uint32_t* offsets, const uint8_t* bytes, const uint32_t* ids, int64_t n, const uint32_t* codes, const uint32_t* arenaOff,
                           int smCount, cudaStream_t s) {
   int grid = (int) std::min<int64_t>(std::max<int64_t>((n + 255) / 256, 1), (int64_t) smCount * 8);
   dictRankedBuildKernel<<<grid, 256, 0, s>>>(d, offsets, bytes, ids, n, codes, arenaOff);
}

} // namespace ldb
