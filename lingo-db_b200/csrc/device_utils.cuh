// device_utils.cuh — value-level device primitives shared by every pipeline kernel (sm_90a).
//
// These are the device twins of what the reference's JIT emits inline per tuple:
//   hash64 / hashCombine          UtilToLLVM/LowerToLLVM.cpp:493-514 (KAT: test/lit/DB/hash.mlir:27-34)
//   128-bit wrapping arithmetic   LLVM `mul/add i128` as produced by DBToStd/LowerToStd.cpp:612-700
//   decimal128 loads (trunc i64)  ArrowToStd.cpp:67-85 + LowerToStd.cpp:111-209
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ldb {

// ---------------------------------------------------------------- 128-bit two's complement, wrapping
struct i128 {
   uint64_t lo;
   int64_t hi;
};
__device__ __forceinline__ i128 make128(int64_t v) { return i128{(uint64_t) v, v >> 63}; }
__device__ __forceinline__ i128 add128(i128 a, i128 b) { // one carry chain (IADD3 / IADD3.X), no compare+select
   i128 r;
   asm("add.cc.u64 %0, %2, %4;\n\taddc.u64 %1, %3, %5;" : "=l"(r.lo), "=l"(r.hi) : "l"(a.lo), "l"(a.hi), "l"(b.lo), "l"(b.hi));
   return r;
}
__device__ __forceinline__ i128 sub128(i128 a, i128 b) {
   i128 r;
   asm("sub.cc.u64 %0, %2, %4;\n\tsubc.u64 %1, %3, %5;" : "=l"(r.lo), "=l"(r.hi) : "l"(a.lo), "l"(a.hi), "l"(b.lo), "l"(b.hi));
   return r;
}
// DateRuntime::extractYear (src/runtime/DateRuntime.cpp:99-101) on a date32 value: civil-from-days, exact for EVERY int32 day.
// days + 719468 leaves int32 for dates past the year 5 879 609, so the shift and the 400-year era are taken in 64 bits (a division by a
// constant: multiply-high, no division loop); the day of the era is below 146 097 and the rest stays 32-bit.  Every year fits int32.
__device__ __forceinline__ int32_t yearOfDays(int32_t days) {
   const int64_t z = (int64_t) days + 719468;
   const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
   const uint32_t doe = (uint32_t) (z - era * 146097);
   const uint32_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
   const uint32_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
   const uint32_t mp = (5 * doy + 2) / 153;
   return (int32_t) ((int64_t) yoe + era * 400 + (mp >= 10 ? 1 : 0));
}
__device__ __forceinline__ bool fitsI32(int64_t v) { return v == (int64_t) (int32_t) v; }
// (a * b) * c for operands that fit int32 (c additionally >= 0): three 32x32→64 multiplies instead of the
// ~25-instruction general 64x64→128 / 128x64 sequence.  Exact; callers take it only when EVERY lane of
// the warp qualifies (warp-uniform branch), otherwise the general wrapping path runs.
__device__ __forceinline__ i128 mul32x32(int32_t a, int32_t b) {
   int64_t p = (int64_t) a * (int64_t) b;
   return i128{(uint64_t) p, p >> 63};
}
__device__ __forceinline__ i128 mul64x32pos(int64_t p, int32_t c) { // p any i64, 0 <= c < 2^31
   int64_t hiPart = (int64_t) (int32_t) (p >> 32) * (int64_t) c;               // signed high half
   uint64_t loPart = (uint64_t) (uint32_t) p * (uint64_t) (uint32_t) c;         // unsigned low half
   i128 r;
   asm("add.cc.u64 %0, %2, %3;\n\taddc.u64 %1, %4, 0;" : "=l"(r.lo), "=l"(r.hi) : "l"(loPart), "l"((uint64_t) hiPart << 32), "l"((uint64_t) (hiPart >> 32)));
   return r;
}
// signed 64 × signed 64 → 128 (exact)
__device__ __forceinline__ i128 mul64x64(int64_t a, int64_t b) {
   i128 r;
   r.lo = (uint64_t) a * (uint64_t) b;
   r.hi = __mul64hi(a, b);
   return r;
}
// i128 × signed 64 → low 128 bits (wrapping, like LLVM mul i128 with a sign-extended operand)
__device__ __forceinline__ i128 mul128x64(i128 a, int64_t b) {
   i128 r;
   uint64_t ub = (uint64_t) b;
   r.lo = a.lo * ub;
   uint64_t hi = __umul64hi(a.lo, ub) + (uint64_t) a.hi * ub;
   if (b < 0) hi -= a.lo; // b's sign extension contributes a.lo * (2^64 - 1 … ) = -a.lo at bit 64
   r.hi = (int64_t) hi;
   return r;
}

// ---------------------------------------------------------------- reference hash
__device__ __forceinline__ uint64_t bswap64(uint64_t x) {
   uint32_t lo = (uint32_t) x, hi = (uint32_t) (x >> 32);
   return ((uint64_t) __byte_perm(lo, 0, 0x0123) << 32) | (uint64_t) __byte_perm(hi, 0, 0x0123);
}
__device__ __forceinline__ uint64_t hash64(uint64_t v) {
   uint64_t m = v * 11400714819323198549ull; // 0x9E3779B97F4A7C55
   return m ^ bswap64(m);
}
__device__ __forceinline__ uint64_t hashCombine(uint64_t newPiece, uint64_t total) { return newPiece ^ bswap64(total); }
__device__ __forceinline__ uint64_t hashI32(int32_t k) { return hash64((uint64_t) (int64_t) k); }

// ---------------------------------------------------------------- streaming loads (read-once column data)
__device__ __forceinline__ int32_t ldStream32(const int32_t* p) {
   int32_t v;
   asm("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(v) : "l"(p));
   return v;
}
__device__ __forceinline__ int64_t ldStream64(const int64_t* p) {
   int64_t v;
   asm("ld.global.nc.L1::no_allocate.s64 %0, [%1];" : "=l"(v) : "l"(p));
   return v;
}

// ---------------------------------------------------------------- TMA bulk copies (cp.async.bulk → SASS UBLKCP) + mbarrier
__device__ __forceinline__ uint32_t smemAddr(const void* p) { return (uint32_t) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbarInit(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smemAddr(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbarInitFence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbarExpectTx(uint64_t* bar, uint32_t bytes) {
   asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smemAddr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbarArrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smemAddr(bar)) : "memory"); }
__device__ __forceinline__ void mbarWait(uint64_t* bar, uint32_t parity) {
   asm volatile(
      "{\n\t.reg .pred p;\n"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n"
      "DONE_%=:\n\t}" ::"r"(smemAddr(bar)),
      "r"(parity)
      : "memory");
}
// the same wait with a pause between polls: a thread that is expected to wait long (the producer lane behind the slowest consumer
// warp) otherwise spends issue slots on try_wait/branch that the compute warps of the SM need (in K4/K5 a
// sizeable share of the issued instructions were poll loops).  sleepNs == 0: plain polling.
__device__ __forceinline__ void mbarWaitPaused(uint64_t* bar, uint32_t parity, uint32_t sleepNs) {
   const uint32_t addr = smemAddr(bar);
   while (true) {
      uint32_t done;
      asm volatile(
         "{\n\t.reg .pred p;\n\t"
         "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
         "selp.u32 %0, 1, 0, p;\n\t}"
         : "=r"(done)
         : "r"(addr), "r"(parity)
         : "memory");
      if (done) return;
      if (sleepNs) __nanosleep(sleepNs);
   }
}
// global → shared bulk copy, completion counted in bytes on `bar`; src/dst 16-B aligned, bytes % 16 == 0
// Column data is read exactly once: L2 evict_first keeps the 50 MB L2 for the hash-table directories and bloom filters.
__device__ __forceinline__ uint64_t evictFirstPolicy() {
   uint64_t pol;
   asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
   return pol;
}
__device__ __forceinline__ void bulkLoad(uint32_t dstSmem, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
   asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dstSmem), "l"(src), "r"(bytes),
                "r"(smemAddr(bar)), "l"(policy)
                : "memory");
}
__device__ __forceinline__ int32_t ldShared32(uint32_t addr) {
   int32_t v;
   asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(addr));
   return v;
}
__device__ __forceinline__ int64_t ldShared64(uint32_t addr) {
   int64_t v;
   asm volatile("ld.shared.s64 %0, [%1];" : "=l"(v) : "r"(addr));
   return v;
}
__device__ __forceinline__ void ldShared64x2(uint32_t addr, int64_t& a, int64_t& b) { // addr 16-byte aligned
   asm volatile("ld.shared.v2.s64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "r"(addr));
}
__device__ __forceinline__ void ldShared32x2(uint32_t addr, uint32_t& a, uint32_t& b) { // addr 8-byte aligned
   asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(a), "=r"(b) : "r"(addr));
}
// ---------------------------------------------------------------- blocked Bloom filter of the join tables
// Three bit positions inside the 32-bit filter word that (h >> 32) selects, from a second multiply of the hash.  (Deriving them from the
// low hash word with one 32-bit multiply saves four instructions per probe but raised the false-positive rate enough to slow K9
// down and gained nothing on K4/K5, which wait on the filter word, not on the ALU.)
__device__ __forceinline__ uint32_t bloomBits(uint64_t h) {
   const uint64_t g = h * 0xD6E8FEB86659FD93ull;
   return (1u << (g >> 59)) | (1u << ((g >> 54) & 31)) | (1u << ((g >> 49) & 31));
}

// ---------------------------------------------------------------- filters
// op mask: bit0 = accept a<b, bit1 = accept a==b, bit2 = accept a>b  (built on the host from LdbFilterOp)
__device__ __forceinline__ bool cmpMask(int64_t a, int64_t b, uint32_t mask) {
   uint32_t rel = a < b ? 1u : (a == b ? 2u : 4u);
   return (rel & mask) != 0;
}

// ---------------------------------------------------------------- warp / block reductions
__device__ __forceinline__ uint64_t shflXor64(uint64_t v, int m) {
   uint32_t lo = __shfl_xor_sync(0xffffffffu, (uint32_t) v, m);
   uint32_t hi = __shfl_xor_sync(0xffffffffu, (uint32_t) (v >> 32), m);
   return ((uint64_t) hi << 32) | lo;
}
__device__ __forceinline__ uint64_t warpSum64(uint64_t v) { // wrapping
#pragma unroll
   for (int m = 16; m > 0; m >>= 1) v += shflXor64(v, m);
   return v;
}
// exact 128-bit warp sum: the low word is split into two 32-bit limbs so that lane sums cannot lose carries
__device__ __forceinline__ i128 warpSum128(i128 v) {
   uint64_t s0 = warpSum64(v.lo & 0xffffffffull);
   uint64_t s1 = warpSum64(v.lo >> 32);
   uint64_t sh = warpSum64((uint64_t) v.hi);
   i128 r;
   uint64_t mid = s1 + (s0 >> 32); // < 2^38
   r.lo = (s0 & 0xffffffffull) | (mid << 32);
   r.hi = (int64_t) (sh + (mid >> 32));
   return r;
}
// 128-bit atomic add as two 64-bit atomics with carry: commutative, exact mod 2^128 once all adds landed
__device__ __forceinline__ void atomicAdd128(unsigned long long* lo, unsigned long long* hi, i128 v) {
   unsigned long long old = atomicAdd(lo, (unsigned long long) v.lo);
   unsigned long long carry = (old + v.lo) < old ? 1ull : 0ull;
   unsigned long long h = (unsigned long long) v.hi + carry;
   if (h != 0) atomicAdd(hi, h);
}

} // namespace ldb
