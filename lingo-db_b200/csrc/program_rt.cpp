// program_rt.cpp — host side of the generic program pipeline (include/ldb_gpu.h "program pipelines"): validates a program,
// binds it batch by batch and launches the interpreter kernel; hash-aggregation states, their read-back / export as a table,
// ORDER BY … LIMIT through the device radix sort.
#include "context.h"
#include "program.h"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <deque>

using namespace ldb;

namespace {
bool isCountKind(int k) { return k == LDB_AGG_COUNT || k == LDB_AGG_COUNT_STAR; }
} // namespace

LdbTable* ldb::addResultTable(LdbContext* ctx, std::string name, std::vector<LdbColumn> columns, LdbBatch b, Scratch& buffers) {
   auto* t = new LdbTable;
   t->ctx = ctx;
   t->name = std::move(name);
   t->columns = std::move(columns);
   t->numRows = b.nRows;
   b.validity.assign(b.data.size(), nullptr);
   b.validityBitOffset.assign(b.data.size(), 0);
   b.owned = buffers.take();
   t->batches.push_back(std::move(b));
   ctx->tables.push_back(t);
   return t;
}

extern "C" {

int ldb_gpu_hashagg_create(LdbContext* ctx, int32_t n_keys, int32_t n_aggs, const LdbProgAgg* aggs, int64_t expected_groups, LdbState** out, LdbError* err) {
   return guarded(err, [&] {
      if (!ctx || !out || (n_aggs > 0 && !aggs)) fail(LDB_ERR_INVALID, "null argument");
      if (n_keys < 0 || n_keys > kProgMaxKeys || n_aggs < 0 || n_aggs > kProgMaxAggs) fail(LDB_ERR_INVALID, "hash aggregation takes 0..4 keys and 0..8 aggregates");
      for (int a = 0; a < n_aggs; a++)
         if (aggs[a].kind < LDB_AGG_SUM || aggs[a].kind > LDB_AGG_ANY) fail(LDB_ERR_INVALID, "unknown aggregate kind");
      LDB_CUDA(cudaSetDevice(ctx->device));
      auto* s = new LdbState;
      s->ctx = ctx;
      s->kind = LDB_STATE_HASHAGG;
      ctx->states.push_back(s);
      auto& h = s->hashagg;
      h.nKeys = n_keys;
      h.nAggs = n_aggs;
      h.entryBytes = (uint32_t) (48 + 16 * n_aggs);
      const uint64_t cap = n_keys == 0 ? 1 : nextPow2((uint64_t) std::max<int64_t>(expected_groups, 8) * 2);
      h.mask = cap - 1;
      h.base = (uint8_t*) ctx->stagingAlloc(cap * h.entryBytes);
      s->allocations.push_back(h.base);
      ctx->launch("hashagg_init", [&] { launchHashAggInit(h, ctx->smCount, ctx->compute); });
      uint8_t* small = (uint8_t*) ctx->stagingAlloc(256);
      s->allocations.push_back(small);
      LDB_CUDA(cudaMemsetAsync(small, 0, 256, ctx->compute));
      h.count = (unsigned long long*) small;
      h.error = (int32_t*) (small + 8);
      for (int a = 0; a < n_aggs; a++) s->aggKinds[a] = aggs[a].kind;
      if (n_keys == 0) { // the one group exists from the start, with the aggregates' identities
         std::vector<uint8_t> e(h.entryBytes, 0);
         *(uint32_t*) e.data() = 2;
         unsigned long long* ea = (unsigned long long*) (e.data() + 48);
         for (int a = 0; a < n_aggs; a++) {
            switch (aggs[a].kind) {
               case LDB_AGG_MIN: // INT128_MAX
                  ea[2 * a] = ~0ull;
                  ea[2 * a + 1] = ~0ull >> 1;
                  break;
               case LDB_AGG_MAX: ea[2 * a + 1] = 1ull << 63; break; // INT128_MIN
               case LDB_AGG_MIN_F64:
               case LDB_AGG_MAX_F64: ea[2 * a] = kF64MinMaxIdentity; break;
               default: break;
            }
         }
         LDB_CUDA(cudaMemcpyAsync(h.base, e.data(), e.size(), cudaMemcpyHostToDevice, ctx->compute));
         unsigned long long one = 1;
         LDB_CUDA(cudaMemcpyAsync(h.count, &one, 8, cudaMemcpyHostToDevice, ctx->compute));
         ctx->syncStream(ctx->compute); // the host buffers above are locals
      }
      *out = s;
   });
}
static void checkHashAgg(LdbState* s) {
   if (!s || s->kind != LDB_STATE_HASHAGG) fail(LDB_ERR_INVALID, "not a hash aggregation state");
}
int ldb_gpu_hashagg_count(LdbState* s, int64_t* n_groups, LdbError* err) {
   return guarded(err, [&] {
      checkHashAgg(s);
      unsigned long long h[2] = {0, 0};
      LDB_CUDA(cudaMemcpyAsync(h, s->hashagg.count, 16, cudaMemcpyDeviceToHost, s->ctx->compute));
      s->ctx->syncStream(s->ctx->compute);
      if ((int32_t) h[1]) fail(LDB_ERR_CAPACITY, "hash aggregation table full: more groups than expected_groups allowed");
      *n_groups = (int64_t) h[0];
   });
}

// export into fresh device columns, allocated in `cols`; returns the row count (synchronises before the export, not after)
struct ExportedGroups {
   int64_t n = 0;
   std::vector<int64_t*> keyCols;
   std::vector<uint8_t*> keyValid, aggCols, aggValid;
};
static ExportedGroups exportGroups(LdbState* s, Scratch& cols) {
   LdbContext* ctx = s->ctx;
   auto& h = s->hashagg;
   int64_t n = 0;
   LdbError e;
   if (ldb_gpu_hashagg_count(s, &n, &e) != LDB_OK) fail(e.code, e.message);
   ExportedGroups g;
   g.n = n;
   const size_t rows = (size_t) std::max<int64_t>(n, 1);
   for (int k = 0; k < h.nKeys; k++) {
      g.keyCols.push_back(cols.alloc<int64_t>(rows * 8));
      g.keyValid.push_back(cols.alloc<uint8_t>(rows));
   }
   uint32_t countMask = 0;
   for (int a = 0; a < h.nAggs; a++) {
      g.aggCols.push_back(cols.alloc<uint8_t>(rows * 16));
      g.aggValid.push_back(cols.alloc<uint8_t>(rows));
      if (isCountKind(s->aggKinds[a])) countMask |= 1u << a;
   }
   unsigned long long* counter = cols.alloc<unsigned long long>(8);
   LDB_CUDA(cudaMemsetAsync(counter, 0, 8, ctx->compute));
   ctx->launch("hashagg_export", [&] { launchHashAggExport(h, g.keyCols.data(), g.keyValid.data(), g.aggCols.data(), g.aggValid.data(), counter, countMask, ctx->smCount, ctx->compute); });
   return g;
}
int ldb_gpu_hashagg_read(LdbState* s, LdbHashAggRow* rows, int64_t max_rows, int64_t* n_rows, LdbError* err) {
   return guarded(err, [&] {
      checkHashAgg(s);
      if (!rows || !n_rows) fail(LDB_ERR_INVALID, "null argument");
      LdbContext* ctx = s->ctx;
      LDB_CUDA(cudaSetDevice(ctx->device));
      Scratch cols(ctx);
      ExportedGroups g = exportGroups(s, cols);
      auto& h = s->hashagg;
      const int64_t n = std::min(g.n, max_rows);
      std::vector<std::vector<int64_t>> keys(h.nKeys, std::vector<int64_t>((size_t) n));
      std::vector<std::vector<uint8_t>> kv(h.nKeys, std::vector<uint8_t>((size_t) n)), av(h.nAggs, std::vector<uint8_t>((size_t) n));
      std::vector<std::vector<LdbI128>> aggs(h.nAggs, std::vector<LdbI128>((size_t) n));
      for (int k = 0; k < h.nKeys && n; k++) {
         LDB_CUDA(cudaMemcpyAsync(keys[k].data(), g.keyCols[k], (size_t) n * 8, cudaMemcpyDeviceToHost, ctx->compute));
         LDB_CUDA(cudaMemcpyAsync(kv[k].data(), g.keyValid[k], (size_t) n, cudaMemcpyDeviceToHost, ctx->compute));
      }
      for (int a = 0; a < h.nAggs && n; a++) {
         LDB_CUDA(cudaMemcpyAsync(aggs[a].data(), g.aggCols[a], (size_t) n * 16, cudaMemcpyDeviceToHost, ctx->compute));
         LDB_CUDA(cudaMemcpyAsync(av[a].data(), g.aggValid[a], (size_t) n, cudaMemcpyDeviceToHost, ctx->compute));
      }
      ctx->syncStream(ctx->compute);
      for (int64_t i = 0; i < n; i++) {
         LdbHashAggRow& r = rows[i];
         memset(&r, 0, sizeof(r));
         for (int k = 0; k < h.nKeys; k++) {
            r.keys[k] = keys[k][(size_t) i];
            if (!kv[k][(size_t) i]) r.key_null_mask |= 1u << k;
         }
         for (int a = 0; a < h.nAggs; a++) {
            r.aggs[a] = aggs[a][(size_t) i];
            if (av[a][(size_t) i]) r.agg_valid_mask |= 1u << a;
         }
      }
      *n_rows = g.n;
   });
}
int ldb_gpu_hashagg_to_table(LdbState* s, const char* name, LdbTable** out, LdbError* err) {
   return guarded(err, [&] {
      checkHashAgg(s);
      if (!out) fail(LDB_ERR_INVALID, "null argument");
      LdbContext* ctx = s->ctx;
      LDB_CUDA(cudaSetDevice(ctx->device));
      Scratch cols(ctx);
      ExportedGroups g = exportGroups(s, cols);
      ctx->syncStream(ctx->compute);
      auto& h = s->hashagg;
      std::vector<LdbColumn> columns;
      LdbBatch b;
      b.nRows = g.n;
      for (int k = 0; k < h.nKeys; k++) {
         columns.push_back({"k" + std::to_string(k), LDB_INT64, 0, 0});
         b.data.push_back(g.keyCols[k]);
         b.bytes.push_back(nullptr);
         b.elemBytes.push_back(8);
         b.validBytes.push_back(g.keyValid[k]);
      }
      for (int a = 0; a < h.nAggs; a++) {
         const int kind = s->aggKinds[a];
         const bool f64 = kind == LDB_AGG_SUM_F64 || kind == LDB_AGG_MIN_F64 || kind == LDB_AGG_MAX_F64;
         columns.push_back({"a" + std::to_string(a), f64 ? LDB_FLOAT64 : LDB_DECIMAL128, 38, 0});
         b.data.push_back(g.aggCols[a]);
         b.bytes.push_back(nullptr);
         b.elemBytes.push_back(16); // doubles keep the 16-byte stride (bits in the low 8 bytes)
         b.validBytes.push_back(g.aggValid[a]);
      }
      *out = addResultTable(ctx, name ? name : "groups", std::move(columns), std::move(b), cols);
   });
}

static_assert(sizeof(ProgramParams) <= 4096, "ProgramParams exceeds the 4 KB kernel-parameter limit");

} // extern "C"

// ---------------------------------------------------------------- string dictionaries
static void checkDict(LdbState* s) {
   if (!s || s->kind != LDB_STATE_DICT) fail(LDB_ERR_INVALID, "not a string dictionary");
}
std::pair<int64_t, int64_t> ldb_gpu_dict_counters_internal(LdbState* s) {
   unsigned long long c[3] = {0, 0, 0};
   LDB_CUDA(cudaMemcpyAsync(c, s->dict.ctr, sizeof(c), cudaMemcpyDeviceToHost, s->ctx->compute));
   s->ctx->syncStream(s->ctx->compute);
   switch ((uint32_t) c[2]) {
      case 0: break;
      case 1: fail(LDB_ERR_CAPACITY, "string dictionary full: more distinct strings than expected_strings allowed (recreate it larger)");
      case 2: fail(LDB_ERR_CAPACITY, "string dictionary arena full: more string bytes than expected_bytes allowed (recreate it larger)");
      case 3: fail(LDB_ERR_CAPACITY, "string dictionary: a code would pass INT32_MAX");
      default: fail(LDB_ERR_CAPACITY, "string dictionary error word " + std::to_string((uint32_t) c[2]));
   }
   return {(int64_t) c[0], (int64_t) c[1]};
}

// row ids of the single-batch table `t` (n rows, n < 2^32) ordered by the keys (column index, descending): a device buffer of n
// uint32 in `scratch`, like the sort's temporaries, so the caller waits for the sort before its scope ends.  The one place that
// knows the string order: ORDER BY, dictionary ranks and unified dictionaries.
uint32_t* ldb::sortRows(Scratch& scratch, LdbTable* t, const std::vector<std::pair<int, int>>& keys, int64_t n) {
   LdbContext* ctx = t->ctx;
   LdbBatch& b = t->batches[0];
   const size_t rows = (size_t) std::max<int64_t>(n, 1);
   uint32_t* dv = scratch.alloc<uint32_t>(rows * 4);
   if (n == 0) return dv;
   unsigned long long* dk = scratch.alloc<unsigned long long>(rows * 8);
   unsigned long long* dk2 = scratch.alloc<unsigned long long>(rows * 8);
   uint32_t* dv2 = scratch.alloc<uint32_t>(rows * 4);
   unsigned int* hist = scratch.alloc<unsigned int>((size_t) ((n + 4095) / 4096) * 256 * 4);
   int32_t* maxLen = scratch.alloc<int32_t>(16);
   int first = 1;
   SortValidity valid{};
   auto pass = [&](int c, int kind, int chunk, int desc) {
      const int digits = kind == 3 ? 1 : 8; // the NULL flag is the lowest digit
      ctx->launch("radix_sort", [&] {
         launchBuildSortWords((const uint8_t*) b.data[c], (const uint8_t*) b.bytes[c], b.elemBytes[c], valid, kind, chunk, n, desc, first, dv, dk, maxLen, ctx->smCount, ctx->compute);
         launchRadixSortPairs(dk, dv, dk2, dv2, n, hist, ctx->smCount, ctx->compute, digits);
      });
      if (digits % 2) {
         std::swap(dk, dk2);
         std::swap(dv, dv2);
      }
      first = 0;
   };
   for (size_t k = keys.size(); k-- > 0;) {
      const int c = keys[k].first, desc = keys[k].second;
      valid.bytes = c < (int) b.validBytes.size() ? b.validBytes[c] : nullptr;
      valid.bitmap = c < (int) b.validity.size() && !valid.bytes ? (const uint8_t*) b.validity[c] : nullptr;
      valid.bitOffset = valid.bitmap ? b.validityBitOffset[c] : 0;
      if (t->columns[c].type != LDB_UTF8) {
         if (b.elemBytes[c] == 16) pass(c, 0, 0, desc); // an i128 cell: its low word first, then the high word
         pass(c, 0, b.elemBytes[c] == 16 ? 1 : 0, desc);
      } else {
         int32_t longest = 0;
         LDB_CUDA(cudaMemsetAsync(maxLen, 0, 4, ctx->compute));
         pass(c, 1, 0, desc); // lengths: the least significant word of a string
         LDB_CUDA(cudaMemcpyAsync(&longest, maxLen, 4, cudaMemcpyDeviceToHost, ctx->compute));
         ctx->syncStream(ctx->compute);
         for (int chunk = (longest + 7) / 8; chunk-- > 0;) pass(c, 2, chunk, desc);
      }
      if (valid.bytes || valid.bitmap) pass(c, 3, 0, desc); // NULL last (ASC) / first (DESC), NULLs tied
   }
   return dv;
}

LdbState* ldb_gpu_dict_new_internal(LdbContext* ctx, int64_t expected_strings, int64_t expected_bytes) {
   auto* s = new LdbState;
   s->ctx = ctx;
   s->kind = LDB_STATE_DICT;
   ctx->states.push_back(s);
   auto alloc = [&](size_t bytes) {
      void* p = ctx->stagingAlloc(std::max<size_t>(bytes, 16));
      s->allocations.push_back(p);
      return p;
   };
   DictDev& dd = s->dict;
   const uint64_t cap = nextPow2((uint64_t) std::max<int64_t>(expected_strings, 8) * 2);
   dd.mask = cap - 1;
   dd.slots = (unsigned long long*) alloc(cap * 8);
   dd.entryOff = (int64_t*) alloc(cap * 8);
   dd.entryLen = (int32_t*) alloc(cap * 4);
   dd.arenaCap = std::max<int64_t>(expected_bytes, 1);
   dd.arena = (uint8_t*) alloc((size_t) dd.arenaCap);
   dd.ctr = (unsigned long long*) alloc(32);
   dd.codeCap = std::min<int64_t>((int64_t) cap, (int64_t) INT32_MAX + 1);
   LDB_CUDA(cudaMemsetAsync(dd.slots, 0, cap * 8, ctx->compute));
   LDB_CUDA(cudaMemsetAsync(dd.ctr, 0, 32, ctx->compute));
   return s;
}

extern "C" {

int ldb_gpu_dict_create(LdbContext* ctx, int64_t expected_strings, int64_t expected_bytes, LdbState** out, LdbError* err) {
   return guarded(err, [&] {
      if (!ctx || !out) fail(LDB_ERR_INVALID, "null argument");
      if (expected_strings < 0 || expected_bytes < 0) fail(LDB_ERR_INVALID, "negative dictionary size");
      if (expected_strings > kDictMaxStrings) fail(LDB_ERR_UNSUPPORTED, "a dictionary holds at most 2^30 expected strings (codes are int32)");
      LDB_CUDA(cudaSetDevice(ctx->device));
      *out = ldb_gpu_dict_new_internal(ctx, expected_strings, expected_bytes);
   });
}
int ldb_gpu_dict_count(LdbState* s, int64_t* n_strings, LdbError* err) {
   return guarded(err, [&] {
      checkDict(s);
      if (!n_strings) fail(LDB_ERR_INVALID, "null argument");
      LDB_CUDA(cudaSetDevice(s->ctx->device));
      *n_strings = ldb_gpu_dict_counters_internal(s).second;
   });
}
int ldb_gpu_dict_to_table(LdbState* s, const char* name, LdbTable** out, LdbError* err) {
   return guarded(err, [&] {
      checkDict(s);
      if (!out) fail(LDB_ERR_INVALID, "null argument");
      LdbContext* ctx = s->ctx;
      LDB_CUDA(cudaSetDevice(ctx->device));
      const std::pair<int64_t, int64_t> used = ldb_gpu_dict_counters_internal(s);
      const int64_t bytes = used.first, n = used.second;
      if (bytes > (int64_t) INT32_MAX) fail(LDB_ERR_UNSUPPORTED, "dictionary strings exceed 2^31 - 1 bytes (utf8 offsets are int32)");
      Scratch cols(ctx), scratch(ctx);
      uint32_t* offsets = cols.alloc<uint32_t>((size_t) (n + 1) * 4);
      uint8_t* data = cols.alloc<uint8_t>((size_t) std::max<int64_t>(bytes, 1));
      int32_t* rank = cols.alloc<int32_t>((size_t) std::max<int64_t>(n, 1) * 4);
      ctx->launch("dict_export", [&] { launchDictExport(s->dict, n, offsets, data, ctx->smCount, ctx->compute); });
      LdbBatch b;
      b.nRows = n;
      b.data = {offsets, rank};
      b.bytes = {data, nullptr};
      b.elemBytes = {4, 4};
      LdbTable* t = addResultTable(ctx, name ? name : "dictionary", {{"str", LDB_UTF8, 0, 0}, {"rank", LDB_INT32, 0, 0}}, std::move(b), cols);
      uint32_t* ids = sortRows(scratch, t, {{0, 0}}, n);
      if (n) ctx->launch("dict_rank", [&] { launchScatterRanks(ids, n, rank, ctx->smCount, ctx->compute); });
      ctx->syncStream(ctx->compute);
      *out = t;
   });
}

// ---------------------------------------------------------------- key-tuple join tables
int ldb_gpu_join_table_create_keys(LdbContext* ctx, int32_t n_keys, int64_t expected_rows, int32_t flags, LdbState** out, LdbError* err) {
   return guarded(err, [&] {
      int devices = 0;
      if (cudaGetDeviceCount(&devices) != cudaSuccess || devices == 0) {
         cudaGetLastError();
         fail(LDB_ERR_NO_DEVICE, "no CUDA device available: the GPU operator runtime has no CPU fallback");
      }
      if (!ctx || !out) fail(LDB_ERR_INVALID, "null argument");
      if (n_keys < 1 || n_keys > kProgMaxKeys) fail(LDB_ERR_INVALID, "a key-tuple join table takes 1..4 keys");
      if (expected_rows < 0) fail(LDB_ERR_INVALID, "negative expected_rows");
      if (expected_rows > ((int64_t) 1 << 36)) fail(LDB_ERR_UNSUPPORTED, "a key-tuple join table holds at most 2^36 expected rows");
      if (ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "key-tuple join tables are not part of captured queries");
      LDB_CUDA(cudaSetDevice(ctx->device));
      auto* s = new LdbState;
      s->ctx = ctx;
      s->kind = LDB_STATE_KEY_JOIN;
      ctx->states.push_back(s);
      auto alloc = [&](size_t bytes) {
         void* p = ctx->stagingAlloc(std::max<size_t>(bytes, 16));
         s->allocations.push_back(p);
         LDB_CUDA(cudaMemsetAsync(p, 0, std::max<size_t>(bytes, 16), ctx->compute));
         return p;
      };
      KeyJoinDev& k = s->keyJoin;
      const uint64_t cap = nextPow2((uint64_t) std::max<int64_t>(expected_rows, 8) * 2); // load <= 0.5, like the other join tables
      k.mask = cap - 1;
      k.nKeys = n_keys;
      k.entryBytes = n_keys <= 2 ? 32 : 48; // {word, payload, keys} padded: one 32-byte sector for 1-2 keys
      k.unique = (flags & LDB_JOIN_UNIQUE) ? 1 : 0;
      k.base = (uint8_t*) alloc(cap * k.entryBytes);
      uint8_t* small = (uint8_t*) alloc(16);
      k.count = (unsigned long long*) small;
      k.error = (int32_t*) (small + 8);
      if (cap >= 4096 && !(flags & LDB_JOIN_NO_BLOOM)) { // the plain tables' filter: 8 bits per directory slot
         const uint64_t words = cap / 4;
         k.bloom = (uint32_t*) alloc(words * 4);
         k.bloomMask = (uint32_t) (words - 1);
      }
      *out = s;
   });
}
} // extern "C"
void ldb_gpu_check_keyjoin_error_internal(LdbState* s) {
   int32_t e = 0;
   LDB_CUDA(cudaMemcpyAsync(&e, s->keyJoin.error, sizeof(e), cudaMemcpyDeviceToHost, s->ctx->compute));
   s->ctx->syncStream(s->ctx->compute);
   switch (e) {
      case 0: return;
      case 1: fail(LDB_ERR_CAPACITY, "key-tuple join table full: more build rows than expected_rows allowed, or more than 65536 entries in one probe run (too many duplicates of one key tuple)");
      case 6: fail(LDB_ERR_CAPACITY, "a probe run of a key-tuple join table is longer than the interpreter's bound of 16384 slots (too many entries share one run)");
      case 7: fail(LDB_ERR_UNSUPPORTED, "a program join build met a key or payload outside int64 (key-tuple join tables store int64 keys and payloads)");
      default: fail(LDB_ERR_INVALID, "key-tuple join table error word " + std::to_string(e));
   }
}

void ldb::bindColumn(ProgCol& pc, const LdbBatch& b, int ci) {
   pc.data = (const uint8_t*) b.data[ci];
   pc.bytes = (const uint8_t*) b.bytes[ci];
   pc.elemBytes = b.elemBytes[ci];
   pc.validity = ci < (int) b.validity.size() ? (const uint8_t*) b.validity[ci] : nullptr;
   pc.bitOffset = ci < (int) b.validityBitOffset.size() ? b.validityBitOffset[ci] : 0;
   pc.validBytes = ci < (int) b.validBytes.size() ? b.validBytes[ci] : nullptr;
}

// One run of a program over the batches of its source, filled step by step by runProgram: the kernel parameters every batch
// shares, where each column comes from, and the states whose error words are read after the launches.
struct ProgramPlan {
   LdbContext* ctx;
   const LdbProgramDesc* d;
   LdbTable* t; // the source
   int nCols = 0;
   ProgramParams base{};
   std::vector<int> colIdx, rowReg;  // per column: its index in its table; the row register of a side column (-1: a source column)
   std::vector<LdbTable*> colTable;
   bool written[kProgMaxRegs] = {}; // registers some instruction writes
   bool usesRowid = false;
   int eachTable = -1; // tables[] index PROBE_EACH reads
   bool probed[kProgMaxTables] = {}, coded[kProgMaxTables] = {}; // tables[k] read by PROBE / PROBE_EACH, by STRCODE
   bool inserted[kProgMaxTables] = {};                           // tables[k] inserted into by STRCODE b = 1
   bool marked[kProgMaxTables] = {};                             // tables[k] marked by MARK
   bool existed[kProgMaxTables] = {};                            // tables[k] read by EXISTS
   // registers written inside an EXISTS block that has ended (they hold whatever its last match left), and the dst registers of ended
   // EXISTS (a verdict there, not a row); a later write outside a block clears both
   bool blockOnly[kProgMaxRegs] = {}, verdict[kProgMaxRegs] = {};
   std::vector<LdbState*> dicts, tupleTables; // tupleTables: key-tuple tables whose error word the run may set

   ProgramPlan(LdbContext* c, const LdbProgramDesc* desc) : ctx(c), d(desc), t(desc->source) {}
   int colType(int c) const { return colTable[c]->columns[colIdx[c]].type; }
   void wantReg(int r, const char* what) const {
      if (r < 0 || r >= kProgMaxRegs || !written[r]) fail(LDB_ERR_INVALID, std::string("program reads an unwritten or out-of-range register (") + what + ")");
      if (blockOnly[r]) fail(LDB_ERR_INVALID, std::string("a register written inside an EXISTS block is read after the block (") + what + ")");
   }
   void wantTupleTable(LdbState* js) const {
      if (js->ctx != ctx) fail(LDB_ERR_INVALID, "key-tuple join table belongs to another context");
      if (ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "key-tuple join tables are not part of captured queries");
   }
};

// the source's and the side tables' columns by name, and the interpreter's limits
static void resolveColumns(ProgramPlan& p, const LdbProgramJoins* j) {
   LdbContext* ctx = p.ctx;
   const LdbProgramDesc* d = p.d;
   if (p.t->ctx != ctx) fail(LDB_ERR_INVALID, "table belongs to another context");
   if (j && (j->n_side_tables < 0 || j->n_side_columns < 0 || (j->n_side_tables > 0 && !j->side_tables) || (j->n_side_columns > 0 && !j->side_columns)))
      fail(LDB_ERR_INVALID, "malformed side-table list");
   const int nSide = j ? j->n_side_columns : 0;
   if (d->n_columns < 0 || d->n_columns + nSide > kProgMaxCols || d->n_instr < 0 || d->n_instr > kProgMaxInstr || d->n_consts < 0 || d->n_consts > kProgMaxConsts ||
       d->n_strings < 0 || d->n_strings > kProgMaxStrings || d->n_tables < 0 || d->n_tables > kProgMaxTables)
      fail(LDB_ERR_UNSUPPORTED, "program exceeds the interpreter's limits (12 source + side columns, 96 instructions, 24 constants, 12 strings, 4 tables)");
   LDB_CUDA(cudaSetDevice(ctx->device));
   p.nCols = d->n_columns + nSide;
   p.base.nCols = p.nCols;
   p.base.nInstr = d->n_instr;
   p.base.nTables = d->n_tables;
   p.base.eachPc = -1;
   p.colIdx.assign((size_t) p.nCols, 0);
   p.rowReg.assign((size_t) p.nCols, -1);
   p.colTable.assign((size_t) p.nCols, p.t);
   for (int c = 0; c < d->n_columns; c++) {
      p.colIdx[c] = p.t->colIndex(d->columns[c]);
      if (p.colIdx[c] < 0) fail(LDB_ERR_INVALID, std::string("unknown column ") + (d->columns[c] ? d->columns[c] : "(null)"));
   }
   for (int k = 0; k < nSide; k++) {
      const LdbSideColumn& sc = j->side_columns[k];
      const int c = d->n_columns + k;
      if (sc.table < 0 || sc.table >= j->n_side_tables || !j->side_tables[sc.table]) fail(LDB_ERR_INVALID, "side column: side table index out of range");
      LdbTable* st = j->side_tables[sc.table];
      if (st->ctx != ctx) fail(LDB_ERR_INVALID, "side table belongs to another context");
      p.colIdx[c] = st->colIndex(sc.column);
      if (p.colIdx[c] < 0) fail(LDB_ERR_INVALID, std::string("unknown side column ") + (sc.column ? sc.column : "(null)"));
      if (sc.row_reg < 0 || sc.row_reg >= kProgMaxRegs) fail(LDB_ERR_INVALID, "side column: row register out of range");
      p.colTable[c] = st;
      p.rowReg[c] = sc.row_reg;
   }
}

// static validation: every register read was written before, every index is in range, types fit the opcode; copies the
// instructions, constants and string constants into the kernel parameters
static void validateInstructions(ProgramPlan& p) {
   const LdbProgramDesc* d = p.d;
   ProgramParams& base = p.base;
   bool beforeEach[kProgMaxRegs] = {};
   // EXISTS: the last instruction of the block being read (-1: none), the EXISTS's dst, the registers written before it and inside it
   int exEnd = -1, exDst = 0;
   bool beforeExists[kProgMaxRegs] = {}, inBlock[kProgMaxRegs] = {};
   bool probedInBlock[kProgMaxTables] = {}; // tables[k] probed inside an EXISTS block (which also runs for keys without a match)
   auto wantCol = [&](int c, const char* what) {
      if (c < 0 || c >= p.nCols) fail(LDB_ERR_INVALID, std::string(what) + ": column index out of range");
      if (p.rowReg[c] >= 0) p.wantReg(p.rowReg[c], "row register of a side column");
      if (p.rowReg[c] >= 0 && p.verdict[p.rowReg[c]]) fail(LDB_ERR_INVALID, "a side column reads an EXISTS result as its row after the EXISTS block (it holds the verdict there)");
   };
   if (d->n_tables > 0 && !d->tables) fail(LDB_ERR_INVALID, "null tables list");
   int tupleKeys[kProgMaxTables] = {}; // tables[k] is a key-tuple join table of this many keys: PROBE reads registers a .. a + n - 1
   for (int k = 0; k < d->n_tables; k++)
      if (d->tables[k] && d->tables[k]->kind == LDB_STATE_KEY_JOIN) tupleKeys[k] = d->tables[k]->keyJoin.nKeys;
   auto wantKeys = [&](const LdbInstr& in) {
      for (int k = 0; k < std::max(tupleKeys[in.arg], 1); k++) p.wantReg(in.a + k, "key");
   };
   for (int i = 0; i < d->n_instr; i++) {
      const LdbInstr& in = d->instr[i];
      if (in.dst >= kProgMaxRegs) fail(LDB_ERR_INVALID, "destination register out of range");
      if (exEnd >= 0) { // inside an EXISTS block: it re-runs per match and must end at its last instruction
         if (in.op == LDB_OP_EXISTS) fail(LDB_ERR_INVALID, "EXISTS blocks do not nest (an EXISTS inside another EXISTS's block)");
         if (in.op == LDB_OP_PROBE_EACH || in.op == LDB_OP_MARK || (in.op == LDB_OP_STRCODE && in.b == 1))
            fail(LDB_ERR_INVALID, "an EXISTS block may not contain PROBE_EACH, MARK or an inserting STRCODE (it runs once per match)");
      }
      switch (in.op) {
         case LDB_OP_LOAD:
            wantCol(in.arg, "LOAD");
            if (p.colType(in.arg) == LDB_UTF8) fail(LDB_ERR_UNSUPPORTED, "LOAD of a string column (strings are operands of STRCMP / STRLIKE / STRKEY8 / STRCODE only)");
            break;
         case LDB_OP_STRCODE:
            if (in.a >= p.nCols || p.colType(in.a) != LDB_UTF8) fail(LDB_ERR_INVALID, "STRCODE needs a utf8 column");
            wantCol(in.a, "STRCODE");
            if (in.arg < 0 || in.arg >= d->n_tables) fail(LDB_ERR_INVALID, "STRCODE: dictionary index out of range");
            if (in.b > 1) fail(LDB_ERR_INVALID, "STRCODE: b is 1 (insert) or 0 (lookup only)");
            p.coded[in.arg] = true;
            p.inserted[in.arg] |= in.b == 1;
            break;
         case LDB_OP_CONST:
            if (in.arg < 0 || in.arg >= d->n_consts) fail(LDB_ERR_INVALID, "CONST: constant index out of range");
            break;
         case LDB_OP_ADD: case LDB_OP_SUB: case LDB_OP_MUL: case LDB_OP_DIV: case LDB_OP_AND: case LDB_OP_OR:
         case LDB_OP_FADD: case LDB_OP_FSUB: case LDB_OP_FMUL: case LDB_OP_FDIV:
            p.wantReg(in.a, "a");
            p.wantReg(in.b, "b");
            break;
         case LDB_OP_CMP: case LDB_OP_FCMP:
            p.wantReg(in.a, "a");
            p.wantReg(in.b, "b");
            if (in.arg < LDB_EQ || in.arg > LDB_GTE) fail(LDB_ERR_INVALID, "CMP: unknown comparison");
            break;
         case LDB_OP_NEG: case LDB_OP_NOT: case LDB_OP_ISNULL: case LDB_OP_I2F: case LDB_OP_YEAR: p.wantReg(in.a, "a"); break;
         case LDB_OP_SELECT:
            p.wantReg(in.a, "a");
            p.wantReg(in.b, "b");
            p.wantReg(in.arg, "condition");
            break;
         case LDB_OP_STRKEY8:
            if (in.a >= p.nCols || p.colType(in.a) != LDB_UTF8) fail(LDB_ERR_INVALID, "STRKEY8 needs a utf8 column");
            wantCol(in.a, "STRKEY8");
            break;
         case LDB_OP_STRCMP: case LDB_OP_STRLIKE:
            if (in.a >= p.nCols || p.colType(in.a) != LDB_UTF8) fail(LDB_ERR_INVALID, "string op needs a utf8 column");
            wantCol(in.a, "string op");
            if (in.arg < 0 || in.arg >= d->n_strings) fail(LDB_ERR_INVALID, "string constant index out of range");
            if (in.op == LDB_OP_STRCMP ? in.b > LDB_GTE : in.b > 2) fail(LDB_ERR_INVALID, "string op: unknown comparison / pattern kind");
            break;
         case LDB_OP_PROBE:
            if (in.arg < 0 || in.arg >= d->n_tables) fail(LDB_ERR_INVALID, "PROBE: table index out of range");
            wantKeys(in);
            p.probed[in.arg] = true;
            if (exEnd >= 0) probedInBlock[in.arg] = true;
            break;
         case LDB_OP_ROWID: p.usesRowid = true; break;
         case LDB_OP_PROBE_EACH:
            if (in.arg < 0 || in.arg >= d->n_tables) fail(LDB_ERR_INVALID, "PROBE_EACH: table index out of range");
            wantKeys(in);
            if (in.b > 1) fail(LDB_ERR_INVALID, "PROBE_EACH: b is 0 (inner) or 1 (left outer)");
            if (base.eachPc >= 0) fail(LDB_ERR_UNSUPPORTED, "at most one PROBE_EACH per program");
            base.eachPc = i;
            p.eachTable = in.arg;
            p.probed[in.arg] = true;
            break;
         case LDB_OP_MARK:
            if (in.arg < 0 || in.arg >= d->n_tables) fail(LDB_ERR_INVALID, "MARK: table index out of range");
            if (!p.probed[in.arg]) fail(LDB_ERR_INVALID, "MARK: no earlier PROBE / PROBE_EACH of the program reads the table it marks");
            if (probedInBlock[in.arg]) fail(LDB_ERR_INVALID, "MARK: the table it marks is probed inside an EXISTS block");
            p.wantReg(in.a, "MARK condition");
            p.marked[in.arg] = true;
            break;
         case LDB_OP_EXISTS:
            if (in.arg < 0 || in.arg >= d->n_tables) fail(LDB_ERR_INVALID, "EXISTS: table index out of range");
            wantKeys(in);
            if (i + in.b >= d->n_instr) fail(LDB_ERR_INVALID, "EXISTS: its residual block of b instructions runs past the end of the program");
            p.existed[in.arg] = true;
            break;
         default: fail(LDB_ERR_UNSUPPORTED, "unknown opcode " + std::to_string(in.op));
      }
      // the instructions after PROBE_EACH run once per match: they may not overwrite what the first pass left for the next one
      if (base.eachPc >= 0 && i > base.eachPc && beforeEach[in.dst]) fail(LDB_ERR_INVALID, "an instruction after PROBE_EACH overwrites a register written at or before it");
      if (exEnd >= 0) { // the block re-runs per match: what was written before the EXISTS (its dst included) must survive it
         if (beforeExists[in.dst]) fail(LDB_ERR_INVALID, "an instruction of an EXISTS block overwrites a register written before the EXISTS");
         inBlock[in.dst] = true;
      } else {
         p.blockOnly[in.dst] = p.verdict[in.dst] = false;
      }
      p.written[in.dst] = true;
      if (in.op == LDB_OP_EXISTS) {
         std::copy(p.written, p.written + kProgMaxRegs, beforeExists);
         std::fill(inBlock, inBlock + kProgMaxRegs, false);
         exDst = in.dst;
         exEnd = in.b ? i + in.b : -1;
         if (!in.b) p.verdict[in.dst] = true;
      } else if (i == exEnd) { // the block ends: after it, its registers and the EXISTS's dst as a row are off limits
         for (int r = 0; r < kProgMaxRegs; r++) p.blockOnly[r] |= inBlock[r];
         p.verdict[exDst] = true;
         exEnd = -1;
      }
      if (base.eachPc == i) std::copy(p.written, p.written + kProgMaxRegs, beforeEach);
      base.instr[i] = ProgInstr{in.op, in.dst, in.a, in.b, in.arg};
   }
   for (int c = 0; c < d->n_consts; c++) {
      base.constLo[c] = d->consts[c].lo;
      base.constHi[c] = d->consts[c].hi;
   }
   for (int c = 0; c < d->n_strings; c++) {
      const size_t n = d->strings[c] ? strlen(d->strings[c]) : 0;
      if (n > (size_t) kProgStringBytes) fail(LDB_ERR_UNSUPPORTED, "string constant longer than 32 bytes");
      memcpy(base.strings[c], d->strings[c], n);
      base.stringLen[c] = (int32_t) n;
   }
}

// ---------------------------------------------------------------- join-table markers (program.h)
// the tables that keep markers: plain single-key, direct-address and key-tuple join tables
static bool markable(const LdbState* s) {
   return s && (s->kind == LDB_STATE_KEY_JOIN || (s->kind == LDB_STATE_JOIN_TABLE && (s->join.stride == 8 || s->join.direct)));
}
static void checkMarkable(LdbState* s) {
   if (s->kind != LDB_STATE_JOIN_TABLE && s->kind != LDB_STATE_KEY_JOIN) fail(LDB_ERR_INVALID, "not a join table");
   if (!markable(s)) fail(LDB_ERR_INVALID, "markers are kept for plain single-key, direct-address and key-tuple join tables (not pair tables or group-join maps)");
   if (s->ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "join-table markers are not part of captured queries");
}
static uint64_t markSlots(const LdbState* s) {
   if (s->kind == LDB_STATE_KEY_JOIN) return s->keyJoin.mask + 1;
   return s->join.direct ? (uint64_t) s->join.range : s->join.mask + 1;
}
// tables[k] is marked by a MARK instruction: its markers, allocated zeroed on first use
static void bindMarks(ProgramPlan& p, int k) {
   LdbState* js = p.d->tables[k];
   if (!markable(js)) fail(LDB_ERR_INVALID, "MARK takes a plain single-key, direct-address or key-tuple join table (not a pair table, a group-join map or a dictionary)");
   if (js->ctx != p.ctx) fail(LDB_ERR_INVALID, "MARK: the join table belongs to another context");
   if (p.d->sink_kind == LDB_SINK_JOIN_BUILD && p.d->sink == js) fail(LDB_ERR_INVALID, "MARK: a program may not mark the join table it builds");
   if (p.ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "programs with MARK are not part of captured queries");
   if (!js->marks) {
      const size_t bytes = std::max<size_t>(markSlots(js), 16);
      js->marks = (uint8_t*) p.ctx->stagingAlloc(bytes);
      js->allocations.push_back(js->marks);
      LDB_CUDA(cudaMemsetAsync(js->marks, 0, bytes, p.ctx->compute));
   }
   p.base.marks[k] = js->marks;
}

// the table slots: plain join tables, key-tuple join tables and string dictionaries
static void bindTables(ProgramPlan& p) {
   LdbContext* ctx = p.ctx;
   const LdbProgramDesc* d = p.d;
   for (int k = 0; k < d->n_tables; k++) {
      LdbState* js = d->tables[k];
      // the table's error word (a probe run at the bound) is read back after the launch, which a captured query cannot do
      if (p.existed[k] && ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "programs with EXISTS are not part of captured queries (the probe-run bound is checked after the launch)");
      if (p.marked[k]) bindMarks(p, k);
      if (js && js->kind == LDB_STATE_KEY_JOIN) {
         if (p.coded[k]) fail(LDB_ERR_INVALID, "STRCODE needs a string dictionary, not a join table");
         p.wantTupleTable(js);
         if (d->sink_kind == LDB_SINK_JOIN_BUILD && d->sink == js) fail(LDB_ERR_INVALID, "a program may not build a key-tuple join table and probe it");
         p.base.keyTables[k] = js->keyJoin;
         if (p.probed[k] || p.existed[k]) p.tupleTables.push_back(js);
         continue;
      }
      if (js && js->kind == LDB_STATE_DICT) {
         if (p.existed[k]) fail(LDB_ERR_INVALID, "EXISTS on a string dictionary (it takes a join table)");
         if (p.probed[k]) fail(LDB_ERR_INVALID, "PROBE / PROBE_EACH on a string dictionary (they take join tables)");
         if (js->ctx != ctx) fail(LDB_ERR_INVALID, "string dictionary belongs to another context");
         if (ctx->capturing) fail(LDB_ERR_UNSUPPORTED, "string dictionaries are not part of captured queries");
         if (js->unified && p.inserted[k]) fail(LDB_ERR_INVALID, "an inserting STRCODE against a unified dictionary (its codes agree across ranks: it takes lookups only)");
         p.base.dicts[k] = js->dict;
         p.dicts.push_back(js);
         continue;
      }
      if (p.coded[k]) fail(LDB_ERR_INVALID, "STRCODE needs a string dictionary, not a join table");
      if (k == p.eachTable && js && js->kind == LDB_STATE_JOIN_TABLE && !(js->join.stride == 8 || js->join.direct))
         fail(LDB_ERR_UNSUPPORTED, "PROBE_EACH takes a plain single-key or direct-address join table (not a pair table or a group-join map)");
      if (p.existed[k] && js && js->kind == LDB_STATE_JOIN_TABLE && !(js->join.stride == 8 || js->join.direct))
         fail(LDB_ERR_UNSUPPORTED, "EXISTS takes a plain single-key, direct-address or key-tuple join table (not a pair table or a group-join map)");
      if (!js || js->kind != LDB_STATE_JOIN_TABLE || js->join.stride == 16) fail(LDB_ERR_INVALID, "PROBE tables are single-key join tables");
      p.base.tables[k] = js->join;
   }
}

// materialize output buffers for `rows` rows (+ the row counter) in `out`, replacing the ones it holds
static void allocOut(ProgramPlan& p, Scratch& out, size_t rows) {
   for (void* q : out.take()) p.ctx->stagingRelease(q);
   for (int c = 0; c < p.d->n_out; c++) {
      p.base.outValues[c] = out.alloc<uint8_t>(rows * 16);
      p.base.outValid[c] = out.alloc<uint8_t>(rows);
   }
   p.base.outCount = out.alloc<unsigned long long>(8);
   LDB_CUDA(cudaMemsetAsync(p.base.outCount, 0, 8, p.ctx->compute));
   p.base.outCapacity = (int64_t) rows;
}

// the filter and the sink: a hash aggregation, a join build (plain or key-tuple table), materialized rows (buffers in `out`) or none
static void bindSink(ProgramPlan& p, Scratch& out) {
   const LdbProgramDesc* d = p.d;
   ProgramParams& base = p.base;
   base.filterReg = d->filter_reg;
   if (d->filter_reg >= 0) p.wantReg(d->filter_reg, "filter");
   base.sinkKind = d->sink_kind;
   LdbState* sink = d->sink;
   if (d->sink_kind == LDB_SINK_HASHAGG) {
      checkHashAgg(sink);
      if (sink->ctx != p.ctx || d->n_keys != sink->hashagg.nKeys || d->n_aggs != sink->hashagg.nAggs) fail(LDB_ERR_INVALID, "key / aggregate count differs from the state's");
      base.nKeys = d->n_keys;
      base.nAggs = d->n_aggs;
      for (int k = 0; k < d->n_keys; k++) {
         p.wantReg(d->key_regs[k], "group key");
         base.keyReg[k] = d->key_regs[k];
      }
      for (int a = 0; a < d->n_aggs; a++) {
         if (d->aggs[a].kind != sink->aggKinds[a]) fail(LDB_ERR_INVALID, "aggregate kind differs from the state's");
         if (d->aggs[a].kind != LDB_AGG_COUNT_STAR) p.wantReg(d->aggs[a].reg, "aggregate input");
         base.aggs[a] = ProgAgg{d->aggs[a].kind, d->aggs[a].reg};
      }
      base.agg = sink->hashagg;
   } else if (d->sink_kind == LDB_SINK_JOIN_BUILD && sink && sink->kind == LDB_STATE_KEY_JOIN) {
      // keys from n_keys / key_regs[]; payloads are int64, so ROWID has no row limit here
      p.wantTupleTable(sink);
      if (d->n_keys != sink->keyJoin.nKeys) fail(LDB_ERR_INVALID, "n_keys differs from the key-tuple join table's key count");
      if (d->build_key_reg != -1) fail(LDB_ERR_INVALID, "a build into a key-tuple join table takes its keys from key_regs (build_key_reg must be -1)");
      base.nKeys = d->n_keys;
      for (int k = 0; k < d->n_keys; k++) {
         p.wantReg(d->key_regs[k], "build key");
         base.keyReg[k] = d->key_regs[k];
      }
      if (d->build_payload_reg >= 0) p.wantReg(d->build_payload_reg, "build payload");
      base.buildKeyReg = -1;
      base.buildPayloadReg = d->build_payload_reg;
      base.keyBuild = sink->keyJoin;
      p.tupleTables.push_back(sink);
   } else if (d->sink_kind == LDB_SINK_JOIN_BUILD) {
      if (!sink || sink->kind != LDB_STATE_JOIN_TABLE || sink->join.stride != 8 || sink->join.direct) fail(LDB_ERR_INVALID, "build sink must be a plain single-key join table");
      if (p.usesRowid && p.t->numRows > (int64_t) INT32_MAX) fail(LDB_ERR_UNSUPPORTED, "ROWID build payloads are int32: the source has 2^31 rows or more");
      p.wantReg(d->build_key_reg, "build key");
      if (d->build_payload_reg >= 0) p.wantReg(d->build_payload_reg, "build payload");
      base.buildKeyReg = d->build_key_reg;
      base.buildPayloadReg = d->build_payload_reg;
      base.build = sink->join;
   } else if (d->sink_kind == LDB_SINK_MATERIALIZE) {
      if (d->n_out < 1 || d->n_out > kProgMaxAggs || !d->out_table) fail(LDB_ERR_INVALID, "materialize needs 1..8 output registers and out_table");
      base.nOut = d->n_out;
      for (int c = 0; c < d->n_out; c++) {
         p.wantReg(d->out_regs[c], "output");
         base.outReg[c] = d->out_regs[c];
      }
      allocOut(p, out, (size_t) std::max<int64_t>(p.t->numRows, 1));
   } else if (d->sink_kind == LDB_SINK_NONE) { // effects only (MARK, STRCODE inserts)
      if (sink) fail(LDB_ERR_INVALID, "LDB_SINK_NONE takes no sink state (sink must be NULL)");
   } else {
      fail(LDB_ERR_INVALID, "unknown sink kind");
   }
}

// side columns: bound once for all batches of the source; a multi-batch side table through a device-resident batch directory
// (in `dirs`)
static void bindSideColumns(ProgramPlan& p, Scratch& dirs) {
   LdbContext* ctx = p.ctx;
   for (int c = p.d->n_columns; c < p.nCols; c++) {
      LdbTable* st = p.colTable[c];
      ProgCol& pc = p.base.cols[c];
      pc.type = p.colType(c);
      pc.rowReg = p.rowReg[c];
      std::vector<ProgSideBatch> dir;
      int64_t first = 0;
      const LdbBatch* only = nullptr;
      for (auto& b : st->batches) {
         ldb_gpu_wait_batch_internal(ctx, &b);
         if (b.nRows > 0) {
            ProgCol one{};
            bindColumn(one, b, p.colIdx[c]);
            dir.push_back(ProgSideBatch{one.data, one.bytes, one.validity, one.validBytes, one.bitOffset, first, one.elemBytes, 0});
            only = &b;
         }
         first += b.nRows;
      }
      pc.sideRows = first;
      pc.nBatches = (int32_t) dir.size();
      if (dir.size() == 1) {
         bindColumn(pc, *only, p.colIdx[c]);
      } else if (dir.size() > 1) {
         ProgSideBatch* dd = dirs.alloc<ProgSideBatch>(dir.size() * sizeof(ProgSideBatch));
         LDB_CUDA(cudaMemcpyAsync(dd, dir.data(), dir.size() * sizeof(ProgSideBatch), cudaMemcpyHostToDevice, ctx->compute));
         pc.dir = dd;
      }
   }
   for (int c = 0; c < p.d->n_columns; c++) p.base.cols[c].rowReg = -1;
}

// one interpreter launch per non-empty batch of the source
static void launchBatches(const ProgramPlan& p) {
   LdbContext* ctx = p.ctx;
   int64_t first = 0;
   for (auto& b : p.t->batches) {
      const int64_t firstRow = first;
      first += b.nRows;
      if (b.nRows == 0) continue;
      ProgramParams pp = p.base;
      pp.nRows = b.nRows;
      pp.firstRow = firstRow;
      for (int c = 0; c < p.d->n_columns; c++) {
         const int ci = p.colIdx[c];
         pp.cols[c].type = p.t->columns[ci].type;
         bindColumn(pp.cols[c], b, ci);
      }
      ldb_gpu_wait_batch_internal(ctx, &b);
      ctx->launch("program", [&] { launchProgram(pp, ctx->smCount, ctx->compute); });
   }
}

// a probe run longer than the bound (PROBE_EACH, EXISTS), or a build that could not store a row (table full, the reserved pair, a key
// or payload outside int32): fail rather than return a truncated match list, a verdict that missed a match or a table with rows missing
// — and a dictionary that could not take a string
static void checkErrorWords(const ProgramPlan& p) {
   const LdbProgramDesc* d = p.d;
   for (LdbState* js : {p.eachTable >= 0 ? d->tables[p.eachTable] : nullptr, d->sink_kind == LDB_SINK_JOIN_BUILD ? d->sink : nullptr})
      if (js && js->kind == LDB_STATE_JOIN_TABLE) ldb_gpu_check_join_error_internal(js);
   for (int k = 0; k < d->n_tables; k++)
      if (p.existed[k] && k != p.eachTable && d->tables[k]->kind == LDB_STATE_JOIN_TABLE) ldb_gpu_check_join_error_internal(d->tables[k]);
   for (LdbState* ks : p.tupleTables) ldb_gpu_check_keyjoin_error_internal(ks); // a full build, a probe run at the bound, a key outside int64
   for (LdbState* ds : p.dicts) ldb_gpu_dict_counters_internal(ds);
}

// the materialized rows as a table that takes over the output buffers of `out` (synchronises)
static LdbTable* materializeResult(ProgramPlan& p, Scratch& out) {
   LdbContext* ctx = p.ctx;
   unsigned long long n = 0;
   LDB_CUDA(cudaMemcpyAsync(&n, p.base.outCount, 8, cudaMemcpyDeviceToHost, ctx->compute));
   ctx->syncStream(ctx->compute);
   if (n > (unsigned long long) p.base.outCapacity) { // PROBE_EACH produced more rows than the source has: regrow and run once more
      allocOut(p, out, (size_t) n);
      launchBatches(p);
      LDB_CUDA(cudaMemcpyAsync(&n, p.base.outCount, 8, cudaMemcpyDeviceToHost, ctx->compute));
      ctx->syncStream(ctx->compute);
      if (n > (unsigned long long) p.base.outCapacity) fail(LDB_ERR_INVALID, "materialize: the rerun produced more rows than the first run");
   }
   std::vector<LdbColumn> columns;
   LdbBatch ob;
   ob.nRows = (int64_t) n;
   for (int c = 0; c < p.d->n_out; c++) {
      columns.push_back({"c" + std::to_string(c), LDB_DECIMAL128, 38, 0});
      ob.data.push_back(p.base.outValues[c]);
      ob.bytes.push_back(nullptr);
      ob.elemBytes.push_back(16);
      ob.validBytes.push_back(p.base.outValid[c]);
   }
   return addResultTable(ctx, p.t->name + "_out", std::move(columns), std::move(ob), out);
}

static void runProgram(LdbContext* ctx, const LdbProgramDesc* d, const LdbProgramJoins* j) {
   if (!ctx || !d || !d->source) fail(LDB_ERR_INVALID, "null argument");
   ProgramPlan p(ctx, d);
   resolveColumns(p, j);
   validateInstructions(p);
   bindTables(p);
   Scratch out(ctx), dirs(ctx);
   bindSink(p, out);
   bindSideColumns(p, dirs);
   launchBatches(p);
   checkErrorWords(p);
   if (d->sink_kind == LDB_SINK_MATERIALIZE) *d->out_table = materializeResult(p, out);
   if (!dirs.empty()) ctx->syncStream(ctx->compute); // the batch directories are read until the last launch ends
}

// ORDER BY … LIMIT over a single-batch table: the first min(n, limit) row ids (limit < 0: all n) of the stable sort by `keys`
static void orderRows(LdbTable* t, const std::vector<std::pair<int, int>>& keys, int64_t limit, int64_t* row_ids, int64_t* n_out) {
   if (t->batches.size() != 1) fail(LDB_ERR_UNSUPPORTED, "ORDER BY runs over single-batch tables (materialised results, exported groups)");
   LdbContext* ctx = t->ctx;
   LdbBatch& b = t->batches[0];
   const int64_t n = b.nRows;
   if (n >= (int64_t) 1 << 32) fail(LDB_ERR_UNSUPPORTED, "ORDER BY handles up to 2^32 - 1 rows");
   LDB_CUDA(cudaSetDevice(ctx->device));
   ldb_gpu_wait_batch_internal(ctx, &b);
   Scratch scratch(ctx);
   const uint32_t* ids = sortRows(scratch, t, keys, n);
   const int64_t m = std::min<int64_t>(n, limit < 0 ? n : limit);
   std::vector<uint32_t> top((size_t) m);
   if (m) LDB_CUDA(cudaMemcpyAsync(top.data(), ids, (size_t) m * 4, cudaMemcpyDeviceToHost, ctx->compute));
   ctx->syncStream(ctx->compute);
   for (int64_t i = 0; i < m; i++) row_ids[i] = top[(size_t) i];
   *n_out = m;
}

// the validity of gathered rows, one run of consecutive row ids at a time, into host_valid (1 = not NULL): one byte per row
// (tables this library made) is copied, an Arrow bitmap has the bytes that hold the run's bits copied and is decoded by finish()
// once the stream has been synchronised, a column without either is all valid
class GatherValidity {
 public:
   GatherValidity(const LdbBatch& b, int c, uint8_t* hostValid) : hostValid_(hostValid) {
      bytes_ = c < (int) b.validBytes.size() ? b.validBytes[c] : nullptr;
      bitmap_ = c < (int) b.validity.size() && !bytes_ ? (const uint8_t*) b.validity[c] : nullptr;
      bitOffset_ = bitmap_ ? b.validityBitOffset[c] : 0;
   }
   // rows row .. row + m - 1 → host_valid[i .. i + m)
   void run(int64_t i, int64_t row, int64_t m, cudaStream_t s) {
      if (!hostValid_) return;
      if (bytes_) {
         LDB_CUDA(cudaMemcpyAsync(hostValid_ + i, bytes_ + row, (size_t) m, cudaMemcpyDeviceToHost, s));
      } else if (bitmap_) {
         const int64_t bit0 = bitOffset_ + row;
         runs_.push_back({i, m, bit0 % 8, std::vector<uint8_t>((size_t) ((bit0 % 8 + m + 7) / 8))});
         LDB_CUDA(cudaMemcpyAsync(runs_.back().bits.data(), bitmap_ + bit0 / 8, runs_.back().bits.size(), cudaMemcpyDeviceToHost, s));
      } else {
         memset(hostValid_ + i, 1, (size_t) m);
      }
   }
   void finish() {
      for (const Run& r : runs_)
         for (int64_t q = 0; q < r.m; q++) hostValid_[r.i + q] = (r.bits[(size_t) ((r.bit0 + q) >> 3)] >> ((r.bit0 + q) & 7)) & 1u;
   }

 private:
   struct Run {
      int64_t i, m, bit0;
      std::vector<uint8_t> bits;
   };
   uint8_t* hostValid_;
   const uint8_t* bytes_;
   const uint8_t* bitmap_;
   int64_t bitOffset_;
   std::deque<Run> runs_; // a deque: the bytes of earlier runs stay put while later runs are added
};

extern "C" {

int ldb_gpu_run_program(LdbContext* ctx, const LdbProgramDesc* d, LdbError* err) {
   return guarded(err, [&] { runProgram(ctx, d, nullptr); });
}
int ldb_gpu_run_program_ex(LdbContext* ctx, const LdbProgramDesc* d, const LdbProgramJoins* joins, LdbError* err) {
   return guarded(err, [&] { runProgram(ctx, d, joins); });
}

// ---------------------------------------------------------------- join-table markers
int ldb_gpu_join_table_marks(LdbState* s, int32_t which, const char* name, LdbTable** out, LdbError* err) {
   return guarded(err, [&] {
      if (!s || !out) fail(LDB_ERR_INVALID, "null argument");
      if (which < -1 || which > 1) fail(LDB_ERR_INVALID, "which is 1 (marked entries), 0 (unmarked entries) or -1 (all entries and a marked column)");
      checkMarkable(s);
      LdbContext* ctx = s->ctx;
      LDB_CUDA(cudaSetDevice(ctx->device));
      int64_t n = 0;
      LdbError e;
      if (ldb_gpu_join_table_count(s, &n, &e) != LDB_OK) fail(e.code, e.message); // the table's error word first
      const bool tuple = s->kind == LDB_STATE_KEY_JOIN;
      const int nKeys = tuple ? s->keyJoin.nKeys : 1;
      const size_t rows = (size_t) std::max<int64_t>(n, 1);
      Scratch cols(ctx), scratch(ctx);
      MarkScanOut o{};
      std::vector<LdbColumn> columns;
      LdbBatch b;
      auto add = [&](const std::string& column, int32_t type, void* data, int32_t elemBytes) {
         columns.push_back({column, type, 0, 0});
         b.data.push_back(data);
         b.bytes.push_back(nullptr);
         b.elemBytes.push_back(elemBytes);
         b.validBytes.push_back(nullptr);
      };
      for (int k = 0; k < nKeys; k++) {
         o.keyCols[k] = cols.alloc<int64_t>(rows * 8);
         add(tuple ? "k" + std::to_string(k) : "key", LDB_INT64, o.keyCols[k], 8);
      }
      o.payload = cols.alloc<int64_t>(rows * 8);
      add("payload", LDB_INT64, o.payload, 8);
      if (which < 0) {
         o.marked = cols.alloc<int32_t>(rows * 4);
         add("marked", LDB_INT32, o.marked, 4);
      }
      o.capacity = n;
      unsigned long long* counter = scratch.alloc<unsigned long long>(8);
      LDB_CUDA(cudaMemsetAsync(counter, 0, 8, ctx->compute));
      ctx->launch("join_marks", [&] { launchJoinMarks(tuple ? JoinTableDev{} : s->join, tuple ? s->keyJoin : KeyJoinDev{}, s->marks, which, o, counter, ctx->smCount, ctx->compute); });
      unsigned long long got = 0;
      LDB_CUDA(cudaMemcpyAsync(&got, counter, 8, cudaMemcpyDeviceToHost, ctx->compute));
      ctx->syncStream(ctx->compute);
      if (got > (unsigned long long) n) fail(LDB_ERR_INVALID, "the join table holds more entries than its count");
      b.nRows = (int64_t) got;
      *out = addResultTable(ctx, name ? name : "marks", std::move(columns), std::move(b), cols);
   });
}
int ldb_gpu_join_table_clear_marks(LdbState* s, LdbError* err) {
   return guarded(err, [&] {
      if (!s) fail(LDB_ERR_INVALID, "null argument");
      checkMarkable(s);
      if (!s->marks) return;
      LDB_CUDA(cudaSetDevice(s->ctx->device));
      LDB_CUDA(cudaMemsetAsync(s->marks, 0, markSlots(s), s->ctx->compute));
   });
}

// ---------------------------------------------------------------- ORDER BY … LIMIT and result gather
int ldb_gpu_table_order_by(LdbTable* t, const char* column, int32_t descending, int64_t limit, int64_t* row_ids, int64_t* n_out, LdbError* err) {
   return guarded(err, [&] {
      if (!t || !row_ids || !n_out) fail(LDB_ERR_INVALID, "null argument");
      const int c = t->colIndex(column);
      if (c < 0) fail(LDB_ERR_INVALID, "unknown column");
      const int type = t->columns[c].type;
      if (type == LDB_UTF8 || type == LDB_FLOAT32 || type == LDB_FLOAT64 || type == LDB_INT8 || type == LDB_INT16) fail(LDB_ERR_UNSUPPORTED, "ORDER BY column must be int32/date32/char(1)/int64/decimal");
      orderRows(t, {{c, descending ? 1 : 0}}, limit, row_ids, n_out);
   });
}
int ldb_gpu_table_gather(LdbTable* t, const char* column, const int64_t* row_ids, int64_t n, void* host_dst, uint8_t* host_valid, LdbError* err) {
   return guarded(err, [&] {
      if (!t || !row_ids || !host_dst) fail(LDB_ERR_INVALID, "null argument");
      LdbContext* ctx = t->ctx;
      const int c = t->colIndex(column);
      if (c < 0) fail(LDB_ERR_INVALID, "unknown column");
      if (t->columns[c].type == LDB_UTF8) fail(LDB_ERR_UNSUPPORTED, "gather reads fixed-width columns");
      if (t->batches.size() != 1) fail(LDB_ERR_UNSUPPORTED, "gather runs over single-batch tables");
      LdbBatch& b = t->batches[0];
      LDB_CUDA(cudaSetDevice(ctx->device));
      ldb_gpu_wait_batch_internal(ctx, &b);
      const size_t w = (size_t) b.elemBytes[c];
      for (int64_t i = 0; i < n; i++)
         if (row_ids[i] < 0 || row_ids[i] >= b.nRows) fail(LDB_ERR_INVALID, "row id out of range");
      // a decimal128 cell staged as 8 bytes (narrowed or packed HOST staging) is read into `narrow` and widened below
      const bool widen = t->columns[c].type == LDB_DECIMAL128 && w == 8;
      std::vector<int64_t> narrow(widen ? (size_t) n : 0);
      uint8_t* dst = widen ? (uint8_t*) narrow.data() : (uint8_t*) host_dst;
      GatherValidity valid(b, c, host_valid);
      // one copy per run of consecutive row ids (a whole column read back in order is one copy)
      for (int64_t i = 0, j; i < n; i = j) {
         for (j = i + 1; j < n && row_ids[j] == row_ids[j - 1] + 1;) j++;
         const size_t m = (size_t) (j - i);
         LDB_CUDA(cudaMemcpyAsync(dst + (size_t) i * w, (const uint8_t*) b.data[c] + (size_t) row_ids[i] * w, m * w, cudaMemcpyDeviceToHost, ctx->compute));
         valid.run(i, row_ids[i], (int64_t) m, ctx->compute);
      }
      ctx->syncStream(ctx->compute);
      valid.finish();
      for (size_t i = 0; i < narrow.size(); i++) {
         const int64_t cell[2] = {narrow[i], narrow[i] >> 63};
         memcpy((uint8_t*) host_dst + i * 16, cell, 16);
      }
   });
}
int ldb_gpu_table_order_by_keys(LdbTable* t, int32_t n_keys, const char* const* columns, const int32_t* descending, int64_t limit, int64_t* row_ids, int64_t* n_out, LdbError* err) {
   return guarded(err, [&] {
      if (!t || !columns || !descending || !row_ids || !n_out) fail(LDB_ERR_INVALID, "null argument");
      if (n_keys < 1) fail(LDB_ERR_INVALID, "ORDER BY needs at least one key");
      std::vector<std::pair<int, int>> keys;
      for (int k = 0; k < n_keys; k++) {
         const int c = t->colIndex(columns[k]);
         if (c < 0) fail(LDB_ERR_INVALID, std::string("unknown column ") + (columns[k] ? columns[k] : "(null)"));
         const int type = t->columns[c].type;
         if (type == LDB_FLOAT32 || type == LDB_FLOAT64 || type == LDB_INT8 || type == LDB_INT16) fail(LDB_ERR_UNSUPPORTED, "ORDER BY column must be int32/date32/char(1)/int64/decimal/utf8");
         keys.push_back({c, descending[k] ? 1 : 0});
      }
      orderRows(t, keys, limit, row_ids, n_out);
   });
}
int ldb_gpu_table_gather_strings(LdbTable* t, const char* column, const int64_t* row_ids, int64_t n, int64_t* host_offsets, void* host_bytes, int64_t bytes_cap, int64_t* bytes_needed,
                                 uint8_t* host_valid, LdbError* err) {
   return guarded(err, [&] {
      if (!t || (n > 0 && !row_ids) || !host_offsets || !bytes_needed || n < 0) fail(LDB_ERR_INVALID, "null argument");
      LdbContext* ctx = t->ctx;
      const int c = t->colIndex(column);
      if (c < 0) fail(LDB_ERR_INVALID, "unknown column");
      if (t->columns[c].type != LDB_UTF8) fail(LDB_ERR_UNSUPPORTED, "gather_strings reads utf8 columns");
      if (t->batches.size() != 1) fail(LDB_ERR_UNSUPPORTED, "gather runs over single-batch tables");
      LdbBatch& b = t->batches[0];
      for (int64_t i = 0; i < n; i++)
         if (row_ids[i] < 0 || row_ids[i] >= b.nRows) fail(LDB_ERR_INVALID, "row id out of range");
      LDB_CUDA(cudaSetDevice(ctx->device));
      ldb_gpu_wait_batch_internal(ctx, &b);
      // runs of consecutive row ids: [first index, end index) → the run's m + 1 offsets at `at` in `offs`
      struct Run {
         int64_t i, j;
         size_t at;
      };
      std::vector<Run> runs;
      for (int64_t i = 0, j; i < n; i = j) {
         for (j = i + 1; j < n && row_ids[j] == row_ids[j - 1] + 1;) j++;
         runs.push_back({i, j, 0});
      }
      std::vector<int32_t> offs;
      for (Run& r : runs) {
         r.at = offs.size();
         offs.resize(offs.size() + (size_t) (r.j - r.i) + 1);
      }
      for (const Run& r : runs)
         LDB_CUDA(cudaMemcpyAsync(offs.data() + r.at, (const int32_t*) b.data[c] + row_ids[r.i], (size_t) (r.j - r.i + 1) * 4, cudaMemcpyDeviceToHost, ctx->compute));
      ctx->syncStream(ctx->compute);
      int64_t total = 0;
      for (const Run& r : runs) total += offs[r.at + (size_t) (r.j - r.i)] - offs[r.at];
      *bytes_needed = total;
      if (total > bytes_cap) fail(LDB_ERR_CAPACITY, "gather_strings: the strings need more than bytes_cap bytes (see bytes_needed)");
      if (total > 0 && !host_bytes) fail(LDB_ERR_INVALID, "null argument");
      GatherValidity valid(b, c, host_valid);
      int64_t pos = 0;
      host_offsets[0] = 0;
      for (const Run& r : runs) {
         const size_t m = (size_t) (r.j - r.i);
         for (size_t q = 0; q < m; q++) host_offsets[r.i + (int64_t) q + 1] = pos + offs[r.at + q + 1] - offs[r.at];
         const int64_t len = offs[r.at + m] - offs[r.at];
         if (len) LDB_CUDA(cudaMemcpyAsync((uint8_t*) host_bytes + pos, (const uint8_t*) b.bytes[c] + offs[r.at], (size_t) len, cudaMemcpyDeviceToHost, ctx->compute));
         pos += len;
         valid.run(r.i, row_ids[r.i], (int64_t) m, ctx->compute);
      }
      ctx->syncStream(ctx->compute);
      valid.finish();
   });
}

} // extern "C"
