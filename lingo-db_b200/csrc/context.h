// context.h — internal definitions of the opaque C-ABI handles (include/ldb_gpu.h).
#pragma once
#include "../../include/ldb_gpu.h"
#include "kernels.h"
#include "program.h"

#include <cuda_runtime.h>
#include <atomic>
#include <condition_variable>
#include <cstdio>
#include <exception>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <stdexcept>
#include <string>
#include <vector>

namespace ldb {

struct CudaError : std::runtime_error {
   int code;
   CudaError(int code, const std::string& m) : std::runtime_error(m), code(code) {}
};
inline void cudaCheck(cudaError_t e, const char* what, const char* file, int line) {
   if (e != cudaSuccess) {
      cudaGetLastError();
      throw CudaError(e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver ? LDB_ERR_NO_DEVICE : LDB_ERR_CUDA,
                      std::string(what) + ": " + cudaGetErrorString(e) + " (" + file + ":" + std::to_string(line) + ")");
   }
}
#define LDB_CUDA(x) ::ldb::cudaCheck((x), #x, __FILE__, __LINE__)
struct ApiError : std::runtime_error {
   int code;
   ApiError(int code, const std::string& m) : std::runtime_error(m), code(code) {}
};
[[noreturn]] inline void fail(int code, const std::string& m) { throw ApiError(code, m); }

// The body of every C-ABI entry point: no exception leaves an extern "C" function.  The status goes to the return value and,
// with its message, to `err` when the caller passed one (LDB_OK and an empty message on success).
template <class Fn>
int guarded(LdbError* err, const Fn& fn) {
   auto set = [&](int code, const char* msg) {
      if (err) {
         err->code = code;
         snprintf(err->message, sizeof(err->message), "%s", msg);
      }
      return code;
   };
   try {
      fn();
      return set(LDB_OK, "");
   } catch (const CudaError& e) {
      return set(e.code, e.what());
   } catch (const ApiError& e) {
      return set(e.code, e.what());
   } catch (const std::exception& e) {
      return set(LDB_ERR_INVALID, e.what());
   }
}

inline uint64_t nextPow2(uint64_t v) {
   v--;
   for (int s = 1; s < 64; s <<= 1) v |= v >> s;
   return v + 1;
}

// Host worker pool used while staging HOST batches (narrowing decimal128 → the 8 bytes the kernels read).
class HostPool {
   std::vector<std::thread> threads;
   std::mutex m;
   std::condition_variable cvStart, cvDone;
   std::function<void(int, int)> job; // (worker, nWorkers)
   uint64_t generation = 0;
   int running = 0;
   bool stop = false;
   void main(int id);

   public:
   explicit HostPool(int n);
   ~HostPool();
   int size() const { return (int) threads.size() + 1; }
   void run(const std::function<void(int, int)>& fn); // caller is worker 0
};
struct PinnedSlot {
   void* host = nullptr;
   cudaEvent_t done = nullptr;
   bool inFlight = false;
};

struct KernelFamilyTimer {
   std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;
   double totalMs = 0;
   int64_t launches = 0;
};

class StagingEngine;
struct PackedBatch;

} // namespace ldb

struct LdbState;
struct LdbTable;

struct LdbGraph;
struct LdbContext {
   LdbGraph* capturing = nullptr; // non-null between ldb_gpu_graph_begin and _end: launches are recorded, not run
   int device = 0;
   int smCount = 0;
   cudaDeviceProp prop{};
   cudaStream_t compute = nullptr, copy = nullptr;
   cudaEvent_t timerStart = nullptr, timerStop = nullptr, computeDone = nullptr;
   int64_t launches = 0;
   bool timing = false;
   std::map<std::string, ldb::KernelFamilyTimer> timers;
   std::vector<cudaEvent_t> eventPool;
   std::vector<LdbState*> states;
   std::vector<LdbTable*> tables;
   std::vector<LdbGraph*> graphs;
   std::map<std::string, LdbState*> namedStates; // states created / registered through serialised steps (step_json.cpp)
   // staging pool for HOST batches: size → free device buffers
   std::multimap<size_t, void*> stagingFree;
   std::map<void*, size_t> stagingSize;
   // narrow staging: decimal128(p<19) HOST columns cross PCIe as 8 bytes/value (the JIT truncates them to i64 anyway)
   bool narrowStaging = true;
   std::unique_ptr<ldb::HostPool> pool;
   static constexpr size_t kPinnedSlotBytes = 32u << 20;
   std::vector<ldb::PinnedSlot> pinned;
   size_t nextPinned = 0;
   std::atomic<int64_t> h2dBytes{0}; // bytes this context copied host→device while staging tables
   // compressed staging (staging.h): HOST batches of >= one block are re-encoded by a pool of independent pipelines
   bool packedStaging = true;
   std::shared_ptr<ldb::StagingEngine> staging;
   std::atomic<uint64_t> stagingGen{0};      // bumped by ldb_gpu_table_clear: workers order their next write after computeDone
   std::atomic<int64_t> stagingLaunches{0};  // unpack kernels launched by the staging workers
   std::atomic<int64_t> rawStagedRows{0};    // rows the raw copiers shipped uncompressed (the rest was packed)
   // encoded column copies of DEVICE batches (encode.cu, LdbBatch::enc): built on their own stream, never captured
   cudaStream_t encodeStream = nullptr;
   int64_t encodedBytes = 0;              // device bytes the copies hold now
   int64_t encodedBudget = INT64_MAX;     // LDB_ENCODED_SCAN_MAX_BYTES: beyond it batches are scanned in Arrow layout
   int64_t encodeLaunches = 0;            // encoder kernels launched (part of ldb_gpu_launch_count)

   // Host waits SLEEP instead of spinning (cudaEventBlockingSync): the container's CPU quota is shared with the staging
   // threads and, on a multi-GPU box, with the other ranks — a spinning waiter would burn a whole CPU of it.
   // Short waits (a query's result read: the stream drains within a few hundred microseconds) poll, long ones sleep.
   cudaEvent_t blockingEv = nullptr;
   void syncStream(cudaStream_t s) {
      if (!blockingEv) LDB_CUDA(cudaEventCreateWithFlags(&blockingEv, cudaEventBlockingSync | cudaEventDisableTiming));
      LDB_CUDA(cudaEventRecord(blockingEv, s));
      for (int spin = 0; spin < 20000; spin++) { // ~0.3 ms of polling
         cudaError_t q = cudaEventQuery(blockingEv);
         if (q == cudaSuccess) return;
         if (q != cudaErrorNotReady) LDB_CUDA(q);
      }
      LDB_CUDA(cudaEventSynchronize(blockingEv));
   }
   // pinned scratch for small result reads: a copy into pageable memory would be staged by the driver and serialise with the host
   void* pinnedScratch = nullptr;
   static constexpr size_t kPinnedScratchBytes = 1u << 20; // the sort exchange reads every rank's samples into it
   void* scratch() {
      if (!pinnedScratch) LDB_CUDA(cudaMallocHost(&pinnedScratch, kPinnedScratchBytes));
      return pinnedScratch;
   }
   void launchCaptured(const char* family, const std::function<void()>& fn); // runtime.cpp
   void* stagingAlloc(size_t bytes);
   void stagingRelease(void* p);
   cudaEvent_t getEvent();
   // wrap one kernel launch: counts it and, when timing is on, brackets it with events on `compute`
   template <class Fn>
   void launch(const char* family, const Fn& fn) {
      if (capturing) {
         launchCaptured(family, [&] { fn(); });
         LDB_CUDA(cudaGetLastError());
         return;
      }
      launches++;
      if (timing) {
         auto& t = timers[family];
         cudaEvent_t a = getEvent(), b = getEvent();
         LDB_CUDA(cudaEventRecord(a, compute));
         fn();
         LDB_CUDA(cudaEventRecord(b, compute));
         t.pending.push_back({a, b});
         t.launches++;
      } else {
         fn();
      }
      LDB_CUDA(cudaGetLastError());
   }
};

namespace ldb {
// The scratch device buffers of one call, from the context's staging pool, given back to it when the scope ends.  A call that
// returns normally has already waited for the kernels that read them (it reads their results on the host); no wait is added
// here because some of these calls run inside a graph capture.  A call that throws may leave such kernels queued: then the
// compute stream is drained first, without throwing (and not while capturing, where nothing runs yet).
class Scratch {
   LdbContext* ctx;
   std::vector<void*> bufs;
   const int uncaught = std::uncaught_exceptions();

   public:
   explicit Scratch(LdbContext* c) : ctx(c) {}
   Scratch(const Scratch&) = delete;
   Scratch& operator=(const Scratch&) = delete;
   ~Scratch() {
      if (bufs.empty()) return;
      if (std::uncaught_exceptions() > uncaught && !ctx->capturing) {
         cudaStreamSynchronize(ctx->compute);
         cudaGetLastError();
      }
      for (void* p : bufs) ctx->stagingRelease(p);
   }
   template <class T = void>
   T* alloc(size_t bytes) {
      bufs.reserve(bufs.size() + 1); // the push_back below cannot throw once the buffer is taken from the pool
      void* p = ctx->stagingAlloc(bytes);
      bufs.push_back(p);
      return (T*) p;
   }
   bool empty() const { return bufs.empty(); }
   // the buffers now belong to the caller (a result table's LdbBatch::owned)
   std::vector<void*> take() {
      std::vector<void*> out;
      out.swap(bufs);
      return out;
   }
};
} // namespace ldb

struct LdbBatch {
   int64_t nRows = 0;
   std::vector<const void*> data;  // per column: values / utf8 offsets (device)
   std::vector<const void*> bytes; // per column: utf8 bytes (device) or null
   std::vector<int32_t> elemBytes; // per column: bytes per value as staged (decimal128: 16, or 8 when narrowed)
   std::vector<const void*> validity;      // per column: Arrow validity bitmap on the device (null = no nulls in this batch)
   std::vector<int64_t> validityBitOffset; // bit index of row 0 inside the bitmap
   std::vector<uint8_t*> validBytes;       // per column: one validity byte per row (tables this library produced), else empty / null
   std::vector<void*> owned;       // staging buffers to give back on clear
   cudaEvent_t ready = nullptr;    // H2D of this batch finished (null for borrowed device batches)
   std::shared_ptr<ldb::PackedBatch> packed; // columns staged through the compressed staging engine (host wait + worker events)
   bool borrowed = false;          // appended as LDB_MEM_DEVICE: the caller's buffers, unchanged while the batch belongs to the table
   // per column: frame-of-reference copy read by the K1/K2 scan instead of the Arrow cells (kernels.h kEncodeTileHeader), empty until
   // the first such pipeline needs it
   struct Encoded {
      uint8_t* data = nullptr;
      int32_t width = 0, tileRows = 0;
      int64_t bytes = 0;
      int64_t min = 0, max = 0; // of the batch's column, for the factored Q1 scan (kernels.h GroupByParams::encMin)
      bool failed = false; // allocation failed or over the budget: this batch is scanned in Arrow layout
   };
   std::vector<Encoded> enc;
};
struct LdbColumn {
   std::string name;
   int32_t type, precision, scale;
};
struct LdbTable {
   LdbContext* ctx;
   std::string name;
   std::vector<LdbColumn> columns;
   std::vector<LdbBatch> batches;
   int64_t numRows = 0;
   // column statistics (min, max) of int32/date32 columns, computed on first use and valid while the table has `rows` rows: the planner
   // asks for them on every query (direct-address join tables), the table does not change between two queries
   struct ColumnRange {
      int64_t rows;
      int32_t lo, hi;
   };
   std::map<int, ColumnRange> ranges;
   int colIndex(const char* n) const {
      if (!n) return -1;
      for (size_t i = 0; i < columns.size(); i++)
         if (columns[i].name == n) return (int) i;
      return -1;
   }
};

// A captured query (CUDA graph of everything enqueued on the compute stream between _begin and _end): one cudaGraphLaunch
// replays memsets, pipeline kernels and peer collectives without per-launch host work.
struct LdbGraph {
   LdbContext* ctx = nullptr;
   cudaGraph_t graph = nullptr;
   cudaGraphExec_t exec = nullptr;
   int64_t kernelsPerLaunch = 0;
   struct Timer {
      std::string family;
      cudaEvent_t a, b; // recorded by the graph itself (external event-record nodes)
   };
   std::vector<Timer> timers;
   bool pendingTimes = false; // the last launch's events were not harvested yet
   std::vector<std::function<void()>> onLaunch; // host-side bookkeeping per replay (peer epoch mirrors)
};

// order the compute stream after the staging of one batch (runtime.cpp)
void ldb_gpu_wait_batch_internal(LdbContext* ctx, const struct LdbBatch* b);
namespace ldb {
// the pointers of column `ci` of batch `b` as a program reads them (validity bitmap or validity bytes included; program_rt.cpp)
void bindColumn(ProgCol& pc, const LdbBatch& b, int ci);
// registers a single-batch table this library made: `b` holds nRows and, per column, data / bytes / elemBytes / validBytes; the table
// takes over the device buffers of `buffers` (program_rt.cpp)
LdbTable* addResultTable(LdbContext* ctx, std::string name, std::vector<LdbColumn> columns, LdbBatch b, Scratch& buffers);
// row ids of the single-batch table `t` (n rows, n < 2^32) ordered by the keys (column index, descending), in `scratch`: ORDER BY,
// dictionary ranks and the union of a unified dictionary (program_rt.cpp)
uint32_t* sortRows(Scratch& scratch, LdbTable* t, const std::vector<std::pair<int, int>>& keys, int64_t n);
// the cell width of a column of `type` in the single-batch tables the exchanges and the window operator make: a decimal in 16 bytes
// whatever width it was staged at
inline int32_t shipCellBytes(int type) {
   switch (type) {
      case LDB_INT8: return 1;
      case LDB_INT16: return 2;
      case LDB_INT64:
      case LDB_FLOAT64: return 8;
      case LDB_DECIMAL128: return 16;
      default: return 4; // int32, date32, fsb4, float32
   }
}
// rows ids[0..n) (null: 0..n-1) of columns `cols` of `t` (any number of batches, at most 16 columns) as a new single-batch LdbBatch whose
// buffers are in `bufs`: fixed-width cells at outBytes[j] bytes (a narrowed decimal widened to 16), validity bytes, utf8 offsets and
// bytes.  An id of 0xffffffff makes a row of NULL cells (zero bytes, validity 0, empty strings).  Synchronises.  The sort exchange, the
// window, set and nested-loop join operators (peer.cu)
LdbBatch permuteRows(LdbTable* t, const std::vector<int>& cols, const int32_t* outBytes, const uint32_t* ids, int64_t n, Scratch& bufs, const char* what);
} // namespace ldb
// builds the missing encoded copies of columns cols[0..n) of a borrowed DEVICE batch (encode.cu) for tiles of `tileRows` rows;
// true when every one of them has a copy.  Runs outside any capture and waits for its work on the host.
bool ldb_gpu_encode_batch_internal(LdbContext* ctx, LdbTable* t, LdbBatch& b, const int* cols, int n, int tileRows);
// frees the encoded copies of a batch (the caller made sure no queued kernel reads them)
void ldb_gpu_free_encoded_internal(LdbContext* ctx, LdbBatch& b);

struct LdbState {
   LdbContext* ctx;
   int32_t kind;
   ldb::GroupTableDev group{}; // SIMPLE / GROUPBY
   ldb::JoinTableDev join{};   // JOIN_TABLE
   ldb::HashAggDev hashagg{};  // HASHAGG
   ldb::DictDev dict{};        // DICT
   ldb::KeyJoinDev keyJoin{};  // KEY_JOIN
   int32_t aggKinds[ldb::kProgMaxAggs] = {};
   int32_t nSide = 0, nAggs = 0;
   bool selfTimed = false; // created inside a captured query: its scan kernel's self-measured time is harvested at read
   uint32_t is64Mask = 0;   // aggregates that are 64-bit sums (COL / ONE): normalised to a sign-extended i64 on read
   uint32_t laneBound = 0;  // aggregates whose width (64 / 128 bits) a pipeline fixed already: a later one must agree
   uint8_t* marks = nullptr; // JOIN_TABLE / KEY_JOIN: one marker byte per directory slot (program.h), from the first program that marks
                             // the table; also in `allocations`
   bool unified = false;     // DICT made by ldb_gpu_dict_unify: its codes agree across ranks, so programs may only look strings up in it
   std::vector<void*> allocations;
};

// a new, empty string dictionary with room for `expected_strings` strings of `expected_bytes` bytes (ldb_gpu_dict_create, program_rt.cpp)
LdbState* ldb_gpu_dict_new_internal(LdbContext* ctx, int64_t expected_strings, int64_t expected_bytes);
// a dictionary's counters {arena bytes, codes}, after its error word is checked: LDB_ERR_CAPACITY when it overflowed (synchronises)
std::pair<int64_t, int64_t> ldb_gpu_dict_counters_internal(LdbState* s);
// reads a join table's error word (synchronises the compute stream) and throws ApiError with the status and message of a
// non-zero code (runtime.cpp); every caller that reports a join table's failure goes through it
void ldb_gpu_check_join_error_internal(LdbState* s);
// the same for a key-tuple join table (LDB_STATE_KEY_JOIN, program_rt.cpp)
void ldb_gpu_check_keyjoin_error_internal(LdbState* s);
// fixes the width of aggregate lane `lane` of a group state from the LdbExprKind summed into it (64-bit COL / ONE, else 128-bit);
// throws ApiError(LDB_ERR_UNSUPPORTED) when an earlier pipeline fixed the other width (runtime.cpp)
void ldb_gpu_bind_lane_width_internal(LdbState* s, int lane, int expr);
// merges read a lane at the width of their TARGET: throws ApiError(LDB_ERR_UNSUPPORTED) while one of its aggregate lanes is unbound
void ldb_gpu_want_bound_lanes_internal(LdbState* s);
