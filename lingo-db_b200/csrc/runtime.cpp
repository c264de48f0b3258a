// runtime.cpp — C++ host runtime behind the C-ABI (include/ldb_gpu.h): context, HBM staging of
// Arrow batches, device state objects, descriptor → kernel dispatch.  Host side of the reference's
// src/runtime surface for the three hot paths; there is NO CPU fallback: without a CUDA device
// every entry point fails with LDB_ERR_NO_DEVICE.
#include "context.h"
#include "peer.h"
#include "staging.h"

#include <algorithm>
#include <cstdio>
#include <cstring>

using namespace ldb;

// ------------------------------------------------------------------------------------------------ helpers
namespace {
size_t elemWidth(int type) {
   switch (type) {
      case LDB_INT32:
      case LDB_DATE32:
      case LDB_FSB4:
      case LDB_UTF8: return 4; // utf8: offsets
      case LDB_INT64:
      case LDB_FLOAT64: return 8;
      case LDB_DECIMAL128: return 16;
      case LDB_INT8: return 1;
      case LDB_INT16: return 2;
      case LDB_FLOAT32: return 4;
   }
   fail(LDB_ERR_INVALID, "unknown physical type");
}
// "YYYY-MM-DD" → days since epoch (constant parsing of Restrictions.cpp:17-25)
int32_t parseDate32(const char* s) {
   int y, m, d;
   if (!s || sscanf(s, "%d-%d-%d", &y, &m, &d) != 3) fail(LDB_ERR_INVALID, "could not parse date");
   y -= m <= 2;
   int era = (y >= 0 ? y : y - 399) / 400;
   unsigned yoe = (unsigned) (y - era * 400);
   unsigned doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
   unsigned doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
   return era * 146097 + (int) doe - 719468;
}
// decimal constant at the column's scale (Restrictions.cpp:455-480)
int64_t parseDecimal(const char* s, int scale) {
   if (!s) fail(LDB_ERR_INVALID, "missing decimal constant");
   bool neg = false;
   size_t i = 0, n = strlen(s);
   if (i < n && (s[i] == '-' || s[i] == '+')) neg = s[i++] == '-';
   __int128 v = 0;
   int sc = 0;
   bool dot = false;
   for (; i < n; i++) {
      if (s[i] == '.') {
         dot = true;
         continue;
      }
      if (s[i] < '0' || s[i] > '9') fail(LDB_ERR_INVALID, "could not parse decimal const");
      v = v * 10 + (s[i] - '0');
      if (dot) sc++;
   }
   for (; sc < scale; sc++) v *= 10;
   for (; sc > scale; sc--) {
      if (v % 10) fail(LDB_ERR_INVALID, "decimal rescale would lose data");
      v /= 10;
   }
   if (v > (__int128) INT64_MAX) fail(LDB_ERR_UNSUPPORTED, "decimal constant beyond 64 bits");
   return (int64_t) (neg ? -v : v);
}
uint32_t opMask(int op) {
   switch (op) {
      case LDB_EQ: return 2;
      case LDB_NEQ: return 5;
      case LDB_LT: return 1;
      case LDB_LTE: return 3;
      case LDB_GT: return 4;
      case LDB_GTE: return 6;
   }
   fail(LDB_ERR_UNSUPPORTED, "unsupported filter op"); // same message as Restrictions.cpp:346
}
} // namespace

namespace {
// order the compute stream after the staging of one batch
void waitBatch(LdbContext* ctx, const LdbBatch& b) {
   // inside a captured query the staging must be COMPLETE (a captured stream cannot depend on uncaptured copy streams): wait on the host
   const bool capturing = ctx->capturing != nullptr;
   if (b.ready) {
      if (capturing) LDB_CUDA(cudaEventSynchronize(b.ready));
      else LDB_CUDA(cudaStreamWaitEvent(ctx->compute, b.ready, 0));
   }
   if (b.packed) { // compressed staging: every task of the batch issued (host), then order the scan after the workers' streams
      StagingEngine::wait(*b.packed);
      for (size_t w = 0; w < b.packed->used.size(); w++) {
         if (!b.packed->used[w]) continue;
         if (capturing) LDB_CUDA(cudaEventSynchronize(ctx->staging->events[w]));
         else LDB_CUDA(cudaStreamWaitEvent(ctx->compute, ctx->staging->events[w], 0));
      }
   }
}
}

void ldb_gpu_wait_batch_internal(LdbContext* ctx, const LdbBatch* b) { waitBatch(ctx, *b); }

// ------------------------------------------------------------------------------------------------ host pool
namespace ldb {
HostPool::HostPool(int n) {
   for (int i = 1; i < n; i++) threads.emplace_back([this, i] { main(i); });
}
HostPool::~HostPool() {
   {
      std::unique_lock<std::mutex> l(m);
      stop = true;
   }
   cvStart.notify_all();
   for (auto& t : threads) t.join();
}
void HostPool::main(int id) {
   uint64_t seen = 0;
   while (true) {
      std::function<void(int, int)> fn;
      {
         std::unique_lock<std::mutex> l(m);
         cvStart.wait(l, [&] { return stop || generation != seen; });
         if (stop) return;
         seen = generation;
         fn = job;
      }
      fn(id, size());
      std::unique_lock<std::mutex> l(m);
      if (--running == 0) cvDone.notify_all();
   }
}
void HostPool::run(const std::function<void(int, int)>& fn) {
   {
      std::unique_lock<std::mutex> l(m);
      job = fn;
      running = (int) threads.size();
      generation++;
   }
   cvStart.notify_all();
   fn(0, size());
   std::unique_lock<std::mutex> l(m);
   cvDone.wait(l, [&] { return running == 0; });
}
} // namespace ldb

// decimal128 cells → their low 8 bytes, `n` values, all pool workers
static void narrowDecimals(LdbContext* ctx, const uint8_t* src, int64_t n, uint64_t* dst) {
   ctx->pool->run([&](int w, int nw) {
      int64_t per = (n + nw - 1) / nw, b = per * w, e = std::min<int64_t>(n, b + per);
      const uint64_t* s = reinterpret_cast<const uint64_t*>(src);
      for (int64_t i = b; i < e; i++) dst[i] = s[2 * i];
   });
}

// ------------------------------------------------------------------------------------------------ context
void* LdbContext::stagingAlloc(size_t bytes) {
   bytes = std::max<size_t>(256, (bytes + 255) & ~size_t(255));
   auto it = stagingFree.lower_bound(bytes);
   if (it != stagingFree.end() && it->first <= bytes + bytes / 4) {
      void* p = it->second;
      stagingFree.erase(it);
      return p;
   }
   void* p = nullptr;
   LDB_CUDA(cudaMalloc(&p, bytes));
   stagingSize[p] = bytes;
   return p;
}
void LdbContext::stagingRelease(void* p) { stagingFree.insert({stagingSize.at(p), p}); }
cudaEvent_t LdbContext::getEvent() {
   cudaEvent_t e;
   if (!eventPool.empty()) {
      e = eventPool.back();
      eventPool.pop_back();
      return e;
   }
   LDB_CUDA(cudaEventCreate(&e));
   return e;
}

// a launch while the compute stream is being captured: bracket it with EXTERNAL event-record nodes so that every replay of the
// graph times the kernel, like the eager path does (ldb_gpu_kernel_time harvests them)
void LdbContext::launchCaptured(const char* family, const std::function<void()>& fn) {
   LdbGraph* g = capturing;
   g->kernelsPerLaunch++;
   static const bool timers = [] {
      const char* e = getenv("LDB_GRAPH_TIMERS");
      return e && e[0] == '1';
   }();
   if (!timers) { // default: no event-record nodes in the graph (each costs ~10-20 us of replay latency); the group-by scan kernel
      fn();       // times itself through %globaltimer instead (LDB_GRAPH_TIMERS=1 brings the event nodes back for every kernel)
      return;
   }
   cudaEvent_t a = nullptr, b = nullptr;
   LDB_CUDA(cudaEventCreate(&a));
   LDB_CUDA(cudaEventCreate(&b));
   g->timers.push_back({family, a, b});
   LDB_CUDA(cudaEventRecordWithFlags(a, compute, cudaEventRecordExternal));
   fn();
   LDB_CUDA(cudaEventRecordWithFlags(b, compute, cudaEventRecordExternal));
}

extern "C" {

int ldb_gpu_context_create(int device, LdbContext** out, LdbError* err) {
   return guarded(err, [&] {
      int n = 0;
      cudaError_t e = cudaGetDeviceCount(&n);
      if (e != cudaSuccess || n == 0) {
         cudaGetLastError();
         fail(LDB_ERR_NO_DEVICE, "no CUDA device available: the GPU operator runtime has no CPU fallback");
      }
      if (device < 0 || device >= n) fail(LDB_ERR_INVALID, "device index out of range");
      LDB_CUDA(cudaSetDevice(device));
      auto ctx = std::make_unique<LdbContext>();
      ctx->device = device;
      LDB_CUDA(cudaGetDeviceProperties(&ctx->prop, device));
      ctx->smCount = ctx->prop.multiProcessorCount;
      LDB_CUDA(cudaStreamCreateWithFlags(&ctx->compute, cudaStreamNonBlocking));
      LDB_CUDA(cudaStreamCreateWithFlags(&ctx->copy, cudaStreamNonBlocking));
      LDB_CUDA(cudaEventCreate(&ctx->timerStart));
      LDB_CUDA(cudaEventCreate(&ctx->timerStop));
      LDB_CUDA(cudaEventCreateWithFlags(&ctx->computeDone, cudaEventDisableTiming));
      if (const char* e = getenv("LDB_NARROW_STAGING")) ctx->narrowStaging = atoi(e) != 0;
      if (const char* e = getenv("LDB_PACKED_STAGING")) ctx->packedStaging = atoi(e) != 0;
      if (const char* e = getenv("LDB_ENCODED_SCAN_MAX_BYTES")) ctx->encodedBudget = std::max<int64_t>(0, atoll(e));
      *out = ctx.release();
   });
}
void ldb_gpu_table_destroy(LdbTable* t);
static void destroyState(LdbState* s) { // device memory goes back to the context's pool
   for (void* p : s->allocations) s->ctx->stagingRelease(p);
   delete s;
}
void ldb_gpu_context_destroy(LdbContext* ctx) {
   if (!ctx) return;
   cudaSetDevice(ctx->device);
   cudaDeviceSynchronize();
   while (!ctx->tables.empty()) ldb_gpu_table_destroy(ctx->tables.back());
   ctx->staging.reset(); // joins the staging workers (their streams are drained first)
   for (auto* s : ctx->states) destroyState(s);
   for (auto& kv : ctx->stagingSize) cudaFree(kv.first);
   for (auto& ps : ctx->pinned) {
      if (ps.host) cudaFreeHost(ps.host);
      if (ps.done) cudaEventDestroy(ps.done);
   }
   for (auto e : ctx->eventPool) cudaEventDestroy(e);
   for (auto& kv : ctx->timers)
      for (auto& pr : kv.second.pending) {
         cudaEventDestroy(pr.first);
         cudaEventDestroy(pr.second);
      }
   cudaEventDestroy(ctx->timerStart);
   cudaEventDestroy(ctx->timerStop);
   cudaEventDestroy(ctx->computeDone);
   if (ctx->blockingEv) cudaEventDestroy(ctx->blockingEv);
   if (ctx->pinnedScratch) cudaFreeHost(ctx->pinnedScratch);
   cudaStreamDestroy(ctx->compute);
   cudaStreamDestroy(ctx->copy);
   if (ctx->encodeStream) cudaStreamDestroy(ctx->encodeStream);
   delete ctx;
}
int ldb_gpu_device_info(LdbContext* ctx, LdbDeviceInfo* out, LdbError* err) {
   return guarded(err, [&] {
      if (!ctx || !out) fail(LDB_ERR_INVALID, "null argument");
      LDB_CUDA(cudaSetDevice(ctx->device));
      memset(out, 0, sizeof(*out));
      out->device = ctx->device;
      out->sm_count = ctx->smCount;
      out->cc_major = ctx->prop.major;
      out->cc_minor = ctx->prop.minor;
      out->l2_bytes = ctx->prop.l2CacheSize;
      size_t fr, tot;
      LDB_CUDA(cudaMemGetInfo(&fr, &tot));
      out->total_mem = (int64_t) tot;
      out->free_mem = (int64_t) fr;
      snprintf(out->name, sizeof(out->name), "%s", ctx->prop.name);
   });
}
int ldb_gpu_synchronize(LdbContext* ctx, LdbError* err) {
   return guarded(err, [&] {
      ctx->syncStream(ctx->copy);
      ctx->syncStream(ctx->compute);
   });
}
void* ldb_gpu_context_stream(LdbContext* ctx) { return ctx ? (void*) ctx->compute : nullptr; }
int64_t ldb_gpu_context_h2d_bytes(LdbContext* ctx) { return ctx ? ctx->h2dBytes.load() : 0; }
int64_t ldb_gpu_context_raw_staged_rows(LdbContext* ctx) { return ctx ? ctx->rawStagedRows.load() : 0; }
int32_t ldb_gpu_effective_cpus(void) { return effectiveCpus(); }
void ldb_gpu_set_tuning(int32_t stages_build, int32_t stages_probe_agg, int32_t stages_probe2, int32_t stages_star, int32_t rows_per_thread_build) {
   Tuning t = tuning();
   t.stagesBuild = stages_build;
   t.stagesProbeAgg = stages_probe_agg;
   t.stagesProbe2 = stages_probe2;
   t.stagesStar = stages_star;
   t.rptBuild = rows_per_thread_build;
   setTuning(t);
}
void ldb_gpu_set_filter_specialisation(int32_t on) {
   Tuning t = tuning();
   t.specialise = on ? 1 : 0;
   setTuning(t);
}
void ldb_gpu_set_encoded_scan(int32_t on) {
   Tuning t = tuning();
   t.encodedScan = on ? 1 : 0;
   setTuning(t);
}
int64_t ldb_gpu_context_encoded_bytes(LdbContext* ctx) { return ctx ? ctx->encodedBytes : 0; }
void ldb_gpu_set_poll_pause(int32_t producer_ns, int32_t consumer_ns) {
   Tuning t = tuning();
   t.producerSleepNs = producer_ns;
   t.consumerSleepNs = consumer_ns;
   setTuning(t);
}
int64_t ldb_gpu_launch_count(LdbContext* ctx) { return ctx ? ctx->launches + ctx->stagingLaunches.load() + ctx->encodeLaunches : 0; }
int ldb_gpu_timer_start(LdbContext* ctx, LdbError* err) {
   return guarded(err, [&] { LDB_CUDA(cudaEventRecord(ctx->timerStart, ctx->compute)); });
}
int ldb_gpu_timer_stop(LdbContext* ctx, float* ms, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaEventRecord(ctx->timerStop, ctx->compute));
      LDB_CUDA(cudaEventSynchronize(ctx->timerStop));
      LDB_CUDA(cudaEventElapsedTime(ms, ctx->timerStart, ctx->timerStop));
   });
}
int ldb_gpu_kernel_time_reset(LdbContext* ctx, int enable, LdbError* err) {
   return guarded(err, [&] {
      ctx->syncStream(ctx->compute);
      for (auto& kv : ctx->timers) {
         for (auto& pr : kv.second.pending) {
            ctx->eventPool.push_back(pr.first);
            ctx->eventPool.push_back(pr.second);
         }
      }
      ctx->timers.clear();
      ctx->timing = enable != 0;
   });
}
static void harvestGraphTimes(LdbGraph* g);
int ldb_gpu_kernel_time(LdbContext* ctx, const char* family, float* ms, int64_t* launches, LdbError* err) {
   return guarded(err, [&] {
      ctx->syncStream(ctx->compute);
      for (LdbGraph* g : ctx->graphs) harvestGraphTimes(g);
      auto it = ctx->timers.find(family);
      if (it == ctx->timers.end()) {
         *ms = 0;
         *launches = 0;
         return;
      }
      auto& t = it->second;
      for (auto& pr : t.pending) {
         float e = 0;
         LDB_CUDA(cudaEventElapsedTime(&e, pr.first, pr.second));
         t.totalMs += e;
         ctx->eventPool.push_back(pr.first);
         ctx->eventPool.push_back(pr.second);
      }
      t.pending.clear();
      *ms = (float) t.totalMs;
      *launches = t.launches;
   });
}

// ------------------------------------------------------------------------------------------------ captured queries (CUDA graphs)
// Replaces nothing in the reference by name: it is the GPU counterpart of "compile once, run many" (the reference JIT-compiles a
// query's main() once, LLVMBackends.cpp:795-867).  Between _begin and _end the compute stream is in capture mode: pipelines over
// DEVICE-resident (or already staged) tables, state creation and peer collectives are recorded; result reads and anything else that
// synchronises must stay outside.  States created inside the capture are re-initialised by every launch and belong to the caller.
static void harvestGraphTimes(LdbGraph* g) {
   if (!g->pendingTimes) return;
   for (auto& t : g->timers) {
      float ms = 0;
      if (cudaEventElapsedTime(&ms, t.a, t.b) != cudaSuccess) {
         cudaGetLastError();
         return; // not finished yet: the caller has not synchronised — keep them pending
      }
      auto& acc = g->ctx->timers[t.family];
      acc.totalMs += ms;
      acc.launches++;
   }
   g->pendingTimes = false;
}
int ldb_gpu_graph_begin(LdbContext* ctx, LdbError* err) {
   return guarded(err, [&] {
      if (!ctx) fail(LDB_ERR_INVALID, "null context");
      if (ctx->capturing) fail(LDB_ERR_INVALID, "a capture is already in progress");
      LDB_CUDA(cudaSetDevice(ctx->device));
      ctx->syncStream(ctx->compute);
      auto* g = new LdbGraph;
      g->ctx = ctx;
      cudaError_t e = cudaStreamBeginCapture(ctx->compute, cudaStreamCaptureModeRelaxed);
      if (e != cudaSuccess) {
         delete g;
         LDB_CUDA(e);
      }
      ctx->capturing = g;
   });
}
int ldb_gpu_graph_end(LdbContext* ctx, LdbGraph** out, LdbError* err) {
   return guarded(err, [&] {
      if (!ctx || !out || !ctx->capturing) fail(LDB_ERR_INVALID, "no capture in progress");
      LdbGraph* g = ctx->capturing;
      ctx->capturing = nullptr;
      cudaError_t e = cudaStreamEndCapture(ctx->compute, &g->graph);
      if (e == cudaSuccess) e = cudaGraphInstantiate(&g->exec, g->graph, 0);
      if (e != cudaSuccess) {
         if (g->graph) cudaGraphDestroy(g->graph);
         delete g;
         LDB_CUDA(e);
      }
      ctx->graphs.push_back(g);
      *out = g;
   });
}
int ldb_gpu_graph_launch(LdbGraph* g, LdbError* err) {
   return guarded(err, [&] {
      if (!g || !g->exec) fail(LDB_ERR_INVALID, "null graph");
      LdbContext* ctx = g->ctx;
      LDB_CUDA(cudaSetDevice(ctx->device));
      if (ctx->timing) harvestGraphTimes(g);
      LDB_CUDA(cudaGraphLaunch(g->exec, ctx->compute));
      ctx->launches += g->kernelsPerLaunch;
      g->pendingTimes = ctx->timing && !g->timers.empty();
      for (auto& f : g->onLaunch) f();
   });
}
void ldb_gpu_graph_destroy(LdbGraph* g) {
   if (!g) return;
   cudaSetDevice(g->ctx->device);
   cudaStreamSynchronize(g->ctx->compute);
   for (auto& t : g->timers) {
      cudaEventDestroy(t.a);
      cudaEventDestroy(t.b);
   }
   auto& gs = g->ctx->graphs;
   gs.erase(std::remove(gs.begin(), gs.end(), g), gs.end());
   if (g->exec) cudaGraphExecDestroy(g->exec);
   if (g->graph) cudaGraphDestroy(g->graph);
   delete g;
}

// ------------------------------------------------------------------------------------------------ tables
int ldb_gpu_table_create(LdbContext* ctx, const char* name, int32_t n_cols, const LdbColumnSchema* schema, LdbTable** out, LdbError* err) {
   return guarded(err, [&] {
      if (!ctx || !schema || !out) fail(LDB_ERR_INVALID, "null argument");
      auto* t = new LdbTable;
      t->ctx = ctx;
      t->name = name ? name : "";
      for (int i = 0; i < n_cols; i++) {
         elemWidth(schema[i].type);
         t->columns.push_back({schema[i].name, schema[i].type, schema[i].precision, schema[i].scale});
      }
      ctx->tables.push_back(t);
      *out = t;
   });
}
int ldb_gpu_table_append_batch(LdbTable* t, int64_t n_rows, const LdbArrayView* columns, const int64_t* utf8_bytes, int32_t location, LdbError* err) {
   return guarded(err, [&] {
      if (!t || !columns) fail(LDB_ERR_INVALID, "null argument");
      LdbContext* ctx = t->ctx;
      LDB_CUDA(cudaSetDevice(ctx->device));
      LdbBatch b;
      b.nRows = n_rows;
      b.borrowed = location == LDB_MEM_DEVICE;
      size_t nc = t->columns.size();
      b.data.resize(nc);
      b.bytes.assign(nc, nullptr);
      b.elemBytes.assign(nc, 0);
      b.validity.assign(nc, nullptr);
      b.validityBitOffset.assign(nc, 0);
      // compressed staging (staging.h): fixed-width HOST columns of batches that span at least one block are re-encoded by
      // the staging engine's independent pipelines (pack on a host thread → H2D on its stream → decode kernel) and this call
      // returns at once; the Arrow buffers must stay valid until the table is cleared (they belong to the table storage)
      const bool packThis = location != LDB_MEM_DEVICE && ctx->packedStaging && n_rows >= kPackBlockRows;
      std::shared_ptr<PackedBatch> pk;
      if (packThis) {
         if (!ctx->staging) {
            // sized by the CPUs this process may burn (cgroup quota!), minus the caller's thread and the raw copiers
            int nt = std::max(2, std::min(64, effectiveCpus() - 2)), nraw = 2;
            if (const char* e = getenv("LDB_STAGING_THREADS")) nt = std::max(1, std::min(256, atoi(e)));
            if (const char* e = getenv("LDB_STAGING_RAW_THREADS")) nraw = std::max(0, std::min(8, atoi(e)));
            ctx->staging = std::make_shared<StagingEngine>(ctx, nt, nraw);
         }
         pk = std::make_shared<PackedBatch>();
         pk->nRows = n_rows;
      }
      for (size_t c = 0; c < nc; c++) {
         const LdbArrayView& av = columns[c];
         if (av.length < n_rows) fail(LDB_ERR_INVALID, "column shorter than the batch");
         // nullable column: keep its validity bitmap (Arrow: bit i of buffers[0], LSB first, ArrayView.offset applies).  Only the
         // program pipeline reads it; the specialised pipelines refuse batches whose touched columns carry one (StagePlan::bind).
         if (av.null_count != 0 && av.buffers[0] && n_rows > 0) {
            const int64_t firstByte = av.offset / 8, nBytes = (av.offset % 8 + n_rows + 7) / 8;
            if (location == LDB_MEM_DEVICE) {
               b.validity[c] = (const uint8_t*) av.buffers[0] + firstByte;
            } else {
               void* dv = ctx->stagingAlloc((size_t) nBytes);
               b.owned.push_back(dv);
               LDB_CUDA(cudaMemcpyAsync(dv, (const uint8_t*) av.buffers[0] + firstByte, (size_t) nBytes, cudaMemcpyHostToDevice, ctx->copy));
               ctx->h2dBytes.fetch_add(nBytes);
               b.validity[c] = dv;
            }
            b.validityBitOffset[c] = av.offset % 8;
         }
         size_t w = elemWidth(t->columns[c].type);
         bool utf8 = t->columns[c].type == LDB_UTF8;
         const uint8_t* src = (const uint8_t*) av.buffers[1] + (size_t) av.offset * w;
         size_t bytes = (size_t) (n_rows + (utf8 ? 1 : 0)) * w;
         b.elemBytes[c] = (int32_t) w;
         const int ty = t->columns[c].type;
         const bool packable = packThis && (ty == LDB_INT32 || ty == LDB_DATE32 || ty == LDB_FSB4 || ty == LDB_INT64 || (ty == LDB_DECIMAL128 && t->columns[c].precision < 19)) && pk->cols.size() < (size_t) kMaxPackCols;
         if (location == LDB_MEM_DEVICE) {
            b.data[c] = src;
            if (utf8) b.bytes[c] = av.buffers[2];
         } else if (packable) {
            const int kind = ty == LDB_DECIMAL128 ? 2 : ty == LDB_INT64 ? 1 : 0;
            const int outBytes = kind == 0 ? 4 : 8;
            uint8_t* dst = (uint8_t*) ctx->stagingAlloc((size_t) n_rows * outBytes);
            b.owned.push_back(dst);
            pk->cols.push_back(PackedBatch::Col{src, kind, (int32_t) w, dst, outBytes});
            b.data[c] = dst;
            b.elemBytes[c] = outBytes;
         } else if (ctx->narrowStaging && t->columns[c].type == LDB_DECIMAL128 && t->columns[c].precision < 19 && n_rows > 0) {
            // narrow on the host into a ring of pinned slots, copy 8 B/value: chunk k+1 is narrowed while chunk k is on the wire
            if (!ctx->pool) {
               int hw = (int) std::thread::hardware_concurrency();
               // measured on the 2x32-core box (128 hw threads), ms per SF100 Q1 e2e step: 6 thr 796, 10 thr 634, 12 thr 531,
               // 16 thr 621, 20 thr 573, 32 thr 946, 64 thr 1544 (no narrowing: 823) → ~hw/10; more threads fight over one NUMA node
               int nt = std::max(2, std::min(16, hw / 10));
               if (const char* e = getenv("LDB_STAGING_THREADS")) nt = std::max(1, atoi(e));
               ctx->pool = std::make_unique<HostPool>(nt);
               ctx->pinned.resize(4);
               for (auto& ps : ctx->pinned) {
                  LDB_CUDA(cudaMallocHost(&ps.host, LdbContext::kPinnedSlotBytes));
                  LDB_CUDA(cudaEventCreateWithFlags(&ps.done, cudaEventDisableTiming));
               }
            }
            uint8_t* dst = (uint8_t*) ctx->stagingAlloc((size_t) n_rows * 8);
            b.owned.push_back(dst);
            const int64_t chunkRows = (int64_t) (LdbContext::kPinnedSlotBytes / 8);
            for (int64_t r0 = 0; r0 < n_rows; r0 += chunkRows) {
               int64_t m = std::min<int64_t>(chunkRows, n_rows - r0);
               PinnedSlot& ps = ctx->pinned[ctx->nextPinned++ % ctx->pinned.size()];
               if (ps.inFlight) LDB_CUDA(cudaEventSynchronize(ps.done));
               narrowDecimals(ctx, src + (size_t) r0 * 16, m, (uint64_t*) ps.host);
               LDB_CUDA(cudaMemcpyAsync(dst + (size_t) r0 * 8, ps.host, (size_t) m * 8, cudaMemcpyHostToDevice, ctx->copy));
               LDB_CUDA(cudaEventRecord(ps.done, ctx->copy));
               ps.inFlight = true;
               ctx->h2dBytes += m * 8;
            }
            b.data[c] = dst;
            b.elemBytes[c] = 8;
         } else {
            void* dst = ctx->stagingAlloc(bytes);
            b.owned.push_back(dst);
            LDB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->copy));
            ctx->h2dBytes += (int64_t) bytes;
            b.data[c] = dst;
            if (utf8) {
               if (!utf8_bytes) fail(LDB_ERR_INVALID, "utf8 column needs utf8_bytes");
               size_t sb = std::max<int64_t>(utf8_bytes[c], 1);
               void* d2 = ctx->stagingAlloc(sb);
               b.owned.push_back(d2);
               LDB_CUDA(cudaMemcpyAsync(d2, av.buffers[2], (size_t) utf8_bytes[c], cudaMemcpyHostToDevice, ctx->copy));
               ctx->h2dBytes += utf8_bytes[c];
               b.bytes[c] = d2;
            }
         }
      }
      if (location != LDB_MEM_DEVICE) {
         b.ready = ctx->getEvent();
         LDB_CUDA(cudaEventRecord(b.ready, ctx->copy));
      }
      if (pk && !pk->cols.empty()) {
         b.packed = pk;
         ctx->staging->submit(pk);
      }
      t->numRows += n_rows;
      t->ranges.clear();
      t->batches.push_back(std::move(b));
   });
}
int ldb_gpu_table_clear(LdbTable* t, LdbError* err) {
   return guarded(err, [&] {
      LdbContext* ctx = t->ctx;
      // staging workers may still be writing into buffers released below: let them finish issuing (host wait, errors ignored)
      for (auto& b : t->batches)
         if (b.packed) {
            try {
               StagingEngine::wait(*b.packed);
            } catch (const std::exception&) {
            }
            for (size_t w = 0; w < b.packed->used.size(); w++)
               if (b.packed->used[w]) LDB_CUDA(cudaStreamWaitEvent(ctx->compute, ctx->staging->events[w], 0));
         }
      // staged buffers may still be read by queued kernels: later copies wait for the compute stream
      LDB_CUDA(cudaEventRecord(ctx->computeDone, ctx->compute));
      LDB_CUDA(cudaStreamWaitEvent(ctx->copy, ctx->computeDone, 0));
      ctx->stagingGen.fetch_add(1);
      bool encoded = false;
      for (auto& b : t->batches) encoded |= !b.enc.empty();
      if (encoded && !ctx->capturing) ctx->syncStream(ctx->compute); // queued scans may still read the encoded copies freed below
      for (auto& b : t->batches) {
         ldb_gpu_free_encoded_internal(ctx, b);
         for (void* p : b.owned) ctx->stagingRelease(p);
         if (b.ready) ctx->eventPool.push_back(b.ready);
      }
      t->batches.clear();
      t->numRows = 0;
      t->ranges.clear();
   });
}
int64_t ldb_gpu_table_num_rows(const LdbTable* t) { return t ? t->numRows : 0; }
void ldb_gpu_table_destroy(LdbTable* t) {
   if (!t) return;
   LdbContext* ctx = t->ctx;
   cudaStreamSynchronize(ctx->compute);
   LdbError e;
   ldb_gpu_table_clear(t, &e);
   ctx->tables.erase(std::remove(ctx->tables.begin(), ctx->tables.end(), t), ctx->tables.end());
   delete t;
}

// ------------------------------------------------------------------------------------------------ states
static void* devAlloc(LdbState* s, size_t bytes, int fillByte) {
   void* p = s->ctx->stagingAlloc(std::max<size_t>(bytes, 16));
   s->allocations.push_back(p);
   LDB_CUDA(cudaMemsetAsync(p, fillByte, std::max<size_t>(bytes, 16), s->ctx->compute));
   return p;
}
static LdbState* newGroupState(LdbContext* ctx, int kind, int nKeys, int nAggs, int capacity) {
   if (nAggs < 1 || nAggs > kMaxAggs) fail(LDB_ERR_INVALID, "n_aggs out of range");
   if (nKeys < 0 || nKeys > kMaxKeys) fail(LDB_ERR_INVALID, "n_keys out of range");
   LDB_CUDA(cudaSetDevice(ctx->device));
   auto* s = new LdbState;
   s->ctx = ctx;
   s->kind = kind;
   ctx->states.push_back(s);
   auto& g = s->group;
   g.capacity = nKeys == 0 ? 2 : (int) nextPow2((uint64_t) std::max(capacity, 16)); // keyless: slot 0 only (2 keeps the accumulators 8-byte aligned inside the image)
   g.nKeys = nKeys;
   g.nAggs = nAggs;
   // one allocation, one memset: the exchange image (state | keys | acc) followed by the error word
   // … then {error word, pad, self-timing words max(~start), max(end)} — kernels.cu scanGroupByKernel
   const size_t image = groupImageBytes(g.capacity);
   uint8_t* base = (uint8_t*) devAlloc(s, image + 32, 0);
   s->selfTimed = ctx->capturing != nullptr; // a state created inside a captured query reports its kernel time through the table
   g.state = (int32_t*) base;
   g.keys = (int32_t*) (base + (size_t) g.capacity * 4);
   g.acc = (unsigned long long*) (base + (size_t) g.capacity * 4 + (size_t) g.capacity * kMaxKeys * 4);
   g.error = (int32_t*) (base + image);
   s->nAggs = nAggs;
   return s;
}
void ldb_gpu_state_destroy(LdbState* s) {
   if (!s) return;
   LdbContext* ctx = s->ctx;
   cudaSetDevice(ctx->device);
   cudaStreamSynchronize(ctx->compute);
   ctx->states.erase(std::remove(ctx->states.begin(), ctx->states.end(), s), ctx->states.end());
   for (auto it = ctx->namedStates.begin(); it != ctx->namedStates.end();) it = it->second == s ? ctx->namedStates.erase(it) : std::next(it);
   destroyState(s);
}
int ldb_gpu_simple_state_create(LdbContext* ctx, int32_t n_aggs, LdbState** out, LdbError* err) {
   return guarded(err, [&] { *out = newGroupState(ctx, LDB_STATE_SIMPLE, 0, n_aggs, 1); });
}
int ldb_gpu_groupby_create(LdbContext* ctx, int32_t n_keys, int32_t n_aggs, int32_t capacity, LdbState** out, LdbError* err) {
   return guarded(err, [&] {
      if (n_keys < 1) fail(LDB_ERR_INVALID, "group-by needs at least one key (use a simple state)");
      *out = newGroupState(ctx, LDB_STATE_GROUPBY, n_keys, n_aggs, capacity);
   });
}
static void checkGroupError(LdbState* s) {
   int32_t e = 0;
   LDB_CUDA(cudaMemcpyAsync(&e, s->group.error, sizeof(e), cudaMemcpyDeviceToHost, s->ctx->compute));
   s->ctx->syncStream(s->ctx->compute);
   if (e) fail(LDB_ERR_CAPACITY, "group-by table overflow: more groups than the declared capacity");
}
int ldb_gpu_simple_state_read(LdbState* s, LdbI128* aggs, LdbError* err) {
   return guarded(err, [&] {
      if (!s || s->kind != LDB_STATE_SIMPLE) fail(LDB_ERR_INVALID, "not a simple state");
      unsigned long long* h = (unsigned long long*) s->ctx->scratch();
      LDB_CUDA(cudaMemcpyAsync(h, s->group.acc, sizeof(unsigned long long) * kMaxAggs * 2, cudaMemcpyDeviceToHost, s->ctx->compute));
      s->ctx->syncStream(s->ctx->compute);
      for (int a = 0; a < s->nAggs; a++) aggs[a] = (s->is64Mask >> a) & 1u ? LdbI128{h[2 * a], (int64_t) h[2 * a] >> 63} : LdbI128{h[2 * a], (int64_t) h[2 * a + 1]};
   });
}
int ldb_gpu_groupby_read(LdbState* s, LdbGroupRow* rows, int32_t max_rows, int32_t* n_rows, LdbError* err) {
   return guarded(err, [&] {
      if (!s || s->kind != LDB_STATE_GROUPBY) fail(LDB_ERR_INVALID, "not a group-by state");
      auto& g = s->group;
      // the table is one allocation (image + error word): one copy, one synchronisation
      const size_t image = groupImageBytes(g.capacity);
      std::vector<uint8_t> pageable;
      uint8_t* host = (uint8_t*) s->ctx->scratch(); // pinned: the copy is asynchronous, the only wait is the one below
      if (image + 32 > LdbContext::kPinnedScratchBytes) {
         pageable.resize(image + 32);
         host = pageable.data();
      }
      LDB_CUDA(cudaMemcpyAsync(host, g.state, image + 32, cudaMemcpyDeviceToHost, s->ctx->compute));
      s->ctx->syncStream(s->ctx->compute);
      if (s->ctx->timing && s->selfTimed) { // captured queries carry no event nodes: the scan kernel timed itself (%globaltimer)
         const unsigned long long inv = *(const unsigned long long*) (host + image + 8), end = *(const unsigned long long*) (host + image + 16);
         if (inv && end > ~inv) {
            auto& acc = s->ctx->timers["scan_groupby"];
            acc.totalMs += (double) (end - ~inv) / 1e6;
            acc.launches++;
         }
      }
      if (*(const int32_t*) (host + image)) fail(LDB_ERR_CAPACITY, "group-by table overflow: more groups than the declared capacity");
      const int32_t* st = (const int32_t*) host;
      const int32_t* keys = (const int32_t*) (host + (size_t) g.capacity * 4);
      const unsigned long long* acc = (const unsigned long long*) (host + (size_t) g.capacity * 4 + (size_t) g.capacity * kMaxKeys * 4);
      int n = 0;
      for (int i = 0; i < g.capacity; i++) {
         if (st[i] != 2) continue;
         if (n < max_rows) {
            LdbGroupRow& r = rows[n];
            memset(&r, 0, sizeof(r));
            for (int k = 0; k < kMaxKeys; k++) r.keys[k] = keys[(size_t) i * kMaxKeys + k];
            for (int a = 0; a < g.nAggs; a++) {
               const unsigned long long lo = acc[((size_t) i * kMaxAggs + a) * 2];
               // 64-bit aggregates wrap at 64 bits; their hi word only collected carries of the two-word atomics → sign-extend lo
               r.aggs[a] = (s->is64Mask >> a) & 1u ? LdbI128{lo, (int64_t) lo >> 63} : LdbI128{lo, (int64_t) acc[((size_t) i * kMaxAggs + a) * 2 + 1]};
            }
         }
         n++;
      }
      *n_rows = n;
   });
}
int ldb_gpu_groupby_merge_rows(LdbState* s, const LdbGroupRow* rows, int32_t n_rows, LdbError* err) {
   return guarded(err, [&] {
      if (!s || (s->kind != LDB_STATE_GROUPBY && s->kind != LDB_STATE_SIMPLE)) fail(LDB_ERR_INVALID, "not a group state");
      ldb_gpu_want_bound_lanes_internal(s);
      if (n_rows <= 0) return;
      LdbContext* ctx = s->ctx;
      std::vector<int32_t> keys((size_t) n_rows * kMaxKeys);
      std::vector<unsigned long long> acc((size_t) n_rows * kMaxAggs * 2, 0);
      for (int r = 0; r < n_rows; r++) {
         for (int k = 0; k < kMaxKeys; k++) keys[(size_t) r * kMaxKeys + k] = rows[r].keys[k];
         for (int a = 0; a < s->group.nAggs; a++) {
            acc[((size_t) r * kMaxAggs + a) * 2] = rows[r].aggs[a].lo;
            acc[((size_t) r * kMaxAggs + a) * 2 + 1] = (unsigned long long) rows[r].aggs[a].hi;
         }
      }
      Scratch scratch(ctx);
      int32_t* dk = scratch.alloc<int32_t>(keys.size() * 4);
      unsigned long long* da = scratch.alloc<unsigned long long>(acc.size() * 8);
      LDB_CUDA(cudaMemcpyAsync(dk, keys.data(), keys.size() * 4, cudaMemcpyHostToDevice, ctx->compute));
      LDB_CUDA(cudaMemcpyAsync(da, acc.data(), acc.size() * 8, cudaMemcpyHostToDevice, ctx->compute));
      ctx->launch("group_merge", [&] { launchGroupMergeRows(s->group, dk, da, n_rows, ctx->compute); });
      ctx->syncStream(ctx->compute);
   });
}

int64_t ldb_gpu_groupby_export_bytes(LdbState* s) { return s ? (int64_t) groupImageBytes(s->group.capacity) : 0; }
int ldb_gpu_groupby_export(LdbState* s, void* dst, LdbError* err) {
   return guarded(err, [&] {
      if (!s || (s->kind != LDB_STATE_GROUPBY && s->kind != LDB_STATE_SIMPLE)) fail(LDB_ERR_INVALID, "not a group state");
      auto& g = s->group; // the table IS the image (newGroupState): one copy
      LDB_CUDA(cudaMemcpyAsync(dst, g.state, groupImageBytes(g.capacity), cudaMemcpyDeviceToDevice, s->ctx->compute));
   });
}
int ldb_gpu_groupby_merge_exported(LdbState* s, const void* src, int32_t n_tables, int32_t skip_index, LdbError* err) {
   return guarded(err, [&] {
      if (!s || (s->kind != LDB_STATE_GROUPBY && s->kind != LDB_STATE_SIMPLE)) fail(LDB_ERR_INVALID, "not a group state");
      ldb_gpu_want_bound_lanes_internal(s);
      LdbContext* ctx = s->ctx;
      ctx->launch("group_merge", [&] { launchGroupMergeImages(s->group, (const uint8_t*) src, n_tables, skip_index, ctx->compute); });
   });
}

int ldb_gpu_join_table_create(LdbContext* ctx, int64_t expected_rows, int32_t unique_keys, int32_t n_side, int32_t n_aggs, LdbState** out, LdbError* err) {
   return guarded(err, [&] {
      if (!ctx || !out) fail(LDB_ERR_INVALID, "null argument");
      if (n_side < 0 || n_side > kMaxSide || n_aggs < 0 || n_aggs > 1) fail(LDB_ERR_INVALID, "n_side/n_aggs out of range");
      LDB_CUDA(cudaSetDevice(ctx->device));
      auto* s = new LdbState;
      s->ctx = ctx;
      s->kind = LDB_STATE_JOIN_TABLE;
      ctx->states.push_back(s);
      // HashIndexedView::build sizes its directory nextPow2(1.25 n) for chained buckets
      // (LazyJoinHashtable.cpp:16); linear probing wants load factor <= 0.5
      uint64_t cap = nextPow2((uint64_t) std::max<int64_t>(expected_rows, 8) * 2);
      auto& j = s->join;
      j.mask = cap - 1;
      j.unique = unique_keys & LDB_JOIN_UNIQUE;
      if (n_side > 0 || n_aggs > 0) { // group-join map: one 32-byte sector per entry
         j.stride = 32;
         j.base = (uint8_t*) ctx->stagingAlloc(cap * 32);
         s->allocations.push_back(j.base);
         ctx->launch("table_init", [&] { launchInitWideTable(j.base, cap, ctx->smCount, ctx->compute); });
      } else {
         j.stride = 8;
         j.base = (uint8_t*) devAlloc(s, cap * 8, 0xff);
      }
      j.count = (unsigned long long*) devAlloc(s, 8, 0);
      j.error = (int32_t*) devAlloc(s, 4, 0);
      if (cap >= 4096 && !(unique_keys & LDB_JOIN_NO_BLOOM)) { // 8 filter bits per directory slot = 16..32 bits per key at load 0.25..0.5
         uint64_t words = cap / 4;
         j.bloom = (uint32_t*) devAlloc(s, words * 4, 0);
         j.bloomMask = (uint32_t) (words - 1);
      }
      s->nSide = n_side;
      s->nAggs = n_aggs;
      *out = s;
   });
}
int ldb_gpu_join_table_create_shared_bloom(LdbContext* ctx, int64_t expected_rows, int32_t unique_keys, LdbComm* comm, int64_t bloom_offset, int64_t* bloom_bytes, LdbState** out, LdbError* err) {
   return guarded(err, [&] {
      const uint64_t cap = nextPow2((uint64_t) std::max<int64_t>(expected_rows, 2048) * 2); // >= 4096 slots: always has a filter
      const uint64_t words = cap / 4;
      if (bloom_bytes) *bloom_bytes = (int64_t) words * 4;
      if (!out) return; // size query
      if (!ctx || !comm) fail(LDB_ERR_INVALID, "null argument");
      if (comm->ctx != ctx) fail(LDB_ERR_INVALID, "comm belongs to another context");
      if (bloom_offset < 0 || bloom_offset % 16 || (size_t) bloom_offset + words * 4 > comm->userBytes) fail(LDB_ERR_CAPACITY, "Bloom filter outside the comm's user heap (create the comm with a larger heap)");
      LDB_CUDA(cudaSetDevice(ctx->device));
      auto* s = new LdbState;
      s->ctx = ctx;
      s->kind = LDB_STATE_JOIN_TABLE;
      ctx->states.push_back(s);
      auto& j = s->join;
      j.mask = cap - 1;
      j.unique = unique_keys & LDB_JOIN_UNIQUE;
      j.stride = 8;
      j.base = (uint8_t*) devAlloc(s, cap * 8, 0xff);
      j.count = (unsigned long long*) devAlloc(s, 8, 0);
      j.error = (int32_t*) devAlloc(s, 4, 0);
      j.bloom = (uint32_t*) (comm->heap + kUserOff + bloom_offset); // owned by the comm's heap, not by the state
      j.bloomMask = (uint32_t) (words - 1);
      LDB_CUDA(cudaMemsetAsync(j.bloom, 0, words * 4, ctx->compute));
      *out = s;
   });
}
int ldb_gpu_join_table_create_pair(LdbContext* ctx, int64_t expected_rows, int32_t unique_keys, LdbState** out, LdbError* err) {
   return guarded(err, [&] {
      if (!ctx || !out) fail(LDB_ERR_INVALID, "null argument");
      LDB_CUDA(cudaSetDevice(ctx->device));
      auto* s = new LdbState;
      s->ctx = ctx;
      s->kind = LDB_STATE_JOIN_TABLE;
      ctx->states.push_back(s);
      uint64_t cap = nextPow2((uint64_t) std::max<int64_t>(expected_rows, 8) * 2);
      auto& j = s->join;
      j.mask = cap - 1;
      j.unique = unique_keys & LDB_JOIN_UNIQUE;
      j.stride = 16;
      j.base = (uint8_t*) devAlloc(s, cap * 16, 0xff);
      j.count = (unsigned long long*) devAlloc(s, 8, 0);
      j.error = (int32_t*) devAlloc(s, 4, 0);
      if (cap >= 4096 && !(unique_keys & LDB_JOIN_NO_BLOOM)) {
         uint64_t words = cap / 4;
         j.bloom = (uint32_t*) devAlloc(s, words * 4, 0);
         j.bloomMask = (uint32_t) (words - 1);
      }
      *out = s;
   });
}
int ldb_gpu_join_table_create_direct(LdbContext* ctx, int32_t key_min, int32_t key_max, LdbState** out, LdbError* err) {
   return guarded(err, [&] {
      if (!ctx || !out) fail(LDB_ERR_INVALID, "null argument");
      if (key_max < key_min) fail(LDB_ERR_INVALID, "empty key range");
      const uint64_t range = (uint64_t) ((int64_t) key_max - (int64_t) key_min) + 1;
      if (range > (1ull << 32) - 1) fail(LDB_ERR_UNSUPPORTED, "key range too wide for a direct-address table");
      LDB_CUDA(cudaSetDevice(ctx->device));
      auto* s = new LdbState;
      s->ctx = ctx;
      s->kind = LDB_STATE_JOIN_TABLE;
      ctx->states.push_back(s);
      auto& j = s->join;
      j.stride = 4;
      j.direct = 1;
      j.unique = 1;
      j.keyMin = key_min;
      j.range = (uint32_t) range;
      j.mask = 0;
      j.base = (uint8_t*) devAlloc(s, range * 4, 0x80); // kDirectEmpty in every slot
      j.count = (unsigned long long*) devAlloc(s, 8, 0);
      j.error = (int32_t*) devAlloc(s, 4, 0);
      *out = s;
   });
}
int ldb_gpu_table_column_range(LdbTable* t, const char* column, int32_t* mn, int32_t* mx, LdbError* err) {
   return guarded(err, [&] {
      if (!t || !mn || !mx) fail(LDB_ERR_INVALID, "null argument");
      LdbContext* ctx = t->ctx;
      int c = t->colIndex(column);
      if (c < 0) fail(LDB_ERR_INVALID, "unknown column");
      if (t->columns[c].type != LDB_INT32 && t->columns[c].type != LDB_DATE32) fail(LDB_ERR_UNSUPPORTED, "column range needs an int32/date32 column");
      if (auto it = t->ranges.find(c); it != t->ranges.end() && it->second.rows == t->numRows && !ctx->capturing) {
         *mn = it->second.lo;
         *mx = it->second.hi;
         return;
      }
      LDB_CUDA(cudaSetDevice(ctx->device));
      int32_t init[2] = {INT32_MAX, INT32_MIN};
      Scratch scratch(ctx);
      int32_t* d = scratch.alloc<int32_t>(8);
      LDB_CUDA(cudaMemcpyAsync(d, init, 8, cudaMemcpyHostToDevice, ctx->compute));
      for (auto& b : t->batches) {
         if (b.nRows == 0) continue;
         waitBatch(ctx, b);
         ctx->launch("column_range", [&] { launchColumnRange((const int32_t*) b.data[c], b.nRows, d, ctx->smCount, ctx->compute); });
      }
      LDB_CUDA(cudaMemcpyAsync(init, d, 8, cudaMemcpyDeviceToHost, ctx->compute));
      ctx->syncStream(ctx->compute);
      *mn = init[0];
      *mx = init[1];
      t->ranges[c] = LdbTable::ColumnRange{t->numRows, init[0], init[1]};
   });
}
static void checkJoinError(LdbState* s) {
   int32_t e = 0;
   LDB_CUDA(cudaMemcpyAsync(&e, s->join.error, sizeof(e), cudaMemcpyDeviceToHost, s->ctx->compute));
   s->ctx->syncStream(s->ctx->compute);
   if (e == 1) fail(LDB_ERR_CAPACITY, "join table full: more build rows than expected_rows allowed");
   if (e == 2) fail(LDB_ERR_INVALID, "duplicate key inserted into a join table declared unique");
   if (e == 3) fail(LDB_ERR_UNSUPPORTED, "the pair (key=-1, payload=-1) cannot be stored in a join table");
   if (e == 4) fail(LDB_ERR_UNSUPPORTED, "join tables with side/aggregate lanes need non-negative inline payloads");
   if (e == 5) fail(LDB_ERR_INVALID, "key outside the declared range of a direct-address table");
   if (e == 6) fail(LDB_ERR_CAPACITY, "PROBE_EACH: a probe run is longer than the interpreter's bound of 16384 slots (an overfull join table)");
   if (e == 7) fail(LDB_ERR_UNSUPPORTED, "a program join build met a key or payload outside int32 (join tables store int32 keys and payloads)");
   if (e == 8) fail(LDB_ERR_CAPACITY, "EXISTS: a probe run is longer than the interpreter's bound of 16384 slots (an overfull join table)");
   if (e != 0) fail(LDB_ERR_INVALID, "join table error word " + std::to_string(e));
}
} // extern "C"
void ldb_gpu_check_join_error_internal(LdbState* s) { checkJoinError(s); }
extern "C" {
int ldb_gpu_join_table_count(LdbState* s, int64_t* n_entries, LdbError* err) {
   return guarded(err, [&] {
      if (!s || (s->kind != LDB_STATE_JOIN_TABLE && s->kind != LDB_STATE_KEY_JOIN)) fail(LDB_ERR_INVALID, "not a join table");
      const bool keys = s->kind == LDB_STATE_KEY_JOIN;
      if (keys) ldb_gpu_check_keyjoin_error_internal(s);
      else checkJoinError(s);
      unsigned long long c = 0;
      LDB_CUDA(cudaMemcpyAsync(&c, keys ? s->keyJoin.count : s->join.count, 8, cudaMemcpyDeviceToHost, s->ctx->compute));
      s->ctx->syncStream(s->ctx->compute);
      *n_entries = (int64_t) c;
   });
}
int ldb_gpu_join_table_bloom(LdbState* s, void** dev_ptr, int64_t* bytes, LdbError* err) {
   return guarded(err, [&] {
      if (!s || s->kind != LDB_STATE_JOIN_TABLE) fail(LDB_ERR_INVALID, "not a join table");
      *dev_ptr = s->join.bloom;
      *bytes = s->join.bloom ? ((int64_t) s->join.bloomMask + 1) * 4 : 0;
   });
}
int ldb_gpu_join_table_topk(LdbState* s, int32_t k, LdbTopKRow* rows, int32_t* n_rows, LdbError* err) {
   return guarded(err, [&] {
      if (!s || s->kind != LDB_STATE_JOIN_TABLE || !s->nAggs) fail(LDB_ERR_INVALID, "not a group-join table");
      if (k < 1 || k > 64) fail(LDB_ERR_INVALID, "k must be in [1, 64]");
      checkJoinError(s);
      LdbContext* ctx = s->ctx;
      int blocks = ctx->smCount * 2;
      size_t bytes = sizeof(TopKRowDev) * (size_t) blocks * k;
      Scratch scratch(ctx);
      TopKRowDev* d = scratch.alloc<TopKRowDev>(bytes);
      ctx->launch("join_topk", [&] { launchJoinTopK(s->join, k, (s->is64Mask & 1u) != 0, d, &blocks, ctx->smCount, ctx->compute); });
      std::vector<TopKRowDev> h((size_t) blocks * k);
      LDB_CUDA(cudaMemcpyAsync(h.data(), d, bytes, cudaMemcpyDeviceToHost, ctx->compute));
      ctx->syncStream(ctx->compute);
      std::vector<TopKRowDev> valid;
      for (auto& r : h)
         if (r.valid) valid.push_back(r);
      std::sort(valid.begin(), valid.end(), [](const TopKRowDev& a, const TopKRowDev& b) {
         if (a.aggHi != b.aggHi) return a.aggHi > b.aggHi;
         if (a.aggLo != b.aggLo) return a.aggLo > b.aggLo;
         if (a.side0 != b.side0) return a.side0 < b.side0;
         return a.key < b.key;
      });
      int n = (int) std::min<size_t>(valid.size(), (size_t) k);
      for (int i = 0; i < n; i++) {
         rows[i].key = valid[i].key;
         rows[i].side[0] = valid[i].side0;
         rows[i].side[1] = valid[i].side1;
         rows[i].pad = 0;
         rows[i].agg = LdbI128{valid[i].aggLo, valid[i].aggHi};
      }
      *n_rows = n;
   });
}

// ------------------------------------------------------------------------------------------------ pipelines
namespace {
struct Resolved {
   LdbTable* t;
   int col(const char* name, std::initializer_list<int> types, const char* role) const {
      int i = t->colIndex(name);
      if (i < 0) fail(LDB_ERR_INVALID, std::string("unknown column ") + (name ? name : "(null)") + " for " + role);
      bool ok = false;
      for (int ty : types) ok |= t->columns[i].type == ty;
      if (!ok) fail(LDB_ERR_UNSUPPORTED, std::string("column ") + name + " has an unsupported physical type for " + role);
      return i;
   }
};
// FilterDescription list → per-column predicate pairs (Restrictions::create, Restrictions.cpp:392-520)
// distinct fixed-width columns a pipeline reads → the staged tile layout (kernels.h StagedCols)
struct StagePlan {
   int n = 0;
   int colIdx[kMaxStagedCols];
   int add(LdbTable* t, int col) {
      for (int i = 0; i < n; i++)
         if (colIdx[i] == col) return i;
      if (n == kMaxStagedCols) fail(LDB_ERR_UNSUPPORTED, "a pipeline may touch at most 8 distinct fixed-width columns");
      colIdx[n] = col;
      return n++;
   }
   void bind(LdbTable* t, const LdbBatch& b, StagedCols& out, int rowsPerThread) const {
      out.n = n;
      out.tileRows = kBlockThreads * rowsPerThread;
      int off = 0;
      bool aligned = true;
      for (int i = 0; i < n; i++) {
         if ((colIdx[i] < (int) b.validity.size() && b.validity[colIdx[i]]) || (colIdx[i] < (int) b.validBytes.size() && b.validBytes[colIdx[i]]))
            fail(LDB_ERR_UNSUPPORTED, "column " + t->columns[colIdx[i]].name + " has NULLs in this batch: the specialised pipelines read non-nullable columns — use the program pipeline (ldb_gpu_run_program)");
         out.base[i] = (const uint8_t*) b.data[colIdx[i]];
         out.elemBytes[i] = b.elemBytes[colIdx[i]]; // as staged: decimal128 is 16, or 8 when the HOST batch was narrowed
         out.smemOffset[i] = off;
         off += out.elemBytes[i] * out.tileRows;
         aligned &= ((uintptr_t) out.base[i] % 16) == 0;
      }
      out.stageBytes = off;
      out.useTma = aligned && n > 0 ? 1 : 0;
      out.producerSleepNs = tuning().producerSleepNs;
      out.consumerSleepNs = tuning().consumerSleepNs;
      out.decBytes = 0; // the kernels are instantiated for ONE decimal cell width per batch
      for (int i = 0; i < n; i++) {
         if (t->columns[colIdx[i]].type != LDB_DECIMAL128) continue;
         if (out.decBytes && out.decBytes != out.elemBytes[i])
            fail(LDB_ERR_UNSUPPORTED, "batch stages decimal columns of different cell widths (a narrowed decimal(p<19) next to a 16-byte decimal(p>=19)): use the program pipeline (ldb_gpu_run_program)");
         out.decBytes = out.elemBytes[i];
      }
      if (!out.decBytes) out.decBytes = 16;
   }
   // the same columns read from the batch's encoded copies (every one of them built by ldb_gpu_encode_batch_internal)
   void bindEncoded(LdbTable* t, const LdbBatch& b, StagedCols& out, int rowsPerThread) const {
      bind(t, b, out, rowsPerThread);
      out.tileHeader = kEncodeTileHeader;
      int off = 0;
      for (int i = 0; i < n; i++) {
         const LdbBatch::Encoded& e = b.enc[colIdx[i]];
         out.base[i] = e.data;
         out.elemBytes[i] = e.width;
         out.smemOffset[i] = off;
         off += e.width * out.tileRows + kEncodeTileHeader;
         out.encShift[i] = e.width == 1 ? 0 : e.width == 2 ? 1 : e.width == 4 ? 2 : 3;
         out.encMask[i] = e.width >= 4 ? ~0u : (1u << (8 * e.width)) - 1u;
      }
      out.stageBytes = off;
      out.useTma = n > 0 ? 1 : 0; // the copies are cudaMalloc'd and every column tile is a multiple of 16 bytes
      out.decBytes = kDecEncoded;
   }
};
struct FilterPlan {
   FilterSet set{};
   int colIdx[kMaxFilterCols];
};
// one constant of a filter, typed by the physical column type (Restrictions::create, Restrictions.cpp:392-520)
static int64_t filterConstant(const LdbColumn& col, bool isInt, const char* str, int64_t ival) {
   switch (col.type) {
      case LDB_INT32:
         if (!isInt) fail(LDB_ERR_INVALID, "integer column needs an integer constant");
         return ival;
      case LDB_DATE32: return parseDate32(str);
      case LDB_FSB4: {
         if (!str || strlen(str) > 4) fail(LDB_ERR_INVALID, "char(1) constant too long");
         int32_t v = 0;
         memcpy(&v, str, strlen(str));
         return v;
      }
      case LDB_DECIMAL128: {
         if (col.precision >= 19) fail(LDB_ERR_UNSUPPORTED, "decimal precision >= 19 is not supported on the GPU path yet");
         if (!isInt) return parseDecimal(str, col.scale);
         __int128 v = ival;
         for (int s = 0; s < col.scale; s++) {
            v *= 10;
            if (v > (__int128) INT64_MAX || v < (__int128) INT64_MIN) fail(LDB_ERR_UNSUPPORTED, "decimal constant beyond 64 bits");
         }
         return (int64_t) v;
      }
      default: fail(LDB_ERR_UNSUPPORTED, "unsupported type in filter");
   }
}
FilterPlan planFilters(LdbTable* t, const LdbFilterDesc* f, int n, StagePlan& sp) {
   FilterPlan p;
   p.set.n = 0;
   for (int i = 0; i < n; i++) {
      int c = t->colIndex(f[i].column);
      if (c < 0) fail(LDB_ERR_INVALID, "unknown column in filter"); // Restrictions.cpp:396
      auto& col = t->columns[c];
      if (f[i].op == LDB_NOTNULL) continue; // batches with nulls are rejected at append time → always true (FirstNotNullFilter fast path, Restrictions.cpp:67-75)
      int kind = col.type == LDB_DECIMAL128 ? COL_DEC128_LO64 : COL_I32;
      if (f[i].op == LDB_IN) {
         if (col.type == LDB_UTF8) fail(LDB_ERR_UNSUPPORTED, "IN over strings is not supported on the GPU path yet");
         if (f[i].n_values < 1 || f[i].n_values > LDB_MAX_IN_VALUES) fail(LDB_ERR_UNSUPPORTED, "IN lists hold 1..8 values on the GPU path");
         if (p.set.n == kMaxFilterCols) fail(LDB_ERR_UNSUPPORTED, "more than 4 filter columns in one pipeline");
         FilterCol& fc = p.set.c[p.set.n];
         memset(&fc, 0, sizeof(fc));
         fc.kind = kind;
         fc.staged = sp.add(t, c);
         fc.maskA = fc.maskB = 7;
         fc.nIn = f[i].n_values;
         for (int k = 0; k < f[i].n_values; k++) fc.inVals[k] = filterConstant(col, f[i].value_is_int != 0, f[i].str_values[k], f[i].int_values[k]);
         p.colIdx[p.set.n++] = c;
         continue;
      }
      int64_t value = 0;
      uint32_t mask = opMask(f[i].op == LDB_CONTAINS ? (int) LDB_EQ : f[i].op); // contains: predicate value (0/1) == 1
      const char* str = nullptr;
      if (col.type == LDB_UTF8) {
         if (f[i].op != LDB_EQ && f[i].op != LDB_NEQ && f[i].op != LDB_CONTAINS) fail(LDB_ERR_UNSUPPORTED, "unsupported filter op for string");
         if (!f[i].str_value || strlen(f[i].str_value) > sizeof(FilterCol::str)) fail(LDB_ERR_UNSUPPORTED, "string constant longer than 24 bytes");
         kind = f[i].op == LDB_CONTAINS ? COL_UTF8_CONTAINS : COL_UTF8_EQ;
         value = 1;
         str = f[i].str_value;
      } else {
         if (f[i].op == LDB_CONTAINS) fail(LDB_ERR_UNSUPPORTED, "LIKE-contains needs a utf8 column");
         value = filterConstant(col, f[i].value_is_int != 0, f[i].str_value, f[i].int_value);
      }
      const bool isUtf8 = kind == COL_UTF8_EQ || kind == COL_UTF8_CONTAINS;
      int slot = -1;
      if (!isUtf8)
         for (int k = 0; k < p.set.n; k++)
            if (p.colIdx[k] == c && p.set.c[k].maskB == 7 && p.set.c[k].nIn == 0) slot = k;
      if (slot >= 0) {
         p.set.c[slot].maskB = mask;
         p.set.c[slot].valB = value;
         continue;
      }
      if (p.set.n == kMaxFilterCols) fail(LDB_ERR_UNSUPPORTED, "more than 4 filter columns in one pipeline");
      FilterCol& fc = p.set.c[p.set.n];
      memset(&fc, 0, sizeof(fc));
      fc.kind = kind;
      fc.staged = isUtf8 ? -1 : sp.add(t, c);
      fc.maskA = mask;
      fc.valA = value;
      fc.maskB = 7;
      fc.valB = 0;
      if (str) {
         fc.strLen = (int32_t) strlen(str);
         memcpy(fc.str, str, fc.strLen);
      }
      p.colIdx[p.set.n++] = c;
   }
   return p;
}
void bindFilters(const FilterPlan& p, const LdbBatch& b, FilterSet& out) {
   out = p.set;
   for (int i = 0; i < out.n; i++) {
      if (out.c[i].kind != COL_UTF8_EQ && out.c[i].kind != COL_UTF8_CONTAINS) continue; // fixed-width filter columns are read from the staged tile
      if (p.colIdx[i] < (int) b.validity.size() && b.validity[p.colIdx[i]]) fail(LDB_ERR_UNSUPPORTED, "string filter column has NULLs in this batch: use the program pipeline (ldb_gpu_run_program)");
      out.c[i].base = b.data[p.colIdx[i]];
      out.c[i].bytes = (const uint8_t*) b.bytes[p.colIdx[i]];
   }
}
// value columns of aggregate expressions, de-duplicated in first-appearance order
struct AggPlan {
   int nValueCols = 0;
   int valueCol[kMaxValueCols];
   int nAggs = 0;
   AggSpec aggs[kMaxAggs];
};
AggPlan planAggs(const Resolved& R, const LdbAggDesc* a, int n) {
   AggPlan p;
   if (n < 1 || n > kMaxAggs) fail(LDB_ERR_INVALID, "n_aggs out of range");
   for (int i = 0; i < n; i++) {
      int used = a[i].expr == LDB_EXPR_COL ? 1 : (a[i].expr == LDB_EXPR_MUL || a[i].expr == LDB_EXPR_MUL_1MINUS) ? 2 : a[i].expr == LDB_EXPR_MUL_1MINUS_1PLUS ? 3 : a[i].expr == LDB_EXPR_ONE ? 0 : -1;
      if (used < 0) fail(LDB_ERR_UNSUPPORTED, "unknown aggregate expression kind");
      p.aggs[i].expr = a[i].expr;
      for (int k = 0; k < 3; k++) p.aggs[i].col[k] = 0;
      for (int k = 0; k < used; k++) {
         int c = R.col(a[i].columns[k], {LDB_DECIMAL128}, "aggregate operand");
         auto& col = R.t->columns[c];
         if (col.precision >= 19 || col.scale != 2) fail(LDB_ERR_UNSUPPORTED, "aggregate operands must be decimal(p<19, 2) on the GPU path");
         int idx = -1;
         for (int v = 0; v < p.nValueCols; v++)
            if (p.valueCol[v] == c) idx = v;
         if (idx < 0) {
            if (p.nValueCols == kMaxValueCols) fail(LDB_ERR_UNSUPPORTED, "more than 4 distinct aggregate operand columns");
            idx = p.nValueCols;
            p.valueCol[p.nValueCols++] = c;
         }
         p.aggs[i].col[k] = idx;
      }
   }
   p.nAggs = n;
   return p;
}
// late-materialised operand columns of a probe pipeline (kernels.h LazyCols): bound per batch, never staged through the tiles
void bindLazy(LdbTable* t, const LdbBatch& b, const int* cols, int n, LazyCols& out) {
   out.n = n;
   for (int i = 0; i < n; i++) {
      if ((cols[i] < (int) b.validity.size() && b.validity[cols[i]]) || (cols[i] < (int) b.validBytes.size() && b.validBytes[cols[i]]))
         fail(LDB_ERR_UNSUPPORTED, "column " + t->columns[cols[i]].name + " has NULLs in this batch: use the program pipeline (ldb_gpu_run_program)");
      out.base[i] = (const uint8_t*) b.data[cols[i]];
      out.elemBytes[i] = b.elemBytes[cols[i]];
   }
}
// An aggregate lane of a state keeps one width for its whole life: a 64-bit SUM (COL / ONE; wraps at 64 bits, read back
// sign-extended) or a 128-bit one.  A pipeline that would add the other kind into the same lane is rejected: the read could not
// tell the two apart.
void bindLaneWidth(LdbState* s, int lane, int expr) {
   const uint32_t bit = 1u << lane;
   const bool is64 = expr == LDB_EXPR_COL || expr == LDB_EXPR_ONE;
   if ((s->laneBound & bit) && ((s->is64Mask & bit) != 0) != is64)
      fail(LDB_ERR_UNSUPPORTED, "aggregate " + std::to_string(lane) + " of this state was summed at another width: 64-bit (COL, ONE) and 128-bit expressions cannot share a lane");
   s->laneBound |= bit;
   if (is64) s->is64Mask |= bit;
}
LdbState* wantState(LdbState* s, int kind, const char* role) {
   if (!s || s->kind != kind) fail(LDB_ERR_INVALID, std::string("wrong or missing state for ") + role);
   return s;
}
LdbState* wantSingleKeyTable(LdbState* s, const char* role) {
   wantState(s, LDB_STATE_JOIN_TABLE, role);
   if (s->join.stride == 16) fail(LDB_ERR_UNSUPPORTED, std::string("composite-key table not supported for ") + role);
   if (s->join.direct) fail(LDB_ERR_UNSUPPORTED, std::string("direct-address table not supported for ") + role);
   return s;
}
} // namespace
} // extern "C"
void ldb_gpu_bind_lane_width_internal(LdbState* s, int lane, int expr) { bindLaneWidth(s, lane, expr); }
void ldb_gpu_want_bound_lanes_internal(LdbState* s) {
   const uint32_t all = (1u << s->group.nAggs) - 1u;
   if ((s->laneBound & all) != all)
      fail(LDB_ERR_UNSUPPORTED, "merge target has an aggregate whose width no pipeline fixed yet: a merged lane is read at its target's width (run a pipeline into the state first)");
}
extern "C" {

int ldb_gpu_run_pipeline(LdbContext* ctx, const LdbPipelineDesc* d, LdbError* err) {
   return guarded(err, [&] {
      if (!ctx || !d || !d->source) fail(LDB_ERR_INVALID, "null argument");
      LdbTable* t = d->source;
      if (t->ctx != ctx) fail(LDB_ERR_INVALID, "table belongs to another context");
      LDB_CUDA(cudaSetDevice(ctx->device));
      Resolved R{t};
      StagePlan sp;
      FilterPlan fp = planFilters(t, d->filters, d->n_filters, sp);
      const char* why = "";
      switch (d->kind) {
         case LDB_PIPE_SCAN_REDUCE:
         case LDB_PIPE_SCAN_GROUPBY: {
            bool keyless = d->kind == LDB_PIPE_SCAN_REDUCE;
            LdbState* sink = wantState(d->sink, keyless ? LDB_STATE_SIMPLE : LDB_STATE_GROUPBY, "sink");
            AggPlan ap = planAggs(R, d->aggs, d->n_aggs);
            if (ap.nAggs != sink->group.nAggs) fail(LDB_ERR_INVALID, "aggregate count differs from the state's");
            for (int a = 0; a < ap.nAggs; a++) bindLaneWidth(sink, a, ap.aggs[a].expr);
            int nKeys = keyless ? 0 : d->n_keys;
            if (nKeys != sink->group.nKeys) fail(LDB_ERR_INVALID, "key count differs from the state's");
            int keyCol[kMaxKeys] = {0, 0};
            int keyStage[kMaxKeys] = {0, 0}, valueStage[kMaxValueCols] = {0, 0, 0, 0};
            for (int k = 0; k < nKeys; k++) {
               keyCol[k] = R.col(d->key_columns[k], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "group key");
               keyStage[k] = sp.add(t, keyCol[k]);
            }
            for (int v = 0; v < ap.nValueCols; v++) valueStage[v] = sp.add(t, ap.valueCol[v]);
            for (auto& b : t->batches) {
               if (b.nRows == 0) continue;
               GroupByParams p{};
               p.src.nRows = b.nRows;
               bindFilters(fp, b, p.src.filters);
               p.nKeys = nKeys;
               for (int k = 0; k < nKeys; k++) p.keyStage[k] = keyStage[k];
               p.nValueCols = ap.nValueCols;
               for (int v = 0; v < ap.nValueCols; v++) p.valueStage[v] = valueStage[v];
               p.nAggs = ap.nAggs;
               for (int a = 0; a < ap.nAggs; a++) p.aggs[a] = ap.aggs[a];
               p.table = sink->group;
               // a borrowed DEVICE batch is scanned from its frame-of-reference copy (built here on first use); HOST-staged
               // batches, signatures without an encoded instantiation and copies that could not be allocated use the Arrow cells
               const bool encoded = tuning().encodedScan && b.borrowed && scanGroupByEncodable(p) &&
                                    ldb_gpu_encode_batch_internal(ctx, t, b, sp.colIdx, sp.n, kBlockThreads * kRowsPerThreadScan);
               if (encoded) {
                  sp.bindEncoded(t, b, p.src.cols, kRowsPerThreadScan);
                  for (int v = 0; v < ap.nValueCols; v++) {
                     const LdbBatch::Encoded& e = b.enc[ap.valueCol[v]];
                     p.encMin[v] = e.min;
                     p.encRange[v] = (uint64_t) e.max - (uint64_t) e.min;
                  }
               } else {
                  sp.bind(t, b, p.src.cols, kRowsPerThreadScan);
               }
               waitBatch(ctx, b);
               bool ok = true;
               ctx->launch(keyless ? "scan_reduce" : "scan_groupby", [&] { ok = launchScanGroupBy(p, ctx->smCount, ctx->compute, &why); });
               if (!ok) fail(LDB_ERR_UNSUPPORTED, why);
               // which Q1 instance ran: the factored one's eager launches also count (without a time) as family "scan_groupby_factored"
               if (encoded && ctx->timing && !ctx->capturing && scanGroupByFactored(p)) ctx->timers["scan_groupby_factored"].launches++;
            }
            break;
         }
         case LDB_PIPE_SCAN_BUILD: {
            LdbState* sink = wantState(d->sink, LDB_STATE_JOIN_TABLE, "sink");
            if (d->n_probes < 0 || d->n_probes > 1) fail(LDB_ERR_UNSUPPORTED, "build pipelines take at most one probe");
            if (d->n_side != sink->nSide) fail(LDB_ERR_INVALID, "side column count differs from the table's");
            int keyCol = R.col(d->build_key_column, {LDB_INT32, LDB_DATE32, LDB_FSB4}, "build key");
            const bool pair = sink->join.stride == 16;
            if (pair != (d->build_key2_column != nullptr)) fail(LDB_ERR_INVALID, "a second build key goes with a composite-key table (and only with one)");
            if (pair && d->n_side) fail(LDB_ERR_UNSUPPORTED, "composite-key tables carry no side lanes");
            if (sink->join.direct && d->n_side) fail(LDB_ERR_UNSUPPORTED, "direct-address tables carry no side lanes");
            int key2Col = pair ? R.col(d->build_key2_column, {LDB_INT32, LDB_DATE32, LDB_FSB4}, "second build key") : -1;
            int payCol = -1, payKind = PAYLOAD_I32;
            if (d->build_payload_column) {
               if (pair) {
                  payCol = R.col(d->build_payload_column, {LDB_INT32, LDB_DATE32, LDB_FSB4, LDB_DECIMAL128}, "build payload");
                  if (t->columns[payCol].type == LDB_DECIMAL128) {
                     if (t->columns[payCol].precision >= 19) fail(LDB_ERR_UNSUPPORTED, "decimal payloads must have precision < 19");
                     payKind = PAYLOAD_DEC_LO64;
                  }
               } else {
                  payCol = R.col(d->build_payload_column, {LDB_INT32, LDB_DATE32, LDB_FSB4}, "build payload");
               }
            }
            if (d->build_payload_expr == LDB_PAYLOAD_YEAR) {
               if (pair || payCol < 0 || t->columns[payCol].type != LDB_DATE32) fail(LDB_ERR_UNSUPPORTED, "year payloads come from a date32 column of a single-key build");
               payKind = PAYLOAD_YEAR_OF_DATE32;
            } else if (d->build_payload_expr != LDB_PAYLOAD_COLUMN) {
               fail(LDB_ERR_UNSUPPORTED, "unknown build payload expression");
            }
            int sideCol[kMaxSide] = {0, 0};
            for (int k = 0; k < d->n_side; k++) sideCol[k] = R.col(d->side_columns[k], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "side payload");
            LdbState* probe = d->n_probes ? wantState(d->probe_states[0], LDB_STATE_JOIN_TABLE, "probe") : nullptr;
            if (probe && (probe->join.stride == 16 || probe->join.direct)) fail(LDB_ERR_UNSUPPORTED, "build pipelines probe single-key hash tables");
            int probeCol = d->n_probes ? R.col(d->probe_key_columns[0], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "probe key") : -1;
            int keyStage = sp.add(t, keyCol), key2Stage = key2Col >= 0 ? sp.add(t, key2Col) : -1, payStage = payCol >= 0 ? sp.add(t, payCol) : -1, probeStage = probeCol >= 0 ? sp.add(t, probeCol) : 0;
            int sideStage[kMaxSide] = {0, 0};
            for (int k = 0; k < d->n_side; k++) sideStage[k] = sp.add(t, sideCol[k]);
            for (auto& b : t->batches) {
               if (b.nRows == 0) continue;
               BuildParams p{};
               p.src.nRows = b.nRows;
               bindFilters(fp, b, p.src.filters);
               sp.bind(t, b, p.src.cols, sink->join.stride == 16 ? kRowsPerThreadStar : tuning().rptBuild); // the pair build keeps 1 row/thread
               p.keyStage = keyStage;
               p.keyStage2 = key2Stage;
               p.payloadStage = payStage;
               p.payloadKind = payKind;
               p.nSide = d->n_side;
               for (int k = 0; k < d->n_side; k++) p.sideStage[k] = sideStage[k];
               p.hasProbe = probe ? 1 : 0;
               if (probe) {
                  p.probe = probe->join;
                  p.probeKeyStage = probeStage;
               }
               p.sink = sink->join;
               waitBatch(ctx, b);
               ctx->launch("join_build", [&] { launchScanBuild(p, ctx->smCount, ctx->compute); });
            }
            break;
         }
         case LDB_PIPE_SCAN_PROBE_AGG: {
            LdbState* table = wantState(d->sink, LDB_STATE_JOIN_TABLE, "group-join map");
            if (!table->nAggs) fail(LDB_ERR_INVALID, "join table was created without aggregate lanes");
            if (d->n_probes != 1 || d->probe_states[0] != table) fail(LDB_ERR_INVALID, "probe-aggregate pipelines probe their own sink");
            AggPlan ap = planAggs(R, d->aggs, 1);
            bindLaneWidth(table, 0, ap.aggs[0].expr); // the top-k ranks a 64-bit lane by its sign-extended value
            int probeCol = R.col(d->probe_key_columns[0], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "probe key");
            int probeStage = sp.add(t, probeCol);
            for (auto& b : t->batches) {
               if (b.nRows == 0) continue;
               ProbeAggParams p{};
               p.src.nRows = b.nRows;
               bindFilters(fp, b, p.src.filters);
               sp.bind(t, b, p.src.cols, kRowsPerThreadProbe);
               p.probeKeyStage = probeStage;
               p.table = table->join;
               p.agg = ap.aggs[0];
               bindLazy(t, b, ap.valueCol, ap.nValueCols, p.values);
               waitBatch(ctx, b);
               bool ok = true;
               ctx->launch("join_probe_agg", [&] { ok = launchScanProbeAgg(p, ctx->smCount, ctx->compute, &why); });
               if (!ok) fail(LDB_ERR_UNSUPPORTED, why);
            }
            break;
         }
         case LDB_PIPE_SCAN_PROBE2_GROUPBY: {
            LdbState* sink = wantState(d->sink, LDB_STATE_GROUPBY, "sink");
            if (sink->group.nKeys != 1 || sink->group.nAggs != 1) fail(LDB_ERR_INVALID, "probe-probe-group sink must have one key and one aggregate");
            if (d->n_probes != 2) fail(LDB_ERR_INVALID, "probe-probe-group pipelines take two probes");
            LdbState* ta = wantSingleKeyTable(d->probe_states[0], "probe A");
            LdbState* tb = wantSingleKeyTable(d->probe_states[1], "probe B");
            AggPlan ap = planAggs(R, d->aggs, 1);
            int ca = R.col(d->probe_key_columns[0], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "probe key A");
            int cb = R.col(d->probe_key_columns[1], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "probe key B");
            int stageA = sp.add(t, ca), stageB = sp.add(t, cb);
            bindLaneWidth(sink, 0, ap.aggs[0].expr);
            for (auto& b : t->batches) {
               if (b.nRows == 0) continue;
               Probe2GroupByParams p{};
               p.src.nRows = b.nRows;
               bindFilters(fp, b, p.src.filters);
               sp.bind(t, b, p.src.cols, kRowsPerThreadProbe);
               p.keyStageA = stageA;
               p.keyStageB = stageB;
               p.tableA = ta->join;
               p.tableB = tb->join;
               p.agg = ap.aggs[0];
               bindLazy(t, b, ap.valueCol, ap.nValueCols, p.values);
               p.groups = sink->group;
               waitBatch(ctx, b);
               bool ok = true;
               ctx->launch("join_probe2_groupby", [&] { ok = launchScanProbe2GroupBy(p, ctx->smCount, ctx->compute, &why); });
               if (!ok) fail(LDB_ERR_UNSUPPORTED, why);
            }
            break;
         }
         case LDB_PIPE_SCAN_MATERIALIZE: {
            if (d->n_out_cols < 1 || d->n_out_cols > kMaxOutCols) fail(LDB_ERR_INVALID, "n_out_cols out of range");
            if (d->n_probes < 0 || d->n_probes > 1) fail(LDB_ERR_UNSUPPORTED, "materialize pipelines take at most one probe");
            if (!d->out_count || d->out_capacity < 0) fail(LDB_ERR_INVALID, "materialize needs out_count and out_capacity");
            LdbState* probe = d->n_probes ? wantSingleKeyTable(d->probe_states[0], "probe") : nullptr;
            int probeStage = 0;
            if (probe) probeStage = sp.add(t, R.col(d->probe_key_columns[0], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "probe key"));
            int outStage[kMaxOutCols], outElem[kMaxOutCols];
            for (int c = 0; c < d->n_out_cols; c++) {
               if (!d->out_columns[c] || !d->out_buffers[c]) fail(LDB_ERR_INVALID, "missing output column or buffer");
               if (std::string(d->out_columns[c]) == "$payload") {
                  if (!probe || d->probe_bloom_only) fail(LDB_ERR_INVALID, "$payload needs a full probe");
                  outStage[c] = -1;
                  outElem[c] = 4;
               } else {
                  int col = R.col(d->out_columns[c], {LDB_INT32, LDB_DATE32, LDB_FSB4, LDB_DECIMAL128}, "output column");
                  outStage[c] = sp.add(t, col);
                  outElem[c] = (int) elemWidth(t->columns[col].type);
               }
            }
            for (auto& b : t->batches) {
               if (b.nRows == 0) continue;
               MaterializeParams p{};
               p.src.nRows = b.nRows;
               bindFilters(fp, b, p.src.filters);
               sp.bind(t, b, p.src.cols, kRowsPerThreadProbe);
               p.hasProbe = probe ? 1 : 0;
               p.bloomOnly = d->probe_bloom_only ? 1 : 0;
               if (probe) p.probe = probe->join;
               p.probeKeyStage = probeStage;
               p.nOut = d->n_out_cols;
               for (int c = 0; c < d->n_out_cols; c++) {
                  p.outStage[c] = outStage[c];
                  p.outElem[c] = outElem[c];
                  p.out[c] = d->out_buffers[c];
               }
               p.capacity = d->out_capacity;
               p.count = (unsigned long long*) d->out_count;
               waitBatch(ctx, b);
               ctx->launch("materialize", [&] { launchScanMaterialize(p, ctx->smCount, ctx->compute); });
            }
            break;
         }
         case LDB_PIPE_SCAN_STAR_PROBE_GROUPBY: {
            LdbState* sink = wantState(d->sink, LDB_STATE_GROUPBY, "sink");
            if (sink->group.nKeys != 2 || sink->group.nAggs != 1) fail(LDB_ERR_INVALID, "star-probe sink must have two keys and one aggregate");
            if (d->n_probes != 3) fail(LDB_ERR_INVALID, "star-probe pipelines take three probes");
            if (d->n_aggs != 1 || d->aggs[0].expr != LDB_EXPR_MUL_1MINUS_MINUS_PAYMUL) fail(LDB_ERR_UNSUPPORTED, "star-probe pipelines aggregate a * (1 - b) - $payload0 * c");
            LdbState* tp = wantState(d->probe_states[0], LDB_STATE_JOIN_TABLE, "probe 0");
            LdbState* ts = wantState(d->probe_states[1], LDB_STATE_JOIN_TABLE, "probe 1");
            LdbState* to = wantState(d->probe_states[2], LDB_STATE_JOIN_TABLE, "probe 2");
            if (tp->join.stride != 16 || !d->probe_key2_columns[0]) fail(LDB_ERR_INVALID, "probe 0 of a star-probe pipeline is a composite-key table");
            if (ts->join.stride == 16 || to->join.stride == 16) fail(LDB_ERR_INVALID, "probes 1 and 2 of a star-probe pipeline are single-key tables");
            StarProbeParams base{};
            base.keyStageP0 = sp.add(t, R.col(d->probe_key_columns[0], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "probe key 0"));
            base.keyStageP1 = sp.add(t, R.col(d->probe_key2_columns[0], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "probe key 0 (second)"));
            base.keyStageS = sp.add(t, R.col(d->probe_key_columns[1], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "probe key 1"));
            base.keyStageO = sp.add(t, R.col(d->probe_key_columns[2], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "probe key 2"));
            int starValueCols[3];
            for (int k = 0; k < 3; k++) {
               int c = R.col(d->aggs[0].columns[k], {LDB_DECIMAL128}, "aggregate operand");
               if (t->columns[c].precision >= 19 || t->columns[c].scale != 2) fail(LDB_ERR_UNSUPPORTED, "aggregate operands must be decimal(p<19, 2) on the GPU path");
               starValueCols[k] = c;
            }
            bindLaneWidth(sink, 0, LDB_EXPR_MUL_1MINUS_MINUS_PAYMUL);
            for (auto& b : t->batches) {
               if (b.nRows == 0) continue;
               StarProbeParams p = base;
               p.src.nRows = b.nRows;
               bindFilters(fp, b, p.src.filters);
               sp.bind(t, b, p.src.cols, tuning().rptStar);
               bindLazy(t, b, starValueCols, 3, p.values);
               p.tableP = tp->join;
               p.tableS = ts->join;
               p.tableO = to->join;
               p.groups = sink->group;
               waitBatch(ctx, b);
               bool ok = true;
               ctx->launch("join_star_probe_groupby", [&] { ok = launchScanStarProbeGroupBy(p, ctx->smCount, ctx->compute, &why); });
               if (!ok) fail(LDB_ERR_UNSUPPORTED, why);
            }
            break;
         }
         case LDB_PIPE_SCAN_PARTITION_SEND: {
            LdbComm* c = d->comm;
            if (!c || c->ctx != ctx) fail(LDB_ERR_INVALID, "partition-send needs a comm of this context");
            if (!c->connected && c->world > 1) fail(LDB_ERR_INVALID, "comm is not connected to its peers yet");
            if (d->n_out_cols < 2 || d->n_out_cols > 4) fail(LDB_ERR_INVALID, "partition-send ships {key, second[, decimal[, decimal]]}");
            if (d->n_probes < 0 || d->n_probes > 1) fail(LDB_ERR_UNSUPPORTED, "partition-send pipelines take at most one probe");
            LdbState* probe = d->n_probes ? wantSingleKeyTable(d->probe_states[0], "probe") : nullptr;
            SendParams base{};
            base.hasProbe = probe ? 1 : 0;
            base.bloomOnly = d->probe_bloom_only ? 1 : 0;
            if (probe) base.probeKeyStage = sp.add(t, R.col(d->probe_key_columns[0], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "probe key"));
            base.keyStage = sp.add(t, R.col(d->out_columns[0], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "partition key"));
            if (d->out_columns[1] && std::string(d->out_columns[1]) == "$payload") {
               if (!probe || d->probe_bloom_only) fail(LDB_ERR_INVALID, "$payload needs a full probe");
               // the full probe is a semi-join (one tuple per row with a match): it cannot say WHICH match's payload to ship
               if (!probe->join.unique) fail(LDB_ERR_UNSUPPORTED, "partition-send ships $payload only from a probe of a unique-key table");
               base.secondStage = -1;
            } else {
               base.secondStage = sp.add(t, R.col(d->out_columns[1], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "second tuple column"));
            }
            base.secondYear = d->build_payload_expr == LDB_PAYLOAD_YEAR ? 1 : 0;
            if (base.secondYear && base.secondStage < 0) fail(LDB_ERR_INVALID, "the year expression applies to a shipped date32 column, not to a probe payload");
            base.nDec = d->n_out_cols - 2;
            int sendDecCols[2] = {0, 0};
            for (int k = 0; k < base.nDec; k++) {
               int col = R.col(d->out_columns[2 + k], {LDB_DECIMAL128}, "decimal tuple column");
               if (t->columns[col].precision >= 19) fail(LDB_ERR_UNSUPPORTED, "shipped decimals must have precision < 19");
               sendDecCols[k] = col;
            }
            const int64_t tupleBytes = 8 * (1 + base.nDec);
            const int64_t region = (int64_t) c->world * d->send_capacity * tupleBytes;
            if (d->send_capacity <= 0 || d->send_offset < 0 || d->send_offset % 16 || (size_t) (d->send_offset + region) > c->userBytes ||
                d->send_cursors_offset < 0 || d->send_cursors_offset % 16 || (size_t) d->send_cursors_offset + 16 * 8 > c->userBytes)
               fail(LDB_ERR_CAPACITY, "receive region / cursors outside the comm's user heap (create the comm with a larger heap)");
            base.world = c->world;
            for (int r = 0; r < c->world; r++) base.dest[r] = c->peerHeap[r] + kUserOff + d->send_offset + (int64_t) c->rank * d->send_capacity * tupleBytes;
            base.capacity = d->send_capacity;
            base.cursors = (unsigned long long*) (c->heap + kUserOff + d->send_cursors_offset);
            base.error = (int32_t*) (base.cursors + 8);
            for (auto& b : t->batches) {
               if (b.nRows == 0) continue;
               SendParams p = base;
               p.src.nRows = b.nRows;
               bindFilters(fp, b, p.src.filters);
               sp.bind(t, b, p.src.cols, kRowsPerThreadProbe);
               bindLazy(t, b, sendDecCols, base.nDec, p.dec);
               if (probe) p.probe = probe->join;
               waitBatch(ctx, b);
               ctx->launch("partition_send", [&] { launchScanPartitionSend(p, ctx->smCount, ctx->compute); });
            }
            break;
         }
         case LDB_PIPE_SCAN_STAR_PROBE_SEND: {
            LdbComm* c = d->comm;
            if (!c || c->ctx != ctx) fail(LDB_ERR_INVALID, "star-probe-send needs a comm of this context");
            if (!c->connected && c->world > 1) fail(LDB_ERR_INVALID, "comm is not connected to its peers yet");
            if (d->n_probes != 2) fail(LDB_ERR_INVALID, "star-probe-send pipelines take two probes (composite-key table, foreign-key table)");
            if (d->n_aggs != 1 || d->aggs[0].expr != LDB_EXPR_MUL_1MINUS_MINUS_PAYMUL) fail(LDB_ERR_UNSUPPORTED, "star-probe-send pipelines ship a * (1 - b) - $payload0 * c");
            if (d->n_out_cols != 1 || !d->out_columns[0]) fail(LDB_ERR_INVALID, "star-probe-send: out_columns[0] names the partition key");
            LdbState* tp = wantState(d->probe_states[0], LDB_STATE_JOIN_TABLE, "probe 0");
            LdbState* ts = wantState(d->probe_states[1], LDB_STATE_JOIN_TABLE, "probe 1");
            if (tp->join.stride != 16 || !d->probe_key2_columns[0]) fail(LDB_ERR_INVALID, "probe 0 of a star-probe-send pipeline is a composite-key table");
            if (ts->join.stride == 16) fail(LDB_ERR_INVALID, "probe 1 of a star-probe-send pipeline is a single-key table");
            StarSendParams base{};
            base.keyStageP0 = sp.add(t, R.col(d->probe_key_columns[0], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "probe key 0"));
            base.keyStageP1 = sp.add(t, R.col(d->probe_key2_columns[0], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "probe key 0 (second)"));
            base.keyStageS = sp.add(t, R.col(d->probe_key_columns[1], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "probe key 1"));
            base.keyStageO = sp.add(t, R.col(d->out_columns[0], {LDB_INT32, LDB_DATE32, LDB_FSB4}, "partition key"));
            int valueCols[3];
            for (int k = 0; k < 3; k++) {
               valueCols[k] = R.col(d->aggs[0].columns[k], {LDB_DECIMAL128}, "aggregate operand");
               if (t->columns[valueCols[k]].precision >= 19 || t->columns[valueCols[k]].scale != 2) fail(LDB_ERR_UNSUPPORTED, "aggregate operands must be decimal(p<19, 2) on the GPU path");
            }
            const int64_t region = (int64_t) c->world * d->send_capacity * 24;
            if (d->send_capacity <= 0 || d->send_offset < 0 || d->send_offset % 16 || (size_t) (d->send_offset + region) > c->userBytes ||
                d->send_cursors_offset < 0 || d->send_cursors_offset % 16 || (size_t) d->send_cursors_offset + 16 * 8 > c->userBytes)
               fail(LDB_ERR_CAPACITY, "receive region / cursors outside the comm's user heap (create the comm with a larger heap)");
            base.world = c->world;
            for (int r = 0; r < c->world; r++) base.dest[r] = c->peerHeap[r] + kUserOff + d->send_offset + (int64_t) c->rank * d->send_capacity * 24;
            base.capacity = d->send_capacity;
            base.cursors = (unsigned long long*) (c->heap + kUserOff + d->send_cursors_offset);
            base.error = (int32_t*) (base.cursors + 8);
            for (auto& b : t->batches) {
               if (b.nRows == 0) continue;
               StarSendParams p = base;
               p.src.nRows = b.nRows;
               bindFilters(fp, b, p.src.filters);
               sp.bind(t, b, p.src.cols, 2);
               bindLazy(t, b, valueCols, 3, p.values);
               p.tableP = tp->join;
               p.tableS = ts->join;
               waitBatch(ctx, b);
               ctx->launch("star_probe_send", [&] { launchScanStarProbeSend(p, ctx->smCount, ctx->compute); });
            }
            break;
         }
         default: fail(LDB_ERR_UNSUPPORTED, "unknown pipeline kind");
      }
   });
}

// ------------------------------------------------------------------------------------------------ repartition / misc
int ldb_gpu_partition_tuples(LdbContext* ctx, const int32_t* keys, const void* const* payload_cols, const int32_t* payload_widths, int32_t n_payload_cols, int64_t n_rows, int32_t n_parts,
                             int32_t* out_keys, void* const* out_payload_cols, int64_t* out_part_offsets, LdbError* err) {
   return guarded(err, [&] {
      if (n_parts < 1 || n_parts > 64) fail(LDB_ERR_INVALID, "n_parts must be in [1, 64]");
      if (n_payload_cols < 0 || n_payload_cols > 4) fail(LDB_ERR_INVALID, "at most 4 payload columns");
      for (int c = 0; c < n_payload_cols; c++)
         if (payload_widths[c] != 4 && payload_widths[c] != 8 && payload_widths[c] != 16) fail(LDB_ERR_INVALID, "payload width must be 4, 8 or 16");
      LDB_CUDA(cudaSetDevice(ctx->device));
      Scratch scratch(ctx);
      unsigned long long* counts = scratch.alloc<unsigned long long>(64 * 8);
      LDB_CUDA(cudaMemsetAsync(counts, 0, 64 * 8, ctx->compute));
      if (n_rows > 0) ctx->launch("partition", [&] { launchPartitionHistogram(keys, n_rows, n_parts, counts, ctx->smCount, ctx->compute); });
      unsigned long long h[64];
      LDB_CUDA(cudaMemcpyAsync(h, counts, 64 * 8, cudaMemcpyDeviceToHost, ctx->compute));
      ctx->syncStream(ctx->compute);
      unsigned long long cursor[64];
      int64_t off = 0;
      for (int p = 0; p < n_parts; p++) {
         out_part_offsets[p] = off;
         cursor[p] = (unsigned long long) off;
         off += (int64_t) h[p];
      }
      out_part_offsets[n_parts] = off;
      LDB_CUDA(cudaMemcpyAsync(counts, cursor, 64 * 8, cudaMemcpyHostToDevice, ctx->compute));
      if (n_rows > 0) ctx->launch("partition", [&] { launchPartitionScatter(keys, payload_cols, payload_widths, n_payload_cols, n_rows, n_parts, counts, out_keys, out_payload_cols, ctx->smCount, ctx->compute); });
      ctx->syncStream(ctx->compute);
   });
}
int ldb_gpu_join_table_insert(LdbContext* ctx, LdbState* table, const int32_t* keys, const int32_t* payloads, const int32_t* const* side_cols, int64_t n_rows, LdbError* err) {
   return guarded(err, [&] {
      wantSingleKeyTable(table, "insert target");
      if (n_rows <= 0) return;
      const int32_t* s0 = table->nSide > 0 && side_cols ? side_cols[0] : nullptr;
      const int32_t* s1 = table->nSide > 1 && side_cols ? side_cols[1] : nullptr;
      ctx->launch("join_build", [&] { launchInsertTuples(table->join, keys, payloads, s0, s1, n_rows, ctx->smCount, ctx->compute); });
   });
}
int ldb_gpu_hash_i64(LdbContext* ctx, const int64_t* a, const int64_t* b, int64_t n, uint64_t* out, LdbError* err) {
   return guarded(err, [&] {
      LDB_CUDA(cudaSetDevice(ctx->device));
      Scratch scratch(ctx);
      int64_t* da = scratch.alloc<int64_t>(n * 8);
      int64_t* db = b ? scratch.alloc<int64_t>(n * 8) : nullptr;
      uint64_t* dout = scratch.alloc<uint64_t>(n * 8);
      LDB_CUDA(cudaMemcpyAsync(da, a, n * 8, cudaMemcpyHostToDevice, ctx->compute));
      if (b) LDB_CUDA(cudaMemcpyAsync(db, b, n * 8, cudaMemcpyHostToDevice, ctx->compute));
      ctx->launch("hash", [&] { launchHashI64(da, db, n, dout, ctx->compute); });
      LDB_CUDA(cudaMemcpyAsync(out, dout, n * 8, cudaMemcpyDeviceToHost, ctx->compute));
      ctx->syncStream(ctx->compute);
   });
}

} // extern "C"
