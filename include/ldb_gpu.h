/* ldb_gpu.h — C-ABI of the H100 backend for LingoDB's three data-parallel hot paths
 * (Arrow scan + predicates/expressions, hash-join build+probe, hash group-by).
 *
 * Why a pipeline-level ABI: in the reference the per-tuple work (predicates, arithmetic, hashing, the
 * bucket probe, the aggregate update) is generated inline by SubOpToControlFlow and JIT-compiled;
 * src/runtime only owns state objects and calls back into JIT'd host function pointers per morsel
 * (DataSourceIteration.h:25, PreAggregationHashtable.h:40, ThreadLocal.h:9-11).  Device code cannot
 * call host function pointers, so this boundary receives DATA (descriptors) where the reference
 * passes CODE.  Each entry point cites the reference interface it replaces.
 *
 * Conventions: plain C, no exceptions; every call returns LDB_OK (0) or an error code and fills
 * `err` (may be NULL).  The C++ shim (integration/GPUPipeline.cpp) rethrows as
 * std::runtime_error to match the reference's convention (e.g. src/runtime/Hashtable.cpp:106).
 * Ownership mirrors ExecutionContext::registerState (include/lingodb/runtime/ExecutionContext.h:111-113):
 * states belong to the context and die with it; callers never free device memory themselves.
 */
#ifndef LDB_GPU_H
#define LDB_GPU_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------ errors */
enum LdbStatus {
   LDB_OK = 0,
   LDB_ERR_CUDA = 1,        /* CUDA runtime failure (reference: CudaUtils.cuh:5-20 prints and exits) */
   LDB_ERR_UNSUPPORTED = 2, /* descriptor does not match a compiled pipeline */
   LDB_ERR_INVALID = 3,     /* bad argument (unknown column, wrong type, NULL handle …) */
   LDB_ERR_CAPACITY = 4,    /* a device table overflowed its declared capacity */
   LDB_ERR_NO_DEVICE = 5    /* no CUDA device: there is NO CPU fallback on this path */
};
typedef struct LdbError {
   int32_t code;
   char message[252];
} LdbError;

/* ------------------------------------------------------------------------------------ context
 * Replaces: runtime::ExecutionContext (state ownership) + the scheduler hand-off
 * (scheduler::awaitChildTask, include/lingodb/scheduler/Scheduler.h:32-33): one context per device,
 * work is issued on the context's CUDA streams instead of worker fibers. */
typedef struct LdbContext LdbContext;
typedef struct LdbDeviceInfo {
   int32_t device, sm_count, cc_major, cc_minor;
   int64_t total_mem, free_mem, l2_bytes;
   char name[64];
} LdbDeviceInfo;
int ldb_gpu_context_create(int device, LdbContext** out, LdbError* err);
void ldb_gpu_context_destroy(LdbContext* ctx);
int ldb_gpu_device_info(LdbContext* ctx, LdbDeviceInfo* out, LdbError* err);
int ldb_gpu_synchronize(LdbContext* ctx, LdbError* err);
/* the CUDA stream (cudaStream_t) every pipeline kernel of this context is launched on, so callers can order their own
 * work (NCCL collectives, allocator frees) after it without a host synchronisation */
void* ldb_gpu_context_stream(LdbContext* ctx);
/* number of kernels this library has launched on the context since creation (bench "gpu_launches") */
int64_t ldb_gpu_launch_count(LdbContext* ctx);
/* CUDA-event timing on the context's compute stream (the stream every pipeline kernel runs on) */
int ldb_gpu_timer_start(LdbContext* ctx, LdbError* err);
int ldb_gpu_timer_stop(LdbContext* ctx, float* milliseconds, LdbError* err);
/* device time (ms) and launch count accumulated by one named kernel family since the last reset;
 * name = "scan_groupby" | "scan_reduce" | "join_build" | "join_probe" | … (roofline leg of bench.py) */
int ldb_gpu_kernel_time(LdbContext* ctx, const char* family, float* ms, int64_t* launches, LdbError* err);
int ldb_gpu_kernel_time_reset(LdbContext* ctx, int enable, LdbError* err);

/* ------------------------------------------------------------------------------------ captured queries
 * "Compile once, run many" (the reference JIT-compiles a query's main() once, src/execution/LLVMBackends.cpp:795-867): between
 * _begin and _end the context's compute stream is captured into a CUDA graph — state creation, pipelines over DEVICE-resident or
 * already staged tables and peer collectives (ldb_gpu_groupby_allmerge, ldb_gpu_comm_barrier) are recorded instead of run; result
 * reads and anything that synchronises stay outside.  ldb_gpu_graph_launch replays the whole sequence with one driver call;
 * states created inside the capture are re-initialised by each replay and are read (ldb_gpu_groupby_read …) after it. */
typedef struct LdbGraph LdbGraph;
int ldb_gpu_graph_begin(LdbContext* ctx, LdbError* err);
int ldb_gpu_graph_end(LdbContext* ctx, LdbGraph** out, LdbError* err);
int ldb_gpu_graph_launch(LdbGraph* graph, LdbError* err);
void ldb_gpu_graph_destroy(LdbGraph* graph);

/* ------------------------------------------------------------------------------------ tables
 * Replaces: ArrayView/BatchView (include/lingodb/runtime/ArrowView.h:8-29), LingoDBTable::TableChunk
 * (src/runtime/storage/LingoDBTable.cpp:200-225) and DataSource::get (src/runtime/DataSourceIteration.cpp:57).
 * LdbArrayView has the exact field layout of lingodb::runtime::ArrayView, so the reference's
 * TableChunk::getArrayView() pointers can be passed through unchanged. */
typedef struct LdbArrayView {
   int64_t length, null_count, offset, n_buffers, n_children;
   const void** buffers; /* [0] validity (may be NULL), [1] values or utf8 offsets, [2] utf8 bytes */
   const struct LdbArrayView** children;
} LdbArrayView;
enum LdbPhysType { LDB_INT32 = 0, LDB_INT64 = 1, LDB_DATE32 = 2, LDB_DECIMAL128 = 3, LDB_FSB4 = 4, LDB_UTF8 = 5,
                   /* read by the program pipeline (ldb_gpu_run_program) only */
                   LDB_INT8 = 6, LDB_INT16 = 7, LDB_FLOAT32 = 8, LDB_FLOAT64 = 9 };
typedef struct LdbColumnSchema {
   const char* name;
   int32_t type; /* LdbPhysType: physical Arrow type as in LingoDBTable.cpp:122-195 */
   int32_t precision, scale;
} LdbColumnSchema;
enum LdbMemLocation { LDB_MEM_HOST = 0, LDB_MEM_DEVICE = 1 };
typedef struct LdbTable LdbTable;
int ldb_gpu_table_create(LdbContext* ctx, const char* name, int32_t n_cols, const LdbColumnSchema* schema, LdbTable** out, LdbError* err);
/* Append one record batch.  HOST buffers are staged to HBM with asynchronous copies on the context's
 * copy stream (the scan of batch k overlaps the copy of batch k+1); DEVICE buffers are borrowed.
 * Borrowed DEVICE buffers must not change while the batch belongs to the table (until ldb_gpu_table_clear /
 * _destroy): the table caches what it derived from them — column min/max statistics and the encoded column copies the
 * scan pipelines read (ldb_gpu_set_encoded_scan).  To change the data, clear the table and append it again.
 * utf8 columns additionally need `utf8_bytes[col]` = size of buffers[2] (0 for other columns). */
int ldb_gpu_table_append_batch(LdbTable* t, int64_t n_rows, const LdbArrayView* columns, const int64_t* utf8_bytes, int32_t location, LdbError* err);
int ldb_gpu_table_clear(LdbTable* t, LdbError* err); /* drop all batches (staging memory is pooled) */
/* Bytes copied host→device by this context's table staging so far.  HOST decimal128(p<19) columns are narrowed on
 * the host to the 8 bytes per value the kernels read (the JIT truncates them to i64, LowerToStd.cpp:111-209), so they
 * cost 8 B/value of PCIe instead of 16; LDB_NARROW_STAGING=0 in the environment disables it. */
int64_t ldb_gpu_context_h2d_bytes(LdbContext* ctx);
/* Compressed staging (csrc/staging.cu): HOST batches of >= 65 536 rows are re-encoded by host threads (frame of reference,
 * 1/2/4/8 bytes per value per 64 Ki-value block) and decoded on the GPU; idle PCIe time is filled by raw copiers that ship
 * Arrow cells unchanged.  rows the raw copiers took so far / CPUs the process may use (cgroup quota aware): */
int64_t ldb_gpu_context_raw_staged_rows(LdbContext* ctx);
int32_t ldb_gpu_effective_cpus(void);
/* experiment hook: depth of the TMA tile pipeline (2..4 stages) of the join-build / probe-aggregate / probe-probe-group / star-probe
 * kernels and the rows per thread of a build tile (1, 2, 4); defaults = measured best, also settable
 * through LDB_STAGES_BUILD / _PROBE_AGG / _PROBE2 / _STAR and LDB_RPT_BUILD */
void ldb_gpu_set_tuning(int32_t stages_build, int32_t stages_probe_agg, int32_t stages_probe2, int32_t stages_star, int32_t rows_per_thread_build);
/* experiment hook: 1 (default) = the join pipelines (build, probe-aggregate, probe-probe-group, star probe) run the instantiation compiled for
 * their filter SHAPE (none / one int32 compare / one int32 range — what the reference's JIT would emit for the same pushed-down predicate);
 * 0 = always the descriptor-driven form.  Results are identical; also settable through LDB_SPECIALISE. */
void ldb_gpu_set_filter_specialisation(int32_t on);
/* 1 (default) = scan-reduce / scan-group-by pipelines (Q6, Q1 signatures) read a DEVICE batch from a frame-of-reference copy of its
 * fixed-width columns (csrc/encode.cu: per 64 Ki-row block a base, values in 1/2/4/8 bytes; Q1 ~12 B/row instead of 76), built
 * once on the first such pipeline that needs it and freed by ldb_gpu_table_clear / _destroy; 0 = Arrow cells only.  Results are
 * identical; also settable through LDB_ENCODED_SCAN.  A copy that cannot be allocated, or that would take the context past
 * LDB_ENCODED_SCAN_MAX_BYTES (environment, read at context creation; default unlimited), leaves its batch in Arrow layout.
 * Bytes the copies of a context hold now: */
void ldb_gpu_set_encoded_scan(int32_t on);
int64_t ldb_gpu_context_encoded_bytes(LdbContext* ctx);
/* experiment hook: nanoseconds the producer lane / the consumer warps of the warp-specialised tile driver pause between two polls of
 * a tile barrier (0 = poll back to back; also LDB_PRODUCER_SLEEP_NS / LDB_CONSUMER_SLEEP_NS) */
void ldb_gpu_set_poll_pause(int32_t producer_ns, int32_t consumer_ns);
int64_t ldb_gpu_table_num_rows(const LdbTable* t);
void ldb_gpu_table_destroy(LdbTable* t);

/* ------------------------------------------------------------------------------------ states
 * Device-resident runtime objects behind the reference's names:
 *   LDB_STATE_SIMPLE      rt::SimpleState (src/runtime/SimpleState.cpp:8-30): keyless aggregates
 *   LDB_STATE_GROUPBY     rt::PreAggregationHashtable(+Fragment) / rt::Hashtable
 *                         (PreAggregationHashtable.cpp:46-170, Hashtable.cpp:10-150): small-domain group-by
 *   LDB_STATE_JOIN_TABLE  rt::GrowingBuffer + rt::HashIndexedView (GrowingBuffer.cpp:39-113,
 *                         LazyJoinHashtable.cpp:12-34): key → payload multimap; with aggregate
 *                         lanes it is the group-join map of SubOpToControlFlow.cpp:2730-2839.
 *   LDB_STATE_KEY_JOIN    rt::HashIndexedView over a key TUPLE (db.hash over the tuple, LowerToStd.cpp:1139-1150):
 *                         1..4 int64 keys → int64 payload, for program pipelines (ldb_gpu_join_table_create_keys).
 * The memory image differs from the CPU objects (open addressing, 32-bit payloads, no tagged
 * pointers): the contract is the same MULTISET of results, not the same bytes (SURVEY §7). */
enum LdbStateKind { LDB_STATE_SIMPLE = 1, LDB_STATE_GROUPBY = 2, LDB_STATE_JOIN_TABLE = 3, LDB_STATE_HASHAGG = 4, LDB_STATE_DICT = 5, LDB_STATE_KEY_JOIN = 6 };
typedef struct LdbState LdbState;
typedef struct LdbI128 {
   uint64_t lo;
   int64_t hi;
} LdbI128;

/* Frees one state early (a query's states die together when its ExecutionContext does,
 * ExecutionContext.cpp:27-40; long-lived contexts release per query with this). */
void ldb_gpu_state_destroy(LdbState* s);

#define LDB_MAX_AGGS 8
#define LDB_MAX_KEYS 2
#define LDB_MAX_SIDE 2

int ldb_gpu_simple_state_create(LdbContext* ctx, int32_t n_aggs, LdbState** out, LdbError* err);
int ldb_gpu_simple_state_read(LdbState* s, LdbI128* aggs /* n_aggs */, LdbError* err);

int ldb_gpu_groupby_create(LdbContext* ctx, int32_t n_keys, int32_t n_aggs, int32_t capacity, LdbState** out, LdbError* err);
typedef struct LdbGroupRow {
   int32_t keys[LDB_MAX_KEYS];
   LdbI128 aggs[LDB_MAX_AGGS];
} LdbGroupRow;
/* rt::PreAggregationHashtable::createIterator + BufferIterator::iterate, for a tiny result */
int ldb_gpu_groupby_read(LdbState* s, LdbGroupRow* rows, int32_t max_rows, int32_t* n_rows, LdbError* err);
/* fold another GPU's partial groups into this state (K7 merge; rt::PreAggregationHashtable::merge).  Every merge (_merge_rows,
 * _merge_exported, ldb_gpu_groupby_allmerge) adds the 128-bit cells per key and carries no width: a merged lane is read at the width
 * of its TARGET (a 64-bit lane as the sign-extended low word).  So the target's lanes must have been bound by a pipeline (LdbAggDesc);
 * a merge into a state with an unbound aggregate lane fails with LDB_ERR_UNSUPPORTED. */
int ldb_gpu_groupby_merge_rows(LdbState* s, const LdbGroupRow* rows, int32_t n_rows, LdbError* err);

/* Multi-GPU merge without a host round trip: copy the table image {state[cap], keys[cap][2], acc[cap][8][2]}
 * into a caller-provided DEVICE buffer (bytes = ldb_gpu_groupby_export_bytes), all-gather it with NCCL,
 * then fold the `n_tables` images (skipping `skip_index`, the caller's own) back into the state. */
int64_t ldb_gpu_groupby_export_bytes(LdbState* s);
int ldb_gpu_groupby_export(LdbState* s, void* dev_dst, LdbError* err);
int ldb_gpu_groupby_merge_exported(LdbState* s, const void* dev_src, int32_t n_tables, int32_t skip_index, LdbError* err);

/* unique_keys is a flag word: LDB_JOIN_UNIQUE = the build keys are unique (a probe stops at its first match, a duplicate
 * insert is an error); LDB_JOIN_NO_BLOOM = no Bloom filter in front of the directory (foreign-key probes that always
 * hit gain nothing from it, and the build saves one random atomic per row). */
enum LdbJoinFlags { LDB_JOIN_UNIQUE = 1, LDB_JOIN_NO_BLOOM = 2 };
/* expected_rows sizes the directory like HashIndexedView::build (nextPow2 of a multiple of n);
 * n_side = int32 payload lanes stored beside the slot; n_aggs = int128 aggregate lanes (group-join) */
int ldb_gpu_join_table_create(LdbContext* ctx, int64_t expected_rows, int32_t unique_keys, int32_t n_side, int32_t n_aggs, LdbState** out, LdbError* err);
/* composite (int32, int32) key → int64 payload (a decimal(p<19) value or an int32); Q9's partsupp side:
 * (ps_partkey, ps_suppkey) → ps_supplycost.  Slot placement uses its own 64-bit mix, not db.hash over the tuple
 * (LowerToStd.cpp:1139-1150), whose XOR-combine clusters correlated keys under open addressing (csrc/kernels.cu). */
int ldb_gpu_join_table_create_pair(LdbContext* ctx, int64_t expected_rows, int32_t unique_keys, LdbState** out, LdbError* err);
/* Direct-address table for DENSE unique int32 keys in [key_min, key_max] (surrogate primary keys): slot = key - key_min
 * holds the int32 payload.  No reference counterpart as an object — it is what the reference's INLJ over a primary-key
 * index degenerates to for dense keys (OptimizeImplementations.cpp:226-244, LingoDBHashIndex.cpp:32-147).  Accepted as the
 * sink of a K3 build without side lanes and as probe 1/2 of a K9 star probe; a key outside the range or a duplicate key
 * fails the build (LDB_ERR_INVALID).  ldb_gpu_table_column_range gives the plan the column's min/max (one streaming pass). */
int ldb_gpu_join_table_create_direct(LdbContext* ctx, int32_t key_min, int32_t key_max, LdbState** out, LdbError* err);
int ldb_gpu_table_column_range(LdbTable* t, const char* column, int32_t* min, int32_t* max, LdbError* err);
/* Key-tuple join table (LDB_STATE_KEY_JOIN): n_keys (1..4) int64 keys → int64 payload, for program pipelines only — built by the
 * JOIN_BUILD sink (keys from LdbProgramDesc.n_keys / key_regs), read by LDB_OP_PROBE / LDB_OP_PROBE_EACH (keys from consecutive
 * registers).  The directory holds nextPow2(2 x expected_rows) entries; a build that overflows it fails with LDB_ERR_CAPACITY, as
 * does an insert that finds no free slot within 65 536 probes (more duplicates of one tuple than that in a multimap).  flags:
 * LDB_JOIN_UNIQUE = set semantics, a duplicate key tuple is dropped (which of the duplicates' payloads is kept is unspecified);
 * LDB_JOIN_NO_BLOOM = no Bloom filter.  Without it the table is a multimap: every duplicate is kept.  ldb_gpu_join_table_count,
 * ldb_gpu_state_destroy, ldb_gpu_register_state and ldb_gpu_find_state take it; the specialised pipelines, serialised steps and every
 * other join-table entry point refuse it (LDB_ERR_INVALID).  Not for captured queries: creating, building or probing one while a
 * capture is in progress fails with LDB_ERR_UNSUPPORTED. */
int ldb_gpu_join_table_create_keys(LdbContext* ctx, int32_t n_keys, int64_t expected_rows, int32_t flags, LdbState** out, LdbError* err);
int ldb_gpu_join_table_count(LdbState* s, int64_t* n_entries, LdbError* err);
/* Join-table markers (LDB_OP_MARK) of a plain single-key, direct-address or key-tuple join table.  ldb_gpu_join_table_marks returns a
 * single-batch DEVICE table over the table's entries: which = 1 the marked ones, 0 the unmarked ones, -1 all of them.  Columns: "key"
 * (int64; a direct-address table's keys are key_min + slot), or "k0".."k{n-1}" for a key-tuple table; "payload" (int64, e.g. a ROWID
 * for side-column reads); with which = -1 also "marked" (int32, 0 / 1).  Row order is unspecified.  A table no program has marked reads
 * as all unmarked; entries inserted after marking start unmarked.  ldb_gpu_join_table_clear_marks unmarks every entry (a table without
 * markers: nothing to do).  Both refuse NULL arguments, other states, pair tables and group-join maps (LDB_ERR_INVALID) and captured
 * queries (LDB_ERR_UNSUPPORTED). */
int ldb_gpu_join_table_marks(LdbState* s, int32_t which, const char* name, LdbTable** out, LdbError* err);
int ldb_gpu_join_table_clear_marks(LdbState* s, LdbError* err);
typedef struct LdbTopKRow {
   int32_t key, side[LDB_MAX_SIDE];
   int32_t pad;
   LdbI128 agg;
} LdbTopKRow;
/* The table's Bloom filter as a DEVICE buffer (NULL/0 for tiny tables): ranks that hold hash partitions of one
 * logical build side OR their filters together (NCCL all_reduce BOR) so every rank can pre-filter its probe side. */
int ldb_gpu_join_table_bloom(LdbState* s, void** dev_ptr, int64_t* bytes, LdbError* err);
/* scan of the group-join map + Heap (include/lingodb/runtime/Heap.h): marked groups ordered by
 * (agg0 desc, side0 asc, key asc), first k; agg0 compares as a signed 128-bit value (a 64-bit SUM sign-extended) */
int ldb_gpu_join_table_topk(LdbState* s, int32_t k, LdbTopKRow* rows, int32_t* n_rows, LdbError* err);

/* ------------------------------------------------------------------------------------ pipelines
 * Replaces: one execution step of the JIT'd main() — rt::DataSourceIteration::iterate(scan_func)
 * (DataSourceIteration.cpp:90-96) plus the inlined per-tuple code of SubOpToControlFlow
 * (scan :1123-1203, probe :2558-2586 + :2254-2313, group-by :3065-3157, reduce :3719-3769).
 * A pipeline = table scan → pushed-down filters → optional hash-table probes → one sink. */
enum LdbFilterOp { LDB_EQ = 0, LDB_NEQ = 1, LDB_LT = 2, LDB_LTE = 3, LDB_GT = 4, LDB_GTE = 5, LDB_NOTNULL = 6, LDB_IN = 7,
                   /* not a TableStorage.h FilterOp: `col like '%str_value%'` on a utf8 column, which the reference evaluates in the
                    * JIT'd selection above the scan (ConstLike → StringRuntime::findMatch, RuntimeFunctions.cpp:60-170,
                    * StringRuntime.cpp:337-345); the GPU scan takes it as one more predicate */
                   LDB_CONTAINS = 8 };
/* FilterDescription (include/lingodb/runtime/storage/TableStorage.h:14-31): column-vs-constant;
 * the constant is a string (dates "YYYY-MM-DD", decimals "0.05", char/varchar text) or an integer */
#define LDB_MAX_IN_VALUES 8
typedef struct LdbFilterDesc {
   const char* column;
   int32_t op;          /* LdbFilterOp */
   int32_t value_is_int;
   const char* str_value;
   int64_t int_value;
   /* LDB_IN (SimpleTypeInFilter, Restrictions.cpp:194-236): up to LDB_MAX_IN_VALUES constants, typed like the single value */
   int32_t n_values;
   const char* str_values[LDB_MAX_IN_VALUES];
   int64_t int_values[LDB_MAX_IN_VALUES];
} LdbFilterDesc;

/* value expressions over decimal(12,2) columns, typed as DBOps.cpp:98-107,221-262 types them */
enum LdbExprKind {
   LDB_EXPR_COL = 0,               /* a                       decimal(12,2)  i64  */
   LDB_EXPR_MUL = 1,               /* a * b                   decimal(24,4)  i128 */
   LDB_EXPR_MUL_1MINUS = 2,        /* a * (1 - b)             decimal(33,4)  i128 */
   LDB_EXPR_MUL_1MINUS_1PLUS = 3,  /* a * (1 - b) * (1 + c)   decimal(38,6)  i128 */
   LDB_EXPR_ONE = 4,               /* count(*) */
   LDB_EXPR_MUL_1MINUS_MINUS_PAYMUL = 5 /* a * (1 - b) - $payload0 * c   decimal(34,4) i128; K9 only ($payload0 = probe 0's int64 payload) */
};
typedef struct LdbAggDesc {
   int32_t expr;            /* LdbExprKind; every aggregate is SUM (count = SUM of ONE); i64 sums (COL, ONE) wrap at 64 bits and
                               are read back sign-extended (LdbI128.hi = lo >> 63) by every sink, the group-join map's top-k included;
                               i128 sums wrap at 128 bits.  An aggregate of a state keeps the width of the first pipeline that
                               summed into it: a later pipeline of the other width fails with LDB_ERR_UNSUPPORTED.  Every group
                               sink binds its lanes: K1/K2 and K4 by their aggregates, K5 lane 0 of the group-join map, and K9,
                               ldb_gpu_probe_received_groupby and _groupby2 lane 0 as 128-bit */
   const char* columns[3];  /* a, b, c */
} LdbAggDesc;

enum LdbPipelineKind {
   /* K1  scan → filters → keyless SUMs → SimpleState                       (Q6) */
   LDB_PIPE_SCAN_REDUCE = 1,
   /* K2  scan → filters → group by ≤2 int32/char keys, SUMs → GroupBy      (Q1) */
   LDB_PIPE_SCAN_GROUPBY = 2,
   /* K3  scan → filters → [probe] → insert {key, payload, side…} → JoinTable
    *     (subop.materialize + create_hash_indexed_view; group-join insert side) */
   LDB_PIPE_SCAN_BUILD = 3,
   /* K5  scan → filters → probe group-join map → atomic SUM into the entry, set marker (Q3) */
   LDB_PIPE_SCAN_PROBE_AGG = 4,
   /* K4  scan → filters → probe A → probe B (payload equality) → group by payload, SUM → GroupBy (Q5) */
   LDB_PIPE_SCAN_PROBE2_GROUPBY = 5,
   /* K8  scan → filters → [probe | Bloom-only semi-join] → append selected columns to dense device buffers
    *     (subop.materialize into a rt::GrowingBuffer, GrowingBuffer.cpp:44, as compacted columns): the
    *     tuple stream that K6 partitions for the all-to-all repartition step */
   LDB_PIPE_SCAN_MATERIALIZE = 6,
   /* K9  scan → filters → probe 0 (composite key, int64 payload) → probe 1 → probe 2 → group by (payload 1, payload 2),
    *     SUM(aggs[0]) with aggs[0].expr = LDB_EXPR_MUL_1MINUS_MINUS_PAYMUL → GroupBy with 2 keys            (Q9) */
   LDB_PIPE_SCAN_STAR_PROBE_GROUPBY = 7,
   /* K10 scan → filters → [probe | Bloom-only semi-join] → radix partition by h64(key) across the ranks of `comm` → tuples stored
    *     straight into the DESTINATION rank's receive region over NVLink (fused partition + exchange; multi-GPU joins).
    *     out_columns[0] = partition/join key (int32), out_columns[1] = second int32 column or "$payload" (build_payload_expr =
    *     LDB_PAYLOAD_YEAR ships extract(year from that date32 column) instead), out_columns[2..3] =
    *     decimal(p<19) columns shipped as their low 8 bytes.  Tuple = 1 + (n_out_cols - 2) eight-byte words.  The receive region of
    *     every rank is heap[send_offset, + world * send_capacity * tuple bytes): sub-region s belongs to source rank s.
    *     send_cursors_offset: heap offset of 16 uint64 (zeroed by the caller): [d] = tuples sent to rank d, [8] = overflow flag.
    *     The full probe is a semi-join: one tuple per qualifying row with at least one match (K8 emits one per match), so "$payload"
    *     needs a probe table created LDB_JOIN_UNIQUE (else LDB_ERR_UNSUPPORTED).  A cursor counts every tuple; only the first
    *     send_capacity of each destination are stored, the rest set the overflow flag. */
   LDB_PIPE_SCAN_PARTITION_SEND = 8,
   /* K11 scan → filters → probe 0 (composite key, int64 payload c; Bloom first) → probe 1 (foreign key → int32 payload g) → the row's
    *     a * (1 - b) - c * d (aggs[0] = LDB_EXPR_MUL_1MINUS_MINUS_PAYMUL) is shipped as {out_columns[0] : 32 | g : 32, lo, hi} (24 bytes)
    *     to the rank that owns h64(out_columns[0]) — the probe side of a star join whose LAST build side is hash-partitioned across
    *     the ranks (Q9's orders).  comm / send_* as for K10; the receiver runs ldb_gpu_probe_received_groupby2. */
   LDB_PIPE_SCAN_STAR_PROBE_SEND = 9
};
/* inline payload of a K3 build: the column's value, or extract(year from <date32 column>) (DateRuntime::extractYear) */
enum LdbPayloadExpr { LDB_PAYLOAD_COLUMN = 0, LDB_PAYLOAD_YEAR = 1 };
#define LDB_MAX_PROBES 3
#define LDB_MAX_OUT_COLS 4
typedef struct LdbPipelineDesc {
   int32_t kind; /* LdbPipelineKind */
   LdbTable* source;
   int32_t n_filters;
   const LdbFilterDesc* filters;
   /* group-by keys (K2) */
   int32_t n_keys;
   const char* key_columns[LDB_MAX_KEYS];
   /* aggregates (K1, K2: n_aggs; K4, K5: aggs[0]) */
   int32_t n_aggs;
   LdbAggDesc aggs[LDB_MAX_AGGS];
   /* probes: probe_key_columns[i] (and probe_key2_columns[i] for a composite-key table) is looked up in
    * probe_states[i] (K3: 0 or 1, K5: 1, K4: 2, K9: 3) */
   int32_t n_probes;
   LdbState* probe_states[LDB_MAX_PROBES];
   const char* probe_key_columns[LDB_MAX_PROBES];
   const char* probe_key2_columns[LDB_MAX_PROBES];
   /* K3 build: inserted key, inline payload (a column, or the probe's payload when NULL and a
    * probe is present, or 0), side payload columns */
   const char* build_key_column;
   const char* build_key2_column;  /* second key column when the sink is a composite-key table, else NULL */
   const char* build_payload_column;
   int32_t build_payload_expr;     /* LdbPayloadExpr */
   int32_t n_side;
   const char* side_columns[LDB_MAX_SIDE];
   LdbState* sink; /* SimpleState | GroupBy | JoinTable (K5: the probed map itself) */
   /* K8 materialize: out_columns[i] names a fixed-width source column, or "$payload" = the inline payload of
    * probe 0; out_buffers[i] are DEVICE buffers of out_capacity rows (column width as in the source schema,
    * 4 bytes for $payload); out_count is a DEVICE uint64 the kernel adds the number of appended rows to
    * (rows beyond out_capacity are counted but not written → the caller regrows and reruns).
    * probe_bloom_only != 0: probe 0 only consults the table's Bloom filter (semi-join reduction before a shuffle) */
   int32_t n_out_cols;
   const char* out_columns[LDB_MAX_OUT_COLS];
   void* out_buffers[LDB_MAX_OUT_COLS];
   int64_t out_capacity;
   uint64_t* out_count;
   int32_t probe_bloom_only;
   /* K10 partition-send */
   struct LdbComm* comm;
   int64_t send_offset, send_capacity, send_cursors_offset;
} LdbPipelineDesc;
int ldb_gpu_run_pipeline(LdbContext* ctx, const LdbPipelineDesc* desc, LdbError* err);

/* ------------------------------------------------------------------------------------ serialised steps
 * One execution step as a DOCUMENT: what a compiler hook (GPUPatternList / handleExecutionStepGPU, SURVEY §8 f1;
 * SubOpToControlFlow.cpp:4254-4394) emits for a scan pipeline and what rt::GPUPipeline::run(VarLen32 descr) receives, like the
 * hex-serialised description DataSource::get receives today (DataSourceIteration.cpp:57-88).  JSON:
 *   {"kind": "scan_groupby", "source": "<table name>", "filters": [{"column", "op", "value" | "values"}], "keys": [...],
 *    "aggs": [{"expr", "columns"}], "probes": [{"state", "key", "key2"}], "build": {"key", "key2", "payload", "payload_expr", "side"},
 *    "sink": {"name", "create": {"type": "simple|groupby|join|join_pair|join_direct", ...}}}
 * Tables are resolved by the name given to ldb_gpu_table_create, states by the names steps gave them (or ldb_gpu_register_state).
 * tests/golden/plans/ holds the five TPC-H plans in this form (q1.json … q9.json). */
int ldb_gpu_step_validate(const char* json, LdbError* err); /* structure only; needs no device */
int ldb_gpu_run_step(LdbContext* ctx, const char* json, LdbError* err);
int ldb_gpu_run_step_hex(LdbContext* ctx, const char* hex_json, LdbError* err);
int ldb_gpu_register_state(LdbContext* ctx, const char* name, LdbState* s, LdbError* err);
LdbState* ldb_gpu_find_state(LdbContext* ctx, const char* name);

/* ------------------------------------------------------------------------------------ program pipelines (generic)
 * The hand-specialised pipelines above cover the TPC-H hot shapes at HBM speed.  Everything else a scan pipeline of the
 * sub-operator dialect can contain runs through ONE kernel that interprets a register program per row (csrc/program.cu):
 *   expressions   db.add/sub/mul/div/cmp/and/or/not/between/case over int8..int64, date32, char(1), decimal(38), float/double
 *                 (LowerToStd.cpp:612-700,851-910; decimal scales are the program writer's job, exactly as the lowering rescales)
 *   nulls         every LOAD tests the column's validity bit (Restrictions.cpp:67-162, LowerToStd.cpp:111-209); SQL three-valued logic
 *   strings       =, <>, <, <=, >, >= against constants, LIKE 'x%' / '%x' / '%x%' (VarLen32Filter, Restrictions.cpp:234-325);
 *                 strings of any length as int32 keys through a string dictionary (LDB_OP_STRCODE)
 *   joins         PROBE: key → payload of a join table, NULL when absent → semi / anti / mark / left-outer joins
 *                 (RelAlgToSubOp.cpp:1129-1206,1340-1588) as a filter or a value; MARK: markers on the matched build entries →
 *                 reversed semi / anti / mark joins, right and full outer joins (RelAlgToSubOp.cpp:1248-1528); EXISTS: a residual
 *                 predicate over each match, reduced to one boolean per probe tuple (anyTuple, RelAlgToSubOp.cpp:1296-1304, used at
 *                 :1360, :1395, :1430, :1506, :1565) → semi / anti / mark joins with a residual and left outer joins with a residual
 *   sinks         hash aggregation with up to 4 (nullable) int64 keys and SUM/COUNT/MIN/MAX/ANY over ANY number of groups
 *                 (rt::PreAggregationHashtable::merge, PreAggregationHashtable.cpp:76-170; rt::Hashtable, Hashtable.cpp:10-150;
 *                 subop.reduce, SubOpToControlFlow.cpp:3540-3769), a join-table build, or compacted output columns.
 * It is slower than the specialised kernels (one thread per row, registers in local memory) — it is the catch-all. */
enum LdbOp {
   LDB_OP_LOAD = 1,    /* dst = columns[arg]                                  (NULL from the validity bit) */
   LDB_OP_CONST = 2,   /* dst = consts[arg] */
   LDB_OP_ADD = 3, LDB_OP_SUB = 4, LDB_OP_MUL = 5, /* wrapping i128 */
   LDB_OP_DIV = 6,     /* truncating signed division; x / 0 = NULL */
   LDB_OP_NEG = 7,
   LDB_OP_CMP = 8,     /* dst = a <arg: LDB_EQ..LDB_GTE> b                    (integers, decimals at equal scale, dates, char(1)) */
   LDB_OP_AND = 9, LDB_OP_OR = 10, LDB_OP_NOT = 11, /* three-valued */
   LDB_OP_ISNULL = 12,
   LDB_OP_SELECT = 13, /* dst = regs[arg] is true ? a : b                     (CASE WHEN) */
   LDB_OP_I2F = 14, LDB_OP_FADD = 15, LDB_OP_FSUB = 16, LDB_OP_FMUL = 17, LDB_OP_FDIV = 18,
   LDB_OP_FCMP = 19,   /* like CMP on doubles */
   LDB_OP_STRCMP = 20, /* dst = columns[a] <b: LDB_EQ..LDB_GTE> strings[arg] */
   LDB_OP_STRLIKE = 21,/* dst = columns[a] LIKE strings[arg]; b = 0 'x%', 1 '%x', 2 '%x%' */
   LDB_OP_YEAR = 22,   /* dst = extract(year from date32 a) */
   LDB_OP_PROBE = 23,  /* dst = payload of int32 key a in tables[arg]; NULL when absent.  On a key-tuple join table of n keys
                          (LDB_STATE_KEY_JOIN) the key is the tuple of registers a, a+1, …, a+n-1 and the payload comes back as int64; a
                          NULL component or one outside int64 never matches, and a probe run that reaches the interpreter's bound of
                          16384 slots fails the call (LDB_ERR_CAPACITY). */
   LDB_OP_STRKEY8 = 24,/* dst = first 8 bytes of columns[a], zero padded, big-endian, as a signed int64 (a group / sort key for short
                          strings: char(n<=8), flags, codes; longer strings take LDB_OP_STRCODE).  It preserves the
                          bytewise string order only while the first byte is below 0x80 (7-bit text): a first byte >= 0x80 makes the
                          key negative, so such strings order before ASCII ones. */
   LDB_OP_ROWID = 25,  /* dst = global row number of the scanned row in its table (a row-id build payload for side-column reads) */
   LDB_OP_PROBE_EACH = 26,/* dst = payload of EACH match of int32 key a in tables[arg] (plain single-key or direct-address tables); the
                             instructions after it, the filter and the sink run once per match.  b = 0 inner join (no match: no tuple),
                             b = 1 left outer join (no match: one tuple with dst NULL).  A NULL key never matches.  At most one per
                             program; later instructions may not overwrite registers written at or before it.  A probe run longer
                             than the interpreter's bound fails the call (LDB_ERR_CAPACITY) rather than dropping matches.  On a
                             key-tuple join table the key is the tuple of registers a .. a+n-1, as for PROBE. */
   LDB_OP_STRCODE = 27,/* dst = int32 code of the utf8 string columns[a] (a source or side column) in the string dictionary tables[arg]
                          (ldb_gpu_dict_create).  b = 1 inserts an absent string, b = 0 only looks up: an absent string gives NULL.  A
                          NULL string gives NULL and is never inserted.  Every instruction runs before the WHERE test, so b = 1 inserts
                          the string of every row it is evaluated on, whether WHERE keeps the row or not.  A code fits int32: it is a
                          hash-aggregation key, a join-build key or payload, a PROBE / PROBE_EACH key (a string equi-join builds with
                          b = 1 and probes with b = 0).  The call fails with LDB_ERR_CAPACITY when the dictionary overflows. */
   LDB_OP_MARK = 28,   /* dst = MARK(a, arg): when a is TRUE and the latest PROBE / PROBE_EACH of tables[arg] for this tuple matched an entry,
                          sets that entry's marker; dst is TRUE when it marked, else FALSE (never NULL).  A NULL or FALSE a, or an
                          unmatched probe (the NULL tuple of a left-outer PROBE_EACH included), marks nothing.  Like STRCODE b = 1 it runs
                          on every tuple it is evaluated on, whether WHERE keeps the tuple or not: a join's residual predicate goes into a.
                          PROBE on a multimap marks ONE of the key's entries; marking every duplicate takes PROBE_EACH.  Markers accumulate
                          over calls until ldb_gpu_join_table_clear_marks; ldb_gpu_join_table_marks reads them back: the build side of
                          reversed semi / anti / mark joins and the unmatched rest of right and full outer joins.  tables[arg] must be read
                          by an earlier PROBE / PROBE_EACH of the program, must not be its JOIN_BUILD sink, and must be a plain single-key,
                          direct-address or key-tuple join table (not a pair table, a group-join map or a dictionary): LDB_ERR_INVALID.
                          Not for captured queries (LDB_ERR_UNSUPPORTED). */
   LDB_OP_EXISTS = 29  /* dst = EXISTS(a, arg, b): does some match of key a in tables[arg] satisfy the residual block, the b instructions
                          that follow?  (the reference's anyTuple, RelAlgToSubOp.cpp:1296-1304, which lowers every semi / anti / mark /
                          outer join whose preserved side is the probe side: :1360, :1395, :1430, :1506, :1565.)  For each match in
                          probe-run order, dst holds the match's payload (a row id for side-column reads) and the block runs; the
                          residual is the register the block's last instruction writes.  The walk stops at the first match whose
                          residual is TRUE (NULL is not TRUE).  A key without a match runs the block once with dst NULL and its residual
                          ignored (so that a warp's lanes stay together; the block has no effects).  After the block dst is TRUE if some
                          match passed, else FALSE, never NULL, and the program continues once.  b = 0: no residual, TRUE when the key
                          has any match.  A NULL key, or one outside the key type, has no match (FALSE).  Semi join: WHERE dst; anti
                          join: WHERE NOT dst; mark join: dst as a value.  tables[arg] is what PROBE_EACH takes: a plain single-key
                          (unique or multimap), direct-address or key-tuple join table (keys a .. a+n-1); a pair table or group-join map
                          fails with LDB_ERR_UNSUPPORTED, a dictionary with LDB_ERR_INVALID.  A probe run longer than the interpreter's
                          bound of 16384 slots fails the call (LDB_ERR_CAPACITY); that is checked after the launch, so programs with
                          EXISTS are not part of captured queries (LDB_ERR_UNSUPPORTED).  LDB_ERR_INVALID: the block runs past n_instr;
                          it contains EXISTS (no nesting), PROBE_EACH, MARK or an inserting STRCODE (PROBE and side-column reads are
                          fine, but no MARK may mark a table probed inside it); it writes a register written before the EXISTS (the
                          block re-runs per match); an instruction, the filter or the sink after the block reads a register written
                          inside it, or a side column reads dst as its row after the block.  Several EXISTS per program may come before
                          or after a PROBE_EACH; after it, they run once per PROBE_EACH match.
                          A left outer join with a residual is composed from EXISTS and PROBE_EACH:
                            v = EXISTS(t, k, residual);  k' = SELECT(v, k, NULL) (NULL: x DIV 0);  m = PROBE_EACH(t, k', b = 1);
                            WHERE (residual' OR ISNULL(m)) AND user_where, residual' = the residual against the PROBE_EACH match m.
                          A probe row yields exactly its matches that pass the residual, or one NULL-extended tuple when none does. */
};
/* SUM wraps at 128 bits; MIN / MAX compare signed 128-bit values; the _F64 kinds work on doubles */
enum LdbAggKind { LDB_AGG_SUM = 1, LDB_AGG_SUM_F64 = 2, LDB_AGG_COUNT = 3, LDB_AGG_COUNT_STAR = 4, LDB_AGG_MIN = 5, LDB_AGG_MAX = 6,
                  LDB_AGG_MIN_F64 = 7, LDB_AGG_MAX_F64 = 8, LDB_AGG_ANY = 9 };
typedef struct LdbInstr {
   uint8_t op, dst, a, b;
   int32_t arg;
} LdbInstr;
#define LDB_PROG_MAX_KEYS 4
typedef struct LdbProgAgg {
   int32_t kind; /* LdbAggKind */
   int32_t reg;
} LdbProgAgg;
/* LDB_SINK_NONE: the program runs for its effects only (LDB_OP_MARK, LDB_OP_STRCODE inserts); `sink` must be NULL */
enum LdbProgramSink { LDB_SINK_HASHAGG = 1, LDB_SINK_JOIN_BUILD = 2, LDB_SINK_MATERIALIZE = 3, LDB_SINK_NONE = 4 };
typedef struct LdbProgramDesc {
   LdbTable* source;
   int32_t n_columns;            /* <= 12 */
   const char* const* columns;
   int32_t n_instr;              /* <= 96, registers 0..47 */
   const LdbInstr* instr;
   int32_t n_consts;             /* <= 24 */
   const LdbI128* consts;
   int32_t n_strings;            /* <= 12, each <= 32 bytes */
   const char* const* strings;
   int32_t n_tables;             /* <= 4 join tables (single int32 key, direct-address, or key-tuple of the same context) for
                                    LDB_OP_PROBE / LDB_OP_PROBE_EACH, or string dictionaries (same context) for LDB_OP_STRCODE; a
                                    dictionary is no PROBE table and a join table no STRCODE dictionary (LDB_ERR_INVALID).  A program
                                    may not probe the key-tuple table it builds (LDB_ERR_INVALID). */
   LdbState* const* tables;
   int32_t filter_reg;           /* the row is kept when this register is TRUE (NULL is not true); -1 = keep all */
   int32_t sink_kind;            /* LdbProgramSink */
   LdbState* sink;               /* HASHAGG state | JOIN_TABLE; NULL for MATERIALIZE and NONE */
   int32_t n_keys;
   int32_t key_regs[LDB_PROG_MAX_KEYS];
   int32_t n_aggs;
   LdbProgAgg aggs[LDB_MAX_AGGS];
   /* JOIN_BUILD: payload_reg -1 = 0.  Rows with a NULL key are not inserted; a NULL payload is stored as 0.  The call fails when a
    * row could not be stored: a non-NULL key or payload outside int32 (LDB_ERR_UNSUPPORTED), a table smaller than the build side
    * (LDB_ERR_CAPACITY), the reserved pair key -1 / payload -1 (LDB_ERR_UNSUPPORTED).
    * Into a key-tuple join table (LDB_STATE_KEY_JOIN) the keys are n_keys / key_regs[] (n_keys must equal the table's key count
    * and build_key_reg must be -1, else LDB_ERR_INVALID); a row with a NULL key component is not inserted; a non-NULL key or
    * payload outside int64 fails the call (LDB_ERR_UNSUPPORTED); ROWID payloads have no row limit. */
   int32_t build_key_reg, build_payload_reg;
   /* MATERIALIZE: out_regs → a new DEVICE table (columns "c0".."cN": decimal128(38,0) cells = the raw i128 / double bits in the
    * low 8 bytes, each with a validity byte); capacity = source rows, regrown to the produced row count (one more run of the
    * program) when a PROBE_EACH yields more tuples than that */
   int32_t n_out;
   int32_t out_regs[LDB_MAX_AGGS];
   LdbTable** out_table;
} LdbProgramDesc;
int ldb_gpu_run_program(LdbContext* ctx, const LdbProgramDesc* desc, LdbError* err);
/* Side columns: columns of OTHER tables ("side tables", same context, any number of batches), read at the row number a register
 * holds — typically a ROWID payload returned by PROBE / PROBE_EACH, so a join can read any number of build-side attributes,
 * decimals and strings included.  A NULL row register (or one outside the side table) reads NULL: outer-join semantics.
 * Side column k takes program column index desc->n_columns + k; source and side columns share the 12-column budget.  LOAD, STRCMP,
 * STRLIKE, STRKEY8 and STRCODE read them like source columns (validity bitmaps and bytes honoured); utf8 side columns are operands of the
 * string ops only.  The row register must be written before the first instruction that reads the column. */
typedef struct LdbSideColumn {
   int32_t table;      /* index into LdbProgramJoins.side_tables */
   const char* column;
   int32_t row_reg;    /* register holding the side table's row number */
} LdbSideColumn;
typedef struct LdbProgramJoins {
   int32_t n_side_tables;
   LdbTable* const* side_tables;
   int32_t n_side_columns;
   const LdbSideColumn* side_columns;
} LdbProgramJoins;
/* ldb_gpu_run_program with side columns (joins may be NULL).  A JOIN_BUILD program that uses ROWID is rejected when its source
 * has 2^31 rows or more and its sink is a plain join table (int32 payloads); a key-tuple join table takes int64 payloads. */
int ldb_gpu_run_program_ex(LdbContext* ctx, const LdbProgramDesc* desc, const LdbProgramJoins* joins, LdbError* err);
/* hash aggregation state sized for `expected_groups` (the directory holds 2x that; LDB_ERR_CAPACITY when it overflows) */
int ldb_gpu_hashagg_create(LdbContext* ctx, int32_t n_keys, int32_t n_aggs, const LdbProgAgg* aggs, int64_t expected_groups, LdbState** out, LdbError* err);
int ldb_gpu_hashagg_count(LdbState* s, int64_t* n_groups, LdbError* err);
typedef struct LdbHashAggRow {
   int64_t keys[LDB_PROG_MAX_KEYS];
   uint32_t key_null_mask, agg_valid_mask; /* bit k: key k IS NULL / bit a: aggregate a is not NULL */
   LdbI128 aggs[LDB_MAX_AGGS];             /* doubles: bits in .lo */
} LdbHashAggRow;
int ldb_gpu_hashagg_read(LdbState* s, LdbHashAggRow* rows, int64_t max_rows, int64_t* n_rows, LdbError* err);
/* the groups as a DEVICE table for the next pipeline (HAVING, joins, top-k): columns k0..k3 (int64, nullable) and a0..a7
 * (decimal128(38,0) raw i128 | float64, nullable) — the scan over the hash table that starts the reference's next pipeline */
int ldb_gpu_hashagg_to_table(LdbState* s, const char* name, LdbTable** out, LdbError* err);
/* ORDER BY <column> [DESC] LIMIT k over a DEVICE/staged table (GrowingBuffer::sort + Heap, GrowingBuffer.cpp:54-78): an LSD radix
 * sort of (order-preserving 64-bit key, row id) on the device; returns the first `limit` row ids (ties keep row order: stable).
 * column types: int32/date32/fsb4/int64/decimal of any precision, ordered by its full value (a 16-byte cell takes two sort passes:
 * low word, then high word).  A materialized column holding double bits (the materialize sink does not record register types)
 * orders by its bit pattern. */
int ldb_gpu_table_order_by(LdbTable* t, const char* column, int32_t descending, int64_t limit, int64_t* row_ids, int64_t* n_out, LdbError* err);
/* read back `n` cells of a fixed-width column at the given row ids (result materialisation of small outputs) */
int ldb_gpu_table_gather(LdbTable* t, const char* column, const int64_t* row_ids, int64_t n, void* host_dst /* n * cell bytes */, uint8_t* host_valid /* n, may be NULL */, LdbError* err);
/* ORDER BY k1 [DESC], k2 [DESC], … LIMIT over a single-batch table of fewer than 2^32 rows: an LSD composition of the stable radix
 * sort (the last key first), so ties on every key keep row order.  Fixed-width keys: the types ldb_gpu_table_order_by takes, in its
 * order (decimals of any precision by their full value; a 16-byte cell costs two sort passes, other fixed-width keys one).  utf8
 * keys order bytewise with unsigned bytes, a proper prefix first (the order of LDB_OP_STRCMP); a utf8 key costs one sort pass for
 * its lengths plus one per 8 bytes of its LONGEST string.  Validity is not consulted: a NULL sorts by the cell it holds.  Returns
 * the first `limit` row ids (all with limit < 0).  Unknown column: LDB_ERR_INVALID. */
int ldb_gpu_table_order_by_keys(LdbTable* t, int32_t n_keys, const char* const* columns, const int32_t* descending, int64_t limit, int64_t* row_ids, int64_t* n_out, LdbError* err);
/* read back `n` utf8 cells of a single-batch table at the given row ids: string i is host_bytes[host_offsets[i] ..
 * host_offsets[i + 1]), host_valid[i] (may be NULL) = 0 for NULL.  One copy per run of consecutive row ids.  When the strings need
 * more than bytes_cap bytes the call fails with LDB_ERR_CAPACITY, sets *bytes_needed and writes nothing else. */
int ldb_gpu_table_gather_strings(LdbTable* t, const char* column, const int64_t* row_ids, int64_t n, int64_t* host_offsets /* n + 1 */, void* host_bytes,
                                 int64_t bytes_cap, int64_t* bytes_needed, uint8_t* host_valid, LdbError* err);

/* String dictionary (LDB_STATE_DICT): a device hash set of byte strings that gives each distinct string a dense int32 code, for
 * LDB_OP_STRCODE — group, join and sort keys over strings of any length.  Codes are 0..n-1 and stable for the dictionary's lifetime
 * (later inserts never renumber); WHICH string gets which code depends on thread timing and is unspecified.  Sized for
 * `expected_strings` (a directory of nextPow2(2 x that) slots) and `expected_bytes` of string data.  When the directory or the byte
 * arena overflows, a probe run passes the interpreter's bound or a code would pass INT32_MAX, the program fails with
 * LDB_ERR_CAPACITY; the contents are then unspecified: recreate the dictionary larger.  No string is dropped silently.  Not for
 * captured queries, serialised steps or multi-GPU: codes belong to one context. */
int ldb_gpu_dict_create(LdbContext* ctx, int64_t expected_strings, int64_t expected_bytes, LdbState** out, LdbError* err);
int ldb_gpu_dict_count(LdbState* s, int64_t* n_strings, LdbError* err);
/* the dictionary as a single-batch DEVICE table, row i = code i: "str" (utf8) the string, "rank" (int32) its position in bytewise
 * order (ldb_gpu_table_order_by_keys' order): ("fetch", dict_table, code, "str") reads a string back, "rank" is an order-preserving
 * key for strings of any length and bytes.  The strings must fit 2^31 - 1 bytes. */
int ldb_gpu_dict_to_table(LdbState* s, const char* name, LdbTable** out, LdbError* err);

/* ------------------------------------------------------------------------------------ repartition (K6)
 * No reference counterpart (the reference is single-process; SURVEY §2 "Parallelism strategies").
 * Radix partition of a fixed-width tuple stream by the top bits of the reference hash h64(key)
 * into per-destination contiguous blocks, ready for an NCCL all-to-all. */
int ldb_gpu_partition_tuples(LdbContext* ctx, const int32_t* keys, const void* const* payload_cols, const int32_t* payload_widths, int32_t n_payload_cols, int64_t n_rows, int32_t n_parts,
                             int32_t* out_keys, void* const* out_payload_cols, int64_t* out_part_offsets /* n_parts+1, host */, LdbError* err);
/* insert already-materialised tuples (e.g. received from peers) into a JoinTable */
int ldb_gpu_join_table_insert(LdbContext* ctx, LdbState* table, const int32_t* keys, const int32_t* payloads, const int32_t* const* side_cols, int64_t n_rows, LdbError* err);

/* ------------------------------------------------------------------------------------ multi-GPU: peer-mapped exchange
 * No reference counterpart (the reference is single-process; SURVEY §2 "Parallelism strategies", §8(e)).  One process per
 * GPU; every rank owns a symmetric heap its peers map through CUDA IPC, and a transfer is a kernel that stores into the
 * peer's HBM over NVLink 5 / NVSwitch and publishes a flag — no NCCL call and no host round trip on the data path
 * (csrc/peer.cu).  Bootstrap: each rank creates its comm, the 64-byte handles are exchanged by the caller (any transport:
 * torch.distributed, MPI, a file) and passed to ldb_gpu_comm_connect in rank order.  Collectives are enqueued on the
 * context's compute stream and must be called by every rank in the same order. */
typedef struct LdbComm LdbComm;
#define LDB_IPC_HANDLE_BYTES 64
int ldb_gpu_comm_create(LdbContext* ctx, int32_t rank, int32_t world, int64_t user_heap_bytes, LdbComm** out, uint8_t* handle_out /* 64 */, LdbError* err);
int ldb_gpu_comm_connect(LdbComm* comm, const uint8_t* all_handles /* world x 64, rank order */, LdbError* err);
/* one process driving several devices (tests): comms[i] is rank i of a world of n */
int ldb_gpu_comm_connect_local(LdbComm** comms, int32_t n, LdbError* err);
void ldb_gpu_comm_destroy(LdbComm* comm);
int32_t ldb_gpu_comm_rank(LdbComm* comm);
int32_t ldb_gpu_comm_world(LdbComm* comm);
int64_t ldb_gpu_comm_reserved_bytes(void); /* control + mailbox bytes in front of the user region */
int64_t ldb_gpu_comm_slot_bytes(void);     /* largest block of ldb_gpu_comm_allgather_small */
/* the user region of this rank's heap (device pointer); the same offset addresses the same region on every peer */
void* ldb_gpu_comm_heap(LdbComm* comm, int64_t* user_bytes);
/* device-side barrier: orders everything this rank stored into peer heaps before it against the peers' later reads */
int ldb_gpu_comm_barrier(LdbComm* comm, LdbError* err);
/* all-gather of one small DEVICE block (multiple of 16 bytes, <= slot bytes); *result = device address of the gathered
 * blocks (rank r at r * slot_bytes), valid until the next-but-one gather */
int ldb_gpu_comm_allgather_small(LdbComm* comm, const void* dev_src, int64_t bytes, void** result, LdbError* err);
/* K7 over NVLink (rt::PreAggregationHashtable::merge across GPUs): every rank pushes its group-table image to every peer
 * and folds the peers' images into its own table — ONE kernel instead of export + all-gather + merge.  Afterwards every
 * rank holds the full result.  SIMPLE and GROUPBY states (capacity <= 1024). */
int ldb_gpu_groupby_allmerge(LdbState* s, LdbComm* comm, LdbError* err);
/* zero / read back (synchronising) a range of this rank's user heap */
int ldb_gpu_comm_heap_zero(LdbComm* comm, int64_t user_offset, int64_t bytes, LdbError* err);
int ldb_gpu_comm_heap_read(LdbComm* comm, int64_t user_offset, int64_t bytes, void* host_dst, LdbError* err);
/* ---- receive side of LDB_PIPE_SCAN_PARTITION_SEND (all offsets are user-heap offsets, identical on every rank)
 * publish: copy this rank's cursors[d] into rank d's counts[rank] (heap[counts_offset + rank * 8]); follow with a barrier */
int ldb_gpu_comm_publish_counts(LdbComm* comm, int64_t cursors_offset, int64_t counts_offset, LdbError* err);
/* insert the {key:32 | payload:32} tuples received from every source (counts read on the device) into a join table */
int ldb_gpu_join_table_insert_received(LdbState* table, LdbComm* comm, int64_t recv_offset, int64_t capacity, int64_t counts_offset, LdbError* err);
/* received {keyA:32 | keyB:32, a, b} tuples → probe A, probe B, payloads equal → group by payload → SUM(a * (1 - b)) (decimal scale `scale`) */
int ldb_gpu_probe_received_groupby(LdbState* table_a, LdbState* table_b, LdbState* groups, LdbComm* comm, int64_t recv_offset, int64_t capacity, int64_t counts_offset, int32_t scale, LdbError* err);
/* received {key:32 | g0:32, lo, hi} tuples (K11) → probe `table` on key (payload = g1) → group by (g0, g1) → SUM of the shipped i128 */
int ldb_gpu_probe_received_groupby2(LdbState* table, LdbState* groups, LdbComm* comm, int64_t recv_offset, int64_t capacity, int64_t counts_offset, LdbError* err);
/* a join table whose Bloom filter lives in the symmetric heap at bloom_offset (so the ranks can OR their partitions' filters
 * together with ldb_gpu_comm_or_reduce); *bloom_bytes = size of the filter (call with out == NULL to query it for expected_rows) */
int ldb_gpu_join_table_create_shared_bloom(LdbContext* ctx, int64_t expected_rows, int32_t unique_keys, LdbComm* comm, int64_t bloom_offset, int64_t* bloom_bytes, LdbState** out, LdbError* err);
/* OR-all-reduce of heap[user_offset, +bytes) across the ranks (Bloom filters of hash partitions); barrier before and after */
int ldb_gpu_comm_or_reduce(LdbComm* comm, int64_t user_offset, int64_t bytes, LdbError* err);
/* synchronises and reports a collective that timed out on a dead peer (LDB_PEER_TIMEOUT_MS, default 20000) */
int ldb_gpu_comm_check(LdbComm* comm, LdbError* err);

/* ------------------------------------------------------------------------------------ value-level hooks
 * Device twins of util.hash_64 / hash_combine (LowerToLLVM.cpp:493-514), exported for the KAT tests:
 * hashes `n` int64 values (optionally combined with a second column) on the GPU. */
int ldb_gpu_hash_i64(LdbContext* ctx, const int64_t* host_values, const int64_t* host_values2, int64_t n, uint64_t* host_out, LdbError* err);

/* ------------------------------------------------------------------------------------ device datagen
 * Device twin of ldb_datagen.h (same tpch_gen.h); fills DEVICE buffers. */
struct LdbGenScale;
struct LdbGenLineitemCols;
struct LdbGenOrdersCols;
struct LdbGenCustomerCols;
struct LdbGenSupplierCols;
struct LdbGenPartCols;
struct LdbGenPartsuppCols;
int ldb_gpu_datagen_lineitem(LdbContext* ctx, const struct LdbGenScale* g, int64_t row_begin, int64_t n_rows, const struct LdbGenLineitemCols* dev_cols, LdbError* err);
int ldb_gpu_datagen_orders(LdbContext* ctx, const struct LdbGenScale* g, int64_t row_begin, int64_t n_rows, const struct LdbGenOrdersCols* dev_cols, LdbError* err);
int ldb_gpu_datagen_customer_fixed(LdbContext* ctx, const struct LdbGenScale* g, int64_t row_begin, int64_t n_rows, const struct LdbGenCustomerCols* dev_cols, int32_t* dev_seg_lengths, LdbError* err);
int ldb_gpu_datagen_customer_bytes(LdbContext* ctx, const struct LdbGenScale* g, int64_t row_begin, int64_t n_rows, const int32_t* dev_offsets, uint8_t* dev_data, LdbError* err);
int ldb_gpu_datagen_supplier(LdbContext* ctx, const struct LdbGenScale* g, int64_t row_begin, int64_t n_rows, const struct LdbGenSupplierCols* dev_cols, LdbError* err);
int ldb_gpu_datagen_part_fixed(LdbContext* ctx, const struct LdbGenScale* g, int64_t row_begin, int64_t n_rows, const struct LdbGenPartCols* dev_cols, int32_t* dev_name_lengths, LdbError* err);
int ldb_gpu_datagen_part_bytes(LdbContext* ctx, const struct LdbGenScale* g, int64_t row_begin, int64_t n_rows, const int32_t* dev_offsets, uint8_t* dev_data, LdbError* err);
int ldb_gpu_datagen_partsupp(LdbContext* ctx, const struct LdbGenScale* g, int64_t row_begin, int64_t n_rows, const struct LdbGenPartsuppCols* dev_cols, LdbError* err);
/* dbgen-faithful variant (ldb_datagen.h, csrc/dbgen_gen.h): lineitem is generated per ORDER at dev_first_row[order] (prefix sum of
 * the line counts); `table` of the two small-table entry points: 0 customer, 1 supplier, 2 part, 3 partsupp (bytes: 0 or 2). */
int ldb_gpu_dbgen_line_counts(LdbContext* ctx, const struct LdbGenScale* g, int64_t order_begin, int64_t n_orders, int32_t* dev_counts, LdbError* err);
int ldb_gpu_dbgen_lineitem(LdbContext* ctx, const struct LdbGenScale* g, int64_t order_begin, int64_t n_orders, const int64_t* dev_first_row, const struct LdbGenLineitemCols* dev_cols, LdbError* err);
int ldb_gpu_dbgen_orders(LdbContext* ctx, const struct LdbGenScale* g, int64_t row_begin, int64_t n_rows, const struct LdbGenOrdersCols* dev_cols, LdbError* err);
int ldb_gpu_dbgen_small_fixed(LdbContext* ctx, const struct LdbGenScale* g, int32_t table, int64_t row_begin, int64_t n_rows, int32_t* dev_key, int32_t* dev_second, uint8_t* dev_decimal, int32_t* dev_lengths, LdbError* err);
int ldb_gpu_dbgen_bytes(LdbContext* ctx, const struct LdbGenScale* g, int32_t table, int64_t row_begin, int64_t n_rows, const int32_t* dev_offsets, uint8_t* dev_data, LdbError* err);

#ifdef __cplusplus
}
#endif
#endif
