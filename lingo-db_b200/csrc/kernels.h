// kernels.h — host-visible parameter blocks and launchers of the sm_90a pipeline kernels (kernels.cu).
// Internal to libldb_gpu.so; the public surface is include/ldb_gpu.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ldb {

constexpr int kMaxFilterCols = 4;
constexpr int kMaxValueCols = 4;
constexpr int kMaxAggs = 8;
constexpr int kMaxKeys = 2;
constexpr int kMaxSide = 2;

enum ColKind : int32_t { COL_I32 = 0, COL_DEC128_LO64 = 1, COL_UTF8_EQ = 2, COL_UTF8_CONTAINS = 3 };

// One pushed-down filter column with up to two predicates (e.g. a range); op masks as in cmpMask().
// utf8 columns evaluate `string == constant` to 1/0 first, then compare that to valA (1).
struct FilterCol {
   const void* base;     // utf8 only: offsets (fixed-width columns are read through the staged tile)
   const uint8_t* bytes; // utf8 data
   int32_t kind;
   int32_t staged;       // index into StagedCols (fixed-width columns), -1 for utf8
   uint32_t maskA, maskB;
   int64_t valA, valB;
   uint8_t str[24];
   int32_t strLen;
   int32_t nIn;        // > 0: IN list (the A/B predicates are unused)
   int64_t inVals[8];
};
struct FilterSet {
   int32_t n;
   FilterCol c[kMaxFilterCols];
};

// ---- small-domain group table (rt::PreAggregationHashtable / SimpleState twin), lives in HBM
struct GroupTableDev {
   int32_t capacity; // power of two (1 for a keyless SimpleState)
   int32_t nKeys, nAggs;
   int32_t* state;           // 0 empty, 1 being written, 2 ready
   int32_t* keys;            // [capacity][kMaxKeys]
   unsigned long long* acc;  // [capacity][kMaxAggs][2] = {lo, hi}
   int32_t* error;           // set to 1 on overflow
};

// The table is ONE allocation laid out as the image ranks exchange: state[cap] | keys[cap][kMaxKeys] | acc[cap][kMaxAggs][2],
// followed by the error word — so an export is a single copy and a peer can be handed the table itself.
__host__ __device__ inline size_t groupImageBytes(int64_t capacity) { return (size_t) capacity * 4 + (size_t) capacity * kMaxKeys * 4 + (size_t) capacity * kMaxAggs * 2 * 8; }

// ---- join table (rt::GrowingBuffer + rt::HashIndexedView twin; with agg lanes: the group-join map)
// Open addressing, slot s at base + s * stride.  Two layouts:
//   stride  8  {key:32, payload:32}                                              plain joins
//   stride 16  {key0:32, key1:32, payload:64}                                     composite (int32,int32) key → int64 payload
//              (Q9's partsupp: (ps_partkey, ps_suppkey) → ps_supplycost); hashed like db.hash over the key pair
//   stride  4  DIRECT-ADDRESS table for dense integer keys (surrogate primary keys: o_orderkey, s_suppkey): slot = key - keyMin,
//              the slot holds the int32 payload (kDirectEmpty = no such key).  No hashing, no CAS retry, no key compare; a
//              build in key order writes sequentially.  Chosen by the plan when (max - min + 1) <= 8 x rows (tpch_plans.cpp).
//   stride 32  {key:32, marker:1|payload:31, side0:32, side1:32, aggLo:64, aggHi:64}  group-join map — ONE 32-byte
//              sector per entry, so an insert (CAS + side lanes) or a probe hit (compare + i128 atomic add + marker)
//              touches a single DRAM sector instead of up to four separate arrays.
// The first 8 bytes all-ones = empty.
struct JoinTableDev {
   uint8_t* base;
   uint32_t stride;
   uint64_t mask;             // capacity - 1
   uint32_t* bloom;           // blocked Bloom filter over the build keys (32-bit blocks, 3 bits/key), sized to stay in L2
   uint32_t bloomMask;        // words - 1
   unsigned long long* count; // inserted entries
   int32_t* error;            // 1 = table full, 2 = duplicate key in a unique table, 3 = unstorable pair, 4 = negative payload in a wide table,
                              // 5 = key outside the declared range of a direct-address table, 6 = a program's PROBE_EACH met a
                              // probe run longer than its bound
   int32_t unique;
   int32_t direct;            // stride 4: direct-address table
   int32_t keyMin;
   uint32_t range;            // number of slots of a direct-address table
};
constexpr int32_t kDirectEmpty = (int32_t) 0x80808080; // byte-fill pattern, so a cudaMemset initialises the table

// The distinct fixed-width columns a pipeline touches.  Every scan kernel streams them tile by tile
// (kTileRows rows) into shared memory with TMA bulk copies (cp.async.bulk + mbarrier, 2 stages), so
// each column byte crosses HBM→SM exactly once and no per-row global address arithmetic is issued.
constexpr int kMaxStagedCols = 8;
constexpr int kBlockThreads = 256;
constexpr int kRowsPerThreadScan = 2;  // K1/K2: arithmetic-heavy, fewer/larger tiles
constexpr int kRowsPerThreadProbe = 2; // K4/K5/K8 (1 row/thread with 2x the CTAs measured slower there on Q3)
constexpr int kRowsPerThreadStar = 1;  // K3/K9 (survivor-queue kernels): small tiles → >= 4 CTAs/SM; they are latency-bound between tiles, not arithmetic-bound
constexpr int kStages = 2;    // default depth of the tile pipeline
constexpr int kMaxStages = 4; // the probe / build kernels are tile-LATENCY bound with 2 (one copy in flight per CTA): they take 3-4
// Tuning knobs read once from the environment (experiments; the defaults are the measured best)
struct Tuning {
   int stagesBuild, stagesProbeAgg, stagesProbe2, stagesStar; // TMA pipeline depth of K3 / K5 / K4 / K9
   int rptBuild;                                              // rows per thread of a K3 tile (1, 2 or 4)
   int rptStar;                                               // rows per thread of a K9 tile (1, 2 or 4)
   int producerSleepNs, consumerSleepNs;                      // pause between mbarrier polls in the warp-specialised tile driver (0 = poll)
   int specialise;                                            // 1: join pipelines run the filter-shape instantiations (kernels.cu FilterShape), 0: descriptor-driven only
   int encodedScan;                                           // 1: K1/K2 scan DEVICE batches from their frame-of-reference copy (LdbBatch::enc), 0: Arrow layout only
};
const Tuning& tuning();
void setTuning(const Tuning& t);

// ---- frame-of-reference encoded column copy (encode.cu), read by K1/K2 in place of the Arrow cells of a DEVICE batch.
// Per column one width W in {1, 2, 4, 8} bytes; per block of kEncodeBlockRows rows a base (the block minimum, int64); a value is
// stored as (v - base) in W bytes, zero-extended on decode (exact modulo 2^64, so int32 columns and the low 8 bytes of a
// decimal(p<19) cell come back bit for bit).  The copy is TILE-FRAMED for the K1/K2 tile of kEncodeTileRows rows: tile t of a
// column starts at t * (kEncodeTileHeader + kEncodeTileRows * W) with a 16-byte header {base of the tile's block, max - min of that
// block} followed by the tile's packed values.  One bulk copy then brings a tile's base with its values, and no thread loads a base from HBM.
constexpr int64_t kEncodeBlockRows = 65536; // = kPackBlockRows of the compressed staging format: a tile never straddles two blocks
// Invariant of the format: the headers of the kEncodeBlockRows / tileRows (= 128) tiles of one block are equal.  A run of F tiles
// starting at a multiple of F, F dividing 128, thus lies in one block and shares one header — the encoded Q1 scan reads F tiles of a
// column with one bulk copy and one header (kernels.cu kEncFrames).
constexpr int kEncodeTileHeader = 16;
constexpr int kDecEncoded = 0; // StagedCols::decBytes / kernel DB parameter of the encoded layout
inline int64_t encodedColumnBytes(int64_t nRows, int width, int tileRows) {
   const int64_t tiles = (nRows + tileRows - 1) / tileRows;
   return ((tiles * kEncodeTileHeader + nRows * width) + 15) / 16 * 16;
}

struct StagedCols {
   int32_t n;
   int32_t tileRows;   // rows per tile = kBlockThreads * rows-per-thread of the kernel
   int32_t stageBytes; // bytes of one stage = sum(elemBytes * tileRows + tileHeader)
   int32_t useTma;     // 0 when a column base is not 16-byte aligned: tiles are then read with plain loads
   int32_t decBytes;   // bytes per decimal128 cell as staged: 16 (Arrow layout), 8 (HOST batch narrowed) or kDecEncoded; selects the kernel instantiation
   int32_t tileHeader; // bytes in front of every column tile: kEncodeTileHeader in the encoded layout, else 0
   int32_t producerSleepNs, consumerSleepNs; // pause between mbarrier polls of the producer lane / the consumer warps (0 = plain polling)
   const uint8_t* base[kMaxStagedCols];
   int32_t elemBytes[kMaxStagedCols];  // 4 (int32/date32/fsb4) or 16 (decimal128); the width W in the encoded layout
   int32_t smemOffset[kMaxStagedCols]; // offset of the column inside a stage
   int32_t encShift[kMaxStagedCols];   // encoded layout: log2(W)
   uint32_t encMask[kMaxStagedCols];   // encoded layout: mask of the low W bytes of a 32-bit word (W <= 4)
};
// LATE-MATERIALISED value columns: a selective probe pipeline (Bloom filter in front, a few percent of the rows survive) streams
// only its key / filter columns through the TMA tiles; the operands of the aggregate are fetched from HBM by the SURVIVORS
// (one 32-byte sector per cell) — Q9's lineitem pipeline then moves 16 B/row + 5 % x 3 sectors instead of 60 B/row.  When every
// row survives the per-warp loads are contiguous, so the traffic is never worse than streaming (only un-prefetched).
constexpr int kMaxLazyCols = 4;
struct LazyCols {
   int32_t n;
   int32_t elemBytes[kMaxLazyCols]; // 16, or 8 when the HOST batch was narrowed
   const uint8_t* base[kMaxLazyCols];
};
struct ScanSource {
   int64_t nRows;
   StagedCols cols;
   FilterSet filters;
};

// aggregate = SUM(expr over value columns); expr kinds mirror LdbExprKind
struct AggSpec {
   int32_t expr;
   int32_t col[3]; // indices into value columns
};
struct GroupByParams {
   ScanSource src;
   int32_t nKeys;
   int32_t keyStage[kMaxKeys];        // staged-column indices
   int32_t nValueCols;
   int32_t valueStage[kMaxValueCols]; // decimal128 (16 B / value)
   int32_t nAggs;
   AggSpec aggs[kMaxAggs];
   GroupTableDev table;
   // encoded layout: the batch's minimum and max - min of value column v (LdbBatch::Encoded), which bound every stage header's
   // block; the factored Q1 scan indexes its per-cell sums by them
   int64_t encMin[kMaxValueCols];
   uint64_t encRange[kMaxValueCols];
   // the factored Q1 scan's cell words, chosen by the launcher from encRange (kernels.cu factoredFold): ep - min_ep splits into its low
   // facShift bits and the rest, and the words are folded into 64-bit sums every facFoldFrames frames, before any of them can overflow
   uint32_t facShift;
   uint32_t facFoldFrames;
};

enum PayloadKind : int32_t { PAYLOAD_I32 = 0, PAYLOAD_YEAR_OF_DATE32 = 1, PAYLOAD_DEC_LO64 = 2 };
struct BuildParams {
   ScanSource src;
   int32_t keyStage;
   int32_t keyStage2;    // pair tables: second key column, else -1
   int32_t payloadStage; // -1: none
   int32_t payloadKind;  // PayloadKind
   int32_t nSide;
   int32_t sideStage[kMaxSide];
   int32_t hasProbe;
   JoinTableDev probe;
   int32_t probeKeyStage;
   JoinTableDev sink;
};

struct ProbeAggParams {
   ScanSource src;
   int32_t probeKeyStage;
   JoinTableDev table;
   AggSpec agg;
   LazyCols values; // operands of the aggregate, in expression order
};

struct Probe2GroupByParams {
   ScanSource src;
   int32_t keyStageA, keyStageB;
   JoinTableDev tableA, tableB;
   AggSpec agg;
   LazyCols values;
   GroupTableDev groups; // keyed by the matched payload
};

// K9: scan → probe P (composite key → int64 payload c) → probe S (→ group key 0) → probe O (→ group key 1)
//     → SUM(a * (1 - b) - c * d) grouped by the two payloads (Q9's lineitem pipeline)
struct StarProbeParams {
   ScanSource src;
   int32_t keyStageP0, keyStageP1, keyStageS, keyStageO;
   JoinTableDev tableP, tableS, tableO;
   LazyCols values;       // a, b, d
   GroupTableDev groups;  // 2 keys, 1 aggregate
};

constexpr int kMaxOutCols = 4;
struct MaterializeParams {
   ScanSource src;
   int32_t hasProbe, bloomOnly;
   JoinTableDev probe;
   int32_t probeKeyStage;
   int32_t nOut;
   int32_t outStage[kMaxOutCols]; // staged column, or -1 = probe payload
   int32_t outElem[kMaxOutCols];  // 4 or 16
   void* out[kMaxOutCols];
   int64_t capacity;
   unsigned long long* count;
};

struct TopKRowDev {
   int32_t key, side0, side1, valid;
   unsigned long long aggLo;
   long long aggHi;
};

// ---- fused repartition (multi-GPU joins): scan → filters → [probe | Bloom semi-join] → radix partition by h64(key) → tuples
// stored STRAIGHT into the destination rank's receive buffer over NVLink (peer-mapped heap, csrc/peer.cu) — no staging copy,
// no collective call.  A tuple is 1..3 eight-byte words: {key:32 | second:32}, then up to two decimal(p<19) values (lo64).
// Every (source, destination) pair owns a sub-region of `capacity` tuples in the destination's buffer, so the only atomics
// are the source's local per-destination cursors (one per destination per tile).
constexpr int kMaxRanks = 8;
struct SendParams {
   ScanSource src;
   int32_t keyStage;
   int32_t secondStage; // staged int32 column, or -1: the probe's payload
   int32_t secondYear;  // ship extract(year from <date32 second column>) instead of the column's value (DateRuntime::extractYear)
   int32_t nDec;
   LazyCols dec; // the shipped decimal columns (fetched for the rows that are sent)
   int32_t hasProbe, bloomOnly;
   JoinTableDev probe;
   int32_t probeKeyStage;
   int32_t world;
   uint8_t* dest[kMaxRanks]; // destination d's receive region, already offset to THIS source's sub-region
   int64_t capacity;         // tuples per sub-region
   unsigned long long* cursors; // [world], device-local, zeroed by the caller
   int32_t* error;              // 6 = a sub-region overflowed
};
void launchScanPartitionSend(const SendParams& p, int smCount, cudaStream_t s);
// K11 star probe + send: scan → composite-key probe P (Bloom first) → foreign-key probe S → the row's contribution
// a * (1 - b) - c * d (c = P's payload) is shipped as {partition key : 32 | S payload : 32, lo, hi} to the rank that owns the
// partition key — the lineitem side of a Q9-shaped join whose third build side (orders) is hash-partitioned across the ranks
struct StarSendParams {
   ScanSource src;
   int32_t keyStageP0, keyStageP1, keyStageS, keyStageO;
   JoinTableDev tableP, tableS;
   LazyCols values; // a, b, d
   int32_t world;
   uint8_t* dest[kMaxRanks];
   int64_t capacity;
   unsigned long long* cursors;
   int32_t* error;
};
void launchScanStarProbeSend(const StarSendParams& p, int smCount, cudaStream_t s);
// received {key | g0, lo, hi} tuples → probe `table` on key (payload = g1) → group by (g0, g1) → SUM of the shipped i128 value
void launchProbeReceivedGroupBy2(const JoinTableDev& table, const GroupTableDev& groups, const uint8_t* recv, int world, int64_t capacity, const unsigned long long* counts, int smCount, cudaStream_t s);
// received tuples of `world` sources (counts[src] tuples each, read from DEVICE memory) → join-table inserts
void launchInsertReceived(const JoinTableDev& t, const uint8_t* recv, int world, int64_t capacity, const unsigned long long* counts, int smCount, cudaStream_t s);
// received {key|keyB, a, b} tuples → probe A on key, probe B on keyB, payloads equal → group by payload → SUM(a * (one - b))
void launchProbeReceivedGroupBy(const JoinTableDev& tableA, const JoinTableDev& tableB, const GroupTableDev& groups, const uint8_t* recv, int world, int64_t capacity,
                                const unsigned long long* counts, int64_t one, int smCount, cudaStream_t s);

// signature → instantiation registry for the group-by kernel; returns false when no compiled shape matches
bool launchScanGroupBy(const GroupByParams& p, int smCount, cudaStream_t s, const char** why);
// true when launchScanGroupBy runs p (bound to the encoded layout) on the factored Q1 instance (kernels.cu factoredFits)
bool scanGroupByFactored(const GroupByParams& p);
// true when launchScanGroupBy has an instantiation of p's signature for the encoded layout (p.src.cols need not be bound yet)
bool scanGroupByEncodable(const GroupByParams& p);
// encoder (encode.cu).  A source column is `n` int32 cells (isI32) or decimal128 cells of which the low 8 bytes are taken.
// Range pass: blockMin[b] = minimum of block b, blockRange[b] = its max - min; stats[kEncodeStats] (caller zeroes them) = {max over
// blocks of (max - min) as unsigned, ~(min ^ 2^63), max ^ 2^63} of the column.
constexpr int kEncodeStats = 3;
void launchEncodeRange(const uint8_t* src, bool isI32, int64_t n, int64_t* blockMin, int64_t* blockRange, unsigned long long* stats, cudaStream_t s);
// Pack pass: writes the tile-framed copy (kernels.h, kEncodeTileHeader) of width `width` for tiles of `tileRows` rows
void launchEncodePack(const uint8_t* src, bool isI32, int64_t n, const int64_t* blockMin, const int64_t* blockRange, int width, int tileRows, uint8_t* dst,
                      cudaStream_t s);
void launchScanBuild(const BuildParams& p, int smCount, cudaStream_t s);
bool launchScanProbeAgg(const ProbeAggParams& p, int smCount, cudaStream_t s, const char** why);
bool launchScanProbe2GroupBy(const Probe2GroupByParams& p, int smCount, cudaStream_t s, const char** why);
bool launchScanStarProbeGroupBy(const StarProbeParams& p, int smCount, cudaStream_t s, const char** why);
void launchScanMaterialize(const MaterializeParams& p, int smCount, cudaStream_t s);
void launchInitWideTable(uint8_t* base, uint64_t capacity, int smCount, cudaStream_t s);
void launchJoinTopK(const JoinTableDev& t, int k, bool agg64, TopKRowDev* out, int* outBlocks, int smCount, cudaStream_t s);
void launchFill64(unsigned long long* p, unsigned long long v, int64_t n, int smCount, cudaStream_t s);
void launchInsertTuples(const JoinTableDev& t, const int32_t* keys, const int32_t* payloads, const int32_t* side0, const int32_t* side1, int64_t n, int smCount, cudaStream_t s);
void launchColumnRange(const int32_t* col, int64_t n, int32_t* minMax /* device: {min, max} */, int smCount, cudaStream_t s);
void launchHashI64(const int64_t* a, const int64_t* b, int64_t n, uint64_t* out, cudaStream_t s);
void launchGroupMergeRows(const GroupTableDev& t, const int32_t* keys, const unsigned long long* acc, int32_t nRows, cudaStream_t s);
void launchGroupMergeImages(const GroupTableDev& t, const uint8_t* images, int nTables, int skip, cudaStream_t s);
// radix partition (K6): histogram + scatter by the top bits of h64(key)
void launchPartitionHistogram(const int32_t* keys, int64_t n, int nParts, unsigned long long* counts, int smCount, cudaStream_t s);
void launchPartitionScatter(const int32_t* keys, const void* const* payloadCols, const int32_t* widths, int nPayload, int64_t n, int nParts, unsigned long long* cursors, int32_t* outKeys, void* const* outPayload, int smCount, cudaStream_t s);

} // namespace ldb
