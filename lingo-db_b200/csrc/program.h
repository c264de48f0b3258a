// program.h — device-side structures of the GENERIC pipeline (program.cu): scan → register program → sink.
//
// The hand-specialised kernels of kernels.cu cover the TPC-H hot shapes at HBM speed; everything else the sub-operator
// dialect can put into a scan pipeline — arbitrary expressions (db.add/sub/mul/div/cmp/and/or/not/between/case,
// LowerToStd.cpp:612-700,851-910), nullable inputs (validity bits, Restrictions.cpp:67-162), i8…i64/float/decimal(38)/string
// operands, SUM/COUNT/MIN/MAX/ANY with SQL null semantics (RelAlgToSubOp.cpp:1809-2025), group-by over millions of groups
// (PreAggregationHashtable.cpp:76-170), semi/anti/mark probes (RelAlgToSubOp.cpp:1129-1206,1340-1588) — runs through ONE
// kernel that interprets a small register program per row.  It is the GPU stand-in for "whatever the JIT would have emitted".
#pragma once
#include "kernels.h"

namespace ldb {

constexpr int kProgMaxInstr = 96;
constexpr int kProgMaxRegs = 48;
constexpr int kProgMaxCols = 12;
constexpr int kProgMaxConsts = 24;
constexpr int kProgMaxStrings = 12;
constexpr int kProgStringBytes = 32;
constexpr int kProgMaxTables = 4;
constexpr int kProgMaxKeys = 4;
constexpr int kProgMaxAggs = 8;
// the identity of MIN_F64 / MAX_F64 cells: the canonical quiet NaN, which every other value replaces (program.cu, f64Better)
constexpr uint64_t kF64MinMaxIdentity = 0x7ff8000000000000ull;

// one batch of a side table (the device-resident batch directory of a side column over a multi-batch table)
struct ProgSideBatch {
   const uint8_t* data;
   const uint8_t* bytes;
   const uint8_t* validity;
   const uint8_t* validBytes;
   int64_t bitOffset;
   int64_t firstRow; // global row number of the batch's row 0
   int32_t elemBytes;
   int32_t pad;
};
struct ProgCol {
   const uint8_t* data;     // values, or utf8 offsets (int32)
   const uint8_t* bytes;    // utf8 data
   const uint8_t* validity; // Arrow validity bitmap (LSB first) or null = no nulls
   const uint8_t* validBytes; // one validity BYTE per row (columns produced by this library: exported groups, materialised rows)
   int64_t bitOffset;       // bit index of row 0 inside `validity`
   int32_t type;            // LdbPhysType
   int32_t elemBytes;       // as staged (decimal128: 16, or 8 when the HOST batch was narrowed)
   // side column: read at the row register rowReg holds instead of the scanned row (-1 = a column of the scanned table).  A
   // single-batch side table uses the fields above; a multi-batch one the directory `dir` of nBatches batches, sorted by firstRow.
   int32_t rowReg;
   int32_t nBatches;
   int64_t sideRows;        // rows of the side table: a NULL row register or one outside 0..sideRows-1 reads NULL
   const ProgSideBatch* dir;
};
struct ProgInstr {
   uint8_t op, dst, a, b;
   int32_t arg;
};
struct ProgAgg {
   int32_t kind; // LdbAggKind
   int32_t reg;
};
// large-domain hash aggregation table (rt::PreAggregationHashtable after merge / rt::Hashtable): open addressing in HBM
//   entry = { state:u32 (0 empty, 1 being written, 2 ready), flags:u32 (bit a: aggregate a has seen a non-null input; bit 8+a: claimed
//             by an ANY; bit 16+k: key k is NULL), pad:u64, keys[4]:i64, aggs[nAggs] x {lo:u64, hi:u64} } = 48 + 16 nAggs bytes
struct HashAggDev {
   uint8_t* base;
   uint64_t mask; // capacity - 1
   uint32_t entryBytes;
   int32_t nKeys, nAggs;
   unsigned long long* count; // groups
   int32_t* error;            // 1 = table full
};
// string dictionary (LDB_STATE_DICT): a concurrent hash set of byte strings → dense int32 codes 0..n-1, in HBM
//   slots[mask + 1]  u64 = {tag:32 (high 32 bits of the string's hash) | state:32}; state 0 empty (the whole word is 0),
//                    kDictWriting while its claimer copies the string, kDictFailed when the claimer gave up, else code + 1
//   entryOff/Len     per code: the string's arena offset and length
//   arena            the strings' bytes, appended in claim order
//   ctr              [0] arena cursor, [1] next code, [2] low 32 bits: error word (1 directory full or probe bound, 2 arena
//                    full, 3 code past INT32_MAX)
struct DictDev {
   unsigned long long* slots;
   uint64_t mask;
   int64_t* entryOff;
   int32_t* entryLen;
   uint8_t* arena;
   unsigned long long* ctr;
   int64_t arenaCap;
   int64_t codeCap; // codes 0..codeCap-1 fit the entry arrays and int32
};
constexpr uint32_t kDictWriting = 0xffffffffu, kDictFailed = 0xfffffffeu;
constexpr int64_t kDictMaxStrings = (int64_t) 1 << 30; // the most strings a dictionary is made for (its codes are int32)
// key-tuple join table (LDB_STATE_KEY_JOIN): 1..4 int64 keys → int64 payload, open addressing in HBM, cap = nextPow2(2 x expected)
//   entry = { word:u64 = tag:32 (high 32 bits of the tuple's hash) | state:32 (0 empty: the whole word is 0, kKeyJoinWriting,
//             kKeyJoinReady), payload:i64, keys[nKeys]:i64 } padded to entryBytes = 32 (1-2 keys: one DRAM sector) or 48 (3-4 keys)
//   error    1 directory full, 6 a probe run reached the interpreter's bound, 7 a build key or payload outside int64
// nKeys == 0 marks an unused descriptor (the table is a plain join table or a dictionary).
struct KeyJoinDev {
   uint8_t* base;
   uint64_t mask;             // capacity - 1
   uint32_t* bloom;           // blocked Bloom filter over the key tuples (as JoinTableDev), or null
   uint32_t bloomMask;
   int32_t nKeys;
   uint32_t entryBytes;
   int32_t unique;            // set semantics: a duplicate tuple is dropped
   unsigned long long* count; // inserted entries
   int32_t* error;
};
constexpr uint32_t kKeyJoinWriting = 1u, kKeyJoinReady = 2u;

// Join-table markers (LDB_OP_MARK): one byte per directory slot of a plain single-key table (mask + 1 slots), per key of a
// direct-address table (range slots) or per entry of a key-tuple table (mask + 1 slots); 0 = unmarked.  Entries never move under open
// addressing, so a marker stays with its entry while more rows are inserted.  Allocated zeroed by the first program that marks the
// table, freed with it; a table without markers reads as all unmarked.
constexpr uint64_t kNoSlot = ~0ull;

// The kernel takes ProgramParams by value (__grid_constant__): 3 744 bytes with the limits above, within the classic 4 096-byte
// kernel-parameter limit (program_rt.cpp checks it at compile time).
struct ProgramParams {
   int64_t nRows;
   int64_t firstRow; // global row number of this batch's row 0 (LDB_OP_ROWID)
   int32_t nCols, nInstr, nTables;
   int32_t eachPc;   // index of the LDB_OP_PROBE_EACH instruction, -1 = none: from there on the program runs once per match
   ProgCol cols[kProgMaxCols];
   ProgInstr instr[kProgMaxInstr];
   unsigned long long constLo[kProgMaxConsts];
   long long constHi[kProgMaxConsts];
   uint8_t strings[kProgMaxStrings][kProgStringBytes];
   int32_t stringLen[kProgMaxStrings];
   JoinTableDev tables[kProgMaxTables];
   DictDev dicts[kProgMaxTables]; // tables[k] is a string dictionary: dicts[k] (LDB_OP_STRCODE)
   KeyJoinDev keyTables[kProgMaxTables]; // tables[k] is a key-tuple join table: keyTables[k] (nKeys > 0; PROBE / PROBE_EACH read its keys
                                         // from registers a .. a + nKeys - 1)
   int32_t filterReg; // -1: every row passes
   int32_t sinkKind;  // 1 hash aggregation, 2 join-table build, 3 materialize
   // sink 1 (and sink 2 into a key-tuple table: its key registers)
   int32_t nKeys, nAggs;
   int32_t keyReg[kProgMaxKeys];
   ProgAgg aggs[kProgMaxAggs];
   HashAggDev agg;
   // sink 2
   int32_t buildKeyReg, buildPayloadReg;
   JoinTableDev build;
   KeyJoinDev keyBuild; // nKeys > 0: the build goes into this key-tuple table instead of `build`
   // sink 3: compacted output columns, 16 bytes per value (i128 / double bits in lo) + 1 validity byte
   int32_t nOut;
   int32_t outReg[kProgMaxAggs];
   uint8_t* outValues[kProgMaxAggs];
   uint8_t* outValid[kProgMaxAggs];
   int64_t outCapacity;
   unsigned long long* outCount;
   // LDB_OP_MARK: the markers of tables[k] when an instruction marks it, else null.  Last, so that the fields every other instance
   // reads keep their offsets; any non-null entry selects the kernel instance that has the MARK code.
   uint8_t* marks[kProgMaxTables];
};
// the entries of one join table (a key-tuple table when k.nKeys > 0, else the plain or direct-address table t) selected by their
// markers: which = 1 marked, 0 unmarked, -1 all (and `marked` gets 0 / 1).  Per selected entry, at a position counted by `counter`:
// its keys (keyCols[0..n)), its payload, its marker.  Positions at or past `capacity` are counted but not written.
struct MarkScanOut {
   int64_t* keyCols[kProgMaxKeys];
   int64_t* payload;
   int32_t* marked; // null unless which = -1
   int64_t capacity;
};
void launchJoinMarks(const JoinTableDev& t, const KeyJoinDev& k, const uint8_t* marks, int which, const MarkScanOut& o, unsigned long long* counter, int smCount, cudaStream_t s);

void launchProgram(const ProgramParams& p, int smCount, cudaStream_t s);
void launchHashAggInit(const HashAggDev& t, int smCount, cudaStream_t s);
// compacts the occupied entries into columnar buffers: keys (int64 + validity byte), aggregates (16 B + validity byte)
void launchHashAggExport(const HashAggDev& t, int64_t* const* keyCols, uint8_t* const* keyValid, uint8_t* const* aggCols, uint8_t* const* aggValid, unsigned long long* counter, uint32_t countAggMask, int smCount, cudaStream_t s);
// Exchange of hash aggregations across the ranks of a comm (ldb_gpu_hashagg_exchange, peer.cu).  Received entries are table entries
// as above, copied whole (state, flags with the seen / claim / key-NULL bits, keys, aggregates): source s's j-th entry sits at
// recv[d] + (s * capacity + j) * entryBytes of rank d.  The owner of a group is ((h >> 32) * world) >> 32 for its placement hash h.
struct HashAggShip {
   uint8_t* recv[8];                  // every rank's receive region (peer-mapped; own at [rank]), kMaxPeers entries
   unsigned long long* cursors;       // send: this rank's per-destination position counters, zeroed before
   const unsigned long long* counts;  // merge: the entries source s sent this rank, published by the sources
   int64_t capacity;                  // entries per source sub-region
   int32_t rank, world;
   int32_t kinds[kProgMaxAggs];       // the aggregates' LdbAggKind
};
void launchHashAggSend(const HashAggDev& local, const HashAggShip& x, int smCount, cudaStream_t s);
// maxReceived: the largest min(counts[s], capacity) (sizes the grid)
void launchHashAggMerge(const HashAggDev& owned, const HashAggShip& x, uint64_t maxReceived, int smCount, cudaStream_t s);
void loadHashAggExchangeKernels(); // loads both kernels now (collective launches must not wait for a lazy module load)
// LSD radix sort of (64-bit key, 32-bit row id) pairs — ORDER BY / top-k over materialised rows (GrowingBuffer::sort, Sorting.cpp):
// its lowest `digits` 8-bit digits, one pass each.  After an even number of passes the result is in keys / vals, after an odd
// number in keysTmp / valsTmp.
void launchRadixSortPairs(unsigned long long* keys, uint32_t* vals, unsigned long long* keysTmp, uint32_t* valsTmp, int64_t n, unsigned int* histScratch, int smCount, cudaStream_t s,
                          int digits = 8);
// a key column's validity: one byte per row, or else an Arrow bitmap read from bit `bitOffset` (both null: no NULLs)
struct SortValidity {
   const uint8_t* bytes;
   const uint8_t* bitmap;
   int64_t bitOffset;
};
// multi-key ORDER BY: the 64-bit sort words of one key at the current permutation `ids` (first = 1: ids := 0..n-1 first).
// kind 0: a fixed-width cell (low 8 bytes, sign bit flipped); kind 1: a utf8 cell's length (the longest is atomicMax'ed into
// *maxLen); kind 2: bytes [8 chunk, 8 chunk + 8) of a utf8 cell, zero padded, big-endian, unsigned; kind 3: 1 for a NULL, else 0.
// A NULL cell's word is 0 in kinds 0-2 (NULLs tie on the value; a NULL string leaves *maxLen alone).  DESC inverts the word.
void launchBuildSortWords(const uint8_t* col, const uint8_t* bytes, int elemBytes, SortValidity valid, int kind, int chunk, int64_t n, int descending, int first,
                          uint32_t* ids, unsigned long long* keys, int32_t* maxLen, int smCount, cudaStream_t s);
void launchScatterRanks(const uint32_t* ids, int64_t n, int32_t* rank, int smCount, cudaStream_t s);
// dictionary → table: offsets[0..n] (exclusive scan of the lengths) and the bytes of code i at offsets[i]
void launchDictExport(const DictDev& d, int64_t n, uint32_t* offsets, uint8_t* bytes, int smCount, cudaStream_t s);
// unified dictionaries (ldb_gpu_dict_unify): dst[i] = src[i] + add for i < n (a received block's offsets into the concatenated column)
void launchDictRebase(const uint32_t* src, int64_t n, uint32_t add, uint32_t* dst, int smCount, cudaStream_t s);
// over the n strings of a utf8 column (offsets, bytes) in sorted order `ids`: codes[i] = the distinct strings before sorted position i,
// arenaOff[i] = their bytes; codes[n] and arenaOff[n] are the totals (n + 1 entries each)
void launchDictUnionRanks(const uint32_t* offsets, const uint8_t* bytes, const uint32_t* ids, int64_t n, uint32_t* codes, uint32_t* arenaOff, int smCount, cudaStream_t s);
// fills a fresh dictionary `d` sized for codes[n] strings of arenaOff[n] bytes: arena and entries in code order, one published slot per
// string on dictCode's probe sequence, ctr = {bytes, strings}
void launchDictRankedBuild(const DictDev& d, const uint32_t* offsets, const uint8_t* bytes, const uint32_t* ids, int64_t n, const uint32_t* codes, const uint32_t* arenaOff,
                           int smCount, cudaStream_t s);

} // namespace ldb
